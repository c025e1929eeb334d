"""DP-DSGD — differentially private decentralized SGD with node-level clipping and Gaussian noise, and DECOR's pairwise
noise that cancels over each edge (Allouah, Koloskova, El Mrini, Guerraoui, Jaggi, *The Privacy Power of Correlated
Noise in Decentralized Learning*, ICML 2024).  No counterpart in the reference.

DSGD's round (mix, gradient at the mixed point, step) with DSGD's step schedule.  Round k of node i:

    alpha_k  = alpha_{k-1} (1 - mu alpha_{k-1})
    theta_i <- sum_j W_ij theta_j^pub                                             (DSGD's mix)
    g_i      = grad loss_i(theta_i)
    f_i      = min(1, C / ||g_i||_2)          (1 when g_i = 0; the norm in float64)
    v_i      = C z_dp xi_i^k + C z_pair sum_{j in N_i^k} s_ij xi_ij^k,   s_ij = +1 if i < j else -1
    theta_i <- theta_i - alpha_k (f_i g_i + v_i);  publish theta_i

``xi`` are standard normal rows on the live elements (0 on padding and slot holes) drawn from a counter-based Philox
stream (ops/consensus_ref.py: dp_noise; the kernels draw the same stream): ``xi_ij`` is keyed by the unordered edge, so
both ends draw it bit for bit without communicating, and the edge terms cancel in the network sum.  ``N_i^k`` is the
neighbor set of round k's graph after link drops.  ``z_pair = 0`` is local-DP DSGD, ``z_dp = z_pair = 0`` clipped DSGD.

The privacy ledger (``rho_eav``, ``rho_all``: ``[N]`` float64 zCDP per node, over the rounds run) is optimizer state
and goes into checkpoints.  ``rho_eav`` is the guarantee against an observer of every published row who knows no pair
secret, ``rho_all`` the one against any observer (DESIGN §2.16).  ``privacy_record()`` reports both with their
epsilons; on a ``ConsensusProblem`` it is also the problem's ``privacy_record`` hook, which ``save_metrics`` writes into
the results file (a foreign problem writes its own results, so there the record is the optimizer's alone).  The
guarantee is node-level: neighboring datasets differ in one node's whole shard.  Floating-point Gaussian sampling is not
a certified DP implementation and Philox is not a cryptographic generator: this simulates the mechanism.  Directed graphs, ``mixing_order: reference`` and
Byzantine attackers are refused.
"""
from __future__ import annotations

import math
import numbers
from typing import Dict

import numpy as np
import torch

from .base import ConsensusOptimizer
from ..problems.base import ConsensusProblem
from ..ops import consensus_ref as ref


def _nonneg(conf, key, default=None, positive=False):
    v = conf.get(key, default)
    if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(float(v)) or float(v) < 0.0 \
            or (positive and float(v) == 0.0):
        raise ValueError(f"dp_dsgd {key} must be finite and {'> 0' if positive else '>= 0'} (got {v!r})")
    return float(v)


class DPDSGD(ConsensusOptimizer):
    alg_name = "dp_dsgd"
    SCALARS = ("alph",)

    def __init__(self, ddl_problem, device, conf):
        if conf.get("mixing_order", "jacobi") != "jacobi":
            raise ValueError("dp_dsgd runs the synchronous (jacobi) mixing order only")
        super().__init__(ddl_problem, device, conf)
        graph = getattr(self.pr, "graph", None)
        if graph is not None and graph.is_directed():
            raise ValueError("dp_dsgd needs an undirected graph (the pairwise noise of an edge cancels between its two "
                             "ends)")
        if conf.get("byzantine") is not None:
            raise ValueError("dp_dsgd does not model Byzantine attackers (clipped_gossip and bridge do)")
        self.alph0 = _nonneg(conf, "alpha0")
        self.mu = _nonneg(conf, "mu", 0.0)
        self.clip = _nonneg(conf, "clip_norm", positive=True)
        self.z_dp = _nonneg(conf, "noise_multiplier")
        self.z_pair = _nonneg(conf, "pair_noise_multiplier", 0.0)
        self.delta = conf.get("target_delta", 1e-5)
        if isinstance(self.delta, bool) or not isinstance(self.delta, numbers.Real) or not 0.0 < self.delta < 1.0:
            raise ValueError(f"dp_dsgd target_delta must be in (0, 1) (got {self.delta!r})")
        seed = conf.get("noise_seed", getattr(self.pr, "seed", 0))
        if isinstance(seed, bool) or not isinstance(seed, numbers.Integral):
            raise ValueError(f"dp_dsgd noise_seed must be an integer (got {seed!r})")
        self.noise_seed = int(seed)
        self.key = ref.dp_key(self.noise_seed)
        # C z rounded once to float64: the factors both implementations multiply the normals by
        self.cz_dp, self.cz_pair = self.clip * self.z_dp, self.clip * self.z_pair
        self.alph = self.alph0
        self.refresh_graph = bool(conf.get("update_graph", True))
        self.live = ref.choco_live(self.arena.layout).numpy()
        N = self.pr.N
        self.rho_eav = np.zeros(N)
        self.rho_all = np.zeros(N)
        self._rho_cache: Dict[bytes, tuple] = {}
        if isinstance(self.pr, ConsensusProblem):     # the results file of a foreign problem is not written here
            self.pr.privacy_record = self.privacy_record

    def alpha_table(self, n=None):
        """alpha of rounds 0..n-1 (default: all ``outer_iterations``), DSGD's schedule."""
        out, a = [], self.alph0
        for _ in range(self.oits if n is None else int(n)):
            a = ref.dsgd_alpha(a, self.mu)
            out.append(a)
        return out

    # -- accountant ------------------------------------------------------------------------------------------------
    def round_rho(self, topo) -> tuple:
        """zCDP cost of one round on ``topo`` per node, (eavesdropper, any observer), cached per graph."""
        r = self._rho_cache.get(topo.key)
        if r is None:
            r = self._rho_cache[topo.key] = ref.dp_rho(topo.W, self.z_dp, self.z_pair)
        return r

    def account(self, topo) -> None:
        """Add one round on ``topo`` to the ledger."""
        eav, allo = self.round_rho(topo)
        self.rho_eav += eav
        self.rho_all += allo

    def privacy_record(self) -> dict:
        """The ``privacy`` entry of the results file: the ledger and both epsilons (maximum over the nodes)."""
        return {"target_delta": float(self.delta), "rounds": int(self.k),
                "rho_eavesdropper": torch.as_tensor(self.rho_eav.copy()),
                "rho_any_observer": torch.as_tensor(self.rho_all.copy()),
                "epsilon_eavesdropper": ref.dp_epsilon(self.rho_eav, self.delta),
                "epsilon_any_observer": ref.dp_epsilon(self.rho_all, self.delta)}

    def state_dict(self) -> Dict:
        sd = super().state_dict()
        sd.update(rho_eav=self.rho_eav.copy(), rho_all=self.rho_all.copy())
        return sd

    def load_state_dict(self, sd: Dict):
        super().load_state_dict(sd)
        self.rho_eav[:] = sd["rho_eav"]
        self.rho_all[:] = sd["rho_all"]

    # -- round -----------------------------------------------------------------------------------------------------
    def noise_rows(self, k: int, topo) -> torch.Tensor:
        """``v`` of the local nodes in round k on ``topo``, float64 ``[L, n_pad]``."""
        pl, n_pad = self.pr.placement, self.arena.n_pad
        v = np.zeros((pl.L, n_pad))
        if self.cz_dp != 0.0 or self.cz_pair != 0.0:
            for l, g in enumerate(pl.local_nodes):
                v[l] = ref.dp_noise(self.key, k, g, topo.neighbors_noself[g], n_pad, self.cz_dp, self.cz_pair,
                                    self.live)
        return torch.as_tensor(v, device=self.device)

    def _round(self, k: int):
        pr, a = self.pr, self.arena
        if self.refresh_graph:
            pr.update_graph()
        topo = pr.topology()
        self.alph = ref.dsgd_alpha(self.alph, self.mu)
        with torch.no_grad():
            a.theta.copy_(ref.dsgd_mix(pr.gather_rows(a.theta), self._rows(topo, topo.W)))
        pr.compute_grads()
        with torch.no_grad():
            f = [ref.dp_clip_factor(float(a.grad[l].double().square().sum()), self.clip) for l in range(a.grad.shape[0])]
            u = a.grad * torch.as_tensor(f, dtype=a.dtype, device=self.device)[:, None]
            if self.cz_dp != 0.0 or self.cz_pair != 0.0:
                u = u + self.noise_rows(k, topo).to(a.dtype)
            ref.dsgd_step_(a.theta, u, self.alph)
        self.account(topo)
