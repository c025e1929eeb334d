"""Fused execution of the consensus optimizers: CUDA-graph round programs.

A round is a short, fixed kernel sequence
    DiNNO:  [fwd/bwd, dinno_update(p)] x primal_iterations
    DSGD :  dsgd_mix, fwd/bwd, dsgd_step
    DSGD with momentum:  dsgd_mix, fwd/bwd, dsgdm_step
    DSGT :  dsgt_mix, fwd/bwd, dsgt_track
    Exact Diffusion:  ed_mix, fwd/bwd, ed_step
    CHOCO-SGD:  choco_mix, fwd/bwd, choco_step
    BEER:  beer_mix, fwd/bwd, beer_step
    SGP:  sgp_mix, fwd/bwd, sgp_step
    Push-DIGing:  pdg_mix, fwd/bwd, pdg_track
    K-GT:  kgt_mix, [fwd/bwd, kgt_step(p)] x local_steps       (local DSGD: dsgd_mix in place of kgt_mix)
    ClippedGossip:  cg_dist, cg_mix, fwd/bwd, cg_step           (clip: none: dsgd_mix, fwd/bwd, cg_step)
    decentralized AMSGrad / AdaGrad:  dadaptive_mix, fwd/bwd, dadaptive_step     (own second moment: dsgd_mix first)
    RelaySum:  relay_mix, fwd/bwd, relay_step
    BRIDGE (trimmed mean / median screening):  bridge_mix, fwd/bwd, cg_step
    PowerGossip:  pg_mix, fwd/bwd, pg_step
    DeTAG:  ag_gossip(s) x gossip_steps, fwd/bwd, detag_track      (every ag_gossip a protocol round)
    GT-HSGD:  dsgt_mix, fwd/bwd, fwd/bwd at theta_prev, hsgd_track   (both fwd/bwd on the same minibatch)
    Gossip-PGA:  pga_sum, pga_mix, fwd/bwd, dsgd_step             (pga_sum returns at once on gossip rounds)
    SlowMo:  pga_sum, pga_mix, slowmo_outer, fwd/bwd, dsgd_step   (base momentum: dsgdm_step; slowmo_outer returns at once
             on gossip rounds)
    DP-DSGD / DECOR:  dsgd_mix, fwd/bwd, dp_norm, dp_step
    Moniqua:  mq_mix, fwd/bwd, mq_step
    SPARQ-SGD:  sparq_mix, [fwd/bwd, sparq_step(p)] x local_steps, sparq_publish
    cross-gradient:  xg_pull, fwd/bwd, fwd/bwd at theta_x[e] x dmax, xg_publish, xg_step   (two protocol rounds)
whose per-round scalars come from device schedules indexed by a device round
counter, so ``R`` consecutive rounds are captured once as a CUDA graph and
replayed between evaluation points with no host work (the reference issues
~800 serial micro-launches per round from Python, SURVEY §3.2).  When the
model has no fused forward/backward kernel the same consensus kernels run
eagerly around an autograd step.
"""
from __future__ import annotations

import gc
import os
from typing import Dict

import torch

from .engine import THETA_ROW_ALGS, ConsensusEngine, schedule_horizon

MAX_ROUNDS_PER_GRAPH = 64
PULL_ROUNDS_PER_GRAPH = 64     # host-fed / staged rounds captured per graph (staging kernel forked inside the graph); a
                               # production chunk (evaluate_frequency rounds, 20 in the PAPER configs) is ONE graph launch


def _nvtx(name):
    """NVTX range per phase (visible in Nsight / torch.profiler traces; no-op cost when not profiling)."""
    return torch.cuda.nvtx.range(name)


def _round_ops(opt, eng, grads, grads_prev, grads_cross):
    with _nvtx(f"consensus_round/{opt.alg_name}"):
        _round_ops_impl(opt, eng, grads, grads_prev, grads_cross)


def _round_ops_impl(opt, eng, grads, grads_prev, grads_cross):
    alg = opt.alg_name
    if eng.sum_mode:
        eng.op.local_sum()   # complete graph: per-rank partial sums feeding the NVLS reduction
    if alg == "dinno":
        for p in range(opt.pits):
            grads(p)
            eng.op.dinno_update(p)
    elif alg == "dsgd":
        eng.op.dsgd_mix()
        grads(0)
        eng.op.dsgd_step()
    elif alg == "dsgdm":
        eng.op.dsgd_mix()
        grads(0)
        eng.op.dsgdm_step()
    elif alg == "dsgt":
        eng.op.dsgt_mix()
        grads(0)
        eng.op.dsgt_track()
    elif alg == "exact_diffusion":
        eng.op.ed_mix()
        grads(0)
        eng.op.ed_step()
    elif alg == "choco_sgd":
        eng.op.choco_mix()
        grads(0)
        eng.op.choco_step()
    elif alg == "beer":
        eng.op.beer_mix()
        grads(0)
        eng.op.beer_step()
    elif alg == "kgt":
        if opt.correction:
            eng.op.kgt_mix()
        else:
            eng.op.dsgd_mix()
        for p in range(opt.local_steps):
            grads(p)
            eng.op.kgt_step(p)
    elif alg == "clipped_gossip":
        if opt.clip == "adaptive":
            eng.op.cg_dist()
            eng.op.cg_mix()
        else:
            eng.op.dsgd_mix()
        grads(0)
        eng.op.cg_step()
    elif alg == "bridge":
        eng.op.bridge_mix()
        grads(0)
        eng.op.cg_step()
    elif alg == "dadaptive":
        if opt.tracking:
            eng.op.dadaptive_mix()
        else:
            eng.op.dsgd_mix()
        grads(0)
        eng.op.dadaptive_step()
    elif alg == "relaysum":
        eng.op.relay_mix()
        grads(0)
        eng.op.relay_step()
    elif alg == "powergossip":
        eng.op.pg_mix()
        grads(0)
        eng.op.pg_step()
    elif alg == "detag":
        for s in range(opt.gossip_steps):
            eng.op.ag_gossip(s)
        grads(0)
        eng.op.detag_track()
    elif alg == "gt_hsgd":
        eng.op.dsgt_mix()
        grads(0)
        grads_prev()
        eng.op.hsgd_track()
    elif alg == "cross_gradient":
        eng.op.xg_pull()
        grads(0)
        for e in range(opt.dmax):
            grads_cross(e)
        eng.op.xg_publish()
        eng.op.xg_step()
    elif alg == "gossip_pga":
        eng.op.pga_sum()
        eng.op.pga_mix()
        grads(0)
        eng.op.dsgd_step()
    elif alg == "slowmo":
        eng.op.pga_sum()
        eng.op.pga_mix()
        eng.op.slowmo_outer()
        grads(0)
        if opt.m is None:
            eng.op.dsgd_step()
        else:
            eng.op.dsgdm_step()
    elif alg == "dp_dsgd":
        eng.op.dsgd_mix()
        grads(0)
        eng.op.dp_norm()
        eng.op.dp_step()
    elif alg == "moniqua":
        eng.op.mq_mix()
        grads(0)
        eng.op.mq_step()
    elif alg == "sparq_sgd":
        eng.op.sparq_mix()
        for p in range(opt.local_steps):
            grads(p)
            eng.op.sparq_step(p)
        eng.op.sparq_publish()
    elif alg == "sgp":
        eng.op.sgp_mix()
        grads(0)
        eng.op.sgp_step()
    elif alg == "push_diging":
        eng.op.pdg_mix()
        grads(0)
        eng.op.pdg_track()
    else:  # pragma: no cover
        raise NameError("Unknown distributed opt algorithm.")


def _collect_before_capture():
    """Collect cyclic garbage before a capture: an unreachable program of an earlier run (optimizer, program and problem
    reference each other) may still own CUDA graphs, and the collector destroying one of them in the middle of a capture
    invalidates that capture."""
    gc.collect()


class _RoundCount:
    """Runs ``_round_ops_impl`` once without a device, as the engine and the gradient callbacks, and counts the round's
    calls: ``ops`` on ``eng.op``, ``draws`` of ``grads(p)`` and ``extra`` of ``grads_prev`` and ``grads_cross``."""

    def __init__(self, opt, sum_mode: bool = False):
        self.sum_mode = sum_mode
        self.op = self
        self.ops = self.draws = self.extra = 0
        _round_ops_impl(opt, self, self._draw, self._extra, self._extra)

    def __getattr__(self, name):       # a kernel of eng.op
        return self._op

    def _op(self, *args):
        self.ops += 1

    def _draw(self, p: int = 0):
        self.draws += 1

    def _extra(self, *args):
        self.extra += 1


def draws_per_round(opt) -> int:
    """Minibatch draws (``grads(p)`` calls) of one round."""
    return _RoundCount(opt).draws


class RoundProgram:
    """Owns the engine and the captured graphs for one optimizer."""

    def __init__(self, opt):
        self.opt = opt
        pr = self.pr = opt.pr
        self.dpr = draws_per_round(opt)
        init_draws = 1 if (opt.alg_name == "dsgt" and opt.init_grads and not opt._initialised) else 0
        graphs = pr.plan_graphs(schedule_horizon(opt), opt.k, self.dpr, init_draws,
                                refresh=getattr(opt, "refresh_graph", True))
        # a problem without a fused forward/backward kernel is captured when its gradient step is (a batched hook over
        # fixed buffers, ReferenceProblemAdapter.capturable_grads); per-node autograd runs eagerly between the kernels
        self.capturable = ((pr.fused is not None or getattr(pr, "capturable_grads", False))
                           and os.environ.get("NNDT_NO_GRAPH", "0") != "1")
        # ---- input pipeline of the fused MNIST problem ------------------------------------------------------------
        pipeline = "resident"
        if pr.fused is not None:
            pipeline = pr.conf.get("input_pipeline", "auto")
            can_stage = hasattr(pr.fused, "enable_host_feed") and self.capturable
            if pipeline == "auto":
                # staged-resident is the faster way to run resident shards (4 % on the headline round): the training
                # kernel reads a compact, L2-resident batch instead of chasing the sampler through HBM
                pipeline = "staged" if can_stage else "resident"
            if not hasattr(pr.fused, "enable_host_feed"):
                pipeline = "resident"
        self.eng = ConsensusEngine(opt, graphs)
        self.graph_plan = graphs
        # evaluation between rounds can use the fused consensus-metric kernel on the published rows where channel 0 holds
        # theta; the others' metric reads the parameter rows (all_theta) at the evaluation points instead
        theta_rows = opt.alg_name in THETA_ROW_ALGS and not getattr(opt, "byzantine", None)
        pr._metric_engine = (self.eng, lambda: opt.k) if theta_rows else None
        self._graphs: Dict[int, torch.cuda.CUDAGraph] = {}
        self.host_mode = False
        self.pipeline = "resident"
        if pr.fused is not None:
            pr.fused.sync_calls_from_host()
            self._deferred_pipeline = None
            if pipeline in ("host", "staged") and hasattr(pr.fused, "enable_host_feed"):
                if init_draws:
                    # DSGT init_grads (optimizers/dsgt.py:33-46 of the reference): the ONE initial gradient draw runs on the
                    # resident shards; the host-fed / staged stream starts at the draw after it (dsgt_init switches over)
                    self._deferred_pipeline = pipeline
                else:
                    self._enable_pipeline(pipeline)

    def _enable_pipeline(self, pipeline: str):
        self.pr.fused.enable_host_feed(self.dpr, source="device" if pipeline == "staged" else "host")
        self.host_mode = True
        self.pipeline = pipeline
        self._stage_set = 0
        self._pull_graphs: Dict = {}
        self._pull_parity = 0
        self._pull_primed = False
        self._side = None

    def launches_per_round(self) -> int:
        """Kernel launches of one communication round (the staging kernel of the host-fed / staged pipelines
        included)."""
        c = _RoundCount(self.opt, self.eng.sum_mode)
        return c.ops + c.draws + c.extra + (1 if self.host_mode else 0)

    def grads(self, p: int = 0):
        pr = self.pr
        if pr.fused is None:
            if self.opt.alg_name == "gt_hsgd":     # autograd: both points in one call (grads_prev has nothing left)
                pr.compute_grads_pair(self.opt.theta_prev, self.opt.grad_prev)
            elif self.opt.alg_name == "cross_gradient":     # autograd: every point in one call (as gt_hsgd)
                pr.compute_grads_multi(self.opt.theta_x, self.opt.grad_x)
            else:
                pr.compute_grads()
        elif self.host_mode:
            pr.fused.direct_ops[self._stage_set][p].train()
        else:
            pr.fused.launch()

    def grads_prev(self):
        """GT-HSGD's second forward/backward, at theta_prev on the minibatch ``grads(0)`` just drew: the prev-point op,
        or the direct one of the current stage set."""
        pr = self.pr
        if pr.fused is None:
            return
        if self.host_mode:
            pr.fused.direct_prev_ops[self._stage_set].train()
        else:
            pr.fused.launch_prev()

    def grads_cross(self, e: int):
        """The cross-gradient forward/backward at ``theta_x[e]`` on the minibatch ``grads(0)`` just drew: cross-point op
        ``e``, or its direct op of the current stage set."""
        pr = self.pr
        if pr.fused is None:
            return
        if self.host_mode:
            pr.fused.cross[e]["direct"][self._stage_set].train()
        else:
            pr.fused.launch_cross(e)

    def _count(self, rounds: int):
        """Host mirror of the device-side draw counters."""
        if self.pr.fused is not None:
            self.pr.count_draws_all(rounds * self.dpr)

    def dsgt_init(self):
        self.grads()
        self.eng.op.dsgt_init()
        if self.pr.fused is not None:
            self.pr.count_draws_all(1)
            if getattr(self, "_deferred_pipeline", None):
                torch.cuda.synchronize(self.pr.device)      # the kernel-owned draw counters have advanced
                self._enable_pipeline(self._deferred_pipeline)
                self._deferred_pipeline = None

    def _capture_pull_graph(self, R: int, parity: int):
        """``R`` host-fed rounds as ONE graph with two branches: while round i computes on the capture stream,
        the staging kernel pulls round i+1's rows out of pinned host memory on a forked stream (device-initiated
        H2D over PCIe); the training kernel stores every step's losses into pinned host memory itself.  No CPU work
        per round at all."""
        fz = self.pr.fused
        if self._side is None:
            self._side = torch.cuda.Stream(device=self.pr.device)
        side = self._side
        _collect_before_capture()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            main = torch.cuda.current_stream(self.pr.device)
            for i in range(R):
                b = (parity + i) & 1
                # set b^1 was last read by round i-1, which precedes this point on `main`
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    fz.gather_ops[b ^ 1].launch()
                self._stage_set = b
                _round_ops(self.opt, self.eng, self.grads, self.grads_prev, self.grads_cross)
                main.wait_stream(side)     # round i+1 consumes what was just staged (also joins the fork)
        return g

    def _pull_graph(self, r: int, parity: int):
        key = (r, parity)
        g = self._pull_graphs.get(key)
        if g is None:
            g = self._pull_graphs[key] = self._capture_pull_graph(r, parity)
        return g

    def _run_pull_graphs(self, rounds: int, capture_only: bool = False):
        fz = self.pr.fused
        if not self._pull_primed:
            fz.gather_ops[self._pull_parity].launch()      # stage the very first round
            self._pull_primed = True
        left, parity = rounds, self._pull_parity
        while left > 0:
            r = min(left, PULL_ROUNDS_PER_GRAPH)
            g = self._pull_graph(r, parity)
            parity = (parity + r) & 1
            left -= r
            if not capture_only:
                g.replay()
                self._pull_parity = parity
                self._count(r)

    def _resident_graph(self, r: int):
        g = self._graphs.get(r)
        if g is None:
            _collect_before_capture()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for _ in range(r):
                    _round_ops(self.opt, self.eng, self.grads, self.grads_prev, self.grads_cross)
            self._graphs[r] = g
        return g

    def drop_graphs(self):
        """Forget the captured resident-round graphs (their kernels read buffers that have been reallocated)."""
        self._graphs.clear()

    def prepare(self, rounds: int):
        """Capture (without executing) every CUDA graph that ``run(rounds)`` will replay from the current state, so a
        following ``run`` issues graph launches only."""
        if not self.capturable:
            return
        if self.host_mode:
            self._run_pull_graphs(rounds, capture_only=True)
            return
        left = rounds
        while left > 0:
            r = min(left, MAX_ROUNDS_PER_GRAPH)
            self._resident_graph(r)
            left -= r

    def run(self, rounds: int):
        """Execute ``rounds`` consecutive rounds starting at the device round counter."""
        if self.opt.k + rounds > self.eng.horizon:
            raise RuntimeError(f"rounds {self.opt.k}..{self.opt.k + rounds - 1} run past the schedule horizon of "
                               f"{self.eng.horizon} rounds")
        if self.eng.dp:         # the privacy ledger follows the planned graph of every round run
            for k in range(self.opt.k, self.opt.k + rounds):
                eav, allo = self.eng.dp[self.eng.gid[k]]
                self.opt.rho_eav += eav
                self.opt.rho_all += allo
        if self.host_mode:
            return self._run_pull_graphs(rounds)
        left = rounds
        while left > 0:
            r = min(left, MAX_ROUNDS_PER_GRAPH)
            if self.capturable:
                self._resident_graph(r).replay()
            else:
                for _ in range(r):
                    _round_ops(self.opt, self.eng, self.grads, self.grads_prev, self.grads_cross)
            self._count(r)
            left -= r

    def sync_back(self):
        """Mirror device-resident optimizer state into the optimizer object: the published rows that are the only live
        copy (``ConsensusEngine.published_rows``) and the host scalars of round k."""
        opt = self.opt
        for row, dst, only in self.eng.published_rows(opt.k):
            if only:
                dst.copy_(row)
        if opt.alg_name == "dinno" and opt.k > 0:
            opt.rho = opt.rho_at(opt.k - 1)
        if hasattr(opt, "alpha_table") and opt.k > 0:
            opt.alph = opt.alpha_table(opt.k)[opt.k - 1]


def run_fused_training(opt, profiler=None):
    pr = opt.pr
    prog = opt.fused_program()
    every = opt._eval_every()
    oits = opt.oits
    while opt.k < oits:
        k = opt.k
        opt._maybe_eval(k)
        if k >= oits - 1:
            nxt = oits
        else:
            nxt = min((k // every + 1) * every, oits - 1)
        if profiler is not None or opt.checkpointer is not None:
            nxt = k + 1 if profiler is not None else min(nxt, opt.checkpointer.next_save_after(k))
        prog.run(nxt - k)
        opt.k = nxt
        if profiler is not None:
            profiler.step()
        if opt.checkpointer is not None:
            prog.sync_back()
            opt.checkpointer.maybe_save(opt)
    torch.cuda.synchronize(pr.device)
    prog.eng.check()
    prog.sync_back()
