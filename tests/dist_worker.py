"""Multi-process worker (launched by torch.distributed.run from test_distributed.py).

Every rank hosts N/world graph nodes of one case of ``CASES``; after a few rounds the gathered parameters must match a
single-process run of the same problem (rank 0 recomputes it locally).  Two comparisons:

* exact: ``torch.equal`` on theta and on every row the optimizer declares in ``STATE``.  The consensus kernels are
  elementwise per node in a fixed neighbor order and the gloo path gathers the same rows, so where nothing sums over
  ranks the placement cannot change a bit.
* close: theta within a tolerance, where a sum-mode mix or an unpinned samples-per-CTA split changes the summation
  order.

``--delayed 1`` (GPUs) stresses the buffer-reuse protocol: every neighbor read is checked against its round tag
(``debug_sequence_check``), rounds are launched one at a time and one rank is held back by a spin kernel before every
other round, so its peers run ahead as far as the protocol lets them.  Cases that allow a changing graph also drop links
every round (fault injection)."""
import argparse
import copy
import os
import sys
from dataclasses import dataclass, field

import networkx as nx
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nn_distributed_training_b200.data.mnist import synthetic_mnist  # noqa: E402
from nn_distributed_training_b200.models import MNISTConvNet  # noqa: E402
from nn_distributed_training_b200.optimizers import build_optimizer  # noqa: E402
from nn_distributed_training_b200.parallel.context import DistContext  # noqa: E402
from nn_distributed_training_b200.problems.dist_mnist_problem import DistMNISTProblem  # noqa: E402
from nn_distributed_training_b200.utils.graph_generation import generate_from_conf  # noqa: E402

METRICS = ["forward_pass_count", "validation_loss", "consensus_error", "top1_accuracy", "current_epoch"]
ROUNDS, DELAYED_ROUNDS = 6, 14


def always(delayed, eng):
    return True


def never(delayed, eng):
    return False


def fused(delayed, eng):
    return eng is not None


def unsummed(delayed, eng):
    """Exact where the fused kernels mix each node's neighbors in a fixed order (pointer-table and delayed runs); a
    sum-mode mix and the PyTorch path may add the rows in another order than one process."""
    return delayed or (eng is not None and not eng.sum_mode)


@dataclass
class Case:
    confs: list                  # optimizer configs, run one after another in one launch
    exact: callable = always     # (delayed, engine or None) -> compare exactly; otherwise close
    directed: bool = False       # --graph names a directed graph (sequence) of graphs_of; push-sum weights w
    link_drops: bool = True      # a delayed run drops links every round (static-graph optimizers refuse that)
    variants: dict = field(default_factory=dict)   # variant flag -> its default
    pin_split: bool = True       # pin samples_per_cta, so both runs sum the same fp32 gradient partials
    close_rows: tuple = ()       # STATE rows held to the close tolerance too
    val_loss: bool = False       # close mode also compares the last validation loss


CASES = {
    "dinno_dsgd_dsgt": Case(
        [{"alg_name": "dinno", "rho_init": 0.5, "rho_scaling": 1.01, "primal_iterations": 2, "primal_optimizer": "adam",
          "persistant_primal_opt": False, "primal_lr_start": 0.005, "primal_lr_finish": 0.0005, "lr_decay_type": "log"},
         {"alg_name": "dsgd", "alpha0": 0.05, "mu": 0.01},
         {"alg_name": "dsgt", "alpha": 0.02, "init_grads": True}],
        exact=never, pin_split=False, val_loss=True),
    "exact_diffusion": Case([{"alg_name": "exact_diffusion", "alpha0": 0.05, "mu": 0.01}], exact=unsummed),
    "dsgdm": Case([{"alg_name": "dsgdm", "alpha0": 0.05, "mu": 0.01, "beta": 0.9, "nesterov": True}], exact=unsummed,
                  variants={"momentum": "quasi_global"}),
    "kgt": Case([{"alg_name": "kgt", "alpha": 0.02, "local_steps": 2}], exact=unsummed, variants={"correction": "1"}),
    "choco_sgd": Case([{"alg_name": "choco_sgd", "alpha0": 0.05, "mu": 0.01, "gamma": 0.5, "compressor": "int8"}],
                      link_drops=False),
    "beer": Case([{"alg_name": "beer", "alpha": 0.05, "gamma": 0.5, "compressor": "int8"}], link_drops=False),
    "sgp": Case([{"alg_name": "sgp", "alpha0": 0.05, "mu": 0.01}], directed=True, link_drops=False),
    "push_diging": Case([{"alg_name": "push_diging", "alpha": 0.05}], directed=True, link_drops=False),
    # the Byzantine nodes are the first and the last node, so the first and the last rank both host an attacker (and the
    # ranks between, on GPUs, none: their step runs without the attack code).  On the fused path the distance partials
    # are per fixed chunk of the row, so an ALIE attacker's reads of its neighbors' rows after the mix see the same rows
    # on any placement.
    "clipped_gossip": Case([{"alg_name": "clipped_gossip", "alpha0": 0.02, "mu": 0.001, "delta": 0.3}], exact=fused,
                           variants={"clip": "adaptive", "attack": "alie"}, close_rows=("pub",)),
}

VARIANTS = {   # variant flag -> the optimizer config it sets, given its value and the node count
    "momentum": lambda v, N: {"momentum": v},
    "correction": lambda v, N: {"correction": bool(int(v))},
    "clip": lambda v, N: {"clip": v},
    "attack": lambda v, N: {"byzantine": {"nodes": [0, N - 1], "attack": v, "scale": 2.0, "z": 1.0}},
}


def _gen(kind, N, **kw):
    return generate_from_conf(dict({"type": kind, "num_nodes": N}, **kw))[1]


def graphs_of(kind, N):
    """The graph of every round: one graph, or a directed sequence the problem steps through."""
    if kind in ("cycle", "wheel", "complete"):
        return [getattr(nx, kind + "_graph")(N)]
    if kind == "switching":
        back = nx.DiGraph()
        back.add_nodes_from(range(N))
        back.add_edges_from((i, (i - 1) % N) for i in range(N))
        return [_gen("directed_cycle", N), _gen("exponential", N), back,
                _gen("random_directed", N, p=0.3, seed=7, gen_attempts=500)]
    if kind == "random_directed":
        return [_gen("random_directed", N, p=0.3, seed=3, gen_attempts=500)]
    return [_gen(kind, N)]


def _regular(g):
    return len({d for _, d in g.out_degree()}) == 1


class SwitchingMNIST(DistMNISTProblem):
    """Round k runs on ``graphs[k % len(graphs)]``: the planned graph sequence of the fused path and ``update_graph``
    of the PyTorch path step through the same list."""

    def __init__(self, graphs, *a, **kw):
        self.graphs = graphs
        self._round_idx = 0
        super().__init__(graphs[0], *a, **kw)

    def plan_graphs(self, oits, k0, draws_per_round, init_draws=0, refresh=True):
        return [self.graphs[k % len(self.graphs)] for k in range(oits)]

    def update_graph(self):
        self.graph = self.graphs[self._round_idx % len(self.graphs)]
        self._round_idx += 1


def make(ctx, case, graphs, conf, backend, delayed, pipeline):
    N = graphs[0].number_of_nodes()
    data = synthetic_mnist(200 * N, seed=3)
    val = synthetic_mnist(128, seed=4)
    shards = [data.select(torch.arange(i * 200, (i + 1) * 200)) for i in range(N)]
    pconf = {"problem_name": "t", "train_batch_size": 32, "val_batch_size": 64, "metrics": METRICS,
             "metrics_config": {"evaluate_frequency": 3}, "optimizer_config": conf}
    if case.pin_split or delayed:
        # the same samples-per-CTA split in the distributed and the single-process run: identical fp32 gradient
        # partials, so the comparison is not blurred by Adam amplifying summation-order round-off
        pconf["samples_per_cta"] = 8
    if pipeline is not None:
        pconf["input_pipeline"] = pipeline
    if delayed and case.link_drops:
        pconf["fault_injection"] = {"link_drop_prob": 0.45, "seed": 3, "from_round": 0, "to_round": DELAYED_ROUNDS}
    torch.manual_seed(5)
    args = (MNISTConvNet(3, 5, 64), torch.nn.NLLLoss(), shards, val, ctx.device, pconf)
    if case.directed:
        return SwitchingMNIST(graphs, *args, ctx=ctx, backend=backend, seed=11)
    return DistMNISTProblem(graphs[0], *args, ctx=ctx, backend=backend, seed=11)


def run_spin_delayed(ctx, opt):
    """Launch the rounds one at a time: the last rank spins ~0.3 ms (many round times) before every odd round and rank 0
    before every third, then check every neighbor read's round tag."""
    from nn_distributed_training_b200.ops import load_ext
    ext = load_ext(required=True)
    slow = ctx.world_size - 1
    for r in range(DELAYED_ROUNDS):
        if ctx.rank == slow and r % 2 == 1:
            ext.spin(600_000)
        if ctx.rank == 0 and r % 3 == 2:
            ext.spin(300_000)
        opt.run_rounds(1)
    torch.cuda.synchronize()
    opt._program.eng.check()             # raises on a stale tag (err == 2) or a spin timeout


def state_rows(pr, opt):
    """theta and every declared row of all N nodes (a row of one value per node, such as push-sum's w, as ``[N, 1]``)."""
    if getattr(opt, "_program", None) is not None:      # the fused path keeps some rows on the device: mirror them
        opt._program.sync_back()
    rows = {"theta": pr.arena.theta}
    rows.update((n, getattr(opt, n)) for n in opt.STATE if getattr(opt, n) is not None)
    return {n: pr.gather_rows(t if t.dim() > 1 else t.view(-1, 1)).cpu() for n, t in rows.items()}


def _bad(x, ref):
    return ((x - ref).abs() > 2e-5 + 2e-3 * ref.abs()).float().mean().item()


def run(ctx, name, case, graph, graphs, conf, backend, delayed, pipeline):
    pr = make(ctx, case, graphs, conf, backend, delayed, pipeline)
    opt = build_optimizer(pr, ctx.device, copy.deepcopy(conf))
    if delayed:
        run_spin_delayed(ctx, opt)
    else:
        opt.train()
    eng = getattr(getattr(opt, "_program", None), "eng", None)
    if eng is not None and "byzantine" in conf:
        assert (eng.t_attack is not None) == any(opt.attack), "attack codes on the wrong ranks"
    rows = state_rows(pr, opt)
    ok = True
    if ctx.is_main:
        solo = DistContext.single(ctx.device)
        pr1 = make(solo, case, graphs, conf, backend, delayed, None if pipeline is None else "resident")
        opt1 = build_optimizer(pr1, solo.device, copy.deepcopy(conf))
        if delayed:
            opt1.run_rounds(DELAYED_ROUNDS)
            torch.cuda.synchronize()
        else:
            opt1.train()
        ref = state_rows(pr1, opt1)
        theta, rtheta = rows["theta"], ref["theta"]
        rel = ((theta - rtheta).norm() / rtheta.norm()).item()
        how = f"{conf['alg_name']} world={ctx.world_size} graph={graph} delayed={int(delayed)}"
        if eng is not None:
            how += f" sum_mode={eng.sum_mode} distinct_graphs={len(eng.topos)}"
        if case.exact(delayed, eng):
            ok = all(torch.equal(rows[n], ref[n]) for n in ref)
            how += " exact"
        elif delayed:
            ok = rel < 1e-5 and len(eng.topos) > 3
        else:
            bad = max(_bad(rows[n], ref[n]) for n in ("theta",) + case.close_rows)
            ok = bad < 5e-3 and rel < 1e-2
            how += f" bad={bad:.2e}"
            if case.val_loss:
                vd = (pr.metrics["validation_loss"][-1] - pr1.metrics["validation_loss"][-1]).abs().max().item()
                ok = ok and vd < 1e-3
                how += f" val_diff={vd:.2e}"
        if case.directed and (len(graphs) > 1 or not _regular(graphs[0])):
            w = ref["w"]           # not doubly stochastic: the push-sum weights must have moved off 1
            ok = ok and not torch.all(w == 1.0)
            how += f" w in [{w.min():.3f}, {w.max():.3f}]"
        print(f"[{name}] {how} rel={rel:.2e} {'OK' if ok else 'MISMATCH'}", flush=True)
    ctx.barrier()
    return ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", required=True, choices=list(CASES))
    ap.add_argument("--cuda", type=int, default=0)
    ap.add_argument("--nodes", type=int, default=6)
    ap.add_argument("--graph", default=None)     # default: cycle, or directed_cycle for a directed case
    ap.add_argument("--pipeline", default=None)  # host: device-initiated staging inside multi-round graphs; the
                                                 # single-process run then uses resident shards
    ap.add_argument("--delayed", type=int, default=0)
    for flag in VARIANTS:
        ap.add_argument("--" + flag, default=None)
    args = ap.parse_args()
    case = CASES[args.case]
    given = {f for f in VARIANTS if getattr(args, f) is not None}
    if not given <= case.variants.keys():
        ap.error(f"case {args.case} takes no {' / '.join('--' + f for f in sorted(given - case.variants.keys()))}")
    graph = args.graph or ("directed_cycle" if case.directed else "cycle")
    graphs = graphs_of(graph, args.nodes)
    ctx = DistContext.from_env(use_cuda=bool(args.cuda))
    ok = True
    for conf in case.confs:
        conf = dict(copy.deepcopy(conf), outer_iterations=DELAYED_ROUNDS if args.delayed else ROUNDS, profile=False)
        for flag, default in case.variants.items():
            conf.update(VARIANTS[flag](getattr(args, flag) or default, args.nodes))
        if args.delayed:
            conf["debug_sequence_check"] = True
        ok = run(ctx, args.case, case, graph, graphs, conf, "fused" if args.cuda else "torch", bool(args.delayed),
                 args.pipeline) and ok
    if ctx.is_main:
        print("DIST_RESULT", "PASS" if ok else "FAIL", flush=True)
    if torch.distributed.is_initialized():
        torch.distributed.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
