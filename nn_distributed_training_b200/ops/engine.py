"""Consensus engine: device tables + fused kernel ops for one optimizer run.

Built once per ``train()``; afterwards a communication round is a fixed sequence
of kernel launches that reads every per-round scalar from device memory, so the
sequence is captured in a CUDA graph and replayed (``round_program.py``).
"""
from __future__ import annotations

import os
from typing import Dict, List

import numpy as np
import torch

from . import load_ext
from .consensus_ref import CHOCO_CODE, choco_live, choco_live_words, ed_weights
from ..optimizers.beer import FIXED_W as BEER_FIXED_W
from ..optimizers.sparq import FIXED_W as SPARQ_FIXED_W
from ..parallel.symm import SymmetricBuffer
from ..utils.graph_generation import Topology

OPT_CODE = {"sgd": 0, "adam": 1, "adamw": 2}


def schedule_horizon(opt) -> int:
    """Rounds the device schedules cover: ``opt.horizon`` (``None``: ``outer_iterations``), at most ``outer_iterations``."""
    H = getattr(opt, "horizon", None)
    H = opt.oits if H is None else int(H)
    if not 1 <= H <= opt.oits:
        raise ValueError(f"schedule horizon {H} outside 1..outer_iterations ({opt.oits})")
    return H


def schedule_tables(opt, H: int):
    """Host (float64) ``rho`` / ``lr`` / ``alpha`` tables of rounds ``[0, H)``: entry k is ``rho_at(k)``, ``lr_at(k)`` and
    ``alpha_table()[k]`` with the configured ``outer_iterations`` (linear and log lr decay depend on it), so a table
    built for a horizon is a prefix of the full one.  A DSGT per-coordinate step leaves ``alpha`` zero (the kernel reads
    the row instead)."""
    rho = np.zeros(H); lr = np.zeros(H); alpha = np.zeros(H)
    if opt.alg_name == "dinno":
        rho[:] = [opt.rho_at(k) for k in range(H)]
        lr[:] = [opt.lr_at(k) for k in range(H)]
    elif hasattr(opt, "alpha_table"):        # a decaying step
        alpha[:] = opt.alpha_table(H)
    elif not torch.is_tensor(opt.alpha):     # DSGT, BEER, Push-DIGing, K-GT, dadaptive, DeTAG, GT-HSGD: a constant step
        alpha[:] = opt.alpha
    return rho, lr, alpha


# Algorithms whose mix has the complete-graph sum mode: channel 0 is theta and every aggregate of the mix is a function
# of the network sum.  The others pull through the pointer table: their rows are codes, numerators with a weight or
# per-edge messages, or a mix clips, screens, noises or averages globally per edge or per round
SUM_MODE_ALGS = frozenset({"dinno", "dsgd", "dsgdm", "dsgt", "exact_diffusion", "kgt", "dadaptive", "gt_hsgd"})
# Algorithms that average the whole network every ``period``-th round (Gossip-PGA's global round: pga_sum, pga_mix): they
# own the fp64 partial sums and sum flags on any graph, need NVLS across ranks, plan the edgeless graph with
# ``gossip: false`` and pull Gossip-PGA's bytes
GLOBAL_AVG_ALGS = frozenset({"gossip_pga", "slowmo"})
# Algorithms whose published channel 0 is theta, so the fused consensus metric can read it (not while Byzantine nodes
# publish attack rows there)
THETA_ROW_ALGS = SUM_MODE_ALGS | GLOBAL_AVG_ALGS | {"dp_dsgd", "clipped_gossip", "bridge"}

# Why an algorithm needs the planned graph sequence to be one fixed graph (and the one in ``opt.topo`` when it holds one)
FIXED_GRAPH = {
    "choco_sgd": "s = sum_j W_ij x_hat_j is only valid for a fixed W",
    "beer": BEER_FIXED_W,
    "sparq_sgd": SPARQ_FIXED_W,
    "relaysum": "its messages relay over one fixed tree",
    "powergossip": "both endpoints of an edge carry its power-iteration vectors from round to round",
    "cross_gradient": "its cross-gradients travel back over the edges of one fixed graph",
    "detag": "Chebyshev acceleration has no guarantee on a changing mixing matrix",
}
# Why an algorithm needs undirected planned graphs
UNDIRECTED = {
    "dp_dsgd": "the pairwise noise of an edge cancels between its two ends",
    "sparq_sgd": "its mix conserves the network sum only with symmetric weights",
    "moniqua": "its mix conserves the network sum only with symmetric weights",
}


def check_plan_graphs(opt, topos: List[Topology]) -> None:
    """The planned topologies of a ``FIXED_GRAPH`` algorithm are one, the graph the optimizer was built on when it holds
    one; those of an ``UNDIRECTED`` algorithm are undirected."""
    alg, topo = opt.alg_name, getattr(opt, "topo", None)
    if alg in FIXED_GRAPH and (len(topos) > 1 or (topo is not None and topos[0].key != topo.key)):
        shape = "tree" if alg == "relaysum" else "graph"
        plan = f"has {len(topos)} topologies" if len(topos) > 1 else f"is not the {shape} the optimizer was built on"
        raise ValueError(f"{alg} needs a fixed {shape}: the planned graph sequence of this problem {plan} "
                         f"({FIXED_GRAPH[alg]})")
    if alg in UNDIRECTED and any(t.directed for t in topos):
        raise ValueError(f"{alg} needs undirected graphs: a planned graph is directed ({UNDIRECTED[alg]})")


WAIT_THREADS = 256     # consensus_device.cuh: THREADS


def partials_stride(n_pad: int, itemsize: int) -> int:
    """fp64 partial sums per row of the norm and distance kernels: one per chunk of ``WAIT_THREADS * (16 / itemsize)``
    elements (a 16-byte vector per thread)."""
    return max(1, -(-n_pad // (WAIT_THREADS * (16 // itemsize))))


def check_wait_capacity(dmax: int, rmax: int) -> None:
    """The round-start wait has one thread per in-neighbor (threads ``0..dmax-1`` of a node's CTA) and one per reader
    of the previous round (``32..32+rmax-1``); a node with more would go on without waiting for the last of them."""
    if dmax > WAIT_THREADS or rmax > WAIT_THREADS - 32:
        raise ValueError(f"a node with {dmax} in-neighbors / {rmax} readers exceeds what the consensus kernels wait "
                         f"for ({WAIT_THREADS} in-neighbors, {WAIT_THREADS - 32} readers)")


CLIP_MAX_DEG = 128     # consensus.h: kClipMaxDeg


def check_clip_capacity(dmax: int) -> None:
    """ClippedGossip's ``clip: adaptive`` mix picks the radius from every neighbor's distance in shared memory, for at
    most ``CLIP_MAX_DEG`` neighbors per node."""
    if dmax > CLIP_MAX_DEG:
        raise ValueError(f"clipped_gossip with clip: adaptive handles at most {CLIP_MAX_DEG} neighbors per node on the "
                         f"fused kernels; the planned graphs have a node with {dmax}")


BRIDGE_MAX_DEG = 16     # consensus.h: kBridgeMaxDeg


def check_bridge_capacity(dmax: int) -> None:
    """BRIDGE's mix screens each element over the neighbor values held in registers, for at most ``BRIDGE_MAX_DEG``
    neighbors per node."""
    if dmax > BRIDGE_MAX_DEG:
        raise ValueError(f"bridge handles at most {BRIDGE_MAX_DEG} neighbors per node on the fused kernels; the planned "
                         f"graphs have a node with {dmax}")


TOPK_CLUSTER = 8              # consensus.h: kTopkCluster
TOPK_ROW_SMEM = 220 * 1024    # consensus.h: kTopkRowSmem


def topk_slice(n_pad: int) -> int:
    """Elements of the row one CTA of the top-k step's cluster holds (consensus_device.cuh: topk_slice)."""
    return -(-(-(-n_pad // TOPK_CLUSTER)) // 32) * 32


def topk_max_row(itemsize: int, chans: int) -> int:
    """The longest row the top-k step selects from: its slices of v and live bits fit ``TOPK_ROW_SMEM``."""
    return 8 * TOPK_ROW_SMEM // (8 * chans * itemsize + 1) // 32 * 32 * TOPK_CLUSTER


def check_topk_capacity(alg: str, n_pad: int, itemsize: int, chans: int) -> None:
    """The top-k step keeps ``v`` of its slice of the row (``chans`` channels) and the slice's live bits in the shared
    memory of each CTA of a ``TOPK_CLUSTER``-CTA cluster, at most ``TOPK_ROW_SMEM`` bytes."""
    sl = topk_slice(n_pad)
    need = chans * sl * itemsize + sl // 8          # the slices of v, then the slice's live words
    if need > TOPK_ROW_SMEM:
        raise ValueError(f"{alg} with compressor topk selects in the shared memory of one {TOPK_CLUSTER}-CTA cluster "
                         f"per node: rows of at most {topk_max_row(itemsize, chans)} elements at this dtype (the row "
                         f"has n_pad = {n_pad}, "
                         f"{need} bytes per CTA against a limit of {TOPK_ROW_SMEM})")


RELAY_MAX_DEG = 16     # consensus.h: kRelayMaxDeg


def check_relay_plan(dmax: int) -> None:
    """RelaySum's step holds a node's received messages in registers, for at most ``RELAY_MAX_DEG`` neighbors (its one
    fixed tree is ``check_plan_graphs``'s)."""
    if dmax > RELAY_MAX_DEG:
        raise ValueError(f"relaysum handles at most {RELAY_MAX_DEG} neighbors per node on the fused kernels; the tree "
                         f"has a node with {dmax}")


PG_MAX_DEG = 16     # consensus.h: kPgMaxDeg


def pg_mix_smem(dmax: int, width: int, itemsize: int) -> int:
    """Dynamic shared memory of pg_mix: the message differences of ``dmax`` neighbor slots."""
    return dmax * width * itemsize


def check_powergossip_capacity(dmax: int, width: int, itemsize: int, optin: int) -> None:
    """PowerGossip's mix keeps a node's message differences (``dmax`` slots of ``width`` elements) in the shared memory
    of each of its CTAs, at most ``optin`` bytes (the device's opt-in limit per block), and its per-edge weights for at
    most ``PG_MAX_DEG`` neighbors."""
    if dmax > PG_MAX_DEG:
        raise ValueError(f"powergossip handles at most {PG_MAX_DEG} neighbors per node on the fused kernels; the graph "
                         f"has a node with {dmax}")
    need = pg_mix_smem(dmax, width, itemsize)
    if need > optin:
        raise ValueError(f"powergossip's mix holds {dmax} message differences of {width} elements in shared memory: "
                         f"{need} bytes per CTA against the device's opt-in limit of {optin} (a model with shorter "
                         f"messages, a graph of lower degree or float32 fits)")


class ConsensusEngine:
    def __init__(self, opt, graphs_per_round: List):
        self.opt = opt
        pr = self.pr = opt.pr
        self.ext = load_ext(required=True)
        dev, a, pl, ctx = pr.device, pr.arena, pr.placement, pr.ctx
        self.dtype = a.dtype
        npdt = np.float32 if self.dtype == torch.float32 else np.float64
        alg = opt.alg_name
        # published channels: channel 0, and channel 1 for a second published row (the tracker y of DSGT, Push-DIGing,
        # DeTAG, GT-HSGD and K-GT with correction, dadaptive's u~ with tracking, BEER's g codes).  RelaySum and
        # PowerGossip publish one message per neighbor: channel e of node i is its message for neighbor j_e.
        # Cross-gradient: channel 0 is theta, channel 1 + e the node's gradient at neighbor j_e's row
        if hasattr(opt, "msg"):
            self.C = opt.dmax
        elif alg == "cross_gradient":
            self.C = 1 + opt.dmax
        else:
            self.C = 2 if (alg == "beer" or getattr(opt, "y", None) is not None
                           or getattr(opt, "ut", None) is not None) else 1
        L, n_pad, oits = pl.L, a.n_pad, opt.oits
        itemsize = a.theta.element_size()
        # DeTAG: every gossip sub-step is a protocol round, p = K k + s, so the device round counter, the flags and the
        # sequence tags count K per gradient round and the schedules hold K entries per gradient round.
        # Cross-gradient: gradient round k is protocol rounds 2k (xg_pull .. xg_publish) and 2k + 1 (xg_step)
        K = self.rounds_per_step = opt.gossip_steps if alg == "detag" else 2 if alg == "cross_gradient" else 1
        # Gossip-PGA's and SlowMo's local SGD (gossip: false) plans the edgeless graph
        if alg in GLOBAL_AVG_ALGS and not opt.gossip:
            edgeless = opt.edgeless_graph()
            graphs_per_round = [edgeless] * len(graphs_per_round)
        # SGP and Push-DIGing mix with the column-stochastic push-sum weights and publish the node's weight w
        push_sum = hasattr(opt, "w")

        # ---- published rows (double buffered, peer mapped when multi-GPU) -----
        # CHOCO-SGD, BEER and Moniqua publish code rows of opt.code_bytes bytes (a multiple of 16) instead of parameter
        # rows, SPARQ-SGD code rows followed by their 16-byte trigger tail (opt.row_bytes); SGP and Push-DIGing rows
        # (both channels) are followed by a 16-byte tail holding the float64 push-sum weight w; PowerGossip's message
        # rows are of the layout's message width
        if hasattr(opt, "row_bytes"):
            self.row_bytes = opt.row_bytes
        elif hasattr(opt, "code_bytes"):
            self.row_bytes = opt.code_bytes
        elif push_sum:
            self.row_bytes = n_pad * itemsize + 16
        elif alg == "powergossip":
            self.row_bytes = opt.lay.width * itemsize
        else:
            self.row_bytes = n_pad * itemsize
        Lmax = max(pl.counts)
        self.pub_buf = SymmetricBuffer((2, self.C, Lmax, self.row_bytes // itemsize), self.dtype, ctx)
        self.pub = self.pub_buf.local
        self.Lpub = Lmax
        k0 = opt.k
        p0 = K * k0                 # the protocol round of gradient round k0
        # round k0 (0, or the round a checkpoint resumed at) is "published" in the parity it will be read from
        if alg == "moniqua" and k0 == 0:
            opt.encode_initial()                    # round 0 reads the codes of theta^0
        if alg == "powergossip":
            self.pub.zero_()                        # messages are zero past their length
        for row, src, _ in self.published_rows(k0):
            row.copy_(src)

        # ---- schedules ----------------------------------------------------------
        H = self.horizon = schedule_horizon(opt)
        rho, lr, alpha = (np.repeat(t, K) for t in schedule_tables(opt, H))
        self.rho = torch.as_tensor(rho.astype(npdt), device=dev)
        self.lr = torch.as_tensor(lr.astype(npdt), device=dev)
        self.alpha = torch.as_tensor(alpha.astype(npdt), device=dev)
        # DSGT with a per-coordinate step: the [n_pad] row replaces the alpha_k schedule in dsgt_mix
        self.alpha_row = None
        if alg == "dsgt" and torch.is_tensor(opt.alpha):
            self.alpha_row = opt.alpha.detach().to(device=dev, dtype=self.dtype).reshape(-1).contiguous()
            if self.alpha_row.numel() != n_pad:
                raise ValueError(f"per-coordinate alpha has {self.alpha_row.numel()} entries for rows of {n_pad}")

        # ---- topology tables ------------------------------------------------------
        topos: List[Topology] = []
        key_to_id: Dict[bytes, int] = {}
        gid = np.zeros(H, dtype=np.int32)
        by_object: Dict[int, int] = {}     # a static plan repeats one graph object: build its topology once
        for k, g in enumerate(graphs_per_round):
            gi = by_object.get(id(g))
            if gi is None:
                t = pr._topo_cache.get(g) if hasattr(pr, "_topo_cache") else Topology(g)
                if t.key not in key_to_id:
                    key_to_id[t.key] = len(topos)
                    topos.append(t)
                gi = by_object[id(g)] = key_to_id[t.key]
            gid[k] = gi
        gid = np.repeat(gid, K)
        self.gid = gid
        self.topos = topos
        G = len(topos)
        if getattr(opt, "compressor", None) == "topk":
            check_topk_capacity(alg, n_pad, itemsize, self.C)
        check_plan_graphs(opt, topos)
        dmax = max(1, max(t.max_degree for t in topos))
        if alg == "bridge":
            check_bridge_capacity(dmax)
        if alg == "relaysum":
            check_relay_plan(dmax)
        if alg == "powergossip":
            props = torch.cuda.get_device_properties(dev)
            check_powergossip_capacity(dmax, opt.lay.width, itemsize,
                                       int(getattr(props, "shared_memory_per_block_optin", 227 * 1024)))
        # reader tables (the out-neighbors the round-start wait also covers) only when a planned graph is directed:
        # on undirected graphs the readers are the neighbors and the kernels take them from deg / nbr_rank
        directed = any(t.directed for t in topos)
        rmax = max(1, max(t.max_readers for t in topos))
        check_wait_capacity(dmax, rmax if directed or G > 1 else 0)    # a static undirected graph has no second wait
        nbr_ptr = np.zeros((G, L, dmax, 2, self.C), dtype=np.int64)
        nbr_w = np.zeros((G, L, dmax), dtype=npdt)
        self_w = np.zeros((G, L), dtype=npdt)
        deg = np.zeros((G, L), dtype=np.int32)
        nbr_rank = -np.ones((G, L, dmax), dtype=np.int32)
        rdr_deg = np.zeros((G, L), dtype=np.int32) if directed else None
        rdr_rank = -np.ones((G, L, rmax), dtype=np.int32) if directed else None
        for gi, t in enumerate(topos):
            rslot = t.reverse_slots() if hasattr(opt, "msg") or alg == "cross_gradient" else None
            # Exact Diffusion (and Moniqua on its base) combines with A = (I + W) / 2 through the same mix kernel; SGP
            # and Push-DIGing with the column-stochastic push-sum weights, over the in-neighbors
            if push_sum:
                Wt = t.push_weights
            else:
                ed = alg == "exact_diffusion" or (alg == "moniqua" and opt.base == "exact_diffusion")
                Wt = ed_weights(t.W) if ed else t.W
            for l, g in enumerate(pl.local_nodes):
                nb = t.neighbors_noself[g]
                deg[gi, l] = len(nb)
                self_w[gi, l] = Wt[g, g]
                for e, j in enumerate(nb):
                    r, lj = int(pl.node_rank[j]), int(pl.node_local[j])
                    nbr_w[gi, l, e] = Wt[g, j]
                    if r != ctx.rank:
                        nbr_rank[gi, l, e] = r
                    for par in range(2):
                        if alg == "cross_gradient":     # theta, and channel 1 + e of the edge: j's gradient here
                            for ch, jch in ((0, 0), (1 + e, 1 + rslot[g][e])):
                                row = (par * self.C + jch) * self.Lpub + lj
                                nbr_ptr[gi, l, e, par, ch] = self.pub_buf.peer_ptrs[r] + row * self.row_bytes
                            continue
                        if rslot is not None:   # channel 0 of the edge: j's message for this node (its reverse slot)
                            row = (par * self.C + rslot[g][e]) * self.Lpub + lj
                            nbr_ptr[gi, l, e, par, 0] = self.pub_buf.peer_ptrs[r] + row * self.row_bytes
                            continue
                        for ch in range(self.C):
                            row = (par * self.C + ch) * self.Lpub + lj
                            nbr_ptr[gi, l, e, par, ch] = self.pub_buf.peer_ptrs[r] + row * self.row_bytes
                if directed:
                    rdr_deg[gi, l] = len(t.readers[g])
                    for e, j in enumerate(t.readers[g]):
                        if int(pl.node_rank[j]) != ctx.rank:
                            rdr_rank[gi, l, e] = int(pl.node_rank[j])
        self.dmax = dmax
        self.t_nbr_ptr = torch.as_tensor(nbr_ptr, device=dev)
        self.t_nbr_w = torch.as_tensor(nbr_w, device=dev)
        self.t_self_w = torch.as_tensor(self_w, device=dev)
        self.t_deg = torch.as_tensor(deg, device=dev)
        self.t_nbr_rank = torch.as_tensor(nbr_rank, device=dev)
        self.t_gid = torch.as_tensor(gid, device=dev)
        self.t_rdr_deg = torch.as_tensor(rdr_deg, device=dev) if directed else None
        self.t_rdr_rank = torch.as_tensor(rdr_rank, device=dev) if directed else None

        # ---- optional protocol self-check (SURVEY 5.2): published rows carry their round, neighbor reads verify it ----
        self.seq_buf = None
        self.t_nbr_seq = None
        if opt.conf.get("debug_sequence_check", False) or os.environ.get("NNDT_SEQ_CHECK") == "1":
            self.seq_buf = SymmetricBuffer((2, Lmax), torch.int32, ctx)
            self.seq_buf.local.fill_(p0 - 1)
            self.seq_buf.local[p0 & 1].fill_(p0)
            nbr_seq = np.zeros((G, L, dmax, 2), dtype=np.int64)
            for gi, t in enumerate(topos):
                for l, g in enumerate(pl.local_nodes):
                    for e, j in enumerate(t.neighbors_noself[g]):
                        r, lj = int(pl.node_rank[j]), int(pl.node_local[j])
                        for par in range(2):
                            nbr_seq[gi, l, e, par] = self.seq_buf.peer_ptrs[r] + (par * Lmax + lj) * 4
            self.t_nbr_seq = torch.as_tensor(nbr_seq, device=dev)

        # ---- counters / flags -----------------------------------------------------
        self.round_ctr = torch.full((1,), p0, dtype=torch.int32, device=dev)
        self.done_ctr = torch.zeros(1, dtype=torch.int32, device=dev)
        self.err = torch.zeros(1, dtype=torch.int32, device=dev)
        self.flag_buf = SymmetricBuffer((max(ctx.world_size, 1),), torch.int32, ctx)
        self.flag_buf.local.fill_(p0)
        peer_flag = np.zeros(max(ctx.world_size, 1), dtype=np.int64)
        for r in range(ctx.world_size):
            peer_flag[r] = self.flag_buf.peer_ptrs[r] + 4 * ctx.rank
        self.t_peer_flag = torch.as_tensor(peer_flag, device=dev)
        # a producer stores "round k published" into each reader's local flag slot; readers spin on local memory
        self.flag_mode = "push"
        # ranks that own a neighbor of a local node in ANY round's graph: the only ones that need this rank's flags
        notify = 0
        remote_node = np.zeros(L, dtype=bool)
        # (directed graphs: the in-neighbors wait for this rank as one of their readers, the readers as an in-neighbor)
        peers = np.concatenate([nbr_rank.ravel(), rdr_rank.ravel()]) if directed else nbr_rank
        for r in np.unique(peers[peers >= 0]):
            notify |= 1 << int(r)
        for l in range(L):
            remote_node[l] = bool((nbr_rank[:, l, :] >= 0).any())
        self.notify_mask = notify
        # launch order of the local nodes: the ones pulling over NVLink first (their CTAs become resident while the
        # preceding forward/backward kernel still runs, which hides the link latency)
        order = np.argsort(~remote_node, kind="stable").astype(np.int32)
        self.t_node_order = torch.as_tensor(order, device=dev)
        if ctx.is_distributed:
            torch.cuda.synchronize(dev)
            ctx.barrier()

        # ---- complete graph: uniform Metropolis weights -> aggregates are functions of the network sum ----
        # (the algorithms outside SUM_MODE_ALGS always pull through the pointer table; complete_graph_mode is ignored.
        # the global rounds of GLOBAL_AVG_ALGS average through the same fp64 partial sums, with sum_mode 0)
        self.sum_mode = (G == 1 and topos[0].is_complete() and pr.N > 1 and alg in SUM_MODE_ALGS
                         and opt.conf.get("complete_graph_mode", "sum") == "sum")
        self.sum_buf = self.sum_flag_buf = None
        sum_mc = None
        if self.sum_mode or alg in GLOBAL_AVG_ALGS:
            self.sum_buf = SymmetricBuffer((2, self.C, n_pad), torch.float64, ctx)   # fp64: S - N*theta cancels in fp32
            self.sum_flag_buf = SymmetricBuffer((max(ctx.world_size, 1),), torch.int32, ctx)
            self.sum_flag_buf.local.fill_(k0)
            if ctx.is_distributed:
                if self.sum_buf.multicast_ptr:
                    sum_mc = self.sum_buf.multicast_ptr      # NVLS: one in-switch reduction per element
                elif alg in GLOBAL_AVG_ALGS:
                    raise ValueError(f"{alg} on more than one rank averages over NVLS (one in-switch reduction of "
                                     f"the fp64 partial sums per global round), and this fabric gives its symmetric "
                                     f"buffer no multicast mapping")
                else:
                    self.sum_mode = False                    # no multicast mapping on this fabric: pointer table
                torch.cuda.synchronize(dev)
                ctx.barrier()
        peer_sum_flag = np.zeros(max(ctx.world_size, 1), dtype=np.int64)
        if self.sum_mode or alg in GLOBAL_AVG_ALGS:
            for r in range(ctx.world_size):
                peer_sum_flag[r] = self.sum_flag_buf.peer_ptrs[r] + 4 * ctx.rank
        self.t_peer_sum_flag = torch.as_tensor(peer_sum_flag, device=dev)

        # ---- gradient source --------------------------------------------------------
        if pr.fused is not None:
            grad_part, S, calls = pr.fused.grad_part, pr.fused.S, pr.fused.calls
            if getattr(pr.fused, "owns_calls", False):
                calls = None       # the forward/backward kernel advances its own draw counters
        else:
            grad_part, S, calls = a.grad, 1, None
        self.S = S

        d = dict(L=L, n_pad=n_pad, S=S, theta=a.theta.data_ptr(), grad_part=grad_part.data_ptr(),
                 pub=self.pub.data_ptr(), C=self.C, nbr_ptr=self.t_nbr_ptr.data_ptr(),
                 nbr_w=self.t_nbr_w.data_ptr(), self_w=self.t_self_w.data_ptr(), deg=self.t_deg.data_ptr(),
                 nbr_rank=self.t_nbr_rank.data_ptr(), dmax=dmax, round_ctr=self.round_ctr.data_ptr(),
                 rho=self.rho.data_ptr(), lr=self.lr.data_ptr(), alpha=self.alpha.data_ptr(),
                 graph_id=self.t_gid.data_ptr(), calls=None if calls is None else calls.data_ptr(),
                 flags=self.flag_buf.local.data_ptr(), peer_flag=self.t_peer_flag.data_ptr(),
                 world=ctx.world_size, rank=ctx.rank, done_ctr=self.done_ctr.data_ptr(), err=self.err.data_ptr(),
                 notify_mask=int(self.notify_mask) if ctx.world_size > 1 else 0,
                 node_order=self.t_node_order.data_ptr() if ctx.world_size > 1 else None)
        self.timeline = None
        if os.environ.get("NNDT_TIMELINE") == "1":       # debug: %globaltimer stamps of the update kernels (scripts/timeline_rounds.py)
            self.timeline = torch.zeros(4096, 16, dtype=torch.int64, device=dev)
            d["timeline"] = self.timeline.data_ptr()
        # the C++ side indexes pub rows with stride L; when ranks host different node counts the
        # published buffer is allocated with the max count, so pass that as the row count of pub
        d["pub_L"] = self.Lpub
        if pr.fused is not None and getattr(pr, "track_tloss", False) and self.dtype == torch.float32:
            # the kernel that consumes a gradient also folds that step's loss into the EMA tracker
            d.update(loss_part=pr.fused.loss_part.data_ptr(), tloss=pr.tloss_local.data_ptr(),
                     tdecay=float(pr.tloss_decay), loss_S=int(pr.fused.loss_part.shape[1]))
            pr.fused.ema_in_kernel = True
        if directed:
            d.update(rdr_deg=self.t_rdr_deg.data_ptr(), rdr_rank=self.t_rdr_rank.data_ptr(), rmax=rmax)
        if self.seq_buf is not None:
            d.update(pub_seq=self.seq_buf.local.data_ptr(), nbr_seq=self.t_nbr_seq.data_ptr())
        if self.sum_mode:
            d.update(sum_mode=1, n_total=pr.N, sum_local=self.sum_buf.local.data_ptr(), sum_mc=sum_mc,
                     sum_flags=self.sum_flag_buf.local.data_ptr(), peer_sum_flag=self.t_peer_sum_flag.data_ptr())
        if alg in GLOBAL_AVG_ALGS:
            d.update(n_total=pr.N, sum_local=self.sum_buf.local.data_ptr(), sum_mc=sum_mc,
                     sum_flags=self.sum_flag_buf.local.data_ptr(), peer_sum_flag=self.t_peer_sum_flag.data_ptr(),
                     period=opt.period, gossip=int(opt.gossip))
        if alg == "slowmo":
            # the outer update's rows, and the base momentum row with its local-mode dsgdm_step arguments
            d.update(anchor=opt.anchor.data_ptr(), slow_u=opt.u.data_ptr(), alpha0=opt.alph0, slow_lr=opt.slow_lr,
                     slow_momentum=opt.slow_momentum, m=None if opt.m is None else opt.m.data_ptr(),
                     beta=opt.base_momentum, quasi_global=0, nesterov=int(opt.nesterov))
        if alg == "dinno":
            d.update(dual=opt.duals.data_ptr(), delta=opt.delta.data_ptr(),
                     m=None if opt.m is None else opt.m.data_ptr(),
                     v=None if opt.v is None else opt.v.data_ptr(),
                     pits=opt.pits, opt=OPT_CODE[opt.opt_kind], persistent=int(opt.persistent))
        if alg == "dsgt":
            d.update(g_old=opt.g.data_ptr(), own_tracker=int(bool(getattr(opt, "own_tracker_step", False))),
                     alpha_row=None if self.alpha_row is None else self.alpha_row.data_ptr())
        if alg == "gt_hsgd":
            # the prev-point partials: the fused problem's second op, or (autograd gradients) the optimizer's grad_prev,
            # one row per node as a.grad
            gpp = pr.fused.grad_part_prev if pr.fused is not None else opt.grad_prev
            d.update(grad_part_prev=gpp.data_ptr(), hsgd_v=opt.v.data_ptr(), theta_prev=opt.theta_prev.data_ptr(),
                     omb=opt.omb)
        self.xmix = self.xg_g = self.t_xg_coef0 = self.t_xg_coef = None
        if alg == "cross_gradient":
            # the round's mixed row and own gradient (dead between rounds); the cross partials: the fused problem's extra
            # ops, or (autograd gradients) the optimizer's grad_x, one row per node and slot; the float64 weights of d
            gx = pr.fused.grad_part_x if pr.fused is not None else opt.grad_x
            self.xmix = torch.zeros(L, n_pad, dtype=self.dtype, device=dev)
            self.xg_g = torch.zeros(L, n_pad, dtype=self.dtype, device=dev)
            self.t_xg_coef0 = opt.coef0.reshape(1, L).contiguous()
            self.t_xg_coef = opt.coef.reshape(1, L, dmax).contiguous()
            d.update(xmix=self.xmix.data_ptr(), theta_x=opt.theta_x.data_ptr(), grad_part_x=gx.data_ptr(),
                     xg_g=self.xg_g.data_ptr(), xg_coef0=self.t_xg_coef0.data_ptr(), xg_coef=self.t_xg_coef.data_ptr())
        if alg == "exact_diffusion":
            d.update(psi=opt.psi.data_ptr())
        if alg == "kgt":
            d.update(local_steps=opt.local_steps, correction=int(opt.correction),
                     corr=opt.c.data_ptr() if opt.correction else None,
                     dacc=opt.d.data_ptr() if opt.correction else None)
        self.omega = self.ymix = None
        if alg == "detag":
            # the sub-step weights in the arena dtype, and Y_K of the last sub-step (dead between rounds)
            self.omega = torch.as_tensor(np.asarray(opt.omega, dtype=npdt), device=dev)
            self.ymix = torch.zeros(L, n_pad, dtype=self.dtype, device=dev)
            d.update(omega=self.omega.data_ptr(), ymix=self.ymix.data_ptr(), g_old=opt.g_old.data_ptr(),
                     gossip_steps=K)
        if alg == "dadaptive":
            d.update(ad_m=opt.m.data_ptr(), ad_v=None if opt.v is None else opt.v.data_ptr(),
                     vhat=opt.vhat.data_ptr(), ut=opt.ut.data_ptr() if opt.tracking else None, beta1=opt.beta1,
                     beta2=opt.beta2, ad_eps=opt.eps, adagrad=int(opt.adagrad), tracking=int(opt.tracking))
        self.t_live = None
        self.dist_part = self.t_attack = self.t_nbr_byz = None
        if hasattr(opt, "byzantine"):     # ClippedGossip, BRIDGE: BRIDGE's step is cg_step, with the same attack tables
            if alg == "clipped_gossip":
                if opt.clip == "adaptive":
                    check_clip_capacity(dmax)
                # fp64 partials of the squared neighbor distances: one per chunk of THREADS * (16 / itemsize) elements
                pstride = partials_stride(n_pad, itemsize)
                self.dist_part = torch.zeros(L * dmax * pstride, dtype=torch.float64, device=dev)
                d.update(dist_part=self.dist_part.data_ptr(), pstride=pstride,
                         clip_adaptive=int(opt.clip == "adaptive"), clip_delta=float(opt.delta))
            else:
                d.update(screen_b=opt.b, screen_median=int(opt.screen == "median"))
            byz = set(opt.byzantine)
            nbr_byz = np.zeros((G, L, dmax), dtype=np.int32)
            for gi, t in enumerate(topos):
                for l, g in enumerate(pl.local_nodes):
                    for e, j in enumerate(t.neighbors_noself[g]):
                        nbr_byz[gi, l, e] = int(j in byz)
            self.t_nbr_byz = torch.as_tensor(nbr_byz, device=dev)
            if any(opt.attack):
                self.t_attack = torch.as_tensor(np.asarray(opt.attack, dtype=np.int32), device=dev)
            d.update(attack_scale=float(opt.scale), attack_z=float(opt.z),
                     attack=None if self.t_attack is None else self.t_attack.data_ptr(),
                     nbr_byz=self.t_nbr_byz.data_ptr())
        self.t_reach = self.rin = None
        if alg == "relaysum":
            # R_i^k - 1 of the local nodes for k = 0 .. diam (exact in either dtype), and the received messages of the
            # round, written by relay_mix and read by relay_step
            self.t_reach = torch.as_tensor(
                (opt.reach[pl.lo: pl.lo + L] - 1).astype(npdt), device=dev).contiguous()
            self.rin = torch.zeros(L, dmax, n_pad, dtype=self.dtype, device=dev)
            d.update(reach=self.t_reach.data_ptr(), rin=self.rin.data_ptr(), diam=opt.diam, relay_n=pr.N)
        self.t_pg_seg = None
        if alg == "powergossip":
            # the segment table {offset, m, n, poff, qoff} and the edge signs; the vectors are the optimizer's own rows,
            # updated in place by pg_mix
            lay = opt.lay
            self.t_pg_seg = torch.as_tensor(np.asarray(lay.segs, dtype=np.int32).reshape(-1, 5), device=dev)
            d.update(pg_vec=opt.vec.data_ptr() if opt.vec.numel() else None, pg_seg=self.t_pg_seg.data_ptr(),
                     pg_sign=opt.sign.data_ptr(), pg_nseg=len(lay.segs), pg_P=lay.P, pg_Q=lay.Q, pg_B=lay.B,
                     pg_W=lay.width, gamma=float(opt.gamma), pg_grid=int(getattr(opt, "pg_grid", 0)))
        # DP-DSGD: ``dp`` is the privacy ledger of the fused path, the zCDP cost of one round on each planned graph
        # (None for the other algorithms)
        self.norm_part = self.t_nbr_id = self.dp = None
        if alg == "dp_dsgd":
            # fp64 partials of sum g^2, one per chunk of THREADS * (16 / itemsize) elements (cg_dist's chunks); the
            # global id of every neighbor slot (the edge streams); the live mask (no noise on padding and slot holes)
            pstride = partials_stride(n_pad, itemsize)
            self.norm_part = torch.zeros(L * pstride, dtype=torch.float64, device=dev)
            nbr_id = np.zeros((G, L, dmax), dtype=np.int32)
            for gi, t in enumerate(topos):
                for l, g in enumerate(pl.local_nodes):
                    for e, j in enumerate(t.neighbors_noself[g]):
                        nbr_id[gi, l, e] = j
            self.t_nbr_id = torch.as_tensor(nbr_id, device=dev)
            live = choco_live(a.layout)
            live = torch.cat([live, live.new_zeros(-n_pad % 32)])      # whole words: a row may be shorter than 32
            self.t_live = choco_live_words(live).to(dev)
            self.dp = [opt.round_rho(t) for t in topos]
            d.update(norm_part=self.norm_part.data_ptr(), pstride=pstride, nbr_id=self.t_nbr_id.data_ptr(),
                     live=self.t_live.data_ptr(), node0=int(pl.lo), clip_norm=float(opt.clip), cz_dp=float(opt.cz_dp),
                     cz_pair=float(opt.cz_pair), dp_key0=int(opt.key[0]), dp_key1=int(opt.key[1]))
        if alg == "dsgdm":
            d.update(m=opt.m.data_ptr(), x_prev=None if opt.x_prev is None else opt.x_prev.data_ptr(), beta=opt.beta,
                     quasi_global=int(opt.quasi_global), nesterov=int(opt.nesterov))
        if alg == "choco_sgd":
            self.t_live = choco_live_words(opt.live).to(dev)
            d.update(x_hat=opt.x_hat.data_ptr(), s=opt.s.data_ptr(), live=self.t_live.data_ptr(), gamma=float(opt.gamma),
                     code=CHOCO_CODE[opt.compressor], code_stride=int(self.row_bytes), topk_k=int(opt.topk_k or 0))
        if alg == "beer":
            self.t_live = choco_live_words(opt.live).to(dev)
            d.update(h=opt.h.data_ptr(), s_h=opt.s_h.data_ptr(), v=opt.v.data_ptr(), g=opt.g.data_ptr(),
                     s_g=opt.s_g.data_ptr(), m_old=opt.m_old.data_ptr(), live=self.t_live.data_ptr(),
                     gamma=float(opt.gamma), code=CHOCO_CODE[opt.compressor], code_stride=int(self.row_bytes),
                     topk_k=int(opt.topk_k or 0))
        # Moniqua: ``mq`` holds the kernels' arguments of the modulo code the published rows carry (range, bit width,
        # rounding keys, margin counters, code row stride; None for the other algorithms)
        self.mq = None
        if alg == "moniqua":
            self.t_live = choco_live_words(opt.live).to(dev)
            self.mq = dict(mq_B=float(opt.B), mq_bits=int(opt.bits), mq_key0=int(opt.key[0]), mq_key1=int(opt.key[1]),
                           mq_margin=opt.margin.data_ptr(), code_stride=int(self.row_bytes))
            d.update(self.mq, psi=None if opt.psi is None else opt.psi.data_ptr(), live=self.t_live.data_ptr(),
                     node0=int(pl.lo))
        self.sparq_thr = None
        if alg == "sparq_sgd":
            # the trigger thresholds (float64 in either dtype), fp64 partials of sum (theta - x_hat)^2 per chunk of
            # THREADS * (16 / itemsize) elements (dp_norm's chunks) and the optimizer's trigger counters
            self.t_live = choco_live_words(opt.live).to(dev)
            self.sparq_thr = torch.as_tensor(opt.threshold_table(H), dtype=torch.float64, device=dev)
            pstride = partials_stride(n_pad, itemsize)
            self.norm_part = torch.zeros(L * pstride, dtype=torch.float64, device=dev)
            d.update(x_hat=opt.x_hat.data_ptr(), s=opt.s.data_ptr(), live=self.t_live.data_ptr(), gamma=float(opt.gamma),
                     code=CHOCO_CODE[opt.compressor], sparq_code_bytes=int(opt.code_bytes),
                     row_stride=int(self.row_bytes), sparq_thr=self.sparq_thr.data_ptr(),
                     norm_part=self.norm_part.data_ptr(), pstride=pstride, sparq_triggers=opt.triggers.data_ptr(),
                     local_steps=int(opt.local_steps))
        if alg == "sgp":
            d.update(x=opt.x.data_ptr(), w=opt.w.data_ptr(), row_stride=int(self.row_bytes))
        if alg == "push_diging":
            d.update(u=opt.u.data_ptr(), w=opt.w.data_ptr(), ysum=opt.ysum.data_ptr(), g_old=opt.g.data_ptr(),
                     row_stride=int(self.row_bytes))
        cls = self.ext.ConsensusOpF32 if self.dtype == torch.float32 else self.ext.ConsensusOpF64
        self.op = cls(d)
        self._keep = d

    def pub_weights(self, par: int) -> torch.Tensor:
        """SGP, Push-DIGing: the float64 push-sum weights in the tails of this rank's published rows of parity ``par``
        (channel 0; a view)."""
        tail = self.pr.arena.n_pad * self.pub.element_size()
        rows = self.pub[par, 0, :self.pr.placement.L].view(torch.uint8)
        return rows[:, tail: tail + 8].view(torch.float64)[:, 0]

    def published_rows(self, k: int):
        """The rows published for round ``k`` that hold optimizer state, as ``(view into pub, optimizer tensor, only)``.
        ``only`` marks a published copy that is the only live one: the kernels update it and not the tensor, so
        ``RoundProgram.sync_back`` copies it back.  ``__init__`` publishes round ``k0`` by copying every tensor in."""
        opt, alg, n_pad = self.opt, self.opt.alg_name, self.pr.arena.n_pad
        par = (self.rounds_per_step * k) & 1        # DeTAG, cross-gradient: the parity of protocol round K k
        pub = self.pub[par, :, :self.pr.placement.L]
        if alg == "beer":
            return [(pub[0].view(torch.uint8), opt.code_h, True), (pub[1].view(torch.uint8), opt.code_g, True)]
        if hasattr(opt, "code"):       # CHOCO-SGD, Moniqua, SPARQ-SGD
            return [(pub[0].view(torch.uint8), opt.code, True)]
        if alg == "sgp":               # the numerators x, and w in the row tail
            return [(pub[0, :, :n_pad], opt.x, False), (self.pub_weights(par), opt.w, False)]
        if alg == "push_diging":       # u with w in its row tail, and y in channel 1
            return [(pub[0, :, :n_pad], opt.u, False), (self.pub_weights(par), opt.w, False),
                    (pub[1, :, :n_pad], opt.y, True)]
        if hasattr(opt, "msg"):        # RelaySum, PowerGossip: the messages, published at the end of round k - 1
            return [(pub.transpose(0, 1), opt.msg, True)]
        if alg == "detag":             # z = theta - alpha y and y
            return [(pub[0], opt.z, True), (pub[1], opt.y, True)]
        if hasattr(opt, "pub"):        # ClippedGossip, BRIDGE: an attacker's published row is not its theta
            return [(pub[0], opt.pub, True)]
        rows = [(pub[0], self.pr.arena.theta, False)]
        if getattr(opt, "y", None) is not None and (alg != "dsgt" or opt._initialised):
            rows.append((pub[1], opt.y, True))        # DSGT once initialised, K-GT with correction, GT-HSGD
        if getattr(opt, "ut", None) is not None:
            rows.append((pub[1], opt.ut, True))       # dadaptive with tracking (its ut row holds the mix's z)
        return rows

    def bytes_per_round(self) -> Dict[str, int]:
        """Bytes one node publishes per round (``row``: one published row) and bytes this rank's nodes pull from their
        neighbors per round (``pulled``: one published row per neighbor edge of the first graph; the own row is not
        counted).  An SGP or Push-DIGing row includes its 16-byte tail.  A K-GT round takes ``local_steps`` gradient
        steps.  dadaptive with tracking publishes two rows (theta and u~), without it one.  ClippedGossip with ``clip: adaptive`` reads every neighbor row twice, once for the distances and once
        for the mix (``clip: none`` once, as DSGD; an ALIE attacker also reads its honest neighbors' rows, not
        counted); BRIDGE reads each neighbor row once, as DSGD.  A PowerGossip node pulls one message per neighbor, of
        ``sum m + biases`` (phase 0) or ``sum n + biases`` (phase 1) elements (unpadded): ``pulled_phase0`` and
        ``pulled_phase1`` report both, ``pulled`` their mean, and ``row`` is the padded message row.  A RelaySum node publishes one message row per neighbor (``row`` counts one) and pulls the one its
        neighbor wrote for it: the pulled bytes are DSGD's.  A DeTAG round gossips ``gossip_steps`` times, each a DSGT
        pull: ``pulled`` counts them all.  A GT-HSGD round exchanges what a DSGT round does.  A Gossip-PGA gossip round
        pulls what a DSGD round does (nothing with ``gossip: false``: the edgeless graph); a global round pulls no row
        and contributes one fp64 partial-sum row per rank (``global_row``, ``n_pad * 8`` bytes) to the NVLS
        reduction, once every ``period`` rounds; SlowMo's outer update adds no traffic, so it pulls Gossip-PGA's
        bytes.  A DP-DSGD round pulls what a DSGD round does: the edge noise is drawn on both ends, and the norm partials stay on the node.  A Moniqua row is the node's code row,
        ``n_pad * bits / 8`` bytes, one per neighbor edge as DSGD's rows; the margin counters stay on the node.  A
        SPARQ-SGD row is the code row and its 16-byte tail (``row``); every neighbor edge pulls the tail each round
        (``tail``) and the code body only when its source triggered: ``pulled_max`` is the round where every neighbor
        triggered, and ``pulled_bytes()`` gives what the mixes actually pulled.  A cross-gradient node pulls each
        neighbor's theta row (``pulled_theta``) and the gradient that neighbor took at its own row (``pulled_cross``), one
        row each per neighbor edge; ``pulled`` is both.  ``grad_evals()`` gives the round's gradient evaluations."""
        deg = int(self.t_deg[0].sum().item())
        alg = self.opt.alg_name
        if alg == "cross_gradient":
            return {"row": int(self.row_bytes), "pulled": 2 * int(self.row_bytes) * deg,
                    "pulled_theta": int(self.row_bytes) * deg, "pulled_cross": int(self.row_bytes) * deg}
        if alg == "sparq_sgd":
            return {"row": int(self.row_bytes), "tail": 16, "pulled_max": int(self.row_bytes) * deg}
        if alg in GLOBAL_AVG_ALGS:
            return {"row": int(self.row_bytes), "pulled": int(self.row_bytes) * deg,
                    "global_row": int(self.pr.arena.n_pad) * 8, "period": int(self.opt.period)}
        if alg == "powergossip":
            lay, itemsize = self.opt.lay, self.pub.element_size()
            p0, p1 = (deg * lay.msg_len(ph) * itemsize for ph in (0, 1))
            return {"row": int(self.row_bytes), "pulled": (p0 + p1) // 2, "pulled_phase0": p0, "pulled_phase1": p1}
        reads = 2 if alg == "clipped_gossip" and self.opt.clip == "adaptive" else 1
        chans = 1 if alg == "relaysum" else self.C
        return {"row": int(self.row_bytes) * chans,
                "pulled": int(self.row_bytes) * chans * deg * reads * self.rounds_per_step}

    def grad_evals(self) -> Dict[str, int]:
        """Forward/backward passes per round over the network: ``useful`` counts the own gradients and one per directed
        edge, ``N + 2|E|``; ``launched`` also the idle slots of nodes below the largest degree, ``N (1 + dmax)``.  Every
        other optimizer evaluates ``draws_per_round`` gradients per node."""
        if self.opt.alg_name == "cross_gradient":
            useful, launched = self.opt.grad_evals()
            return {"useful": useful, "launched": launched}
        from .round_program import draws_per_round
        n = self.pr.N * draws_per_round(self.opt)
        return {"useful": n, "launched": n}

    def pulled_bytes(self) -> int:
        """SPARQ-SGD: the bytes the mixes of the rounds run so far pulled over the whole network, exact, from the
        trigger counters and the fixed degrees (optimizers/sparq.py: pulled_bytes)."""
        return self.opt.pulled_bytes()

    def consensus_metric(self, k: int):
        """Fused consensus-error metric (csrc/consensus.cu: consensus_metric_kernel) on the rows published
        for round ``k``: every rank pulls all N rows (local or NVLink peer) and produces the distance rows of
        its own nodes; returns (pairwise [N, N], to-mean [N, 1]) gathered over ranks, as float64 CPU tensors."""
        pr, pl, ctx, dev = self.pr, self.pr.placement, self.pr.ctx, self.pr.device
        N, L, n_pad = pr.N, pl.L, self.pr.arena.n_pad
        par = k & 1
        itemsize = self.pub.element_size()
        rows = np.zeros(N, dtype=np.int64)
        for g in range(N):
            r, lj = int(pl.node_rank[g]), int(pl.node_local[g])
            rows[g] = self.pub_buf.peer_ptrs[r] + ((par * self.C) * self.Lpub + lj) * n_pad * itemsize
        t_rows = torch.as_tensor(rows, device=dev)
        inv = torch.empty(N, dtype=torch.float64, device=dev)
        pair = torch.empty(L, N, dtype=torch.float64, device=dev)
        mean = torch.empty(L, dtype=torch.float64, device=dev)
        if ctx.is_distributed:
            torch.cuda.synchronize(dev)
            ctx.barrier()              # every rank's rows of round k are published and quiescent
        self.ext.consensus_metric(self.dtype == torch.float64, t_rows.data_ptr(), N, n_pad, pl.lo, L,
                                  inv.data_ptr(), pair.data_ptr(), mean.data_ptr())
        d_all = pr.gather_rows(pair).cpu()
        d_mean = pr.gather_rows(mean.reshape(-1, 1)).cpu()
        if ctx.is_distributed:
            ctx.barrier()              # nobody starts overwriting published rows while a peer still reads
        return d_all, d_mean

    def check(self):
        e = int(self.err.item())
        if e == 2:
            raise RuntimeError("sequence check failed: a neighbor row was read that is not tagged with the current round")
        if e != 0:
            raise RuntimeError("consensus kernel timed out waiting for a peer's published round")
