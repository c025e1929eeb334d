"""The checkpoint state of every consensus optimizer: the key set and value kinds of ``state_dict()`` after two rounds,
and a save -> fresh optimizer -> load -> save round trip that reproduces every value exactly (tensors bit for bit,
scalars with their Python type)."""
import copy

import networkx as nx
import pytest
import torch

from nn_distributed_training_b200.data.mnist import synthetic_mnist
from nn_distributed_training_b200.models import MNISTConvNet
from nn_distributed_training_b200.optimizers import build_optimizer
from nn_distributed_training_b200.problems.dist_mnist_problem import DistMNISTProblem
from nn_distributed_training_b200.utils.graph_generation import generate_from_conf

T, NONE = "tensor", "none"
BASE = {"k": int, "theta": T}
DINNO = {"alg_name": "dinno", "rho_init": 0.5, "rho_scaling": 1.01, "primal_iterations": 2,
         "persistant_primal_opt": False, "primal_lr_start": 0.005, "primal_lr_finish": 0.0005, "lr_decay_type": "log"}
DSGDM = {"alg_name": "dsgdm", "alpha0": 0.05, "mu": 0.01, "beta": 0.9, "nesterov": True}
KGT = {"alg_name": "kgt", "alpha": 0.02, "local_steps": 2}
BYZANTINE = {"nodes": [0], "attack": "alie", "scale": 2.0, "z": 1.0}

# name: (optimizer config, directed graph, per-coordinate DSGT step, the expected kinds beyond k and theta)
CASES = {
    "dinno-adam": (dict(DINNO, primal_optimizer="adam"), False, False,
                   {"rho": float, "t": int, "duals": T, "m": T, "v": T}),
    "dinno-sgd": (dict(DINNO, primal_optimizer="sgd"), False, False,
                  {"rho": float, "t": int, "duals": T, "m": NONE, "v": NONE}),
    "dsgd": ({"alg_name": "dsgd", "alpha0": 0.05, "mu": 0.01}, False, False, {"alph": float}),
    "dsgdm-local": (dict(DSGDM, momentum="local"), False, False, {"alph": float, "m": T}),
    "dsgdm-quasi_global": (dict(DSGDM, momentum="quasi_global"), False, False, {"alph": float, "m": T, "x_prev": T}),
    "dsgt-scalar": ({"alg_name": "dsgt", "alpha": 0.02, "init_grads": True}, False, False,
                    {"initialised": bool, "alpha": float, "y": T, "g": T}),
    "dsgt-per_coordinate": ({"alg_name": "dsgt", "alpha": 0.02, "init_grads": True}, False, True,
                            {"initialised": bool, "alpha": T, "y": T, "g": T}),
    "exact_diffusion": ({"alg_name": "exact_diffusion", "alpha0": 0.05, "mu": 0.01}, False, False,
                        {"alph": float, "psi": T}),
    "choco_sgd-int8": ({"alg_name": "choco_sgd", "alpha0": 0.05, "mu": 0.01, "gamma": 0.5, "compressor": "int8"},
                       False, False, {"alph": float, "x_hat": T, "s": T, "code": T}),
    "beer-int8": ({"alg_name": "beer", "alpha": 0.05, "gamma": 0.5, "compressor": "int8"}, False, False,
                  {n: T for n in ("h", "s_h", "v", "g", "s_g", "m_old", "code_h", "code_g")}),
    "sgp-directed": ({"alg_name": "sgp", "alpha0": 0.05, "mu": 0.01}, True, False, {"alph": float, "x": T, "w": T}),
    "push_diging-directed": ({"alg_name": "push_diging", "alpha": 0.05}, True, False,
                             {"u": T, "w": T, "y": T, "g": T}),
    "kgt-correction": (dict(KGT, correction=True), False, False, {"c": T, "y": T}),
    "kgt-local_dsgd": (dict(KGT, correction=False), False, False, {}),
    "clipped_gossip-alie": ({"alg_name": "clipped_gossip", "alpha0": 0.02, "mu": 0.001, "clip": "adaptive",
                             "delta": 0.3, "byzantine": BYZANTINE}, False, False, {"alph": float, "pub": T}),
}


def _kind(v):
    return T if torch.is_tensor(v) else NONE if v is None else type(v)


def _optimizer(conf, directed, per_coordinate, N=4, M=64):
    conf = dict(copy.deepcopy(conf), outer_iterations=4, profile=False)
    graph = generate_from_conf({"type": "directed_cycle", "num_nodes": N})[1] if directed else nx.wheel_graph(N)
    torch.manual_seed(0)
    data = synthetic_mnist(M * N, seed=3)
    shards = [data.select(torch.arange(i * M, (i + 1) * M)) for i in range(N)]
    pconf = {"problem_name": "t", "train_batch_size": 16, "val_batch_size": 32, "metrics": ["forward_pass_count"],
             "metrics_config": {"evaluate_frequency": 1000}, "optimizer_config": conf}
    pr = DistMNISTProblem(graph, MNISTConvNet(3, 5, 64), torch.nn.NLLLoss(), shards, synthetic_mnist(32, seed=4), "cpu",
                          pconf, backend="torch", seed=7)
    opt = build_optimizer(pr, "cpu", conf)
    if per_coordinate:
        a = opt.arena
        opt.alpha = torch.linspace(0.01, 0.03, a.n_pad, dtype=a.dtype)
    return opt


@pytest.mark.parametrize("case", list(CASES))
def test_state_dict_keys_kinds_and_round_trip(case):
    conf, directed, per_coordinate, kinds = CASES[case]
    opt = _optimizer(conf, directed, per_coordinate)
    opt.run_rounds(2)
    sd = opt.state_dict()
    assert {k: _kind(v) for k, v in sd.items()} == dict(BASE, **kinds)
    assert sd["k"] == 2

    fresh = _optimizer(conf, directed, False)
    fresh.load_state_dict(copy.deepcopy(sd))
    back = fresh.state_dict()
    assert back.keys() == sd.keys()
    for k, v in sd.items():
        if torch.is_tensor(v):
            assert torch.is_tensor(back[k]) and back[k].dtype == v.dtype and torch.equal(back[k], v), k
        else:
            assert type(back[k]) is type(v) and back[k] == v, k
