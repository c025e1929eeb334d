"""Distributed MNIST experiment runner (reference: experiments/dist_mnist_ex.py).

    python -m nn_distributed_training_b200.experiments.dist_mnist_ex <config.yaml>
    torchrun --nproc-per-node 8 -m nn_distributed_training_b200.experiments.dist_mnist_ex <config.yaml>
"""
from __future__ import annotations

import copy
import os
import sys

import torch

from . import common
from ..data.mnist import load_mnist
from ..models import MNISTConvNet
from ..ops import local_train
from ..problems import DistMNISTProblem
from ..utils import graph_generation
from ..utils.config import load_experiment


def train_solo(model, loss, train_set, val_set, device, conf):
    """No-communication baseline: one node trains alone (reference :22-62)."""
    model = model.to(device)
    opt = common.make_solo_optimizer(model, conf)
    dtype = next(model.parameters()).dtype
    train, val = train_set.to(device), val_set.to(device)
    n, bs = len(train), int(conf["train_batch_size"])
    for _ in range(int(conf["epochs"])):
        perm = torch.randperm(n, device=device)
        for a in range(0, n, bs):
            idx = perm[a: a + bs]
            opt.zero_grad()
            l = loss(model(train.inputs(idx, dtype)), train.targets(idx))
            l.backward()
            opt.step()
    with torch.no_grad():
        vb = int(conf["val_batch_size"])
        val_loss, correct = 0.0, 0
        for a in range(0, len(val), vb):
            idx = torch.arange(a, min(len(val), a + vb), device=device)
            out = model(val.inputs(idx, dtype))
            val_loss += loss(out, val.targets(idx)).item()
            correct += out.argmax(dim=1).eq(val.targets(idx)).sum().item()
    return {"validation_loss": val_loss / len(val), "validation_accuracy": correct / len(val)}


def split_random(train, N, generator=None):
    """Equal random shards; unlike the reference (:108-112, SURVEY Q8) a remainder is
    distributed instead of raising."""
    perm = torch.randperm(len(train), generator=generator)
    return [train.select(chunk) for chunk in perm.chunk(N)]


def split_hetero(train, N):
    """Classes partitioned across nodes exactly as the reference does (:113-127): with
    ``len(classes) % N != 0`` trailing classes are unused (SURVEY Q7)."""
    classes = torch.unique(train.y)
    if N > len(classes):
        raise NameError("Hetero MNIST N > 10 not supported.")
    node_classes = torch.split(classes, int(len(classes) / N))
    out = []
    for i in range(N):
        keep = torch.isin(train.y, node_classes[i]).nonzero().reshape(-1)
        out.append(train.select(keep))
    return out


def experiment(yaml_pth):
    conf_dict = load_experiment(yaml_pth, "mnist")
    exp_conf = conf_dict["experiment"]
    ctx = common.make_context(exp_conf)
    output_dir = common.setup_output(exp_conf, yaml_pth, ctx)

    N, graph = graph_generation.generate_from_conf(exp_conf["graph"])
    graph = ctx.broadcast_object(graph)
    if exp_conf["writeout"] and ctx.is_main:
        common.write_gpickle(graph, os.path.join(output_dir, "graph.gpickle"))

    train, src = load_mnist(exp_conf["data_dir"], train=True, source=exp_conf.get("data_source", "auto"))
    val, _ = load_mnist(exp_conf["data_dir"], train=False, source=exp_conf.get("data_source", "auto"))
    if ctx.is_main:
        print(f"MNIST source: {src} ({len(train)} train / {len(val)} val)")
    if exp_conf["data_split_type"] == "random":
        gen = torch.Generator().manual_seed(int(exp_conf.get("seed", 0)))
        train_subsets = split_random(train, N, gen)
    else:
        train_subsets = split_hetero(train, N)

    model_conf = exp_conf["model"]
    torch.manual_seed(int(exp_conf.get("seed", 0)))
    dtype = {"float32": torch.float32, "float64": torch.float64}[exp_conf.get("dtype", "float32")]
    base_model = MNISTConvNet(model_conf["num_filters"], model_conf["kernel_size"], model_conf["linear_width"], dtype=dtype)
    base_loss = common.make_loss(exp_conf["loss"])

    solo_confs = exp_conf["individual_training"]
    if solo_confs["train_solo"] and ctx.is_main:
        print("Performing individual training ...")
        solo_results = {}
        if solo_confs["backend"] == "fused":
            solo_results = local_train.solo_mnist(base_model, base_loss, train_subsets, val, ctx.device, solo_confs,
                                                  seed=int(exp_conf.get("seed", 0)))
        for i in range(N):
            if solo_confs["backend"] == "torch":
                solo_results[i] = train_solo(copy.deepcopy(base_model), base_loss, train_subsets[i], val, ctx.device,
                                             solo_confs)
            if solo_confs["verbose"]:
                print("Node {} - Validation Acc = {:.4f}".format(i, solo_results[i]["validation_accuracy"]))
        if exp_conf["writeout"]:
            torch.save(solo_results, os.path.join(output_dir, "solo_results.pt"))
    ctx.barrier()

    for prob_key, prob_conf in conf_dict["problem_configs"].items():
        prob = DistMNISTProblem(graph, base_model, base_loss, train_subsets, val, ctx.device, prob_conf,
                                ctx=ctx, seed=int(exp_conf.get("seed", 0)))
        prob.data_source = src          # stored in <problem>_results.pt: synthetic runs stay distinguishable from MNIST runs
        common.run_problem(prob, prob_conf, exp_conf, ctx)
    return conf_dict


def main(argv=None):
    argv = sys.argv if argv is None else argv
    yaml_pth = argv[1]
    if not os.path.exists(yaml_pth):
        raise NameError("YAML configuration file does not exist, exiting!")
    experiment(yaml_pth)


if __name__ == "__main__":
    main()
