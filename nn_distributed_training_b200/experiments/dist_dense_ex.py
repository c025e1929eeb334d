"""Offline lidar density mapping runner (reference: experiments/dist_dense_ex.py)."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

from . import common
from . import density_common as dc
from ..floorplans.lidar import RandomPoseLidarDataset, TrajectoryLidarDataset
from ..models import FourierNet
from ..problems import DistDensityProblem
from ..utils import graph_generation
from ..utils.config import load_experiment


def experiment(yaml_pth):
    conf_dict = load_experiment(yaml_pth, "density")
    exp_conf = conf_dict["experiment"]
    ctx = common.make_context(exp_conf)
    output_dir = common.setup_output(exp_conf, yaml_pth, ctx)
    if "seed" in exp_conf:
        torch.manual_seed(exp_conf["seed"])
        np.random.seed(exp_conf["seed"])

    N, graph = graph_generation.generate_from_conf(exp_conf["graph"])
    graph = ctx.broadcast_object(graph)
    if exp_conf["writeout"] and ctx.is_main:
        common.write_gpickle(graph, os.path.join(output_dir, "graph.gpickle"))

    data_conf = exp_conf["data"]
    if ctx.is_main:
        print("Loading the data ...")
    data_dir = dc.resolve_data_dir(data_conf, ctx)
    lidar = dc.make_lidar(data_conf, data_dir, clipped=bool(data_conf.get("clipped_lidar", False)), device=ctx.device)
    if data_conf["split_type"] == "random":
        train_subsets = [RandomPoseLidarDataset(lidar, data_conf["num_scans"], round_density=data_conf["round_density"])
                         for _ in range(N)]
    elif data_conf["split_type"] == "trajectory":
        paths = dc.waypoint_files(data_dir, data_conf["waypoint_subdir"])
        if N > len(paths):
            raise NameError("Requested more nodes than there are waypoint files."
                            "Requested {} nodes, and found {} waypoint files.".format(N, len(paths)))
        train_subsets = [TrajectoryLidarDataset(lidar, np.load(paths[i]), data_conf["spline_res"],
                                                round_density=data_conf["round_density"]) for i in range(N)]
    else:
        raise NameError("Unknown data split type. Must be either (random, trajectory).")
    if ctx.is_main:
        for i in range(N):
            print("Node ", i, "train set size: ", len(train_subsets[i]))
    val_set = RandomPoseLidarDataset(lidar, data_conf["num_validation_scans"], round_density=data_conf["round_density"])

    model_conf = exp_conf["model"]
    dtype = {"float32": torch.float32, "float64": torch.float64}[exp_conf.get("dtype", "float32")]
    base_model = FourierNet(model_conf["shape"], scale=model_conf["scale"], dtype=dtype)
    base_loss = common.make_loss(exp_conf["loss"])

    solo_confs = exp_conf["individual_training"]
    if solo_confs["train_solo"] and ctx.is_main:
        print("Performing individual training ...")
        solo = dc.solo_results(base_model, base_loss, train_subsets[:N], val_set, ctx.device, solo_confs,
                               seed=int(exp_conf.get("seed", 0)))
        for i in range(N):
            if solo_confs["verbose"]:
                print("Node {} - Validation loss = {:.4f}".format(i, solo[i]["validation_loss"]))
        if exp_conf["writeout"]:
            torch.save(solo, os.path.join(output_dir, "solo_results.pt"))
    ctx.barrier()

    for prob_key, prob_conf in conf_dict["problem_configs"].items():
        if prob_conf["optimizer_config"]["alg_name"] not in ("dinno", "dsgt", "dsgd", "dsgdm", "exact_diffusion", "choco_sgd",
                                                             "beer", "sgp", "push_diging", "kgt",
                                                             "clipped_gossip", "dadaptive", "relaysum",
                                                             "bridge", "powergossip", "detag", "gt_hsgd",
                                                             "gossip_pga", "dp_dsgd", "moniqua", "cross_gradient",
                                                             "slowmo"):
            raise NameError("Unknown distributed opt algorithm.")
        prob = DistDensityProblem(graph, base_model, base_loss, train_subsets, val_set, ctx.device, prob_conf,
                                  ctx=ctx, seed=int(exp_conf.get("seed", 0)))
        common.run_problem(prob, prob_conf, exp_conf, ctx)
    return conf_dict


def main(argv=None):
    argv = sys.argv if argv is None else argv
    if not os.path.exists(argv[1]):
        raise NameError("YAML configuration file does not exist, exiting!")
    experiment(argv[1])


if __name__ == "__main__":
    main()
