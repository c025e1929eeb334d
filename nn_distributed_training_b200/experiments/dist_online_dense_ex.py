"""Online lidar density mapping with a time-varying robot communication graph
(reference: experiments/dist_online_dense_ex.py)."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

from . import common
from . import density_common as dc
from ..floorplans.lidar import OnlineTrajectoryLidarDataset, RandomPoseLidarDataset
from ..models import FourierNet
from ..problems import DistOnlineDensityProblem
from ..utils.config import load_experiment


def experiment(yaml_pth):
    conf_dict = load_experiment(yaml_pth, "online_density")
    exp_conf = conf_dict["experiment"]
    ctx = common.make_context(exp_conf)
    torch.manual_seed(exp_conf["seed"])
    np.random.seed(exp_conf["seed"])
    output_dir = common.setup_output(exp_conf, yaml_pth, ctx)

    data_conf = exp_conf["data"]
    if ctx.is_main:
        print("Loading the data ...")
    data_dir = dc.resolve_data_dir(data_conf, ctx)
    lidar = dc.make_lidar(data_conf, data_dir, device=ctx.device)
    paths = dc.waypoint_files(data_dir, data_conf["waypoint_subdir"])
    N = int(data_conf.get("num_nodes", len(paths)))   # reference: one node per waypoint file (:136-139)
    if N > len(paths) or N == 0:
        raise NameError("Requested more nodes than there are waypoint files."
                        "Requested {} nodes, and found {} waypoint files.".format(N, len(paths)))
    train_subsets = [OnlineTrajectoryLidarDataset(lidar, np.load(paths[i]), data_conf["spline_res"],
                                                  data_conf["num_scans_in_window"],
                                                  round_density=data_conf["round_density"],
                                                  seed=int(exp_conf["seed"]), node=i) for i in range(N)]
    if ctx.is_main:
        for i in range(N):
            print()
            print("Node ", i, "train set size: ", len(train_subsets[i]))
            print("Node", i, "hd ratio: {:.4f}".format(
                (torch.sum(train_subsets[i].scans[:, 2] == 1.0) / train_subsets[i].scans.shape[0]).item()))
    val_set = RandomPoseLidarDataset(lidar, data_conf["num_validation_scans"], round_density=data_conf["round_density"])

    model_conf = exp_conf["model"]
    dtype = {"float32": torch.float32, "float64": torch.float64}[exp_conf.get("dtype", "float32")]
    base_model = FourierNet(model_conf["shape"], scale=model_conf["scale"], dtype=dtype)
    base_loss = common.make_loss(exp_conf["loss"])

    solo_confs = exp_conf["individual_training"]
    if solo_confs["train_solo"] and ctx.is_main:
        print("Performing individual training ...")
        solo = dc.solo_results(base_model, base_loss, train_subsets, val_set, ctx.device, solo_confs,
                               seed=int(exp_conf["seed"]))
        for i in range(N):
            if solo_confs["verbose"]:
                print("Node {} - Validation loss = {:.4f}".format(i, solo[i]["validation_loss"]))
        if exp_conf["writeout"]:
            torch.save(solo, os.path.join(output_dir, "solo_results.pt"))
    ctx.barrier()

    for prob_key, prob_conf in conf_dict["problem_configs"].items():
        prob = DistOnlineDensityProblem(base_model, base_loss, train_subsets, val_set, ctx.device, prob_conf,
                                        ctx=ctx, seed=int(exp_conf["seed"]))
        common.run_problem(prob, prob_conf, exp_conf, ctx)
    return conf_dict


def main(argv=None):
    argv = sys.argv if argv is None else argv
    if not os.path.exists(argv[1]):
        raise NameError("YAML configuration file does not exist, exiting!")
    experiment(argv[1])


if __name__ == "__main__":
    main()
