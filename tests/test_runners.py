"""End-to-end runner tests on CPU with small configs (plumbing / API / output-layout parity)."""
import copy
import glob
import os

import numpy as np
import pytest
import torch
import yaml

from nn_distributed_training_b200.experiments import dist_mnist_ex, dist_online_dense_ex, dist_dense_ex, dist_mnist_scaling
from nn_distributed_training_b200.utils.config import ConfigError, load_experiment, validate_optimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXP = os.path.join(ROOT, "experiments")


def _write(tmp_path, name, conf):
    p = os.path.join(tmp_path, name)
    with open(p, "w") as f:
        yaml.safe_dump(conf, f)
    return p


def _load(name):
    with open(os.path.join(EXP, name)) as f:
        return yaml.safe_load(f)


def test_all_shipped_yamls_validate():
    kinds = {"dist_mnist_PAPER.yaml": "mnist", "dist_mnist_anim.yaml": "mnist", "dist_mnist_template.yaml": "mnist",
             "dist_mnist_8gpu.yaml": "mnist", "dist_mnist_scaling.yaml": "mnist_scaling",
             "dist_online_dense_PAPER.yaml": "online_density", "dist_online_dense_anim.yaml": "online_density",
             "dist_online_dense_synthetic.yaml": "online_density", "dist_dense_v2.yaml": "density"}
    for name, kind in kinds.items():
        conf = load_experiment(os.path.join(EXP, name), kind)
        assert conf["experiment"]["name"]


def test_config_errors_are_explicit():
    with pytest.raises(ConfigError, match="alg_name"):
        validate_optimizer({"outer_iterations": 3})
    with pytest.raises(ConfigError, match="rho_init"):
        validate_optimizer({"alg_name": "dinno", "outer_iterations": 3, "primal_iterations": 1, "primal_lr_start": 1e-3})
    # the README's legacy names still load
    c = validate_optimizer({"alg_name": "cadmm", "rho": 0.5, "primal_lr": 1e-3, "outer_iterations": 3, "primal_iterations": 1})
    assert c["alg_name"] == "dinno" and c["rho_init"] == 0.5 and c["lr_decay_type"] == "constant"
    # extension keys are checked too
    from nn_distributed_training_b200.utils.config import validate_problem
    base = {"problem_name": "p", "train_batch_size": 8, "val_batch_size": 8, "metrics": ["validation_loss"],
            "metrics_config": {"evaluate_frequency": 1},
            "optimizer_config": {"alg_name": "dsgd", "alpha0": 0.1, "mu": 0.0, "outer_iterations": 2}}
    assert validate_problem(dict(base, input_pipeline="staged", samples_per_cta=5), "p", "mnist")["input_pipeline"] == "staged"
    validate_problem(dict(base, input_pipeline="host", host_gather="gpu_pull", host_loss="mirror"), "p", "mnist")
    with pytest.raises(ConfigError, match="input_pipeline"):
        validate_problem(dict(base, input_pipeline="disk"), "p", "mnist")
    with pytest.raises(ConfigError, match="samples_per_cta"):
        validate_problem(dict(base, samples_per_cta=12), "p", "mnist")
    with pytest.raises(ConfigError, match="host_gather"):
        validate_problem(dict(base, host_gather="cpu_loader"), "p", "mnist")
    with pytest.raises(ConfigError, match="host_loss"):
        validate_problem(dict(base, host_loss="memcpy"), "p", "mnist")
    with pytest.raises(ConfigError, match="fault_injection"):
        validate_problem(dict(base, fault_injection={"link_drop_prob": 1.5}), "p", "mnist")


def test_mnist_template_runs_and_writes_reference_layout(tmp_path, monkeypatch):
    """BASELINE config 1: dist_mnist_ex.py + dist_mnist_template.yaml, DSGD, 2 nodes, CPU."""
    import nn_distributed_training_b200.data.mnist as M
    monkeypatch.setattr(M, "load_mnist", lambda d, train, **k: (M.synthetic_mnist(512 if train else 128, seed=int(train)), "synthetic"))
    monkeypatch.setattr(dist_mnist_ex, "load_mnist", M.load_mnist)
    conf = _load("dist_mnist_template.yaml")
    conf["experiment"].update(output_metadir=str(tmp_path), writeout=True)
    oc = conf["problem_configs"]["problem1"]["optimizer_config"]
    oc["outer_iterations"] = 6
    conf["problem_configs"]["problem1"]["metrics_config"]["evaluate_frequency"] = 2
    conf["problem_configs"]["problem2"] = copy.deepcopy(conf["problem_configs"]["problem1"])
    conf["problem_configs"]["problem2"].update(problem_name="dinno")
    conf["problem_configs"]["problem2"]["optimizer_config"] = {
        "alg_name": "dinno", "rho_init": 0.5, "rho_scaling": 1.0003, "outer_iterations": 4, "primal_iterations": 2,
        "primal_optimizer": "adam", "persistant_primal_opt": False, "primal_lr_start": 0.005,
        "primal_lr_finish": 0.0005, "lr_decay_type": "log", "profile": False,
        "checkpoint_every": 2}
    dist_mnist_ex.experiment(_write(str(tmp_path), "c.yaml", conf))
    outs = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_template"))
    assert len(outs) == 1
    files = set(os.listdir(outs[0]))
    assert {"graph.gpickle", "dsgd_results.pt", "dinno_results.pt"} <= files
    assert any(f.endswith(".yaml") for f in files)
    # checkpoints go to the STABLE sibling <metadir>/<name>_ckpt (the output directory is time-stamped)
    assert os.path.exists(os.path.join(str(tmp_path), "dist_mnist_template_ckpt", "dinno_ckpt_rank0.pt"))
    res = torch.load(os.path.join(outs[0], "dsgd_results.pt"), weights_only=False)
    assert res.pop("data_source") == "synthetic"
    assert set(res) == {"forward_pass_count", "validation_loss", "consensus_error", "top1_accuracy", "current_epoch"}
    assert len(res["validation_loss"]) == 4          # rounds 0, 2, 4 and the last (5)
    assert res["validation_loss"][0].shape == (2,)
    d_all, d_mean = res["consensus_error"][0]
    assert d_all.shape == (2, 2) and d_mean.shape == (2, 1)
    assert res["forward_pass_count"] == [0, 128, 256, 320]
    from nn_distributed_training_b200.experiments.common import read_gpickle
    assert read_gpickle(os.path.join(outs[0], "graph.gpickle")).number_of_nodes() == 2


def test_two_invocation_resume_through_the_yaml_runner(tmp_path, monkeypatch):
    """`checkpoint_every` in a first invocation, the same YAML with `resume: true` (and no checkpoint_every: the
    ADVICE r1 ZeroDivisionError case) in a second one: the resumed run continues at the saved round and ends exactly
    where an uninterrupted run ends."""
    import nn_distributed_training_b200.data.mnist as M
    monkeypatch.setattr(M, "load_mnist", lambda d, train, **k: (M.synthetic_mnist(512 if train else 128, seed=int(train)), "synthetic"))
    monkeypatch.setattr(dist_mnist_ex, "load_mnist", M.load_mnist)

    def run(tag, oits, **extra):
        conf = _load("dist_mnist_template.yaml")
        meta = str(tmp_path / tag)
        os.makedirs(meta, exist_ok=True)
        conf["experiment"].update(output_metadir=meta, writeout=True)
        pc = conf["problem_configs"]["problem1"]
        pc["metrics_config"]["evaluate_frequency"] = 2
        pc["optimizer_config"].update(outer_iterations=oits, **extra)
        dist_mnist_ex.experiment(_write(meta, f"c{oits}{len(extra)}.yaml", conf))
        out = sorted(glob.glob(os.path.join(meta, "*_dist_mnist_template")))[-1]
        return torch.load(os.path.join(out, "dsgd_results.pt"), weights_only=False)

    full = run("full", 6)
    run("split", 4, checkpoint_every=2)
    import time
    time.sleep(1.0)
    resumed = run("split", 6, resume=True)
    assert resumed["forward_pass_count"][-1] == full["forward_pass_count"][-1]
    assert torch.equal(resumed["validation_loss"][-1], full["validation_loss"][-1])
    assert torch.equal(resumed["top1_accuracy"][-1], full["top1_accuracy"][-1])
    # the first invocation evaluated at 0, 2 and its last round 3; the resumed one adds 4 and 5
    assert len(resumed["validation_loss"]) == 5


@pytest.fixture(scope="module")
def synthetic_dir(tmp_path_factory):
    from nn_distributed_training_b200.floorplans.synthetic import write_dataset
    d = str(tmp_path_factory.mktemp("floor"))
    write_dataset(d, n_paths=4, seed=0)
    return d


def _small_density_conf(name, synthetic_dir, tmp_path):
    conf = _load(name)
    e = conf["experiment"]
    e.update(output_metadir=str(tmp_path), use_cuda=False)
    e["data"].update(data_dir=synthetic_dir, num_beams=8, beam_samps=10, collision_samps=20, spline_res=4,
                     num_validation_scans=20, border_width=8)
    e["model"]["shape"] = [2, 32, 16, 1]
    e["individual_training"].update(train_solo=True, train_batch_size=500, val_batch_size=500, epochs=1)
    return conf


def test_online_density_runner_dynamic_graph(tmp_path, synthetic_dir):
    conf = _small_density_conf("dist_online_dense_PAPER.yaml", synthetic_dir, tmp_path)
    conf["experiment"]["data"].update(num_scans_in_window=10, num_nodes=3)
    for k, pc in conf["problem_configs"].items():
        pc.update(train_batch_size=300, val_batch_size=400, comm_radius=300.0)
        pc["metrics"] = pc["metrics"] + ["current_position", "current_graph"]
        pc["metrics_config"].update(evaluate_frequency=3)
        pc["optimizer_config"]["outer_iterations"] = 7
    dist_online_dense_ex.experiment(_write(str(tmp_path), "o.yaml", conf))
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_online_dense_PAPER"))[0]
    files = set(os.listdir(out))
    assert {"solo_results.pt", "dinno_log_results.pt", "dsgt_results.pt", "dsgd_results.pt",
            "dinno_log_models.pt", "dsgt_models.pt", "dsgd_models.pt"} <= files
    res = torch.load(os.path.join(out, "dinno_log_results.pt"), weights_only=False)
    assert res["mesh_inputs"].shape[1] == 2
    assert len(res["mesh_grid_density"]) == 1                      # mesh_only_at_end
    assert res["mesh_grid_density"][0].shape == (3, res["mesh_inputs"].shape[0], 1)
    assert len(res["validation_loss"]) == 3 and res["validation_loss"][0].shape == (3,)
    pos = np.stack(res["current_position"])
    assert pos.shape == (3, 3, 2) and not np.allclose(pos[0], pos[-1])   # robots moved: windows advanced
    assert res["train_loss_moving_average"][-1].min() > 0
    models = torch.load(os.path.join(out, "dinno_log_models.pt"), weights_only=False)
    assert set(models) == {0, 1, 2} and "seq.0.linear.weight" in models[0]
    # density animation (visualization/animations/density_anim.ipynb) from the saved mesh evaluations
    from nn_distributed_training_b200.visualization import animations
    frames = animations.density_frames(res, node=1, scale=1)
    assert len(frames) == 1 and frames[0].size[0] > 10
    gif = animations.save_gif(frames * 2, os.path.join(str(tmp_path), "d.gif"))
    assert os.path.getsize(gif) > 100
    # static figures of the notebooks without matplotlib: curves, density panel next to the ground truth, lidar figure
    from nn_distributed_training_b200.floorplans.lidar import Lidar2D, OnlineTrajectoryLidarDataset
    from nn_distributed_training_b200.visualization import figures, load_results
    assert os.path.getsize(figures.curves_figure(out, os.path.join(str(tmp_path), "curves.png"), 3)) > 500
    lidar = Lidar2D(os.path.join(synthetic_dir, "floor_img.png"), 8, 0.2, 10, 1.0, 20, 3, border_width=8)
    allres = load_results(out)
    panel = figures.density_panel(allres, os.path.join(str(tmp_path), "panel.png"), lidar=lidar, node=0)
    from PIL import Image
    assert Image.open(panel).size[0] > Image.open(panel).size[1]          # ground truth + 3 algorithms side by side
    paths = sorted(glob.glob(os.path.join(synthetic_dir, "tight_paths", "*.npy")))[:2]
    dsets = [OnlineTrajectoryLidarDataset(lidar, np.load(p), 4, 10, seed=0, node=i) for i, p in enumerate(paths)]
    fig = figures.lidar_figure(lidar, dsets, os.path.join(str(tmp_path), "lidar.png"))
    cols = {c for _, c in Image.open(fig).getcolors(maxcolors=1 << 20)}
    assert (255, 215, 0) in cols and (0, 0, 139) in cols                 # occupied (gold) and free (dark blue) samples drawn
    assert os.path.getsize(figures.compare_runs_figure([out, out], os.path.join(str(tmp_path), "cmp.png"), 3,
                                                       key="validation_loss")) > 500


def test_offline_density_runner(tmp_path, synthetic_dir):
    conf = _small_density_conf("dist_dense_v2.yaml", synthetic_dir, tmp_path)
    conf["experiment"]["graph"].update(num_nodes=3, p=0.9)
    conf["experiment"]["individual_training"]["train_solo"] = False
    pc = conf["problem_configs"]["problem1"]
    pc.update(train_batch_size=300, val_batch_size=400)
    pc["metrics_config"]["evaluate_frequency"] = 2
    pc["optimizer_config"].update(outer_iterations=4, primal_iterations=2)
    dist_dense_ex.experiment(_write(str(tmp_path), "d.yaml", conf))
    out = glob.glob(os.path.join(str(tmp_path), "*_dist_dense_v2"))[0]
    res = torch.load(os.path.join(out, "dinno_results.pt"), weights_only=False)
    assert res["consensus_error"][0].shape == (3, 3)                # offline stores the pairwise matrix only
    assert len(res["mesh_grid_density"]) == 3


def test_scaling_runner(tmp_path, monkeypatch):
    import nn_distributed_training_b200.data.mnist as M
    monkeypatch.setattr(dist_mnist_scaling, "load_mnist",
                        lambda d, train, **k: (M.synthetic_mnist(600 if train else 100, seed=int(train)), "synthetic"))
    conf = _load("dist_mnist_scaling.yaml")
    conf["experiment"].update(output_metadir=str(tmp_path), use_cuda=False, seed=1)
    conf["experiment"]["scaling"].update(min_N=4, max_N=6, num_trials=2, target_fied=1.0)
    conf["problem"]["optimizer_config"].update(outer_iterations=3)
    conf["problem"]["metrics_config"]["evaluate_frequency"] = 2
    dist_mnist_scaling.experiment(_write(str(tmp_path), "s.yaml", conf))
    out = glob.glob(os.path.join(str(tmp_path), "*_scaling_dinno_const_fied"))[0]
    assert {"0.gpickle", "1.gpickle", "0_results.pt", "1_results.pt"} <= set(os.listdir(out))
    # the table behind visualization/scaling_plots.ipynb
    from nn_distributed_training_b200.visualization.animations import scaling_table
    rows = scaling_table(out, evaluate_frequency=2, thresholds=(0.0, 2.0))
    assert [r["trial"] for r in rows] == [0, 1] and all(4 <= r["N"] <= 6 and r["fiedler"] > 0 for r in rows)
    assert all(r["rounds_to_0"] == 0 and r["rounds_to_200"] is None for r in rows)


def test_visualization_summary_and_tools(tmp_path, monkeypatch):
    """Result inspection works on the files the runners write; waypoint tool builds valid paths."""
    import nn_distributed_training_b200.data.mnist as M
    from nn_distributed_training_b200.visualization import load_results, rounds_to_threshold, summarize_run
    monkeypatch.setattr(dist_mnist_ex, "load_mnist",
                        lambda d, train, **k: (M.synthetic_mnist(512 if train else 128, seed=int(train)), "synthetic"))
    conf = _load("dist_mnist_template.yaml")
    conf["experiment"].update(output_metadir=str(tmp_path), writeout=True)
    conf["problem_configs"]["problem1"]["optimizer_config"]["outer_iterations"] = 5
    conf["problem_configs"]["problem1"]["metrics_config"]["evaluate_frequency"] = 2
    conf["problem_configs"]["problem1"]["metrics"] = list(conf["problem_configs"]["problem1"]["metrics"]) + ["validation_as_vector"]
    dist_mnist_ex.experiment(_write(str(tmp_path), "c.yaml", conf))
    run = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_template"))[0]
    # animations of visualization/animations/mnist_anim.ipynb: digit grid framed by correctness, accuracy curve
    from nn_distributed_training_b200.visualization import animations
    m = load_results(run)["dsgd"]
    val = M.synthetic_mnist(128, seed=0)
    frames = animations.mnist_grid_frames(m, val.x.reshape(128, -1), node=1, grid=(4, 5), cell=20, border=2)
    assert len(frames) == len(m["validation_as_vector"]) and frames[0].size == (100, 80)
    inds = animations.pick_grid_indices(m["validation_as_vector"], num_total=20)
    assert inds.numel() == 20 and inds.unique().numel() == 20
    acc_frames = animations.accuracy_frames(m, evaluate_frequency=2, centralized=0.985)
    assert len(acc_frames) == len(m["top1_accuracy"])
    assert os.path.getsize(animations.save_gif(frames, os.path.join(str(tmp_path), "m.gif"))) > 100
    s = summarize_run(run)
    assert "dsgd" in s and 0.0 <= s["dsgd"]["final_top1_mean"] <= 1.0
    r = rounds_to_threshold(load_results(run)["dsgd"], 0.0, 2)
    assert r == 0
    # waypoint authoring without a GUI
    from nn_distributed_training_b200.floorplans.spline_paths import point_selector as ps
    from nn_distributed_training_b200.floorplans.synthetic import make_floorplan
    from PIL import Image
    img, geo = make_floorplan(seed=0)
    p = os.path.join(str(tmp_path), "floor.png")
    Image.fromarray(img, mode="L").save(p)
    c = geo["centers"][(0, 0)]
    pts = ";".join(f"{c[0] + dx},{c[1] + dy}" for dx, dy in [(-30, -30), (30, -30), (30, 30), (-30, 30), (-30, -20)])
    out = os.path.join(str(tmp_path), "wp.npy")
    ps.main(["x", p, out, "--points", pts, "--open"])
    wp = np.load(out)
    assert wp.shape == (5, 2) and np.abs(wp).max() <= 1.0


def test_waypoint_path_editor_model(tmp_path):
    """The editing operations of the polygon waypoint editor (reference floorplans/spline_paths/point_selector.py: drag,
    'i' insert on an edge, 'd' delete, closed loop, numbered save) on the GUI-free model."""
    from nn_distributed_training_b200.floorplans.spline_paths.point_selector import WaypointPath, point_segment_distance
    assert abs(point_segment_distance((0, 1), (-1, 0), (1, 0)) - 1.0) < 1e-12
    assert abs(point_segment_distance((3, 0), (-1, 0), (1, 0)) - 2.0) < 1e-12
    # pixel space = 100 x data space, pick tolerance 5 px
    path = WaypointPath(np.array([[0.0, 0.0], [1.0, 0.0], [1.0, 1.0], [0.0, 1.0]]), epsilon=5.0, to_pixels=lambda a: 100.0 * np.asarray(a))
    assert path.xy.shape == (5, 2) and np.allclose(path.xy[0], path.xy[-1]) and path.n_vertices == 4
    assert path.hit_test((1.02, 0.01)) == 1 and path.hit_test((0.5, 0.5)) is None
    # dragging the first vertex drags the closing duplicate with it
    path.move(0, (-0.1, -0.1))
    assert np.allclose(path.xy[0], path.xy[-1]) and np.allclose(path.xy[0], [-0.1, -0.1])
    # insert on the edge (1,0)-(1,1); a point away from every edge is refused
    assert path.insert((0.5, 0.5)) is None
    ind = path.insert((1.01, 0.5))
    assert ind == 2 and path.n_vertices == 5 and np.allclose(path.xy[2], [1.01, 0.5])
    # delete an interior vertex and the first vertex (the loop stays closed)
    assert path.delete(2) and path.n_vertices == 4
    assert path.delete(0) and path.n_vertices == 3 and np.allclose(path.xy[0], path.xy[-1])
    assert not path.delete(1)                                  # a loop keeps at least three vertices
    traj = path.spline(10)
    assert traj.shape == (10 * (len(path.xy) - 1), 2) and np.isfinite(traj).all()
    d = str(tmp_path / "tight_paths")
    assert path.save(d).endswith("1.npy") and path.save(d).endswith("2.npy")
    assert np.allclose(np.load(os.path.join(d, "2.npy")), path.xy)
    # the shipped reference paths load into the editor model unchanged
    ref = os.path.join(ROOT, "floorplans", "32_data", "tight_paths", "1.npy")
    if os.path.exists(ref):
        wp = np.load(ref)
        assert WaypointPath(wp).xy.shape[0] in (len(wp), len(wp) + 1)


def test_centralized_baseline(monkeypatch):
    import nn_distributed_training_b200.data.mnist as M
    from nn_distributed_training_b200.experiments import centralized
    from nn_distributed_training_b200.models import MNISTConvNet
    tr, va = M.synthetic_mnist(600, seed=0), M.synthetic_mnist(200, seed=1)
    torch.manual_seed(0)
    hist = centralized.train_centralized(MNISTConvNet(3, 5, 64), torch.nn.NLLLoss(), tr, va, "cpu", epochs=2, lr=0.005,
                                         batch=50, verbose=False)
    assert hist[-1]["top1_accuracy"] > 0.5 and hist[-1]["validation_loss"] < hist[0]["validation_loss"] * 1.5


def test_profile_key_writes_a_profiler_trace(tmp_path, monkeypatch):
    """``optimizer_config.profile: true`` (SURVEY 5.1): the runner wraps training in torch.profiler with the
    reference's schedule and every optimizer calls ``profiler.step()`` once per round -> a trace directory
    ``<problem_name>opt_profile`` appears in the run's output directory."""
    import nn_distributed_training_b200.data.mnist as M
    monkeypatch.setattr(dist_mnist_ex, "load_mnist",
                        lambda d, train, **k: (M.synthetic_mnist(256 if train else 64, seed=int(train)), "synthetic"))
    conf = _load("dist_mnist_template.yaml")
    conf["experiment"].update(output_metadir=str(tmp_path), writeout=True)
    pc = conf["problem_configs"]["problem1"]
    pc["optimizer_config"].update(outer_iterations=6, profile=True)      # wait 1 + warmup 1 + active 3 -> one trace
    pc["metrics_config"]["evaluate_frequency"] = 100
    dist_mnist_ex.experiment(_write(str(tmp_path), "p.yaml", conf))
    run = glob.glob(os.path.join(str(tmp_path), "*_dist_mnist_template"))[0]
    prof_dir = os.path.join(run, pc["problem_name"] + "opt_profile")
    assert os.path.isdir(prof_dir) and len(os.listdir(prof_dir)) >= 1


def test_fail_fast_guards(tmp_path, synthetic_dir, monkeypatch, capsys):
    """The reference's runtime guards (SURVEY §4) are kept: hetero split with N > 10, more nodes than waypoint
    files, NaN in the online forward pass, and the disconnected-graph warning (which does not stop the run)."""
    import nn_distributed_training_b200.data.mnist as M
    # hetero split cannot serve more nodes than classes
    with pytest.raises(NameError, match="Hetero"):
        dist_mnist_ex.split_hetero(M.synthetic_mnist(200, seed=0), 11)
    # more robots than waypoint files (4 in the synthetic directory)
    conf = _small_density_conf("dist_online_dense_PAPER.yaml", synthetic_dir, tmp_path)
    conf["experiment"]["data"].update(num_scans_in_window=10, num_nodes=9)
    with pytest.raises(NameError, match="waypoint files"):
        dist_online_dense_ex.experiment(_write(str(tmp_path), "too_many.yaml", conf))
    # online problem: tiny comm radius -> warning only; NaN parameters -> fail fast
    from nn_distributed_training_b200.floorplans.lidar import Lidar2D, OnlineTrajectoryLidarDataset, RandomPoseLidarDataset
    from nn_distributed_training_b200.models import FourierNet
    from nn_distributed_training_b200.optimizers import DSGD
    from nn_distributed_training_b200.problems import DistOnlineDensityProblem
    lidar = Lidar2D(os.path.join(synthetic_dir, "floor_img.png"), 8, 0.2, 10, 1.0, 20, 3, border_width=8)
    paths = sorted(glob.glob(os.path.join(synthetic_dir, "tight_paths", "*.npy")))[:3]
    train = [OnlineTrajectoryLidarDataset(lidar, np.load(p), 4, 10, seed=0, node=i) for i, p in enumerate(paths)]
    val = RandomPoseLidarDataset(lidar, 10)
    oc = {"alg_name": "dsgd", "alpha0": 0.01, "mu": 0.0, "outer_iterations": 2, "profile": False}
    pconf = {"problem_name": "g", "train_batch_size": 100, "val_batch_size": 200, "comm_radius": 1e-3, "dynamic_graph": True,
             "save_models": False, "metrics": ["validation_loss"], "metrics_config": {"evaluate_frequency": 1, "tloss_decay": 0.2,
                                                                                     "mesh_only_at_end": True},
             "optimizer_config": oc}
    torch.manual_seed(0)
    pr = DistOnlineDensityProblem(FourierNet([2, 16, 8, 1], 0.05), torch.nn.BCELoss(), train, val, "cpu", pconf)
    assert "not connected" in capsys.readouterr().out
    DSGD(pr, "cpu", oc).train()                      # isolated nodes take local steps
    assert torch.isfinite(pr.arena.theta).all()
    pr.arena.theta[1].fill_(float("nan"))
    with pytest.raises(NameError, match="NaN"):
        pr.local_batch_loss(1)


def test_cubi_preproc_writes_the_reference_artefacts(tmp_path):
    """floorplans/cubi_preproc.py: per-image SDF tensors (negative inside the bright region, height-normalised, zero on
    the boundary), pzcounts.pt and a 90/10 split_sets.pt — the files the reference's script produces."""
    from PIL import Image
    from nn_distributed_training_b200.floorplans import cubi_preproc as cp
    src, dst = tmp_path / "src", tmp_path / "dst"
    src.mkdir()
    for i in range(10):
        a = np.zeros((80, 120), dtype=np.uint8)
        a[20 + i: 60, 30: 90 - i] = 255                       # bright rectangle on a dark page
        Image.fromarray(a, mode="L").save(str(src / f"plan{i}.png"))
    split = cp.main(["x", str(src), str(dst), "--sidelen", "40", "--seed", "0"])
    assert len(split["train"]) == 9 and len(split["test"]) == 1
    assert sorted(split["train"] + split["test"]) == sorted(f"plan{i}.pt" for i in range(10))
    counts = torch.load(str(dst / "pzcounts.pt"), weights_only=False)
    sdf = torch.load(str(dst / "plan0.pt"), weights_only=False)
    assert sdf.shape == (40, 60) and sdf.dtype == torch.float32   # shorter side -> 40, aspect kept
    assert counts["plan0.pt"] == {"npixels": 2400, "nzeros": int((sdf == 0).sum())} and counts["plan0.pt"]["nzeros"] > 0
    assert sdf[20, 30] < 0 and sdf[2, 2] > 0                      # inside the rectangle / outside
    assert abs(float(sdf[2, 2])) <= 1.5 and float(sdf.abs().max()) < 1.5   # normalised by the image height
    # --no-overwrite keeps existing tensors
    before = os.path.getmtime(str(dst / "plan3.pt"))
    cp.main(["x", str(src), str(dst), "--sidelen", "40", "--no-overwrite"])
    assert os.path.getmtime(str(dst / "plan3.pt")) == before


def test_centralized_baselines(tmp_path, synthetic_dir, monkeypatch):
    """centralized/*.ipynb equivalents: one model on the union of every node's data, for the MNIST and the lidar-density
    configs (the dotted "Centralized" reference lines of the figures)."""
    import nn_distributed_training_b200.data.mnist as M
    from nn_distributed_training_b200.experiments import centralized
    monkeypatch.setattr(centralized, "load_mnist",
                        lambda d, train, **k: (M.synthetic_mnist(600 if train else 200, seed=int(train)), "synthetic"))
    conf = _load("dist_mnist_template.yaml")
    conf["experiment"].update(output_metadir=str(tmp_path), use_cuda=False)
    conf["experiment"]["individual_training"].update(epochs=2, lr=0.005, train_batch_size=50, val_batch_size=100)
    torch.manual_seed(0)
    hist = centralized.centralized_mnist(_write(str(tmp_path), "cm.yaml", conf))
    assert len(hist) == 2 and hist[-1]["top1_accuracy"] > 0.3
    dconf = _small_density_conf("dist_online_dense_PAPER.yaml", synthetic_dir, tmp_path)
    dconf["experiment"]["individual_training"].update(epochs=1)
    hist = centralized.centralized_density(_write(str(tmp_path), "cd.yaml", dconf), online=True)
    assert len(hist) == 1 and np.isfinite(hist[0]["validation_loss"]) and hist[0]["top1_accuracy"] is None
