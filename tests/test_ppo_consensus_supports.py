"""How ``consensus_backend`` / ``--consensus`` reach the distributed-PPO trainers, which configurations the fused
consensus refuses, and the schedule horizon of the fused engine.  No GPU needed: everything here runs before a launch,
and the schedules are built on the host."""
import math

import numpy as np
import pytest
import torch

from consensus_oracle import dsgd_alpha_table, lr_table, rho_table
from nn_distributed_training_b200.ops.engine import schedule_horizon as engine_horizon, schedule_tables
from nn_distributed_training_b200.optimizers import DSGD, DiNNO
from nn_distributed_training_b200.rl import DSGDPPO, DSGTPPO, DiNNOPPO
from nn_distributed_training_b200.rl.consensus_ppo import schedule_horizon
from nn_distributed_training_b200.rl.train_common import common_conf, make_problem, parse_args

DINNO = dict(rho_init=1.0, rho_scaling=1.0, primal_lr_start=3e-4, primal_lr_finish=1e-3, lr_decay_type="constant",
             persistant_primal_opt=False, primal_iterations=5, outer_iterations=10_000_000)
TRAINERS = [(DiNNOPPO, DINNO), (DSGDPPO, dict(alpha0=3e-4, mu=0.0)),
            (DSGTPPO, dict(alpha_actor=3e-4, alpha_critic=1e-3, init_grads=False))]


def _problem(extra=()):
    args = parse_args(["--num_envs", "2", "--device", "cpu", "--no_writeout", "--seed", "0", *extra])
    pr, _ = make_problem(args)
    return pr, common_conf(args)


def test_consensus_flag_parses_and_defaults_to_torch():
    assert parse_args([]).consensus == "torch"
    assert parse_args(["--consensus", "cuda"]).consensus == "cuda"
    assert common_conf(parse_args([]))["consensus_backend"] == "torch"
    assert common_conf(parse_args(["--consensus", "cuda"]))["consensus_backend"] == "fused"
    with pytest.raises(SystemExit):
        parse_args(["--consensus", "fused"])


@pytest.mark.parametrize("cls,conf", TRAINERS)
def test_trainers_default_to_torch_consensus(cls, conf):
    pr, common = _problem()
    tr = cls(pr, "cpu", dict(common, **conf))
    assert tr.inner.conf["consensus_backend"] == "torch" and not tr.fused and not pr.fixed_batch
    assert not tr.inner._use_engine()
    common.pop("consensus_backend")
    tr = cls(pr, "cpu", dict(common, **conf))      # a conf without the key: torch as well
    assert tr.inner.conf["consensus_backend"] == "torch" and not tr.fused


@pytest.mark.parametrize("cls,conf", TRAINERS)
def test_fused_consensus_on_a_cpu_device_names_the_device(cls, conf):
    pr, common = _problem(["--consensus", "cuda"])
    with pytest.raises(ValueError, match="CUDA device.*cpu"):
        cls(pr, "cpu", dict(common, **conf))


def test_fused_consensus_with_reference_mixing_order_names_it():
    pr, common = _problem(["--consensus", "cuda"])
    with pytest.raises(ValueError, match="mixing_order 'reference'"):
        DSGTPPO(pr, "cpu", dict(common, alpha=1e-3, mixing_order="reference"))


def test_unknown_consensus_backend_is_refused():
    pr, common = _problem()
    with pytest.raises(ValueError, match="consensus_backend"):
        DSGDPPO(pr, "cpu", dict(common, alpha0=1e-3, mu=0.0, consensus_backend="cuda"))


@pytest.mark.parametrize("cls,conf", TRAINERS)
@pytest.mark.parametrize("max_rl,outer", [(10_000_000, None), (6000, None), (6001, None), (10_000_000, 7)])
def test_schedule_horizon(cls, conf, max_rl, outer):
    pr, common = _problem()
    c = dict(common, **conf, max_rl_timesteps=max_rl)
    if outer is not None:
        c["outer_iterations"] = outer
    tr = cls(pr, "cpu", c)
    rpi = 1 if cls is DiNNOPPO else pr.n_updates_per_iteration
    its = min(c.get("outer_iterations", 10 ** 12), math.ceil(max_rl / pr.timesteps_per_batch))
    H = schedule_horizon(c, pr, tr.inner.oits, tr.rounds_per_iteration())
    assert tr.rounds_per_iteration() == rpi
    assert H == min(tr.inner.oits, its * rpi)
    if outer is None:
        assert H == its * rpi


@pytest.mark.parametrize("kind", ["constant", "linear", "log"])
def test_dinno_schedules_for_a_horizon_are_a_prefix_of_the_full_tables(kind):
    pr, _ = _problem()
    conf = dict(DINNO, lr_decay_type=kind, primal_lr_start=3e-3, primal_lr_finish=1e-5, rho_scaling=1.0003,
                alg_name="dinno", primal_optimizer="adam", consensus_backend="torch")
    opt = DiNNO(pr, "cpu", conf)
    H = 25_000
    opt.horizon = H
    assert engine_horizon(opt) == H
    rho, lr, alpha = schedule_tables(opt, H)
    assert rho.shape == lr.shape == alpha.shape == (H,)
    full_lr = lr_table(conf, conf["outer_iterations"])       # 10M entries, decay over all of them
    np.testing.assert_allclose(lr, full_lr[:H], rtol=1e-14, atol=0)
    np.testing.assert_allclose(rho, rho_table(conf, H), rtol=1e-13, atol=0)
    assert np.array_equal(lr, [opt.lr_at(k) for k in range(H)]) and np.array_equal(rho, [opt.rho_at(k) for k in range(H)])
    if kind != "constant":
        assert lr[-1] != full_lr[-1] and abs(lr[1] - lr[0]) < abs(full_lr[0] - full_lr[-1]) * 1e-5
    assert not alpha.any()


def test_dsgd_schedule_for_a_horizon_is_a_prefix_of_the_full_table():
    pr, _ = _problem()
    conf = dict(alpha0=0.05, mu=0.5, outer_iterations=10_000_000, alg_name="dsgd", consensus_backend="torch")
    opt = DSGD(pr, "cpu", conf)
    H = 4000
    opt.horizon = H
    rho, lr, alpha = schedule_tables(opt, H)
    assert np.array_equal(alpha, np.asarray(opt.alpha_table(H)))
    np.testing.assert_allclose(alpha, dsgd_alpha_table(0.05, 0.5, 2 * H)[:H], rtol=1e-14, atol=0)
    assert not rho.any() and not lr.any()


def test_horizon_outside_outer_iterations_is_refused():
    pr, _ = _problem()
    opt = DSGD(pr, "cpu", dict(alpha0=0.05, mu=0.0, outer_iterations=10, consensus_backend="torch"))
    opt.horizon = 11
    with pytest.raises(ValueError, match="horizon"):
        engine_horizon(opt)


def test_dsgt_per_coordinate_step_leaves_the_alpha_schedule_empty():
    pr, common = _problem()
    tr = DSGTPPO(pr, "cpu", dict(common, alpha_actor=3e-4, alpha_critic=1e-3))
    assert torch.is_tensor(tr.inner.alpha) and tr.inner.own_tracker_step
    _, _, alpha = schedule_tables(tr.inner, 10)
    assert not alpha.any()
    tr = DSGTPPO(pr, "cpu", dict(common, alpha=2e-3))
    _, _, alpha = schedule_tables(tr.inner, 10)
    assert np.array_equal(alpha, np.full(10, 2e-3))
