"""Typed view of the experiment YAML files.

The reference passes ``yaml.safe_load`` dicts straight down and fails with ``KeyError``
on anything missing (SURVEY §5.6).  Here every key the code reads is declared with its type
and (where the reference had none) a default; unknown optimizer/metric names fail at load time
with the offending path, and the validated dicts that flow down keep the reference's layout
(``experiment`` / ``problem_configs.<key>.optimizer_config``) so existing YAMLs load unchanged.
"""
from __future__ import annotations

import copy
from typing import Any, Dict, Iterable, Optional

import yaml

import math

from ..ops.consensus_ref import (BRIDGE_SCREENS, CHOCO_COMPRESSORS, DADAPTIVE_VARIANTS, MQ_BASES, MQ_BITS,
                                 SPARQ_COMPRESSORS, TOPK_RATIO_DEFAULT)

REQUIRED = object()

ALGS = ("dinno", "dsgd", "dsgdm", "dsgt", "exact_diffusion", "choco_sgd", "beer", "sgp", "push_diging", "kgt",
        "clipped_gossip", "dadaptive", "relaysum", "bridge", "powergossip", "detag", "gt_hsgd", "gossip_pga", "dp_dsgd",
        "moniqua", "sparq_sgd", "cross_gradient", "slowmo")
# the algorithms that model Byzantine attackers (byzantine: {nodes, attack, scale, z})
BYZANTINE_ALGS = ("clipped_gossip", "bridge")
# graph types that generate an nx.DiGraph (utils/graph_generation.py); only the push-sum algorithms run on them
DIRECTED_GRAPH_TYPES = ("directed_cycle", "exponential", "random_directed")
DIRECTED_ALGS = ("sgp", "push_diging")
MOMENTUM_MODES = ("local", "quasi_global")
MNIST_METRICS = ("forward_pass_count", "validation_loss", "consensus_error", "top1_accuracy",
                 "current_epoch", "validation_as_vector")
DENSITY_METRICS = ("forward_pass_count", "validation_loss", "consensus_error", "mesh_grid_density",
                   "current_epoch", "train_loss_moving_average", "current_position", "current_graph")

OPT_SCHEMA = {
    "dinno": {"rho_init": REQUIRED, "rho_scaling": 1.0, "outer_iterations": REQUIRED,
              "primal_iterations": REQUIRED, "primal_optimizer": "adam", "persistant_primal_opt": False,
              "primal_lr_start": REQUIRED, "primal_lr_finish": None, "lr_decay_type": "constant",
              "profile": False},
    "dsgd": {"alpha0": REQUIRED, "mu": REQUIRED, "outer_iterations": REQUIRED, "profile": False},
    "dsgdm": {"alpha0": REQUIRED, "mu": 0.0, "beta": REQUIRED, "momentum": REQUIRED, "nesterov": False,
              "outer_iterations": REQUIRED, "profile": False, "update_graph": True},
    "dsgt": {"alpha": REQUIRED, "init_grads": True, "outer_iterations": REQUIRED, "profile": False},
    "exact_diffusion": {"alpha0": REQUIRED, "mu": 0.0, "outer_iterations": REQUIRED, "profile": False},
    "choco_sgd": {"alpha0": REQUIRED, "mu": 0.0, "gamma": REQUIRED, "compressor": REQUIRED,
                  "outer_iterations": REQUIRED, "profile": False},
    "beer": {"alpha": REQUIRED, "gamma": REQUIRED, "compressor": REQUIRED, "outer_iterations": REQUIRED, "profile": False},
    "sgp": {"alpha0": REQUIRED, "mu": 0.0, "outer_iterations": REQUIRED, "profile": False, "update_graph": True},
    "push_diging": {"alpha": REQUIRED, "outer_iterations": REQUIRED, "profile": False, "update_graph": True},
    "kgt": {"alpha": REQUIRED, "local_steps": REQUIRED, "correction": True, "outer_iterations": REQUIRED,
            "profile": False, "update_graph": True},
    "clipped_gossip": {"alpha0": REQUIRED, "mu": 0.0, "clip": REQUIRED, "outer_iterations": REQUIRED, "profile": False,
                       "update_graph": True},
    # beta2 (default DADAPTIVE_BETA2) is filled in for variant amsgrad only
    "dadaptive": {"alpha": REQUIRED, "variant": REQUIRED, "tracking": True, "beta1": 0.9, "eps": 1e-8,
                  "outer_iterations": REQUIRED, "profile": False, "update_graph": True},
    "relaysum": {"alpha0": REQUIRED, "mu": REQUIRED, "outer_iterations": REQUIRED, "profile": False},
    # b is required with screen trimmed_mean and refused with median
    "bridge": {"alpha0": REQUIRED, "mu": 0.0, "screen": REQUIRED, "outer_iterations": REQUIRED, "profile": False,
               "update_graph": True},
    "powergossip": {"alpha0": REQUIRED, "mu": 0.0, "gamma": REQUIRED, "outer_iterations": REQUIRED, "profile": False},
    "detag": {"alpha": REQUIRED, "gossip_steps": REQUIRED, "accelerate": True, "outer_iterations": REQUIRED,
              "profile": False},
    "gt_hsgd": {"alpha": REQUIRED, "beta": REQUIRED, "outer_iterations": REQUIRED, "update_graph": True,
                "profile": False},
    "gossip_pga": {"alpha0": REQUIRED, "mu": 0.0, "period": REQUIRED, "gossip": True, "outer_iterations": REQUIRED,
                   "update_graph": True, "profile": False},
    # noise_seed defaults to the problem's seed (filled in by the optimizer, which knows it)
    "dp_dsgd": {"alpha0": REQUIRED, "mu": 0.0, "clip_norm": REQUIRED, "noise_multiplier": REQUIRED,
                "pair_noise_multiplier": 0.0, "target_delta": 1e-5, "outer_iterations": REQUIRED, "update_graph": True,
                "profile": False},
    # rounding_seed defaults to the problem's seed (filled in by the optimizer, which knows it)
    "moniqua": {"alpha0": REQUIRED, "mu": 0.0, "bits": REQUIRED, "theta_bound": REQUIRED, "base": "dsgd",
                "outer_iterations": REQUIRED, "update_graph": True, "profile": False},
    "sparq_sgd": {"alpha0": REQUIRED, "mu": 0.0, "gamma": REQUIRED, "compressor": REQUIRED, "threshold": REQUIRED,
                  "local_steps": 1, "threshold_growth": 0.0, "outer_iterations": REQUIRED, "profile": False},
    "cross_gradient": {"alpha0": REQUIRED, "mu": 0.0, "cross_weight": REQUIRED, "outer_iterations": REQUIRED,
                       "profile": False},
    "slowmo": {"alpha0": REQUIRED, "mu": 0.0, "period": REQUIRED, "gossip": True, "slow_momentum": REQUIRED,
               "slow_lr": 1.0, "base_momentum": 0.0, "nesterov": False, "outer_iterations": REQUIRED,
               "update_graph": True, "profile": False},
}
DADAPTIVE_BETA2 = 0.999
# framework extensions accepted in every optimizer_config
OPT_EXTRA = ("mixing_order", "update_graph", "consensus_backend", "persistent_follows_schedule",
             "checkpoint_every", "checkpoint_dir", "resume")


class ConfigError(ValueError):
    pass


def _check_compressor(c: Dict[str, Any], path: str) -> None:
    """CHOCO-SGD / BEER: the compressor, and ``topk_ratio`` (default ``TOPK_RATIO_DEFAULT``) with ``topk`` only."""
    if c["compressor"] not in CHOCO_COMPRESSORS:
        raise ConfigError(f"{path}.compressor must be one of {'|'.join(CHOCO_COMPRESSORS)} (got {c['compressor']!r})")
    if c["compressor"] != "topk":
        if "topk_ratio" in c:
            raise ConfigError(f"{path}.topk_ratio applies to compressor topk only (compressor is {c['compressor']!r})")
        return
    r = c.setdefault("topk_ratio", TOPK_RATIO_DEFAULT)
    if isinstance(r, bool) or not isinstance(r, (int, float)) or not 0.0 < float(r) <= 1.0:
        raise ConfigError(f"{path}.topk_ratio must be in (0, 1] (got {r!r})")


def _real(x) -> bool:
    return not isinstance(x, bool) and isinstance(x, (int, float))


def _check_dadaptive(c: Dict[str, Any], path: str) -> None:
    """Decentralized AMSGrad / AdaGrad: the variant, the tracking switch, the moment coefficients (``beta2`` with
    amsgrad only, default ``DADAPTIVE_BETA2``), ``eps`` and the step."""
    if c["variant"] not in DADAPTIVE_VARIANTS:
        raise ConfigError(f"{path}.variant must be one of {'|'.join(DADAPTIVE_VARIANTS)} (got {c['variant']!r})")
    if not isinstance(c["tracking"], bool):
        raise ConfigError(f"{path}.tracking must be true or false (got {c['tracking']!r})")
    if c["variant"] == "adagrad":
        if "beta2" in c:
            raise ConfigError(f"{path}.beta2 applies to variant amsgrad only (variant is 'adagrad')")
    else:
        c.setdefault("beta2", DADAPTIVE_BETA2)
    for key in ("beta1", "beta2"):
        if key in c and (not _real(c[key]) or not 0.0 <= float(c[key]) < 1.0):
            raise ConfigError(f"{path}.{key} must be in [0, 1) (got {c[key]!r})")
    if not _real(c["eps"]) or not (math.isfinite(float(c["eps"])) and float(c["eps"]) > 0.0):
        raise ConfigError(f"{path}.eps must be finite and > 0 (got {c['eps']!r})")
    if not _real(c["alpha"]) or not float(c["alpha"]) > 0.0:
        raise ConfigError(f"{path}.alpha must be > 0 (got {c['alpha']!r})")


RELAYSUM_KEYS = ("alg_name", "alpha0", "mu", "outer_iterations", "profile")


def _check_relaysum(c: Dict[str, Any], path: str) -> None:
    """RelaySum: DSGD's step schedule and no other key (RelaySum/Grad and momentum are not implemented)."""
    for key in c:
        if key not in RELAYSUM_KEYS and key not in OPT_EXTRA and key != "debug_sequence_check":
            raise ConfigError(f"{path}.{key}: relaysum takes no key {key!r} (its keys are alpha0, mu and "
                              f"outer_iterations)")
    if not _real(c["alpha0"]) or not float(c["alpha0"]) > 0.0:
        raise ConfigError(f"{path}.alpha0 must be > 0 (got {c['alpha0']!r})")
    if not _real(c["mu"]) or not float(c["mu"]) >= 0.0:
        raise ConfigError(f"{path}.mu must be >= 0 (got {c['mu']!r})")


POWERGOSSIP_KEYS = ("alg_name", "alpha0", "mu", "gamma", "outer_iterations", "profile")


def _check_powergossip(c: Dict[str, Any], path: str) -> None:
    """PowerGossip: DSGD's step schedule, the consensus step ``gamma`` in (0, 1], and no other key (higher ranks are not
    implemented)."""
    for key in c:
        if key not in POWERGOSSIP_KEYS and key not in OPT_EXTRA and key != "debug_sequence_check":
            raise ConfigError(f"{path}.{key}: powergossip takes no key {key!r} (its keys are alpha0, mu, gamma and "
                              f"outer_iterations)")
    if not _real(c["alpha0"]) or not (math.isfinite(float(c["alpha0"])) and float(c["alpha0"]) >= 0.0):
        raise ConfigError(f"{path}.alpha0 must be finite and >= 0 (got {c['alpha0']!r})")
    if not _real(c["mu"]) or not (math.isfinite(float(c["mu"])) and float(c["mu"]) >= 0.0):
        raise ConfigError(f"{path}.mu must be finite and >= 0 (got {c['mu']!r})")
    g = c["gamma"]
    if not _real(g) or not (math.isfinite(float(g)) and 0.0 < float(g) <= 1.0):
        raise ConfigError(f"{path}.gamma must be finite and in (0, 1] (got {g!r})")


DETAG_KEYS = ("alg_name", "alpha", "gossip_steps", "accelerate", "outer_iterations", "profile")


def _check_detag(c: Dict[str, Any], path: str) -> None:
    """DeTAG: the step ``alpha`` (finite, > 0), ``gossip_steps`` (an integer >= 1), ``accelerate`` (a bool) and no other
    key."""
    for key in c:
        if key not in DETAG_KEYS and key not in OPT_EXTRA and key != "debug_sequence_check":
            raise ConfigError(f"{path}.{key}: detag takes no key {key!r} (its keys are alpha, gossip_steps, accelerate "
                              f"and outer_iterations)")
    if not _real(c["alpha"]) or not (math.isfinite(float(c["alpha"])) and float(c["alpha"]) > 0.0):
        raise ConfigError(f"{path}.alpha must be finite and > 0 (got {c['alpha']!r})")
    ks = c["gossip_steps"]
    if isinstance(ks, bool) or not isinstance(ks, int) or ks < 1:
        raise ConfigError(f"{path}.gossip_steps must be an integer >= 1 (got {ks!r})")
    if not isinstance(c["accelerate"], bool):
        raise ConfigError(f"{path}.accelerate must be true or false (got {c['accelerate']!r})")


GT_HSGD_KEYS = ("alg_name", "alpha", "beta", "outer_iterations", "update_graph", "profile")


def _check_gt_hsgd(c: Dict[str, Any], path: str) -> None:
    """GT-HSGD: the step ``alpha`` (finite, > 0), the mixing weight ``beta`` (finite, in (0, 1]) and no other key."""
    for key in c:
        if key not in GT_HSGD_KEYS and key not in OPT_EXTRA and key != "debug_sequence_check":
            raise ConfigError(f"{path}.{key}: gt_hsgd takes no key {key!r} (its keys are alpha, beta, outer_iterations "
                              f"and update_graph)")
    if not _real(c["alpha"]) or not (math.isfinite(float(c["alpha"])) and float(c["alpha"]) > 0.0):
        raise ConfigError(f"{path}.alpha must be finite and > 0 (got {c['alpha']!r})")
    if not _real(c["beta"]) or not (math.isfinite(float(c["beta"])) and 0.0 < float(c["beta"]) <= 1.0):
        raise ConfigError(f"{path}.beta must be finite and in (0, 1] (got {c['beta']!r})")


GOSSIP_PGA_KEYS = ("alg_name", "alpha0", "mu", "period", "gossip", "outer_iterations", "update_graph", "profile")


def _check_gossip_pga(c: Dict[str, Any], path: str) -> None:
    """Gossip-PGA: DSGD's step schedule (``alpha0`` and ``mu`` finite, >= 0), ``period`` (an integer >= 1), ``gossip``
    (a bool) and no other key."""
    for key in c:
        if key not in GOSSIP_PGA_KEYS and key not in OPT_EXTRA and key != "debug_sequence_check":
            raise ConfigError(f"{path}.{key}: gossip_pga takes no key {key!r} (its keys are alpha0, mu, period, gossip, "
                              f"outer_iterations and update_graph)")
    for key in ("alpha0", "mu"):
        if not _real(c[key]) or not (math.isfinite(float(c[key])) and float(c[key]) >= 0.0):
            raise ConfigError(f"{path}.{key} must be finite and >= 0 (got {c[key]!r})")
    p = c["period"]
    if isinstance(p, bool) or not isinstance(p, int) or p < 1:
        raise ConfigError(f"{path}.period must be an integer >= 1 (got {p!r})")
    if not isinstance(c["gossip"], bool):
        raise ConfigError(f"{path}.gossip must be true or false (got {c['gossip']!r})")


SLOWMO_KEYS = ("alg_name", "alpha0", "mu", "period", "gossip", "slow_momentum", "slow_lr", "base_momentum", "nesterov",
               "outer_iterations", "update_graph", "profile")


def _check_slowmo(c: Dict[str, Any], path: str) -> None:
    """SlowMo: Gossip-PGA's keys with ``alpha0`` > 0 (the slow step divides by the step size), ``slow_momentum`` and
    ``base_momentum`` in [0, 1), ``slow_lr`` (finite, > 0), ``nesterov`` (a bool) and no other key.  A schedule that
    reaches a step <= 0 is refused when the optimizer is built."""
    for key in c:
        if key not in SLOWMO_KEYS and key not in OPT_EXTRA and key != "debug_sequence_check":
            raise ConfigError(f"{path}.{key}: slowmo takes no key {key!r} (its keys are alpha0, mu, period, gossip, "
                              f"slow_momentum, slow_lr, base_momentum, nesterov, outer_iterations and update_graph)")
    if not _real(c["alpha0"]) or not (math.isfinite(float(c["alpha0"])) and float(c["alpha0"]) > 0.0):
        raise ConfigError(f"{path}.alpha0 must be finite and > 0 (got {c['alpha0']!r})")
    if not _real(c["mu"]) or not (math.isfinite(float(c["mu"])) and float(c["mu"]) >= 0.0):
        raise ConfigError(f"{path}.mu must be finite and >= 0 (got {c['mu']!r})")
    p = c["period"]
    if isinstance(p, bool) or not isinstance(p, int) or p < 1:
        raise ConfigError(f"{path}.period must be an integer >= 1 (got {p!r})")
    for key in ("slow_momentum", "base_momentum"):
        if not _real(c[key]) or not 0.0 <= float(c[key]) < 1.0:
            raise ConfigError(f"{path}.{key} must be in [0, 1) (got {c[key]!r})")
    if not _real(c["slow_lr"]) or not (math.isfinite(float(c["slow_lr"])) and float(c["slow_lr"]) > 0.0):
        raise ConfigError(f"{path}.slow_lr must be finite and > 0 (got {c['slow_lr']!r})")
    for key in ("gossip", "nesterov"):
        if not isinstance(c[key], bool):
            raise ConfigError(f"{path}.{key} must be true or false (got {c[key]!r})")


CROSS_GRADIENT_KEYS = ("alg_name", "alpha0", "mu", "cross_weight", "outer_iterations", "profile")


def _check_cross_gradient(c: Dict[str, Any], path: str) -> None:
    """Cross-gradient gossip: DSGD's step schedule (``alpha0`` and ``mu`` finite, >= 0), ``cross_weight`` (finite, in
    [0, 1]) and no other key."""
    for key in c:
        if key not in CROSS_GRADIENT_KEYS and key not in OPT_EXTRA and key != "debug_sequence_check":
            raise ConfigError(f"{path}.{key}: cross_gradient takes no key {key!r} (its keys are alpha0, mu, cross_weight "
                              f"and outer_iterations)")
    for key in ("alpha0", "mu"):
        if not _real(c[key]) or not (math.isfinite(float(c[key])) and float(c[key]) >= 0.0):
            raise ConfigError(f"{path}.{key} must be finite and >= 0 (got {c[key]!r})")
    w = c["cross_weight"]
    if not _real(w) or not (math.isfinite(float(w)) and 0.0 <= float(w) <= 1.0):
        raise ConfigError(f"{path}.cross_weight must be finite and in [0, 1] (got {w!r})")


def _check_fixed_graph(c: Dict[str, Any], path: str, kind: str) -> None:
    """Cross-gradient gossip sends each gradient back over the edge it came from, on one fixed graph: link drops and the
    online-density runner's moving graph are refused."""
    if c["optimizer_config"]["alg_name"] != "cross_gradient":
        return
    if c.get("fault_injection"):
        raise ConfigError(f"{path}.fault_injection: cross_gradient needs a fixed graph (link drops change it during the "
                          f"run)")
    if kind == "online_density":
        raise ConfigError(f"{path}.optimizer_config.alg_name: cross_gradient needs a fixed graph, and the online-density "
                          f"runner moves the graph with the agents (the offline density runner is supported)")


DP_DSGD_KEYS = ("alg_name", "alpha0", "mu", "clip_norm", "noise_multiplier", "pair_noise_multiplier", "target_delta",
                "noise_seed", "outer_iterations", "update_graph", "profile")


def _check_dp_dsgd(c: Dict[str, Any], path: str) -> None:
    """DP-DSGD: DSGD's step schedule (``alpha0`` and ``mu`` finite, >= 0), ``clip_norm`` (finite, > 0), the multipliers
    (finite, >= 0), ``target_delta`` in (0, 1), an integer ``noise_seed`` and no other key.  ClippedGossip's ``clip`` and
    ``delta`` mean something else and are refused here."""
    for key in c:
        if key not in DP_DSGD_KEYS and key not in OPT_EXTRA and key != "debug_sequence_check":
            raise ConfigError(f"{path}.{key}: dp_dsgd takes no key {key!r} (its keys are alpha0, mu, clip_norm, "
                              f"noise_multiplier, pair_noise_multiplier, target_delta, noise_seed, outer_iterations and "
                              f"update_graph)")
    for key in ("alpha0", "mu", "noise_multiplier", "pair_noise_multiplier"):
        if not _real(c[key]) or not (math.isfinite(float(c[key])) and float(c[key]) >= 0.0):
            raise ConfigError(f"{path}.{key} must be finite and >= 0 (got {c[key]!r})")
    if not _real(c["clip_norm"]) or not (math.isfinite(float(c["clip_norm"])) and float(c["clip_norm"]) > 0.0):
        raise ConfigError(f"{path}.clip_norm must be finite and > 0 (got {c['clip_norm']!r})")
    if not _real(c["target_delta"]) or not 0.0 < float(c["target_delta"]) < 1.0:
        raise ConfigError(f"{path}.target_delta must be in (0, 1) (got {c['target_delta']!r})")
    s = c.get("noise_seed", 0)
    if isinstance(s, bool) or not isinstance(s, int):
        raise ConfigError(f"{path}.noise_seed must be an integer (got {s!r})")


MONIQUA_KEYS = ("alg_name", "alpha0", "mu", "bits", "theta_bound", "base", "rounding_seed", "outer_iterations",
                "update_graph", "profile")


def _check_moniqua(c: Dict[str, Any], path: str) -> None:
    """Moniqua: DSGD's step schedule (``alpha0`` and ``mu`` finite, >= 0), ``bits`` (2, 4 or 8, not a bool),
    ``theta_bound`` (finite, > 0), the ``base``, an integer ``rounding_seed`` and no other key."""
    for key in c:
        if key not in MONIQUA_KEYS and key not in OPT_EXTRA and key != "debug_sequence_check":
            raise ConfigError(f"{path}.{key}: moniqua takes no key {key!r} (its keys are alpha0, mu, bits, theta_bound, "
                              f"base, rounding_seed, outer_iterations and update_graph)")
    for key in ("alpha0", "mu"):
        if not _real(c[key]) or not (math.isfinite(float(c[key])) and float(c[key]) >= 0.0):
            raise ConfigError(f"{path}.{key} must be finite and >= 0 (got {c[key]!r})")
    b = c["bits"]
    if isinstance(b, bool) or not isinstance(b, int) or b not in MQ_BITS:
        raise ConfigError(f"{path}.bits must be one of {'|'.join(map(str, MQ_BITS))} (got {b!r})")
    tb = c["theta_bound"]
    if not _real(tb) or not (math.isfinite(float(tb)) and float(tb) > 0.0):
        raise ConfigError(f"{path}.theta_bound must be finite and > 0 (got {tb!r})")
    if c["base"] not in MQ_BASES:
        raise ConfigError(f"{path}.base must be one of {'|'.join(MQ_BASES)} (got {c['base']!r})")
    s = c.get("rounding_seed", 0)
    if isinstance(s, bool) or not isinstance(s, int):
        raise ConfigError(f"{path}.rounding_seed must be an integer (got {s!r})")


SPARQ_KEYS = ("alg_name", "alpha0", "mu", "gamma", "compressor", "threshold", "local_steps", "threshold_growth",
              "outer_iterations", "update_graph", "profile")


def _check_sparq(c: Dict[str, Any], path: str) -> None:
    """SPARQ-SGD: DSGD's step schedule (``alpha0`` and ``mu`` finite, >= 0), ``gamma`` in (0, 1], a compressor of none,
    int8 or sign, ``threshold`` (finite, >= 0), ``threshold_growth`` in [0, 1), ``local_steps`` (an integer >= 1), a
    fixed graph and no other key."""
    for key in c:
        if key not in SPARQ_KEYS and key not in OPT_EXTRA and key != "debug_sequence_check":
            raise ConfigError(f"{path}.{key}: sparq_sgd takes no key {key!r} (its keys are alpha0, mu, gamma, "
                              f"compressor, threshold, threshold_growth, local_steps and outer_iterations)")
    for key in ("alpha0", "mu", "threshold"):
        if not _real(c[key]) or not (math.isfinite(float(c[key])) and float(c[key]) >= 0.0):
            raise ConfigError(f"{path}.{key} must be finite and >= 0 (got {c[key]!r})")
    g = c["gamma"]
    if not _real(g) or not (math.isfinite(float(g)) and 0.0 < float(g) <= 1.0):
        raise ConfigError(f"{path}.gamma must be finite and in (0, 1] (got {g!r})")
    if c["compressor"] == "topk":
        raise ConfigError(f"{path}.compressor: sparq_sgd has no topk compressor (the top-k code is selected by a "
                          f"cluster kernel that has no trigger); use none|int8|sign")
    if c["compressor"] not in SPARQ_COMPRESSORS:
        raise ConfigError(f"{path}.compressor must be one of {'|'.join(SPARQ_COMPRESSORS)} (got {c['compressor']!r})")
    tg = c["threshold_growth"]
    if not _real(tg) or not 0.0 <= float(tg) < 1.0:
        raise ConfigError(f"{path}.threshold_growth must be in [0, 1) (got {tg!r})")
    h = c["local_steps"]
    if isinstance(h, bool) or not isinstance(h, int) or h < 1:
        raise ConfigError(f"{path}.local_steps must be an integer >= 1 (got {h!r})")
    # s = sum_j W_ij x_hat_j is only valid for a fixed W: the graph is never refreshed
    if c.setdefault("update_graph", False):
        raise ConfigError(f"{path}.update_graph: sparq_sgd needs a fixed graph (its sum of the neighbors' estimates "
                          f"is only valid for a fixed mixing matrix)")


def _check_bridge(c: Dict[str, Any], path: str) -> None:
    """BRIDGE: the screen, and ``b`` (an integer >= 0) with ``trimmed_mean`` only."""
    if c["screen"] not in BRIDGE_SCREENS:
        raise ConfigError(f"{path}.screen must be one of {'|'.join(BRIDGE_SCREENS)} (got {c['screen']!r})")
    if c["screen"] == "median":
        if "b" in c:
            raise ConfigError(f"{path}.b applies to screen trimmed_mean only (screen is 'median')")
        return
    if "b" not in c:
        raise ConfigError(f"missing required key {path}.b (screen: trimmed_mean)")
    b = c["b"]
    if isinstance(b, bool) or not isinstance(b, int) or b < 0:
        raise ConfigError(f"{path}.b must be an integer >= 0 (got {b!r})")


def _fill(d: Dict[str, Any], schema: Dict[str, Any], path: str, extra: Iterable[str] = ()) -> Dict[str, Any]:
    out = dict(d)
    for k, dflt in schema.items():
        if k not in out:
            if dflt is REQUIRED:
                raise ConfigError(f"missing required key {path}.{k}")
            out[k] = copy.deepcopy(dflt)
    return out


def validate_optimizer(conf: Dict[str, Any], path: str = "optimizer_config") -> Dict[str, Any]:
    if "alg_name" not in conf:
        raise ConfigError(f"missing required key {path}.alg_name")
    alg = conf["alg_name"]
    if alg == "cadmm":   # the README's older name for DiNNO (README.md:33,156)
        alg = "dinno"
    if alg not in ALGS:
        raise ConfigError(f"{path}.alg_name: unknown algorithm {alg!r} (expected one of {ALGS})")
    c = dict(conf, alg_name=alg)
    if alg == "dinno":
        # accept the stale schema of dist_dense_v2.yaml (`primal_lr`, SURVEY C16)
        if "primal_lr" in c and "primal_lr_start" not in c:
            c["primal_lr_start"] = c["primal_lr"]
        if "rho" in c and "rho_init" not in c:
            c["rho_init"] = c["rho"]
    c = _fill(c, OPT_SCHEMA[alg], path)
    if alg == "dinno":
        if c["primal_lr_finish"] is None:
            c["primal_lr_finish"] = c["primal_lr_start"]
        if c["lr_decay_type"] not in ("constant", "linear", "log"):
            raise ConfigError(f"{path}.lr_decay_type: {c['lr_decay_type']!r}")
        if c["primal_optimizer"] not in ("adam", "sgd", "adamw"):
            raise ConfigError(f"{path}.primal_optimizer: {c['primal_optimizer']!r}")
    if "byzantine" in c and alg not in BYZANTINE_ALGS:
        raise ConfigError(f"{path}.byzantine: Byzantine attackers are modelled by alg_name clipped_gossip only, or "
                          f"bridge (alg_name is {alg!r})")
    if (alg in ("dsgdm", "exact_diffusion", "choco_sgd", "beer", "sgp", "push_diging", "kgt", "clipped_gossip",
                "dadaptive", "relaysum", "bridge", "powergossip", "detag", "gt_hsgd", "gossip_pga", "dp_dsgd",
                "moniqua", "sparq_sgd", "cross_gradient", "slowmo")
            and c.get("mixing_order", "jacobi") != "jacobi"):
        raise ConfigError(f"{path}.mixing_order: {alg} runs the synchronous 'jacobi' order only "
                          f"(got {c['mixing_order']!r})")
    if alg == "dsgdm":
        if not 0.0 <= float(c["beta"]) < 1.0:
            raise ConfigError(f"{path}.beta must be in [0, 1) (got {c['beta']!r})")
        if c["momentum"] not in MOMENTUM_MODES:
            raise ConfigError(f"{path}.momentum must be one of {'|'.join(MOMENTUM_MODES)} (got {c['momentum']!r})")
    if alg == "choco_sgd":
        if not 0.0 < float(c["gamma"]) <= 1.0:
            raise ConfigError(f"{path}.gamma must be in (0, 1] (got {c['gamma']!r})")
        _check_compressor(c, path)
        # s = sum_j W_ij x_hat_j is only valid for a fixed W: the graph is never refreshed
        if c.setdefault("update_graph", False):
            raise ConfigError(f"{path}.update_graph: choco_sgd needs a fixed graph (its sum of the neighbors' estimates "
                              f"is only valid for a fixed mixing matrix)")
    if alg == "beer":
        if not 0.0 < float(c["gamma"]) <= 1.0:
            raise ConfigError(f"{path}.gamma must be in (0, 1] (got {c['gamma']!r})")
        _check_compressor(c, path)
        # s_h = sum_j W_ij h_j and s_g = sum_j W_ij g_j are only valid for a fixed W: the graph is never refreshed
        if c.setdefault("update_graph", False):
            raise ConfigError(f"{path}.update_graph: beer needs a fixed graph (its sums of the neighbors' estimates "
                              f"are only valid for a fixed mixing matrix)")
    if alg == "kgt":
        ls = c["local_steps"]
        if isinstance(ls, bool) or not isinstance(ls, int) or ls < 1:
            raise ConfigError(f"{path}.local_steps must be an integer >= 1 (got {ls!r})")
        if not float(c["alpha"]) > 0.0:
            raise ConfigError(f"{path}.alpha must be > 0 (got {c['alpha']!r})")
        if not isinstance(c["correction"], bool):
            raise ConfigError(f"{path}.correction must be true or false (got {c['correction']!r})")
    if alg == "dadaptive":
        _check_dadaptive(c, path)
    if alg == "relaysum":
        _check_relaysum(c, path)
    if alg == "clipped_gossip":
        if c["clip"] not in ("none", "adaptive"):
            raise ConfigError(f"{path}.clip must be one of none|adaptive (got {c['clip']!r})")
        if c["clip"] == "adaptive":
            if "delta" not in c:
                raise ConfigError(f"missing required key {path}.delta (clip: adaptive)")
            dl = c["delta"]
            if isinstance(dl, bool) or not isinstance(dl, (int, float)) or not 0.0 <= float(dl) < 1.0:
                raise ConfigError(f"{path}.delta must be in [0, 1) (got {dl!r})")
    if alg == "bridge":
        _check_bridge(c, path)
    if alg == "powergossip":
        _check_powergossip(c, path)
    if alg == "detag":
        _check_detag(c, path)
    if alg == "gt_hsgd":
        _check_gt_hsgd(c, path)
    if alg == "gossip_pga":
        _check_gossip_pga(c, path)
    if alg == "dp_dsgd":
        _check_dp_dsgd(c, path)
    if alg == "moniqua":
        _check_moniqua(c, path)
    if alg == "sparq_sgd":
        _check_sparq(c, path)
    if alg == "cross_gradient":
        _check_cross_gradient(c, path)
    if alg == "slowmo":
        _check_slowmo(c, path)
    if alg in BYZANTINE_ALGS and c.get("byzantine") is not None:
        from ..optimizers.clipped_gossip import check_byzantine
        try:
            check_byzantine(c["byzantine"], None)
        except ValueError as e:
            raise ConfigError(f"{path}.{e}") from None
    if int(c["outer_iterations"]) <= 0:
        raise ConfigError(f"{path}.outer_iterations must be positive")
    return c


# extension keys of a problem config (absent from the reference's schema) and their legal values
PROBLEM_CHOICES = {
    "input_pipeline": ("auto", "resident", "staged", "host"),
    "host_gather": ("gpu_pull",),
    "host_loss": ("mirror",),
}


def _check_extensions(c: Dict[str, Any], path: str) -> None:
    for k, legal in PROBLEM_CHOICES.items():
        if k in c and c[k] not in legal:
            raise ConfigError(f"{path}.{k} must be one of {'|'.join(legal)} (got {c[k]!r})")
    if "samples_per_cta" in c and not (c["samples_per_cta"] == 0 or 4 <= int(c["samples_per_cta"]) <= 8):
        raise ConfigError(f"{path}.samples_per_cta must be 0 (automatic) or 4..8")
    f = c.get("fault_injection")
    if f is not None:
        if not isinstance(f, dict) or not 0.0 <= float(f.get("link_drop_prob", 0.0)) <= 1.0:
            raise ConfigError(f"{path}.fault_injection needs link_drop_prob in [0, 1]")


def validate_problem(conf: Dict[str, Any], path: str, kind: str) -> Dict[str, Any]:
    c = _fill(conf, {"problem_name": REQUIRED, "train_batch_size": REQUIRED, "val_batch_size": REQUIRED,
                     "metrics": REQUIRED, "metrics_config": REQUIRED, "optimizer_config": REQUIRED,
                     "verbose_evals": True}, path)
    _check_extensions(c, path)
    allowed = MNIST_METRICS if kind == "mnist" else DENSITY_METRICS
    for m in c["metrics"]:
        if m not in allowed:
            raise ConfigError(f"{path}.metrics: unknown metric {m!r} for a {kind} problem")
    mc = dict(c["metrics_config"])
    if "evaluate_frequency" not in mc:
        raise ConfigError(f"missing required key {path}.metrics_config.evaluate_frequency")
    if kind == "online_density":
        mc.setdefault("tloss_decay", 0.2)
        mc.setdefault("mesh_only_at_end", True)
        c = _fill(c, {"comm_radius": REQUIRED, "dynamic_graph": True, "save_models": False}, path)
    c["metrics_config"] = mc
    c["optimizer_config"] = validate_optimizer(c["optimizer_config"], path + ".optimizer_config")
    _check_fixed_graph(c, path, kind)
    return c


SOLO_DEFAULT = {"train_solo": False, "optimizer": "adam", "lr": 0.005, "epochs": 1,
                "train_batch_size": 100, "val_batch_size": 100, "verbose": True, "backend": "torch"}
# torch: per-node autograd; fused: every node at once on the sm_90a kernels (ops/local_train.py)
SOLO_BACKENDS = ("torch", "fused")


def validate_experiment(conf: Dict[str, Any], kind: str) -> Dict[str, Any]:
    """``kind``: mnist | mnist_scaling | density | online_density."""
    if "experiment" not in conf:
        raise ConfigError("missing top-level key `experiment`")
    out = copy.deepcopy(conf)
    exp = _fill(out["experiment"], {"name": REQUIRED, "output_metadir": REQUIRED, "writeout": True,
                                     "use_cuda": True, "loss": REQUIRED, "model": REQUIRED}, "experiment")
    if kind in ("mnist", "density"):
        exp = _fill(exp, {"graph": REQUIRED}, "experiment")
    if kind in ("mnist", "density", "online_density"):
        exp["individual_training"] = _fill(exp.get("individual_training", {}), SOLO_DEFAULT,
                                           "experiment.individual_training")
        if exp["individual_training"]["backend"] not in SOLO_BACKENDS:
            raise ConfigError(f"experiment.individual_training.backend must be one of {'|'.join(SOLO_BACKENDS)} "
                              f"(got {exp['individual_training']['backend']!r})")
    if kind == "mnist":
        exp = _fill(exp, {"data_dir": "../data/", "data_split_type": "random"}, "experiment")
        if exp["data_split_type"] not in ("random", "hetero"):
            raise ConfigError("experiment.data_split_type must be random|hetero")
    if kind == "mnist_scaling":
        exp = _fill(exp, {"data_dir": "../data/", "scaling": REQUIRED}, "experiment")
    if kind.startswith("mnist"):
        exp.setdefault("data_source", "auto")
        if exp["data_source"] not in ("auto", "mnist", "synthetic", "synthetic_hard"):
            raise ConfigError("experiment.data_source must be auto|mnist|synthetic|synthetic_hard")
        if exp.get("dtype", "float32") not in ("float32", "float64"):
            raise ConfigError("experiment.dtype must be float32|float64")
    if kind in ("density", "online_density"):
        exp = _fill(exp, {"data": REQUIRED}, "experiment")
        if kind == "online_density":
            exp.setdefault("seed", 0)
    out["experiment"] = exp
    pk = "mnist" if kind.startswith("mnist") else kind
    if kind == "mnist_scaling":
        out["problem"] = validate_problem(dict(out.get("problem", {}), problem_name=out.get("problem", {}).get("problem_name", "trial")),
                                          "problem", pk)
    else:
        if not out.get("problem_configs"):
            raise ConfigError("missing top-level key `problem_configs`")
        out["problem_configs"] = {k: validate_problem(v, f"problem_configs.{k}", pk)
                                  for k, v in out["problem_configs"].items()}
    _check_directed_graph(out)
    _check_byzantine_nodes(out)
    return out


def _check_byzantine_nodes(conf: Dict[str, Any]) -> None:
    """Byzantine node ids against the node count of ``experiment.graph``: in range, and not every node."""
    g = conf["experiment"].get("graph")
    if not isinstance(g, dict) or "num_nodes" not in g:
        return
    from ..optimizers.clipped_gossip import check_byzantine
    probs = conf.get("problem_configs") or ({"problem": conf["problem"]} if "problem" in conf else {})
    for k, p in probs.items():
        byz = p["optimizer_config"].get("byzantine")
        if byz is not None:
            path = f"problem_configs.{k}" if "problem_configs" in conf else k
            try:
                check_byzantine(byz, int(g["num_nodes"]))
            except ValueError as e:
                raise ConfigError(f"{path}.optimizer_config.{e}") from None


def _check_directed_graph(conf: Dict[str, Any]) -> None:
    """A directed ``experiment.graph`` has no Metropolis matrix: only the push-sum algorithms (SGP, Push-DIGing) run on
    it, and link-drop fault injection (which drops undirected edges) does not apply to it."""
    g = conf["experiment"].get("graph")
    if not isinstance(g, dict) or g.get("type") not in DIRECTED_GRAPH_TYPES:
        return
    probs = conf.get("problem_configs") or ({"problem": conf["problem"]} if "problem" in conf else {})
    for k, p in probs.items():
        path = f"problem_configs.{k}" if "problem_configs" in conf else k
        alg = p["optimizer_config"]["alg_name"]
        if alg not in DIRECTED_ALGS:
            raise ConfigError(f"experiment.graph.type: the directed graph {g['type']!r} runs with alg_name "
                              f"{' or '.join(DIRECTED_ALGS)} only ({path}.optimizer_config.alg_name is {alg!r})")
        if p.get("fault_injection"):
            raise ConfigError(f"{path}.fault_injection: link-drop fault injection drops undirected edges and does not "
                              f"apply to the directed graph {g['type']!r}")


def load_experiment(yaml_pth: str, kind: str) -> Dict[str, Any]:
    with open(yaml_pth) as f:
        raw = yaml.safe_load(f)
    return validate_experiment(raw, kind)
