"""gym_jiminy's observer blocks (python/gym_jiminy/common/gym_jiminy/common/blocks) for the batched PD envs:
`MahonyFilter` with its full option set and `BodyObserver`.

Both are stateful and refresh at every observer breakpoint, several times per env-step, so they run inside the step
kernel right after the filter's update, at the (re)start refresh and at every sensor breakpoint, on the measured values
(`BatchedEngine.set_mahony_filter_full`, `BatchedEngine.set_body_observer`).  The classes below carry the reference's
constructor arguments; the PD envs take them as `mahony=` and `body_observer=` and return the reference's observation
layout: `features.<name> = {"quat", ["rpy"], "omega"}` with `[n_env, k, nimu]` leaves, and the filter's state
`states.<name> = {"bias"}`.  One IMU per robot and `update_ratio = 1` only.
"""
from __future__ import annotations

import math
from typing import Any, Callable, Dict, List, Optional, Sequence, Union

import numpy as np

from . import core

_MAHONY_PATHS = ("gym_jiminy.common.blocks.MahonyFilter", "gym_jiminy.common.blocks.mahony_filter.MahonyFilter")
_BODY_PATHS = ("gym_jiminy.common.blocks.BodyObserver", "gym_jiminy.common.blocks.body_orientation_observer.BodyObserver")
_OTHER_OBSERVERS = ("DeformationEstimator", "QuantityObserver")
_DEFAULT_QUAT_KEY = ("features", "mahony_filter", "quat")
_DEFAULT_OMEGA_KEY = ("features", "mahony_filter", "omega")


def _gain(x: Union[float, Sequence[float]], name: str) -> float:
    a = np.asarray(x, dtype=np.float64).ravel()
    if a.size != 1:
        raise NotImplementedError(f"{name}: one gain per IMU, and the batched envs handle one IMU per robot")
    return float(a[0])


def _check_update_ratio(update_ratio: int) -> None:
    if int(update_ratio) != 1:
        raise NotImplementedError("observer blocks run at every sensor refresh: only update_ratio = 1 is supported")


class MahonyFilter:
    """`MahonyFilter(kp=1.0, ki=0.1, *, ignore_twist=False, exact_init=True, compute_rpy=False, update_ratio=1)`
    (blocks/mahony_filter.py:138-226), named `name` in the observation."""

    def __init__(self, kp: Union[float, Sequence[float]] = 1.0, ki: Union[float, Sequence[float]] = 0.1, *,
                 ignore_twist: bool = False, exact_init: bool = True, compute_rpy: bool = False, update_ratio: int = 1,
                 name: str = "mahony_filter"):
        _check_update_ratio(update_ratio)
        self.kp, self.ki = _gain(kp, "kp"), _gain(ki, "ki")
        self.ignore_twist, self.exact_init, self.compute_rpy = bool(ignore_twist), bool(exact_init), bool(compute_rpy)
        self.name = str(name)

    def __eq__(self, other: object) -> bool:
        return isinstance(other, MahonyFilter) and vars(self) == vars(other)

    def __repr__(self) -> str:
        return f"MahonyFilter({', '.join(f'{k}={v!r}' for k, v in vars(self).items())})"

    def configure(self, engine: core.BatchedEngine) -> None:
        engine.set_mahony_filter_full(self.kp, self.ki, self.exact_init, self.ignore_twist, self.compute_rpy)


class BodyObserver:
    """`BodyObserver(*, nested_imu_quat_key, nested_imu_omega_key, twist_time_constant=None, compute_rpy=True,
    update_ratio=1)` (blocks/body_orientation_observer.py:84-188), named `name` in the observation.  The nested keys must
    be the defaults: the body observer reads the MahonyFilter named `mahony_filter`."""

    def __init__(self, *, nested_imu_quat_key: Sequence[str] = _DEFAULT_QUAT_KEY,
                 nested_imu_omega_key: Sequence[str] = _DEFAULT_OMEGA_KEY, twist_time_constant: Optional[float] = None,
                 compute_rpy: bool = True, update_ratio: int = 1, name: str = "body_observer"):
        _check_update_ratio(update_ratio)
        if tuple(nested_imu_quat_key) != _DEFAULT_QUAT_KEY or tuple(nested_imu_omega_key) != _DEFAULT_OMEGA_KEY:
            raise NotImplementedError("the body observer reads features.mahony_filter.quat / omega only")
        if twist_time_constant is not None:
            twist_time_constant = float(twist_time_constant)
            if not math.isfinite(twist_time_constant) or twist_time_constant < 0.0:
                raise ValueError("twist_time_constant must be None, 0 or finite and positive")
        self.twist_time_constant, self.compute_rpy, self.name = twist_time_constant, bool(compute_rpy), str(name)

    def __eq__(self, other: object) -> bool:
        return isinstance(other, BodyObserver) and vars(self) == vars(other)

    def __repr__(self) -> str:
        return f"BodyObserver({', '.join(f'{k}={v!r}' for k, v in vars(self).items())})"

    def configure(self, engine: core.BatchedEngine) -> None:
        engine.set_body_observer(True, self.twist_time_constant, self.compute_rpy)


def observation_shapes(mahony: MahonyFilter, body: Optional[BodyObserver], nimu: int) -> Dict[str, Dict[str, Any]]:
    """The `features` and `states` entries the observers add, as per-env shapes."""
    feats = {mahony.name: _feature_shapes(mahony.compute_rpy, nimu)}
    if body is not None:
        feats[body.name] = _feature_shapes(body.compute_rpy, nimu)
    return {"features": feats, "states": {mahony.name: {"bias": (3, nimu)}}}


def _feature_shapes(rpy: bool, nimu: int) -> Dict[str, Any]:
    out = {"quat": (4, nimu)}
    if rpy:
        out["rpy"] = (3, nimu)
    out["omega"] = (3, nimu)
    return out


def has_record(mahony: MahonyFilter, body: Optional[BodyObserver]) -> bool:
    """Whether the observation reads the observer record (jb_get_observers)."""
    return mahony.compute_rpy or body is not None


def observation(mahony: MahonyFilter, body: Optional[BodyObserver], state, record, copy: Callable) -> Dict[str, Dict[str, Any]]:
    """The observers' leaves from the filter's state [n_env, nimu, 10] and the observer record [n_env, nimu, OBSV_N]
    (numpy arrays or torch tensors; `copy` detaches a leaf from its buffer)."""
    def fields(a, lo, k):
        return copy(a[:, :, lo:lo + k].swapaxes(1, 2))

    feat = {"quat": fields(state, 0, 4)}
    if mahony.compute_rpy:
        feat["rpy"] = fields(record, core.OBSV_MAHONY_RPY, 3)
    feat["omega"] = fields(state, 7, 3)
    feats = {mahony.name: feat}
    if body is not None:
        b = {"quat": fields(record, core.OBSV_BODY_QUAT, 4)}
        if body.compute_rpy:
            b["rpy"] = fields(record, core.OBSV_BODY_RPY, 3)
        b["omega"] = fields(record, core.OBSV_BODY_OMEGA, 3)
        feats[body.name] = b
    return {"features": feats, "states": {mahony.name: {"bias": fields(state, 4, 3)}}}


def stack_leaves(mahony: MahonyFilter, body: Optional[BodyObserver]) -> Dict[tuple, int]:
    """Observation path -> stacked leaf code (jb_set_obs_stack) of every observer leaf."""
    m = mahony.name
    out = {("features", m, "quat"): core.STACK_MAHONY, ("features", m, "omega"): core.STACK_MAHONY_OMEGA,
           ("states", m, "bias"): core.STACK_MAHONY_BIAS}
    if mahony.compute_rpy:
        out[("features", m, "rpy")] = core.STACK_MAHONY_RPY
    if body is not None:
        out[("features", body.name, "quat")] = core.STACK_BODY_QUAT
        out[("features", body.name, "omega")] = core.STACK_BODY_OMEGA
        if body.compute_rpy:
            out[("features", body.name, "rpy")] = core.STACK_BODY_RPY
    return out


def from_config(layers_config: Sequence[dict]) -> List[Union[MahonyFilter, BodyObserver]]:
    """The observer layers of the `layers_config` list of a reference pipeline config (`{"block": {"cls": path, "kwargs":
    {...}}}`), in order.  Controller blocks are the envs' constructor arguments and are skipped, as are wrapper-only
    layers; another observer class raises NotImplementedError."""
    found: List[Union[MahonyFilter, BodyObserver]] = []
    for layer in layers_config:
        block = layer.get("block") or {}
        cls = block.get("cls")
        if cls is None:
            continue
        cls, kwargs = str(cls), dict(block.get("kwargs") or {})
        if cls in _MAHONY_PATHS:
            found.append(MahonyFilter(**kwargs))
        elif cls in _BODY_PATHS:
            found.append(BodyObserver(**kwargs))
        elif cls.rsplit(".", 1)[-1] in _OTHER_OBSERVERS:
            raise NotImplementedError(f"observer block '{cls}' is not supported on the batched envs")
    return found
