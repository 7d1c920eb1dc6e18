"""gym_jiminy's `StackObservation` wrapper (python/gym_jiminy/common/gym_jiminy/common/wrappers/observation_stack.py) for
the batched envs.

The reference updates its frames at every observer refresh, i.e. several times per env-step (`observe_dt = control_dt`),
so the stacking cannot be done on the observations an env-step returns: the step kernel does it, at every sensor
breakpoint, right after the MahonyFilter update (`BatchedEngine.set_obs_stack`).  This module resolves the wrapper's
arguments against an env's observation tree and reads the wrapper entry of a reference pipeline config.

Each stacked leaf of the observation is replaced by its frames `[n_env, num_stack, *leaf shape]`, oldest first.  The
leaves that can be stacked are `t`, a sensor-type block of `measurements`, `actions.pd_controller` (PD envs built with
`augment_observation=True`), `states.pd_controller`, `features.mahony_filter` and the leaves of the observer blocks
(`jiminy_b200.observers`: the filter's `quat`, `rpy`, `omega` and state `bias`, the body observer's `quat`, `rpy` and
`omega`); any other selected leaf, the agent's
`states.agent.q / v` included (and so the reference's default of every leaf), raises NotImplementedError.
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Sequence, Tuple, Union

from . import core

LEAVES = {
    ("t",): core.STACK_T,
    ("measurements", "ImuSensor"): core.STACK_IMU,
    ("measurements", "ForceSensor"): core.STACK_FORCE,
    ("measurements", "EncoderSensor"): core.STACK_ENCODER,
    ("measurements", "EffortSensor"): core.STACK_EFFORT,
    ("measurements", "ContactSensor"): core.STACK_CONTACT,
    ("actions", "pd_controller"): core.STACK_PD_ACTION,
    ("states", "pd_controller"): core.STACK_PD_STATE,
    ("features", "mahony_filter"): core.STACK_MAHONY,
}

_CLASS_PATHS = ("gym_jiminy.common.wrappers.StackObservation",
                "gym_jiminy.common.wrappers.observation_stack.StackObservation")


def leaf_paths(obs: Dict[str, Any], prefix: Tuple[str, ...] = ()) -> List[Tuple[str, ...]]:
    """Paths of the leaves of a nested observation dict, in its order."""
    out: List[Tuple[str, ...]] = []
    for key, value in obs.items():
        if isinstance(value, dict):
            out += leaf_paths(value, prefix + (key,))
        else:
            out.append(prefix + (key,))
    return out


class StackObservation:
    """`StackObservation(num_stack, nested_filter_keys=None, skip_frames_ratio=-1)` with the reference's arguments:
    `nested_filter_keys` lists nested paths (a key or a sequence of keys); every leaf under one of them is stacked
    (None: every leaf).  `skip_frames_ratio`: observer refreshes skipped between two stack updates, -1 for one update per
    env-step."""

    def __init__(self, num_stack: int, nested_filter_keys: Optional[Sequence[Union[str, Sequence[str]]]] = None,
                 skip_frames_ratio: int = -1):
        if int(num_stack) < 1:
            raise ValueError("num_stack must be at least 1")
        if int(skip_frames_ratio) < -1:
            raise ValueError("skip_frames_ratio must be -1 or positive")
        if isinstance(nested_filter_keys, str):
            raise ValueError("nested_filter_keys must be a sequence of nested paths")
        self.num_stack, self.skip_frames_ratio = int(num_stack), int(skip_frames_ratio)
        self.nested_filter_keys = None if nested_filter_keys is None else \
            [(k,) if isinstance(k, (str, int)) else tuple(k) for k in nested_filter_keys]

    def resolve(self, obs: Dict[str, Any], extra: Optional[Dict[Tuple[str, ...], int]] = None
                ) -> List[Tuple[Tuple[str, ...], int]]:
        """(path, leaf code) of every stacked leaf of the observation `obs`, in its order (`observation_stack.py:96-105`);
        `extra` maps the paths of the env's observer leaves (`jiminy_b200.observers.stack_leaves`) to their codes."""
        known = LEAVES if not extra else {**LEAVES, **extra}
        paths = leaf_paths(obs)
        keys = self.nested_filter_keys if self.nested_filter_keys is not None else [(k,) for k in obs]
        chosen = [p for p in paths if any(p[:len(e)] == e for e in keys)]
        if not chosen:
            raise ValueError("At least one observation leaf must be stacked.")
        for p in chosen:
            if p not in known:
                raise NotImplementedError(f"stacking the observation leaf {'.'.join(map(str, p))} is not supported on the "
                                          f"batched envs (supported: {', '.join('.'.join(k) for k in known)})")
        return [(p, known[p]) for p in chosen]


def from_config(layers_config: Sequence[dict]) -> Optional[StackObservation]:
    """The `StackObservation` entry of the `layers_config` list of a reference pipeline config (`{"wrapper": {"cls": path,
    "kwargs": {...}}}`), or None without one.  A layer whose wrapper names another class raises NotImplementedError; the
    block layers (a `block` and the kwargs of its default wrapper) are the envs' constructor arguments and are skipped."""
    found = None
    for layer in layers_config:
        wrapper = layer.get("wrapper") or {}
        cls = wrapper.get("cls")
        if cls is None:
            continue
        if str(cls) not in _CLASS_PATHS:
            raise NotImplementedError(f"wrapper '{cls}' is not supported on the batched envs")
        if found is not None:
            raise NotImplementedError("only one StackObservation wrapper is supported")
        found = StackObservation(**dict(wrapper.get("kwargs") or {}))
    return found
