"""Reward and termination compositions: the trajectory-free terms of gym_jiminy (`gym_jiminy.common.compositions`), with
the reference's semantics, restated in numpy.

The numpy evaluator (`Compositions`) is what the host envs run after every env-step, and the reference the device kernel
(`jb_compositions_device`) is tested against.  It computes what the kernel computes, operation for operation: sums and
products in the same order and without contraction into fused multiply-adds, so that both give the same bits.  The
exceptions are the math-library functions: `pow` (the radial basis function of `MinimizeMechanicalPowerConsumption`, an
L^p mixture of order other than 1, a geometric mean of more than one value) and `sin` / `cos` / `atan2` (roll and
pitch), whose device and host versions may differ by a few ulp.

Semantics (bases/compositions.py, bases/pipeline.py:778-829 of the reference):
- the env's own rule runs first (`envs.terminated_truncated`); when it ends the episode, no condition is evaluated;
- the termination conditions run in order and stop at the first that fires; `info["terminated"]` holds its index
  (-1: none); every supported condition terminates, so `info["truncated"]` is always -1;
- a condition is skipped (it continues) while `t < grace_period`, or when `training_only` is set and the env is not
  training; a quantity outside `[low, high]` ends the episode (`_array_contains`: a bound that is None is not checked;
  for an array quantity, roll and pitch, a NaN is out of bounds, for a scalar one it is not);
- every reward term here is non-terminal: on a terminal step it is not evaluated, and a mixture skips the components that
  were not; a reward that nothing evaluated is 0.0;
- `info[name]` holds each term's value per env: the reward's value, 1.0 / 0.0 for a condition that fired / continued,
  NaN where the term was not evaluated.

The power terms average over a per-env stack of `max(ceil(horizon / step_dt), 1) + 1` entries (`StackedQuantity`): it is
emptied at every (re)start of the env and takes the power of the state it starts from, then one entry per env-step,
whether the term is evaluated or not; the mean sums the entries oldest first.  The power uses the command held since the
last controller update (the motor efforts `RobotState.command` holds: the PD block's torque in PD mode, the action in
effort mode) and the motor-side velocities.
"""
from __future__ import annotations

import math
from enum import IntEnum
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np

CUTOFF_ESP = 1.0e-2

# node kinds of the device spec (include/jiminy_b200.h, jb_set_compositions)
_SURVIVE, _POWER, _ADDITIVE, _MULTIPLICATIVE = 1, 2, 3, 4
_ROLL_PITCH, _FALLING, _FLYING, _SAFETY, _POWER_TERM = 10, 11, 12, 13, 14
MAX_NODES = 32


class EnergyGenerationMode(IntEnum):
    """What happens to the energy a motor generates when braking (quantities/generic.py)."""
    CHARGE = 0
    LOST_EACH = 1
    LOST_GLOBAL = 2
    PENALIZE = 3


def _mode(x) -> EnergyGenerationMode:
    return EnergyGenerationMode[x.upper()] if isinstance(x, str) else EnergyGenerationMode(int(x))


# ------------------------------------------------------------------ terms
class SurviveReward:
    """1.0 at every non-terminal step."""
    name = "reward_survive"
    kind = _SURVIVE

    def __init__(self):
        pass


class MinimizeMechanicalPowerConsumption:
    """radial_basis_function(average mechanical power over `horizon`, cutoff, order=2)."""
    name = "reward_power_consumption"
    kind = _POWER

    def __init__(self, cutoff: float, horizon: float, generator_mode=EnergyGenerationMode.CHARGE):
        self.cutoff, self.horizon, self.generator_mode = float(cutoff), float(horizon), _mode(generator_mode)
        if not (self.cutoff > 0.0 and math.isfinite(self.cutoff)):
            raise ValueError("'cutoff' must be strictly positive.")
        if not (self.horizon > 0.0 and math.isfinite(self.horizon)):
            raise ValueError("'horizon' must be strictly positive.")


class _Mixture:
    kind = 0

    def __init__(self, name: str, components: Sequence):
        if not components:
            raise ValueError("At least one reward component must be specified.")
        self.name, self.components = str(name), tuple(components)


class AdditiveMixtureReward(_Mixture):
    """weighted_norm(weights, order, component values), `order` a positive number or 'inf'.  Components of weight 0 are
    dropped, as in the reference."""
    kind = _ADDITIVE

    def __init__(self, name: str, components: Sequence, order: Union[int, float, str] = 1, weights: Optional[Sequence[float]] = None):
        if weights is None:
            weights = (1.0 / len(components),) * len(components)
        order = float("inf") if order == "inf" else float(order)
        if not order > 0.0:
            raise ValueError("'order' must be strictly positive or 'inf'.")
        if len(weights) != len(components):
            raise ValueError("Exactly one weight per reward component must be specified.")
        weights = [float(w) for w in weights]
        if any(not (w >= 0.0 and math.isfinite(w)) for w in weights):
            raise ValueError("The weights must be finite and non-negative.")
        kept = [(w, c) for w, c in zip(weights, components) if w > 0.0]
        if not kept:
            raise ValueError("At least one reward component must have a positive weight.")
        super().__init__(name, [c for _, c in kept])
        self.order, self.weights = order, tuple(w for w, _ in kept)


class MultiplicativeMixtureReward(_Mixture):
    """geometric_mean(component values)."""
    kind = _MULTIPLICATIVE


class _Termination:
    kind = 0
    name = ""

    def __init__(self, grace_period: float, training_only: bool):
        self.grace_period, self.training_only = float(grace_period), bool(training_only)
        if not (self.grace_period >= 0.0 and math.isfinite(self.grace_period)):
            raise ValueError("'grace_period' must be finite and non-negative.")


def _bound(x, n: int, what: str) -> np.ndarray:
    if x is None:
        return np.full(n, np.nan)
    b = np.asarray(x, dtype=np.float64).reshape(-1)
    if b.size == 1 and n > 1:
        b = np.full(n, b[0])
    if b.size != n:
        raise ValueError(f"'{what}' must hold {n} value(s), not {b.size}.")
    if np.isnan(b).any():
        raise ValueError(f"'{what}' must not hold NaN (None means no bound).")
    return b


class BaseRollPitchTermination(_Termination):
    """Roll and pitch of the root joint (matrix_to_rpy of the base rotation matrix) outside [low, high] (2 values each)."""
    name = "termination_base_roll_pitch"
    kind = _ROLL_PITCH

    def __init__(self, low, high, grace_period: float = 0.0, training_only: bool = False):
        super().__init__(grace_period, training_only)
        self.low, self.high = _bound(low, 2, "low"), _bound(high, 2, "high")


class FallingTermination(_Termination):
    """Base height relative to the lowest contact frame (BaseRelativeHeight) under `min_base_height`."""
    name = "termination_base_height"
    kind = _FALLING

    def __init__(self, min_base_height: float, grace_period: float = 0.0, training_only: bool = False):
        super().__init__(grace_period, training_only)
        self.min_base_height = float(_bound(min_base_height, 1, "min_base_height")[0])


class FlyingTermination(_Termination):
    """Height of the lowest contact frame above the flat ground over `max_height`."""
    name = "termination_flying"
    kind = _FLYING

    def __init__(self, max_height: float, grace_period: float = 0.0, training_only: bool = False):
        super().__init__(grace_period, training_only)
        self.max_height = float(_bound(max_height, 1, "max_height")[0])


class MechanicalSafetyTermination(_Termination):
    """An actuated joint within `position_margin` of a bound while moving towards it faster than `velocity_max`."""
    name = "termination_mechanical_safety"
    kind = _SAFETY

    def __init__(self, position_margin: float, velocity_max: float, grace_period: float = 0.0, training_only: bool = False):
        super().__init__(grace_period, training_only)
        self.position_margin = float(_bound(position_margin, 1, "position_margin")[0])
        self.velocity_max = float(_bound(velocity_max, 1, "velocity_max")[0])


class MechanicalPowerConsumptionTermination(_Termination):
    """Mechanical power (instantaneous, or averaged over `horizon`) over `max_power`."""
    name = "termination_power_consumption"
    kind = _POWER_TERM

    def __init__(self, max_power: float, horizon: Optional[float] = None, generator_mode=EnergyGenerationMode.CHARGE,
                 grace_period: float = 0.0, training_only: bool = False):
        super().__init__(grace_period, training_only)
        self.max_power = float(_bound(max_power, 1, "max_power")[0])
        self.horizon = None if horizon is None else float(horizon)
        if self.horizon is not None and not (self.horizon > 0.0 and math.isfinite(self.horizon)):
            raise ValueError("'horizon' must be strictly positive.")
        self.generator_mode = _mode(generator_mode)


REWARDS = (SurviveReward, MinimizeMechanicalPowerConsumption, AdditiveMixtureReward, MultiplicativeMixtureReward)
TERMINATIONS = (BaseRollPitchTermination, FallingTermination, FlyingTermination, MechanicalSafetyTermination,
                MechanicalPowerConsumptionTermination)


def from_config(config: dict) -> Tuple[Optional[object], Tuple]:
    """(reward, terminations) from the `reward` / `terminations` sections of a reference env config (`{"cls": path,
    "kwargs": {...}}`, nested components included), written with the reference's class paths
    (`gym_jiminy.common.compositions.<Class>`, or its `generic` / `locomotion` / `mixin` submodule).  Any other class
    raises NotImplementedError."""
    known = {c.__name__: c for c in REWARDS + TERMINATIONS}

    def make(entry):
        path = str(entry["cls"])
        mod, _, cls = path.rpartition(".")
        if cls not in known or mod not in ("gym_jiminy.common.compositions", "gym_jiminy.common.compositions.generic",
                                           "gym_jiminy.common.compositions.locomotion", "gym_jiminy.common.compositions.mixin"):
            raise NotImplementedError(f"composition '{path}' is not supported on the batched envs")
        kw = dict(entry.get("kwargs") or {})
        if "components" in kw:
            kw["components"] = [make(c) for c in kw["components"]]
        return known[cls](**kw)

    reward = make(config["reward"]) if config.get("reward") is not None else None
    terms = tuple(make(t) for t in config.get("terminations") or ())
    if reward is not None and not isinstance(reward, REWARDS):
        raise ValueError("'reward' must be a reward")
    if any(not isinstance(t, TERMINATIONS) for t in terms):
        raise ValueError("'terminations' must hold termination conditions")
    return reward, terms


# ------------------------------------------------------------------ numpy restatements of the reference's functions
def quat_to_matrix(quat: np.ndarray) -> np.ndarray:
    """Rotation matrices [n, 3, 3] of quaternions [n, 4] (x, y, z, w): Eigen's toRotationMatrix, as pinocchio computes it."""
    x, y, z, w = (quat[:, k] for k in range(4))
    tx, ty, tz = x + x, y + y, z + z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return np.stack([np.stack([1.0 - (tyy + tzz), txy - twz, txz + twy], -1),
                     np.stack([txy + twz, 1.0 - (txx + tzz), tyz - twx], -1),
                     np.stack([txz - twy, tyz + twx, 1.0 - (txx + tyy)], -1)], -2)


def matrix_to_rpy(mat: np.ndarray) -> np.ndarray:
    """Roll, pitch, yaw [n, 3] of rotation matrices [n, 3, 3] (utils/math.py matrix_to_rpy: Eigen's eulerAngles(2, 1, 0))."""
    cos_pitch = np.sqrt(mat[:, 2, 2] * mat[:, 2, 2] + mat[:, 2, 1] * mat[:, 2, 1])
    pitch = np.arctan2(-mat[:, 2, 0], cos_pitch)
    yaw = np.arctan2(mat[:, 1, 0], mat[:, 0, 0])
    sy, cy = np.sin(yaw), np.cos(yaw)
    roll = np.arctan2(sy * mat[:, 0, 2] - cy * mat[:, 1, 2], cy * mat[:, 1, 1] - sy * mat[:, 0, 1])
    return np.stack([roll, pitch, yaw], -1)


def compute_power(generator_mode, motor_velocities: np.ndarray, motor_efforts: np.ndarray) -> np.ndarray:
    """Mechanical power [n] of motor-side velocities and efforts [n, nmotors] (quantities/generic.py compute_power),
    summed motor after motor."""
    mode = int(generator_mode)
    total = np.zeros(motor_velocities.shape[0])
    for m in range(motor_velocities.shape[1]):
        p = motor_velocities[:, m] * motor_efforts[:, m]
        if mode == EnergyGenerationMode.LOST_EACH:
            p = np.where(p < 0.0, 0.0, p)
        elif mode == EnergyGenerationMode.PENALIZE:
            p = np.abs(p)
        total = total + p
    if mode == EnergyGenerationMode.LOST_GLOBAL:
        total = np.where(total < 0.0, 0.0, total)
    return total


def radial_basis_function(error: np.ndarray, cutoff: float) -> np.ndarray:
    """compositions/mixin.py radial_basis_function for a scalar error per env (order 2): CUTOFF_ESP ** (e^2 / cutoff^2)."""
    return np.power(CUTOFF_ESP, (error * error) / (cutoff * cutoff))


def weighted_norm(weights: Sequence[float], order: float, values: Sequence[Optional[float]]) -> Optional[float]:
    """compositions/mixin.py weighted_norm: the L^order norm of the values that are not None (None if there is none)."""
    total, any_value = 0.0, False
    for value, weight in zip(values, weights):
        if value is None:
            continue
        if order == float("inf"):
            total = weight * value if not any_value else max(total, weight * value)
        else:
            total += weight * (value if order == 1.0 else math.pow(value, order))
        any_value = True
    if not any_value:
        return None
    return total if order in (1.0, float("inf")) else math.pow(total, 1.0 / order)


def geometric_mean(values: Sequence[Optional[float]]) -> Optional[float]:
    """compositions/mixin.py geometric_mean of the values that are not None (None if there is none)."""
    total, n = 1.0, 0
    for value in values:
        if value is not None:
            total *= value
            n += 1
    return None if n == 0 else (total if n == 1 else math.pow(total, 1.0 / n))


def max_stack(horizon: float, step_dt: float) -> int:
    """Entries of the stack of AverageMechanicalPowerConsumption (quantities/generic.py)."""
    return max(int(np.ceil(horizon / step_dt)), 1) + 1


# ------------------------------------------------------------------ the evaluator
class Compositions:
    """A reward tree and termination conditions, flattened into the device spec and evaluated per env with numpy.
    `robot`: the batch's robot table; `height_min`: the env's own base-height rule (None: none); `training`: the env's
    training flag (`training_only` conditions run only when it is set)."""

    def __init__(self, reward, terminations: Sequence, robot, n_env: int, step_dt: float, simulation_duration_max: float,
                 height_min: Optional[float], training: bool = True):
        reward = SurviveReward() if reward is None else reward
        if not isinstance(reward, REWARDS):
            raise ValueError(f"'reward' must be one of {[c.__name__ for c in REWARDS]}, not {type(reward).__name__}")
        self.nodes: List = []

        def post_order(r):
            if not isinstance(r, REWARDS):
                raise ValueError(f"reward component {type(r).__name__} is not a reward")
            for c in getattr(r, "components", ()):
                post_order(c)
            self.nodes.append(r)
        post_order(reward)
        self.n_reward = len(self.nodes)
        for t in terminations:
            if not isinstance(t, TERMINATIONS):
                raise ValueError(f"{type(t).__name__} is not a supported termination condition")
            self.nodes.append(t)
        if len(self.nodes) > MAX_NODES:
            raise ValueError(f"at most {MAX_NODES} reward and termination terms")
        names = [n.name for n in self.nodes]
        if len(set(names)) != len(names):
            raise ValueError(f"the names of the terms must be unique: {names}")
        if any(isinstance(t, (FallingTermination, FlyingTermination)) for t in terminations) and not robot.contact_frame_names:
            raise ValueError("falling / flying terminations need contact frames")
        self.robot, self.n_env, self.step_dt = robot, n_env, float(step_dt)
        self.simulation_duration_max, self.height_min, self.training = float(simulation_duration_max), height_min, bool(training)
        self.names = names
        self.needs_contacts = any(isinstance(t, (FallingTermination, FlyingTermination)) for t in terminations)
        # the spec of jb_set_compositions
        n = len(self.nodes)
        self.node_int, self.node_dbl = np.zeros((n, 4), np.int32), np.zeros((n, 8))
        weights, self.stack_size = [], np.zeros(n, np.int64)
        for i, node in enumerate(self.nodes):
            ni, nd = self.node_int[i], self.node_dbl[i]
            ni[0] = node.kind
            nd[1:5] = np.nan
            if isinstance(node, _Mixture):
                ni[1] = len(node.components)
                if isinstance(node, AdditiveMixtureReward):
                    nd[1] = node.order
                    weights += node.weights
            if isinstance(node, _Termination):
                nd[0], ni[3] = node.grace_period, int(node.training_only)
            if isinstance(node, MinimizeMechanicalPowerConsumption):
                ni[2], nd[1], nd[2] = int(node.generator_mode), node.cutoff, node.horizon
            elif isinstance(node, BaseRollPitchTermination):
                nd[1:3], nd[3:5] = node.low, node.high
            elif isinstance(node, FallingTermination):
                nd[1] = node.min_base_height
            elif isinstance(node, FlyingTermination):
                nd[3] = node.max_height
            elif isinstance(node, MechanicalSafetyTermination):
                nd[1], nd[2] = node.position_margin, node.velocity_max
            elif isinstance(node, MechanicalPowerConsumptionTermination):
                ni[2], nd[3] = int(node.generator_mode), node.max_power
                nd[2] = np.nan if node.horizon is None else node.horizon
            horizon = getattr(node, "horizon", None)
            if horizon is not None:
                self.stack_size[i] = max_stack(horizon, self.step_dt)
        self.weights = np.array(weights, dtype=np.float64)
        iq = [robot.idx_q[m.joint] for m in robot.motors]
        iv = [robot.idx_v[m.joint] for m in robot.motors]
        self.motor_int = np.array([iq, iv], dtype=np.int32).T.reshape(-1, 2)
        self.motor_dbl = np.array([[m.reduction for m in robot.motors], robot.q_lower[iq], robot.q_upper[iq]]).T.reshape(-1, 3)
        self.env_dbl = np.array([self.step_dt, self.simulation_duration_max, np.nan if height_min is None else height_min])
        # per-env power stacks
        self.stacks = {i: np.zeros((n_env, int(m))) for i, m in enumerate(self.stack_size) if m}
        self.count = np.zeros((n, n_env), np.int64)

    def upload(self, engine) -> None:
        """The spec to the batch (`jb_set_compositions`); empties the device stacks."""
        engine.set_compositions(self.node_int, self.node_dbl, self.n_reward, self.weights, self.motor_int, self.motor_dbl,
                                self.env_dbl, self.training)

    # ---- quantities
    def power(self, node, v: np.ndarray, command: np.ndarray) -> np.ndarray:
        vm = v[:, self.motor_int[:, 1]] * self.motor_dbl[:, 0]
        return compute_power(node.generator_mode, vm, command)

    def _mean(self, i: int) -> np.ndarray:
        st, M, cnt = self.stacks[i], int(self.stack_size[i]), self.count[i]
        n = np.minimum(cnt, M)
        first = np.where(cnt < M, 0, cnt % M)
        s = np.zeros(self.n_env)
        rows = np.arange(self.n_env)
        for k in range(M):
            s = np.where(k < n, s + st[rows, (first + k) % M], s)
        return s / n

    def seed(self, mask: Optional[np.ndarray], v: np.ndarray, command: np.ndarray) -> None:
        """The envs of `mask` (None: all) have just (re)started: their stacks are emptied and take the power of the state
        (v [n_env, nv], held command [n_env, nmotors]) they start from."""
        sel = np.ones(self.n_env, bool) if mask is None else np.asarray(mask).astype(bool)
        for i in self.stacks:
            p = self.power(self.nodes[i], v, command)
            self.stacks[i][sel, 0] = p[sel]
            self.count[i, sel] = 1

    def evaluate(self, t: np.ndarray, q: np.ndarray, v: np.ndarray, command: np.ndarray, terminated: np.ndarray,
                 truncated: np.ndarray, contact_positions: Optional[np.ndarray] = None):
        """After an env-step: push the power of the accepted state on every stack, then run the termination conditions
        behind the env's own (terminated, truncated) and the reward tree.  Returns (reward, terminated, truncated, info)
        with info["terminated"] / info["truncated"] (index of the condition, -1: none) and info[name] per term."""
        n = self.n_env
        rows = np.arange(n)
        for i, st in self.stacks.items():
            M = int(self.stack_size[i])
            st[rows, self.count[i] % M] = self.power(self.nodes[i], v, command)
            self.count[i] += 1
        terminated, truncated = np.array(terminated, bool), np.array(truncated, bool)
        fired = np.full(n, -1, np.int32)
        values = np.full((len(self.nodes), n), np.nan)
        pending = ~(terminated | truncated)
        zmin = None
        if self.needs_contacts:
            z = contact_positions[:, :, 2]
            zmin = np.full(n, np.inf)
            for k in range(z.shape[1]):
                zmin = np.where((z[:, k] < zmin) | np.isnan(z[:, k]), z[:, k], zmin)
        for j, node in enumerate(self.nodes[self.n_reward:]):
            i = self.n_reward + j
            skip = (node.training_only and not self.training) | (t < node.grace_period)
            nd = self.node_dbl[i]
            lo, hi = nd[1], nd[3]
            if isinstance(node, BaseRollPitchTermination):
                rpy = matrix_to_rpy(quat_to_matrix(q[:, 3:7]))
                hit = np.zeros(n, bool)
                for k in range(2):
                    if not np.isnan(nd[1 + k]):
                        hit |= ~(nd[1 + k] <= rpy[:, k])
                    if not np.isnan(nd[3 + k]):
                        hit |= ~(rpy[:, k] <= nd[3 + k])
            elif isinstance(node, MechanicalSafetyTermination):
                hit = np.zeros(n, bool)
                for m in range(len(self.motor_int)):
                    qj, vj = q[:, self.motor_int[m, 0]], v[:, self.motor_int[m, 1]]
                    _, qlo, qhi = self.motor_dbl[m]
                    hit |= ((qj - qlo < nd[1]) & (vj < -nd[2])) | ((qhi - qj < nd[1]) & (vj > nd[2]))
            else:
                if isinstance(node, MechanicalPowerConsumptionTermination):
                    x = self._mean(i) if self.stack_size[i] else self.power(node, v, command)
                else:
                    x = q[:, 2] - zmin if isinstance(node, FallingTermination) else zmin
                hit = np.zeros(n, bool)
                if not np.isnan(lo):
                    hit |= lo > x
                if not np.isnan(hi):
                    hit |= x > hi
            hit &= ~skip
            values[i] = np.where(pending, np.where(hit, 1.0, 0.0), np.nan)
            newly = pending & hit
            fired[newly] = j
            terminated |= newly
            pending &= ~hit
        # the reward tree, per env (a terminal step evaluates nothing)
        reward = np.zeros(n)
        live = np.flatnonzero(~terminated)
        node_values = {}
        for i, node in enumerate(self.nodes[:self.n_reward]):
            if isinstance(node, SurviveReward):
                node_values[i] = np.ones(n)
            elif isinstance(node, MinimizeMechanicalPowerConsumption):
                node_values[i] = radial_basis_function(self._mean(i), node.cutoff)
            values[i] = np.nan
        for e in live:
            stack: List[Optional[float]] = []
            wk = 0
            for i, node in enumerate(self.nodes[:self.n_reward]):
                if isinstance(node, _Mixture):
                    k = len(node.components)
                    parts, stack = stack[-k:], stack[:-k]
                    if isinstance(node, AdditiveMixtureReward):
                        x = weighted_norm(self.weights[wk:wk + k], node.order, parts)
                        wk += k
                    else:
                        x = geometric_mean(parts)
                else:
                    x = float(node_values[i][e])
                stack.append(x)
                values[i, e] = np.nan if x is None else x
            reward[e] = 0.0 if stack[-1] is None else stack[-1]
        info: Dict[str, np.ndarray] = {"terminated": fired, "truncated": np.full(n, -1, np.int32)}
        for i, name in enumerate(self.names):
            info[name] = values[i]
        return reward, terminated, truncated, info


def contact_positions(models: Sequence, q: np.ndarray) -> np.ndarray:
    """World positions [n_env, ncontacts, 3] of the contact frames of every env (`robots.frame_placements`), env `e` on
    `models[e]` (its own model table)."""
    from .robots import frame_placements
    names = models[0].contact_frame_names
    out = np.empty((len(q), len(names), 3))
    for e, (m, qe) in enumerate(zip(models, q)):
        pl = frame_placements(m, qe, names)
        out[e] = [pl[nm].p for nm in names]
    return out
