"""Batched counterpart of `gym_jiminy.common.envs.BaseJiminyEnv` / `WalkerJiminyEnv` for the
accelerated path: `reset()` / `step(action)` over N lockstep envs, one kernel launch per step.

Mirrors the reference flow (python/gym_jiminy/common/gym_jiminy/common/envs/generic.py:521-880):
`reset` samples an initial state (`_sample_state`: neutral posture + perturbation, feet on the
ground, :1300-1335) and starts the engine (:673-690); `step` copies the action into the controller
buffer (:806), advances the engine by `step_dt` (:810), refreshes the observation (:834),
evaluates termination (:846-875; `WalkerJiminyEnv.has_terminated`: base height under a threshold,
locomotion.py:380-400) and truncation (numerical failure -> the reference raises and the env
truncates, generic.py:809-817).  Terminated / truncated envs are restarted with a masked `start`,
which is what a vectorised gym env does between steps.

The observation is the reference's `{"t", "states": {"agent": {"q", "v"}}, "measurements": {...}}`
nested dict with a leading env axis; sensor matrices are `[n_env, n_fields, n_sensors]` views of
the flat sensor row.
"""
from __future__ import annotations

import functools
from typing import Any, Dict, Optional, Tuple

import numpy as np

from . import core, scenarios
from .model import RobotTable

SENSOR_FIELDS = {"ImuSensor": 6, "ForceSensor": 6, "EncoderSensor": 2, "EffortSensor": 1, "ContactSensor": 3}


def terminated_truncated(q, status, num_steps, step_dt: float, simulation_duration_max: float, height_min: Optional[float]):
    """Per-env (terminated, truncated) after an env-step, for numpy arrays or torch tensors alike: terminated = base height
    under `height_min` (`WalkerJiminyEnv.has_terminated`, locomotion.py:380-400), truncated = a failure bit of the status
    word (JB_ENV_JOINT_LIMIT only reports that a bound constraint has been active: not a failure) or the time limit.
    `num_steps` must be a float64 (or int64 numpy) array."""
    truncated = ((status & ~core.JB_ENV_JOINT_LIMIT) != 0) | (num_steps * step_dt >= simulation_duration_max)
    terminated = (q[:, 2] < height_min) if height_min is not None else (truncated & False)
    return terminated, truncated


def pd_gains(scenario: scenarios.Scenario, kp, kd):
    kp = scenario.kp if kp is None else kp
    kd = scenario.kd if kd is None else kd
    if kp is None:
        raise ValueError("PD gains are needed (scenario without PD gains and no kp / kd given)")
    return kp, kd


class without_plain_pd:
    """Hides the scenario's PD gains while the base env is built: the `PDController` block replaces the plain PD law."""

    def __init__(self, scenario: scenarios.Scenario):
        self.sc, self.gains = scenario, (scenario.kp, scenario.kd)

    def __enter__(self):
        self.sc.kp = self.sc.kd = None

    def __exit__(self, *exc):
        self.sc.kp, self.sc.kd = self.gains
        return False


def configure_pd_blocks(env, kp, kd, joint_position_margin: float, joint_velocity_limit: float,
                        joint_acceleration_limit: Optional[float], safety: Optional[Dict[str, float]], order: int,
                        joint_velocity_deadband: float, mahony: Optional[Tuple[float, float]], training: bool) -> Optional[np.ndarray]:
    """`MotorSafetyLimit` -> `PDController` -> `MahonyFilter` on `env.engine` from the constructor arguments of
    `PDControlBatchedEnv`, with the bounds the reference's block constructors derive from them
    (blocks/proportional_derivative_controller.py:301-450, :560-640; blocks/motor_safety_limit.py:112-175).  Sets
    `env.command_state_lower / upper` [3, nmotors], `env.action_low / high` and `env._mahony`; returns the `PDAdapter`'s
    motor velocity dead band (None in training mode)."""
    rob, nm, dt = env.robot, env.robot.nmotors, env.step_dt
    kp, kd = np.broadcast_to(kp, (nm,)).astype(np.float64), np.broadcast_to(kd, (nm,)).astype(np.float64)
    ratio = np.array([m.reduction for m in rob.motors])
    iq = np.array([rob.idx_q[m.joint] for m in rob.motors])
    q_lo, q_hi = rob.q_lower[iq] * ratio, rob.q_upper[iq] * ratio          # motor-side position limits
    v_hw = np.array([m.velocity_limit for m in rob.motors])
    effort = np.array([m.effort_limit for m in rob.motors])
    # PDController.__init__ (:405-436)
    vel = np.minimum(v_hw, ratio * joint_velocity_limit)
    if joint_acceleration_limit is None:
        acc = np.minimum(2.0 * vel / dt, effort / (kp * dt * np.maximum(dt, kd)))
    else:
        acc = ratio * joint_acceleration_limit
    env.command_state_lower = np.stack([q_lo + ratio * joint_position_margin, -vel, -acc])
    env.command_state_upper = np.stack([q_hi - ratio * joint_position_margin, vel, acc])
    table = None
    if safety is not None:      # MotorSafetyLimit.__init__ (:161-175)
        if safety["soft_position_margin"] < 0.0 or safety["soft_velocity_max"] < 0.0:
            raise ValueError("Soft position margin and maximum velocity must be positive.")
        table = np.stack([np.full(nm, float(safety["kp"])), np.full(nm, float(safety["kd"])),
                          q_lo + ratio * safety["soft_position_margin"], q_hi - ratio * safety["soft_position_margin"],
                          np.minimum(v_hw, ratio * safety["soft_velocity_max"])])
    env.engine.set_pd_controller_full(kp, kd, env.command_state_lower, env.command_state_upper, table)
    if mahony is not None:
        env.engine.set_mahony_filter(*mahony)
    env._mahony = mahony is not None
    if order not in (0, 1):
        raise ValueError("Derivative order of the action out-of-bounds.")
    env.action_low, env.action_high = env.command_state_lower[order], env.command_state_upper[order]
    return None if training else ratio * joint_velocity_deadband      # PDAdapter._setup: evaluation mode only (:619-621)


class BatchedJiminyEnv:
    def __init__(self, scenario: scenarios.Scenario, device: int = 0, height_threshold_ratio: float = 0.5,
                 simulation_duration_max: float = 20.0, api_: Optional[core.Api] = None):
        self.sc = scenario
        self.robot: RobotTable = scenario.robot
        self.n_env, self.step_dt = scenario.n_env, scenario.step_dt
        self.engine = core.BatchedEngine(self.robot, scenario.options, self.n_env, device=device, api_=api_)
        if scenario.kp is not None:
            self.engine.set_pd_controller(scenario.kp, scenario.kd)
        self.simulation_duration_max = simulation_duration_max
        self._height_min = height_threshold_ratio * float(np.mean(scenario.q0[:, 2])) if self.robot.has_freeflyer else None
        self._layout = self.robot.sensor_layout()
        self._sens = np.zeros((self.n_env, max(self.engine.width, 1)))
        self.num_steps = np.zeros(self.n_env, dtype=np.int64)
        self._rng = np.random.default_rng(scenario.seed)
        lim = np.array([m.effort_limit for m in self.robot.motors]) if self.robot.nmotors else np.zeros(0)
        # action space bounds: motor effort limits (generic.py:344-361) or, in PD mode, joint position bounds
        if scenario.kp is None:
            self.action_low, self.action_high = -lim, lim
        else:
            iq = np.array([self.robot.idx_q[m.joint] for m in self.robot.motors])
            self.action_low, self.action_high = self.robot.q_lower[iq], self.robot.q_upper[iq]
        self._started = False

    # ------------------------------------------------------------------ helpers
    def _observation(self) -> Dict[str, Any]:
        t, q, v, _ = self.engine.get_state()
        sens = np.empty_like(self._sens)      # a fresh matrix per observation: earlier observations stay valid
        self.engine.get_sensors(sens)
        meas = {}
        for name, nf in SENSOR_FIELDS.items():
            off, _, ns = self._layout[name]
            if ns:
                meas[name] = sens[:, off:off + nf * ns].reshape(self.n_env, nf, ns)
        return {"t": t, "states": {"agent": {"q": q, "v": v}}, "measurements": meas}

    def _sample_state(self, n: int) -> Tuple[np.ndarray, np.ndarray]:
        """Fresh draws from the scenario's initial-state distribution (perturbed posture, feet on ground)."""
        sc = scenarios.make(self.sc.name, n, seed=int(self._rng.integers(0, 2 ** 31 - 1)))
        return sc.q0, sc.v0

    # ------------------------------------------------------------------ gym API
    def reset(self, mask: Optional[np.ndarray] = None) -> Tuple[Dict[str, Any], Dict[str, Any]]:
        if mask is None or not self._started:
            q0, v0 = (self.sc.q0, self.sc.v0) if not self._started else self._sample_state(self.n_env)
            self.engine.set_command(self.sc.target0)
            self.engine.start(q0, v0)
            self.num_steps[:] = 0
            self._started = True
        elif mask.any():
            q0, v0 = self._sample_state(self.n_env)
            self.engine.start(q0, v0, mask=mask)
            self.num_steps[mask.astype(bool)] = 0
        return self._observation(), {}

    def step(self, action: np.ndarray):
        """action: [n_env, nmotors] efforts (or position targets in PD mode).  Returns the gymnasium
        5-tuple with per-env arrays; terminated / truncated envs are restarted before returning."""
        if not self._started:
            raise core.BadControlFlow("No simulation running. Please call `reset` before `step`.")
        action = np.clip(np.asarray(action, dtype=np.float64), self.action_low, self.action_high)
        self.engine.set_command(action)
        self.engine.step(self.step_dt)
        obs = self._observation()
        self.num_steps += 1
        status = self.engine.get_status()
        terminated, truncated = terminated_truncated(obs["states"]["agent"]["q"], status, self.num_steps, self.step_dt,
                                                     self.simulation_duration_max, self._height_min)
        reward = np.where(terminated, 0.0, 1.0)          # SurviveReward
        info = {"status": status}
        done = terminated | truncated
        if done.any():
            # gymnasium vector-env convention: finished envs return their first observation after the restart, the
            # terminal one goes to info["final_observation"] (valid where info["_final_observation"])
            info["final_observation"], info["_final_observation"] = obs, done
            obs, _ = self.reset(mask=done.astype(np.uint8))
        return obs, reward, terminated, truncated, info

    def close(self) -> None:
        self.engine.close()


class PDControlBatchedEnv(BatchedJiminyEnv):
    """Batched counterpart of the `*PDControlJiminyEnv` pipelines that `build_pipeline` assembles in the reference
    (e.g. `AtlasPDControlJiminyEnv`, python/gym_jiminy/envs/gym_jiminy/envs/atlas.py:239-295):
    `MotorSafetyLimit` -> `PDController(update_ratio=1)` -> `PDAdapter(update_ratio=-1)` -> `MahonyFilter`.
    The controller, the safety limits and the observer run inside the step kernel; the adapter is evaluated on the
    host once per env-step (jiminy_b200/blocks.py).  Constructor arguments and the bounds derived from them follow the
    reference's block constructors (blocks/proportional_derivative_controller.py:301-450, :560-640;
    blocks/motor_safety_limit.py:112-175).  The action is the adapter's: target motor velocities (order 1) or
    positions (order 0) at the end of the step, within the controller's command-state bounds."""

    def __init__(self, scenario: scenarios.Scenario, *, kp=None, kd=None, joint_position_margin: float = 0.0,
                 joint_velocity_limit: float = float("inf"), joint_acceleration_limit: Optional[float] = None,
                 safety: Optional[Dict[str, float]] = None, order: int = 1, joint_velocity_deadband: float = 0.0,
                 is_instantaneous: bool = False, mahony: Optional[Tuple[float, float]] = None, training: bool = True, **kw):
        from .blocks import PDAdapter
        kp, kd = pd_gains(scenario, kp, kd)
        with without_plain_pd(scenario):          # the base class must not install the plain PD law
            super().__init__(scenario, **kw)
        deadband = configure_pd_blocks(self, kp, kd, joint_position_margin, joint_velocity_limit, joint_acceleration_limit,
                                       safety, order, joint_velocity_deadband, mahony, training)
        self.adapter = PDAdapter(self.engine, self.command_state_lower, self.command_state_upper, order=order,
                                 is_instantaneous=is_instantaneous, velocity_deadband=deadband, step_dt=self.step_dt)

    def _observation(self) -> Dict[str, Any]:
        obs = super()._observation()
        obs["states"]["pd_controller"] = self.engine.get_pd_controller_state()[:, :2]       # PDController.get_state (:488-489)
        if self._mahony:
            obs["features"] = {"mahony_filter": np.swapaxes(self.engine.get_mahony_filter()[:, :, :4], 1, 2)}   # [n, 4, n_imu]
        return obs

    def reset(self, mask: Optional[np.ndarray] = None):
        if mask is None or not self._started:
            # no simulation running: the adapter's dt is 0, the target accelerations stay 0 (:652-662)
            self.engine.set_command(np.zeros((self.n_env, self.robot.nmotors)))
            q0, v0 = (self.sc.q0, self.sc.v0) if not self._started else self._sample_state(self.n_env)
            self.engine.start(q0, v0)
            self.num_steps[:] = 0
            self._started = True
            return self._observation(), {}
        return super().reset(mask)

    def step(self, action: np.ndarray):
        if not self._started:
            raise core.BadControlFlow("No simulation running. Please call `reset` before `step`.")
        action = np.clip(np.asarray(action, dtype=np.float64), self.action_low, self.action_high)
        self.adapter.apply(action)
        self.engine.step(self.step_dt)
        obs = self._observation()
        self.num_steps += 1
        status = self.engine.get_status()
        terminated, truncated = terminated_truncated(obs["states"]["agent"]["q"], status, self.num_steps, self.step_dt,
                                                     self.simulation_duration_max, self._height_min)
        reward = np.where(terminated, 0.0, 1.0)
        done = terminated | truncated
        info = {"status": status}
        if done.any():
            info["final_observation"], info["_final_observation"] = obs, done
            obs, _ = self.reset(mask=done.astype(np.uint8))
        return obs, reward, terminated, truncated, info


def flatten_observation(obs: Dict[str, Any], nested_keys, low=None, high=None) -> np.ndarray:
    """`FilterObservation` + `NormalizeObservation(ignore_unbounded=True)` + `FlattenObservation`
    (gym_jiminy/common/wrappers) for a batched nested observation: the leaves named by `nested_keys` (tuples of
    keys), each rescaled to [-1, 1] by its own finite bounds when `low` / `high` give them (dicts keyed like
    `nested_keys`), flattened per env and concatenated in the order of `nested_keys` -> [n_env, width].  Torch leaves
    (`torch_envs`) give a torch tensor on their device, with the same values."""
    out = []
    for key in nested_keys:
        leaf = obs
        for k in key:
            leaf = leaf[k]
        if type(leaf).__module__.startswith("torch"):
            return _flatten_observation_torch(obs, nested_keys, low, high)
        leaf = np.asarray(leaf, dtype=np.float64)
        x = leaf.reshape(leaf.shape[0], -1)
        if low is not None and key in low:
            lo, hi = np.asarray(low[key], dtype=np.float64).ravel(), np.asarray(high[key], dtype=np.float64).ravel()
            ok = np.isfinite(lo) & np.isfinite(hi)
            scale = np.where(ok, 2.0 / np.where(ok, hi - lo, 1.0), 1.0)
            x = np.where(ok, (x - np.where(ok, lo, 0.0)) * scale - 1.0, x)
        out.append(x)
    return np.concatenate(out, axis=1)


def _flatten_observation_torch(obs: Dict[str, Any], nested_keys, low=None, high=None):
    import torch
    out = []
    for key in nested_keys:
        leaf = obs
        for k in key:
            leaf = leaf[k]
        x = leaf.to(torch.float64).reshape(leaf.shape[0], -1)
        if low is not None and key in low:
            lo, hi = np.asarray(low[key], dtype=np.float64).ravel(), np.asarray(high[key], dtype=np.float64).ravel()
            ok, shift, scale = _torch_bounds(lo.tobytes(), hi.tobytes(), str(x.device))
            x = torch.where(ok, (x - shift) * scale - 1.0, x)
        out.append(x)
    return torch.cat(out, dim=1)


@functools.lru_cache(maxsize=64)
def _torch_bounds(lo_bytes: bytes, hi_bytes: bytes, device: str):
    """The bounds are host constants: the scale is derived in numpy, exactly as in the numpy path, and moved to the device
    once (a host-to-device copy per observation would synchronise the caller's stream)."""
    import torch
    lo, hi = np.frombuffer(lo_bytes, dtype=np.float64), np.frombuffer(hi_bytes, dtype=np.float64)
    ok = np.isfinite(lo) & np.isfinite(hi)
    scale = np.where(ok, 2.0 / np.where(ok, hi - lo, 1.0), 1.0)
    f64 = dict(device=device, dtype=torch.float64)
    return torch.as_tensor(ok, device=device), torch.as_tensor(np.where(ok, lo, 0.0), **f64), torch.as_tensor(scale, **f64)
