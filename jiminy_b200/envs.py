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
from typing import Any, Dict, Optional, Sequence, Tuple, Union

import numpy as np

from . import compositions, core, model_randomisation, observers, scenarios, sensor_randomisation
from .observation_stack import StackObservation
from .observers import BodyObserver, MahonyFilter
from .disturbance import from_std_ratio
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
                        joint_velocity_deadband: float, mahony, training: bool,
                        body_observer: Optional[BodyObserver] = None) -> Optional[np.ndarray]:
    """`MotorSafetyLimit` -> `PDController` -> `MahonyFilter` (-> `BodyObserver`) on `env.engine` from the constructor
    arguments of `PDControlBatchedEnv`, with the bounds the reference's block constructors derive from them
    (blocks/proportional_derivative_controller.py:301-450, :560-640; blocks/motor_safety_limit.py:112-175).  Sets
    `env.command_state_lower / upper` [3, nmotors], `env.action_low / high`, `env._mahony` and, for the object form of
    `mahony`, `env._observers` (the filter and the body observer, else None); returns the `PDAdapter`'s motor velocity
    dead band (None in training mode)."""
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
    env._observers = None
    if isinstance(mahony, MahonyFilter):
        mahony.configure(env.engine)
        if body_observer is not None:
            body_observer.configure(env.engine)
        env._observers = (mahony, body_observer)
    elif body_observer is not None:
        raise ValueError("body_observer needs the MahonyFilter object form of `mahony`")
    elif mahony is not None:
        env.engine.set_mahony_filter(*mahony)
    env._mahony = mahony is not None
    if order not in (0, 1):
        raise ValueError("Derivative order of the action out-of-bounds.")
    env.action_low, env.action_high = env.command_state_lower[order], env.command_state_upper[order]
    return None if training else ratio * joint_velocity_deadband      # PDAdapter._setup: evaluation mode only (:619-621)


class BatchedJiminyEnv:
    training = True     # `training_only` termination conditions run (the PD envs take it as an argument)

    def __init__(self, scenario: scenarios.Scenario, device: int = 0, height_threshold_ratio: float = 0.5,
                 simulation_duration_max: float = 20.0, api_: Optional[core.Api] = None, std_ratio: Optional[dict] = None,
                 model_bias_std: Optional[dict] = None, reward=None, terminations: Sequence = (),
                 stack: Optional[StackObservation] = None):
        """`std_ratio`: the reference walker env's randomisation ratios.  None or {}: none; "disturbance": r, the walker
        disturbance forces (`jiminy_b200.disturbance`); "sensors": r, noise, bias, delay and jitter of every sensor and a
        new seed of its generators (`jiminy_b200.sensor_randomisation`); "model": r, stiffness and damping of every
        flexibility joint (`jiminy_b200.model_randomisation`; NotImplementedError on a robot without one).
        `model_bias_std`: the body biases of the robot options `massBodiesBiasStd`, `centerOfMassPositionBodiesBiasStd`,
        `inertiaBodiesBiasStd`, `relativePositionBodiesBiasStd` (standard deviations; None, {} or zeros: none), drawn per
        env around the nominal model (`model_randomisation.ModelBiasRandomisation`).  All are re-drawn for every env that
        (re)starts.
        `reward` / `terminations`: the reward and the extra termination conditions of the reference's composed env
        (`jiminy_b200.compositions`; `compositions.from_config` reads them from a reference env config).  The defaults,
        `SurviveReward` and no extra condition, are the env's plain behaviour.
        `stack`: gym_jiminy's `StackObservation` wrapper (`jiminy_b200.observation_stack`; `observation_stack.from_config`
        reads it from a reference pipeline config): each stacked leaf of the observation becomes its frames
        `[n_env, num_stack, ...]`, updated by the step kernel at every observer refresh.  None: no stacking."""
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
        self.disturbance = from_std_ratio(self.robot, std_ratio, simulation_duration_max)
        if self.disturbance is not None:
            self.disturbance.register(self.engine)
            self._disturbance_rng = np.random.default_rng([scenario.seed, 0xD157])
        self.sensor_randomisation = sensor_randomisation.from_std_ratio(self.robot.sensor_layout(), std_ratio)
        if self.sensor_randomisation is not None:
            self.sensor_randomisation.register(self.engine)
            self._sensor_rng = np.random.default_rng([scenario.seed, 0x5E45])
            self.sensor_rows: Optional[Dict[str, np.ndarray]] = None      # the options and seed every env runs with
        self.model_randomisation = model_randomisation.from_std_ratio(self.robot, std_ratio)
        if self.model_randomisation is not None:
            self.model_randomisation.register(self.engine)
            self._model_rng = np.random.default_rng([scenario.seed, 0xF1E8])
            self.model_rows: Optional[np.ndarray] = None     # the flexibility rows every env runs with [n_env, n_flex, 6]
        self.model_bias = model_randomisation.from_model_bias_std(self.robot, model_bias_std)
        if self.model_bias is not None:
            self.model_bias.register(self.engine)
            self._model_bias_rng = np.random.default_rng([scenario.seed, 0xB1A5])
            self.model_bias_rows: Optional[np.ndarray] = None     # the body rows every env runs with [n_env, njoints, 13]
        self.compositions = None
        if reward is not None or len(terminations):
            self.compositions = compositions.Compositions(reward, terminations, self.robot, self.n_env, self.step_dt,
                                                          simulation_duration_max, self._height_min, self.training)
        self._started = False
        self._setup_stack(stack)

    # ------------------------------------------------------------------ helpers
    def _obs_shapes(self) -> Dict[str, Any]:
        """The observation tree with the per-env shape of every leaf, in the order of `_observation`."""
        meas = {name: (nf, self._layout[name][2]) for name, nf in SENSOR_FIELDS.items() if self._layout[name][2]}
        return {"t": (), "states": {"agent": {"q": (self.robot.nq,), "v": (self.robot.nv,)}}, "measurements": meas}

    def _setup_stack(self, stack: Optional[StackObservation]) -> None:
        """Resolves the stacked leaves against the observation tree and configures the step kernel's stacking;
        `_stack_leaves` holds (path, first column, width, per-env shape) of each in the frame."""
        self.stack, self._stack_leaves = stack, []
        if stack is None:
            return
        shapes = self._obs_shapes()
        obs_blocks = getattr(self, "_observers", None)
        leaves = stack.resolve(shapes, observers.stack_leaves(*obs_blocks) if obs_blocks is not None else None)
        self.engine.set_obs_stack(stack.num_stack, stack.skip_frames_ratio, [code for _, code in leaves])
        col = 0
        for path, code in leaves:
            shape = shapes
            for k in path:
                shape = shape[k]
            width = self.engine.stack_leaf_width(code)
            self._stack_leaves.append((path, col, width, tuple(shape)))
            col += width

    def _apply_stack(self, obs: Dict[str, Any], frames) -> Dict[str, Any]:
        """Replaces each stacked leaf of `obs` by its frames, from `frames` [n_env, num_stack, frame width] (numpy or torch)."""
        for path, col, width, shape in self._stack_leaves:
            node = obs
            for k in path[:-1]:
                node = node[k]
            node[path[-1]] = frames[:, :, col:col + width].reshape((self.n_env, self.stack.num_stack) + shape)
        return obs

    def _observation(self) -> Dict[str, Any]:
        obs = self._plain_observation()
        return self._apply_stack(obs, self.engine.get_obs_stack()) if self._stack_leaves else obs

    def _plain_observation(self) -> Dict[str, Any]:
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

    def _redraw_disturbance(self, mask: Optional[np.ndarray]) -> None:
        """New disturbance rows for the envs about to (re)start (`_setup` runs at every reset, locomotion.py:298-330)."""
        if self.disturbance is not None:
            draw = self.disturbance.draw_numpy(self._disturbance_rng, self.n_env)
            self.disturbance.apply_host(self.engine, draw, mask)

    def _redraw_sensors(self, mask: Optional[np.ndarray]) -> None:
        """New sensor options and seeds for the envs about to (re)start (`_setup`, locomotion.py:264-286)."""
        if self.sensor_randomisation is not None:
            draw = self.sensor_randomisation.draw_numpy(self._sensor_rng, self.n_env)
            if mask is not None and self.sensor_rows is not None:
                sel = np.asarray(mask).astype(bool)
                draw = {k: np.where(sel.reshape((-1,) + (1,) * (v.ndim - 1)), v, self.sensor_rows[k]) for k, v in draw.items()}
            self.sensor_rows = draw
            self.sensor_randomisation.apply_host(self.engine, draw, mask)

    def _redraw_model(self, mask: Optional[np.ndarray]) -> None:
        """New flexibility stiffness and damping for the envs about to (re)start (`_setup`, locomotion.py:288-296)."""
        if self.model_randomisation is not None:
            draw = self.model_randomisation.draw_numpy(self._model_rng, self.n_env)
            if mask is not None and self.model_rows is not None:
                draw = np.where(np.asarray(mask).astype(bool)[:, None, None], draw, self.model_rows)
            self.model_rows = draw
            self.model_randomisation.apply_host(self.engine, draw, mask)

    def _redraw_model_bias(self, mask: Optional[np.ndarray]) -> None:
        """New body biases for the envs about to (re)start (Model::reset re-draws them at every reset, model.cc:398-416)."""
        if self.model_bias is not None:
            if mask is None or self.model_bias_rows is None:
                draw = self.model_bias.draw_numpy(self._model_bias_rng, self.n_env)
            else:
                # only the restarting envs draw: the transformation costs host time per row
                sel = np.flatnonzero(np.asarray(mask))
                draw = self.model_bias_rows.copy()
                draw[sel] = self.model_bias.draw_numpy(self._model_bias_rng, len(sel))
            self.model_bias_rows = draw
            self.model_bias.apply_host(self.engine, draw, mask)

    # ------------------------------------------------------------------ gym API
    def reset(self, mask: Optional[np.ndarray] = None) -> Tuple[Dict[str, Any], Dict[str, Any]]:
        if mask is None or not self._started:
            mask = None
            q0, v0 = (self.sc.q0, self.sc.v0) if not self._started else self._sample_state(self.n_env)
            self.engine.set_command(self.sc.target0)
            self._redraw_disturbance(None)
            self._redraw_sensors(None)
            self._redraw_model(None)
            self._redraw_model_bias(None)
            self.engine.start(q0, v0)
            self.num_steps[:] = 0
            self._started = True
        elif mask.any():
            q0, v0 = self._sample_state(self.n_env)
            self._redraw_disturbance(mask)
            self._redraw_sensors(mask)
            self._redraw_model(mask)
            self._redraw_model_bias(mask)
            self.engine.start(q0, v0, mask=mask)
            self.num_steps[mask.astype(bool)] = 0
        self._seed_compositions(mask)
        return self._observation(), {}

    def _seed_compositions(self, mask: Optional[np.ndarray]) -> None:
        """The power stacks of the envs that have just (re)started (None: all) take the power of their start state."""
        if self.compositions is not None:
            self.compositions.seed(mask, self.engine.get_state()[2], self.engine.get_stepper_state()[1])

    def _reward_done(self, obs, status):
        """Reward, terminated, truncated and info after an env-step: the env's own rule, then the compositions if any."""
        q = obs["states"]["agent"]["q"]
        terminated, truncated = terminated_truncated(q, status, self.num_steps, self.step_dt, self.simulation_duration_max,
                                                     self._height_min)
        info = {"status": status}
        if self.compositions is None:
            return np.where(terminated, 0.0, 1.0), terminated, truncated, info      # SurviveReward
        comp = self.compositions
        contacts = None
        if comp.needs_contacts:
            models = [self.engine.model(e) for e in range(self.n_env)] if self.model_bias is not None else [self.robot] * self.n_env
            contacts = compositions.contact_positions(models, q)
        reward, terminated, truncated, extra = comp.evaluate(obs["t"], q, obs["states"]["agent"]["v"],
                                                             self.engine.get_stepper_state()[1], terminated, truncated, contacts)
        info.update(extra)
        return reward, terminated, truncated, info

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
        reward, terminated, truncated, info = self._reward_done(obs, self.engine.get_status())
        done = terminated | truncated
        if done.any():
            # gymnasium vector-env convention: finished envs return their first observation after the restart, the
            # terminal one goes to info["final_observation"] (valid where info["_final_observation"])
            info["final_observation"], info["_final_observation"] = obs, done
            obs, _ = self.reset(mask=done.astype(np.uint8))
        return obs, reward, terminated, truncated, info

    def close(self) -> None:
        self.engine.close()


def pd_obs_shapes(env, shapes: Dict[str, Any]) -> Dict[str, Any]:
    """The leaves a PD env adds to the observation tree of `_obs_shapes`, in the order of its `_observation`."""
    nm = env.robot.nmotors
    shapes["states"]["pd_controller"] = (2, nm)
    nimu = env.robot.sensor_layout()["ImuSensor"][2]
    if env._observers is not None:
        extra = observers.observation_shapes(*env._observers, nimu)
        shapes["states"].update(extra["states"])
        shapes["features"] = extra["features"]
    elif env._mahony:
        shapes["features"] = {"mahony_filter": (4, nimu)}
    if env.augment_observation:
        shapes["actions"] = {"pd_controller": (nm,)}
    return shapes


class PDControlBatchedEnv(BatchedJiminyEnv):
    """Batched counterpart of the `*PDControlJiminyEnv` pipelines that `build_pipeline` assembles in the reference
    (e.g. `AtlasPDControlJiminyEnv`, python/gym_jiminy/envs/gym_jiminy/envs/atlas.py:239-295):
    `MotorSafetyLimit` -> `PDController(update_ratio=1)` -> `PDAdapter(update_ratio=-1)` -> `MahonyFilter`.
    The controller, the safety limits and the observer run inside the step kernel; the adapter is evaluated on the
    host once per env-step (jiminy_b200/blocks.py).  Constructor arguments and the bounds derived from them follow the
    reference's block constructors (blocks/proportional_derivative_controller.py:301-450, :560-640;
    blocks/motor_safety_limit.py:112-175).  The action is the adapter's: target motor velocities (order 1) or
    positions (order 0) at the end of the step, within the controller's command-state bounds.
    `augment_observation=True` adds the controller's action, the target accelerations of the env-step
    (`obs["actions"]["pd_controller"]`), as the reference's `ControlledJiminyEnv` does (bases/pipeline.py:1134-1141).
    `mahony`: `(kp, ki)` for the filter's default path, observed as the quaternion array `features.mahony_filter`
    [n_env, 4, nimu]; or a `jiminy_b200.observers.MahonyFilter`, observed with the reference's layout
    (`features.<name> = {"quat", ["rpy"], "omega"}`, `states.<name> = {"bias"}`), which `body_observer` (a
    `jiminy_b200.observers.BodyObserver`, `features.<name> = {"quat", ["rpy"], "omega"}`) needs."""

    def __init__(self, scenario: scenarios.Scenario, *, kp=None, kd=None, joint_position_margin: float = 0.0,
                 joint_velocity_limit: float = float("inf"), joint_acceleration_limit: Optional[float] = None,
                 safety: Optional[Dict[str, float]] = None, order: int = 1, joint_velocity_deadband: float = 0.0,
                 is_instantaneous: bool = False, mahony: Union[None, Tuple[float, float], MahonyFilter] = None,
                 training: bool = True, augment_observation: bool = False, stack: Optional[StackObservation] = None,
                 body_observer: Optional[BodyObserver] = None, **kw):
        from .blocks import PDAdapter
        kp, kd = pd_gains(scenario, kp, kd)
        self.training = training
        self.augment_observation = augment_observation
        with without_plain_pd(scenario):          # the base class must not install the plain PD law
            super().__init__(scenario, **kw)
        deadband = configure_pd_blocks(self, kp, kd, joint_position_margin, joint_velocity_limit, joint_acceleration_limit,
                                       safety, order, joint_velocity_deadband, mahony, training, body_observer)
        self._setup_stack(stack)
        self.adapter = PDAdapter(self.engine, self.command_state_lower, self.command_state_upper, order=order,
                                 is_instantaneous=is_instantaneous, velocity_deadband=deadband, step_dt=self.step_dt)

    def _obs_shapes(self) -> Dict[str, Any]:
        return pd_obs_shapes(self, super()._obs_shapes())

    def _plain_observation(self) -> Dict[str, Any]:
        obs = super()._plain_observation()
        obs["states"]["pd_controller"] = self.engine.get_pd_controller_state()[:, :2]       # PDController.get_state (:488-489)
        if self._observers is not None:
            record = self.engine.get_observers() if observers.has_record(*self._observers) else None
            extra = observers.observation(*self._observers, self.engine.get_mahony_filter(), record, np.ascontiguousarray)
            obs["states"].update(extra["states"])
            obs["features"] = extra["features"]
        elif self._mahony:
            obs["features"] = {"mahony_filter": np.swapaxes(self.engine.get_mahony_filter()[:, :, :4], 1, 2)}   # [n, 4, n_imu]
        if self.augment_observation:
            obs["actions"] = {"pd_controller": self.engine.get_efforts()[2]}      # the block's action (pipeline.py:1134-1141)
        return obs

    def reset(self, mask: Optional[np.ndarray] = None):
        if mask is None or not self._started:
            # no simulation running: the adapter's dt is 0, the target accelerations stay 0 (:652-662)
            self.engine.set_command(np.zeros((self.n_env, self.robot.nmotors)))
            q0, v0 = (self.sc.q0, self.sc.v0) if not self._started else self._sample_state(self.n_env)
            self._redraw_disturbance(None)
            self._redraw_sensors(None)
            self._redraw_model(None)
            self._redraw_model_bias(None)
            self.engine.start(q0, v0)
            self.num_steps[:] = 0
            self._started = True
            self._seed_compositions(None)
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
        reward, terminated, truncated, info = self._reward_done(obs, self.engine.get_status())
        done = terminated | truncated
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
