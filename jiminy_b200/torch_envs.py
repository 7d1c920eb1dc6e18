"""Device-resident counterparts of `envs.BatchedJiminyEnv` / `envs.PDControlBatchedEnv` for a policy on the same GPU:
`reset()` / `step(action)` take and return torch tensors on the batch's device, and `step` never synchronises with the
host.

What differs from the host envs is only where the work runs:
- the action is clipped on the device and handed to the step kernel (`jb_set_command_device`) or, in PD mode, to the
  device `PDAdapter` kernel (`jb_pd_adapter_device`), which writes the target accelerations in place;
- the observation is read from the batch's device buffers (`jb_device_views`, `jb_state_ptrs`, `jb_device_block_views`,
  `jb_device_obs_views` for the stacked frames of `stack=` and the PD action of `augment_observation=True`): fresh tensors
  per observation, the same nested dict as the host envs;
- termination, truncation and `SurviveReward` are evaluated on the device with the host envs' rule
  (`envs.terminated_truncated`); with `reward` / `terminations` (`jiminy_b200.compositions`), a contact-frame pass
  (`jb_contact_positions_device`) and one composition kernel (`jb_compositions_device`) evaluate the env's rule, the
  termination conditions and the reward tree instead, and a second launch of that kernel behind the masked restart
  reseeds the power stacks of the restarted envs;
- finished envs are restarted by a masked `jb_start_device` that is enqueued at EVERY step with the done mask as a device
  tensor: envs outside the mask leave at the top of the launch, so no host decision depends on device data.

Restart states.  The host env draws a fresh sample of the scenario's initial-state distribution at every restart event
(`scenarios.make`: a perturbed posture with the feet put on the ground by forward kinematics on the host).  By default
the restart rows are drawn on the device, with replacement, from a fixed bank `reset_states=(q [B, nq], v [B, nv])`; the
default bank is one such sample of `n_env` rows.  The bank is validated once on the host.  `info["reset_rows"]` gives the
bank row each env restarted from (-1: not restarted).  This is the one semantic difference from the host env.
`reset_states="sample"` removes it: at every step `n_env` fresh rows of the distribution are drawn with the env's torch
generator (`Scenario.draw_initial_torch`) and the masked restart is `jb_start_device_on_ground`, which puts each
restarted env's feet on the ground by forward kinematics in the start kernel (`robots.ground_base_height` on the
device).  There is no bank, so `info["reset_rows"]` is not returned; the next observation holds the placed states.

Disturbance.  With `std_ratio={"disturbance": r}` the walker disturbance (`jiminy_b200.disturbance`) of the envs in the
done mask is re-drawn with a torch generator on the device and written by the device setters before the masked restart,
at every step.  `env.disturbance_rows` holds the impulse schedule and process tables every env currently runs with
(device tensors, `WalkerDisturbance.draw_torch` layout), so that a run can be replayed through the host setters.  The
impulse setter's checks (NaN, t < 0, dt < 1e-10) flag a rejected row's env NOT_STARTED | BAD_START, but the masked restart
enqueued right after it clears that flag and the env runs on with its previous impulse row: the sampler never draws such a
row (t >= 1.75 s, dt = 10 ms, finite wrenches), so nothing here depends on the flag.

Sensors.  With `std_ratio={"sensors": r}` the sensor options (noise, bias, delay, jitter) and engine seeds of the envs in
the done mask are re-drawn the same way (`jiminy_b200.sensor_randomisation`) and written by
`jb_set_sensor_options_env_device` and `jb_set_seeds_device` before the masked restart, which latches them.
`env.sensor_rows` holds the options and seed every env currently runs with.  The sampler never draws a row the setter
would reject (its delays stay below the bound the buffer was sized for).

Model.  With `std_ratio={"model": r}` the stiffness and damping of every flexibility joint of the envs in the done mask are
re-drawn the same way (`jiminy_b200.model_randomisation`) and written by `jb_set_flexibility_env_device` before the
masked restart, which latches them.  `env.model_rows` holds the rows every env currently runs with.  The sampler never
draws a row the setter would reject (the ratio is checked against the nominal values at construction).

Model biases.  With `model_bias_std` (the standard deviations of `massBodiesBiasStd`, `centerOfMassPositionBodiesBiasStd`,
`inertiaBodiesBiasStd`, `relativePositionBodiesBiasStd`) the masses, centres of mass, inertias and joint-placement
translations of the envs in the done mask are re-drawn around the nominal model with the env's torch generator
(`model_randomisation.ModelBiasRandomisation`) and written by `jb_set_model_env_device` before the masked restart, which
latches them.  `env.model_bias_rows` holds the rows every env currently runs with.  The restart bank, like the host envs'
restarts, is grounded on the nominal model; only `reset_states="sample"` grounds each env on its own biased model, inside
the start kernel.

Streams.  All work runs on the batch's own stream (`torch.cuda.ExternalStream(engine.stream())`).  On entry it waits
for the caller's current stream; on exit the caller's current stream waits for it.  With the CPU emulation of the
library (`api_` given), device memory is host memory: the env then runs on `torch_device="cpu"`, without streams.
"""
from __future__ import annotations

import contextlib
import ctypes as C
from typing import Any, Dict, Optional, Tuple, Union

import numpy as np
import torch

from . import core, envs, observers, scenarios
from .parallel import _DevArray

_CTYPES = {torch.float64: C.c_double, torch.int32: C.c_int32}
_TYPESTR = {torch.float64: "<f8", torch.int32: "<i4"}


def validate_reset_states(robot, q: np.ndarray, v: np.ndarray) -> None:
    """The input checks of `Engine::start` (engine.cc:1007-1037) on every row of a restart bank."""
    if q.ndim != 2 or v.ndim != 2 or q.shape[1] != robot.nq or v.shape[1] != robot.nv or q.shape[0] != v.shape[0] or not len(q):
        raise ValueError(f"reset_states must be (q [B, {robot.nq}], v [B, {robot.nv}]) with B >= 1")
    eps = 2.220446049250313e-16
    if np.isnan(q).any():
        raise ValueError("reset_states: a configuration contains NaN.")
    if ((q - robot.q_upper > eps) | (robot.q_lower - q > eps)).any():
        raise ValueError("reset_states: a configuration is out of bounds.")
    if np.isnan(v).any():
        raise ValueError("reset_states: a velocity contains NaN.")


class DeviceBatchedEnv(envs.BatchedJiminyEnv):
    """`BatchedJiminyEnv` with torch actions and observations on the batch's device and the restart on the device.
    Extra arguments: `reset_states` (restart bank, or "sample" for fresh grounded draws: see the module docstring) and
    `torch_device` (default: cuda:<device>, or cpu with the emulated library)."""

    def __init__(self, scenario: scenarios.Scenario, reset_states: Union[None, str, Tuple[np.ndarray, np.ndarray]] = None,
                 torch_device=None, **kw):
        super().__init__(scenario, **kw)
        self._init_device(reset_states, torch_device, kw.get("api_"))

    # ------------------------------------------------------------------ set-up
    def _init_device(self, reset_states, torch_device, api_) -> None:
        eng, n = self.engine, self.n_env
        if torch_device is None:
            torch_device = "cpu" if api_ is not None else torch.device("cuda", eng.device)
        self.torch_device = dev = torch.device(torch_device)
        self._emulated = dev.type == "cpu"
        self._stream = None if self._emulated else torch.cuda.ExternalStream(eng.stream(), device=dev)
        # the default bank: one sample of the distribution the host env's `_sample_state` draws from
        seed = int(np.random.default_rng([self.sc.seed, 0x5EED]).integers(0, 2 ** 31 - 1))
        f64 = dict(dtype=torch.float64, device=dev)
        self._sample_restarts = isinstance(reset_states, str)
        if self._sample_restarts:
            if reset_states != "sample":
                raise ValueError(f"reset_states must be None, 'sample' or (q, v), not {reset_states!r}")
            self.reset_states = None
        else:
            if reset_states is None:
                bank = scenarios.make(self.sc.name, n, seed=seed)
                reset_states = (bank.q0, bank.v0)
            q_bank = np.ascontiguousarray(reset_states[0], dtype=np.float64)
            v_bank = np.ascontiguousarray(reset_states[1], dtype=np.float64)
            validate_reset_states(self.robot, q_bank, v_bank)
            self.reset_states = (torch.as_tensor(q_bank, **f64), torch.as_tensor(v_bank, **f64))
        self._gen = torch.Generator(device=dev)
        self._gen.manual_seed(seed)
        # inputs of the launches, kept alive between steps (every use is ordered on the batch stream)
        nm = max(self.robot.nmotors, 1)
        self._action = torch.zeros((n, nm), **f64)
        self._q_start, self._v_start = torch.zeros((n, self.robot.nq), **f64), torch.zeros((n, self.robot.nv), **f64)
        self._mask = torch.zeros(n, dtype=torch.uint8, device=dev)
        if self.disturbance is not None:
            # the tables and schedule every env currently runs with, drawn on the device (`env.disturbance_rows`)
            self._disturbance_gen = torch.Generator(device=dev)
            self._disturbance_gen.manual_seed(int(np.random.default_rng([self.sc.seed, 0xD157]).integers(0, 2 ** 31 - 1)))
            with self._on_batch_stream():     # the draw's first use of its kernels on the batch stream happens here
                self.disturbance_rows = self.disturbance.draw_torch(self._disturbance_gen, n, dev)
        if self.sensor_randomisation is not None:
            self._sensor_gen = torch.Generator(device=dev)
            self._sensor_gen.manual_seed(int(np.random.default_rng([self.sc.seed, 0x5E45]).integers(0, 2 ** 31 - 1)))
            with self._on_batch_stream():
                self.sensor_rows = self.sensor_randomisation.draw_torch(self._sensor_gen, n, dev)
        if self.model_randomisation is not None:
            self._model_gen = torch.Generator(device=dev)
            self._model_gen.manual_seed(int(np.random.default_rng([self.sc.seed, 0xF1E8]).integers(0, 2 ** 31 - 1)))
            with self._on_batch_stream():
                self.model_rows = self.model_randomisation.draw_torch(self._model_gen, n, dev)
        if self.model_bias is not None:
            self._model_bias_gen = torch.Generator(device=dev)
            self._model_bias_gen.manual_seed(int(np.random.default_rng([self.sc.seed, 0xB1A5]).integers(0, 2 ** 31 - 1)))
            with self._on_batch_stream():
                self.model_bias_rows = self.model_bias.draw_torch(self._model_bias_gen, n, dev)
        self.num_steps = torch.zeros(n, dtype=torch.int64, device=dev)
        # zero-copy views of the batch's device buffers
        ptr = eng.device_state_ptrs()
        status, pd_state, mahony = eng.device_block_views()
        self._t = self._view(ptr["t"], (n,))
        self._qv = self._view(ptr["qv"], (n, self.robot.nq + self.robot.nv))
        self._sensors = self._view(ptr["sensors"], (n, eng.width)) if eng.width else torch.zeros((n, 0), **f64)
        self._status = self._view(status, (n,), torch.int32)
        self._pd_state = self._view(pd_state, (n, 3, self.robot.nmotors)) if pd_state else None
        nimu = self.robot.sensor_layout()["ImuSensor"][2]
        self._mahony_state = self._view(mahony, (n, nimu, 10)) if mahony else None
        record = eng.device_observer_views()
        self._observer_record = self._view(record, (n, nimu, core.OBSV_N)) if record else None
        stack, command = eng.device_obs_views()
        self._command = self._view(command, (n, self.robot.nmotors)) if self.robot.nmotors else None
        self._stack_frames = self._view(stack, (n,) + eng.stack_shape) if self._stack_leaves else None
        self._set_action_bounds()
        if self.compositions is not None:
            # the spec is uploaded once; the launches' outputs live in these buffers, cloned for the caller at every step
            comp = self.compositions
            comp.upload(eng)
            nc = len(self.robot.contact_frame_names)
            self._contacts = torch.full((n, max(nc, 1), 3), float("nan"), **f64)
            self._comp_reward = torch.zeros(n, **f64)
            self._comp_done = torch.zeros((2, n), dtype=torch.bool, device=dev)
            self._comp_index = torch.full((2, n), -1, dtype=torch.int32, device=dev)
            self._comp_values = torch.full((len(comp.nodes), n), float("nan"), **f64)
            self._all = torch.ones(n, dtype=torch.uint8, device=dev)

    def _set_action_bounds(self) -> None:
        f64 = dict(dtype=torch.float64, device=self.torch_device)
        self._low = torch.as_tensor(np.asarray(self.action_low, dtype=np.float64), **f64)
        self._high = torch.as_tensor(np.asarray(self.action_high, dtype=np.float64), **f64)

    def _view(self, ptr: int, shape, dtype=torch.float64) -> torch.Tensor:
        if self._emulated:     # the emulated library's device memory is host memory
            arr = np.ctypeslib.as_array(C.cast(C.c_void_p(ptr), C.POINTER(_CTYPES[dtype])), shape=tuple(shape))
            return torch.from_numpy(arr)
        return torch.as_tensor(_DevArray(ptr, shape, _TYPESTR[dtype]), device=self.torch_device)

    @contextlib.contextmanager
    def _on_batch_stream(self):
        """Runs the body on the batch stream, ordered after the caller's current stream and before its later work."""
        if self._stream is None:
            yield None
            return
        caller = torch.cuda.current_stream(self.torch_device)
        self._stream.wait_stream(caller)
        with torch.cuda.stream(self._stream):
            yield caller
        caller.wait_stream(self._stream)

    @staticmethod
    def _hand_over(caller, tensors) -> None:
        # tensors made on the batch stream and used on the caller's: the allocator must not recycle them early
        if caller is not None:
            for x in tensors:
                x.record_stream(caller)

    # ------------------------------------------------------------------ observation
    def _observation(self) -> Dict[str, Any]:
        obs = self._plain_observation()
        return self._apply_stack(obs, self._stack_frames.clone()) if self._stack_leaves else obs

    def _plain_observation(self) -> Dict[str, Any]:
        nq = self.robot.nq
        qv, sens = self._qv.clone(), self._sensors.clone()      # fresh tensors: earlier observations stay valid
        meas = {}
        for name, nf in envs.SENSOR_FIELDS.items():
            off, _, ns = self._layout[name]
            if ns:
                meas[name] = sens[:, off:off + nf * ns].reshape(self.n_env, nf, ns)
        return {"t": self._t.clone(), "states": {"agent": {"q": qv[:, :nq], "v": qv[:, nq:]}}, "measurements": meas}

    @staticmethod
    def _leaves(obs):
        for x in obs.values():
            if isinstance(x, dict):
                yield from DeviceBatchedEnv._leaves(x)
            else:
                yield x

    # ------------------------------------------------------------------ commands and restarts
    def _apply_action(self, action: torch.Tensor) -> None:
        self.engine.set_command_device(self._action.data_ptr())

    def _first_command(self) -> None:
        self.engine.set_command(self.sc.target0)

    def _redraw_disturbance(self, done: Optional[torch.Tensor]) -> None:
        """New disturbance rows for the envs of `done` (None: all), drawn on the device and written by the device setters
        with the mask in `self._mask`; `disturbance_rows` keeps what every env runs with."""
        if self.disturbance is None:
            return
        new = self.disturbance.draw_torch(self._disturbance_gen, self.n_env, self.torch_device)
        rows = self.disturbance_rows
        if done is None:
            for k in rows:
                rows[k].copy_(new[k])
        else:
            for k in ("t", "dt", "wrench"):
                sel = done.view(1, -1, *([1] * (rows[k].dim() - 2)))
                rows[k].copy_(torch.where(sel, new[k], rows[k]))
            for k in ("values", "grads"):
                rows[k].copy_(torch.where(done.view(-1, 1), new[k], rows[k]))
        self.disturbance.apply_device(self.engine, rows, None if done is None else self._mask.data_ptr())

    def _redraw_sensors(self, done: Optional[torch.Tensor]) -> None:
        """New sensor options and seeds for the envs of `done` (None: all), drawn on the device and written by the device
        setters with the mask in `self._mask`; `sensor_rows` keeps what every env runs with."""
        if self.sensor_randomisation is None:
            return
        new = self.sensor_randomisation.draw_torch(self._sensor_gen, self.n_env, self.torch_device)
        rows = self.sensor_rows
        for k in rows:
            rows[k].copy_(new[k] if done is None else torch.where(done.view(-1, *([1] * (rows[k].dim() - 1))), new[k], rows[k]))
        self.sensor_randomisation.apply_device(self.engine, rows, None if done is None else self._mask.data_ptr())

    def _redraw_model(self, done: Optional[torch.Tensor]) -> None:
        """New flexibility stiffness and damping for the envs of `done` (None: all), drawn on the device and written by the
        device setter with the mask in `self._mask`; `model_rows` keeps what every env runs with."""
        if self.model_randomisation is None:
            return
        new = self.model_randomisation.draw_torch(self._model_gen, self.n_env, self.torch_device)
        self.model_rows.copy_(new if done is None else torch.where(done.view(-1, 1, 1), new, self.model_rows))
        self.model_randomisation.apply_device(self.engine, self.model_rows, None if done is None else self._mask.data_ptr())

    def _redraw_model_bias(self, done: Optional[torch.Tensor]) -> None:
        """New body biases for the envs of `done` (None: all), drawn on the device and written by the device setter with
        the mask in `self._mask`; `model_bias_rows` keeps what every env runs with."""
        if self.model_bias is None:
            return
        new = self.model_bias.draw_torch(self._model_bias_gen, self.n_env, self.torch_device)
        self.model_bias_rows.copy_(new if done is None else torch.where(done.view(-1, 1, 1), new, self.model_bias_rows))
        self.model_bias.apply_device(self.engine, self.model_bias_rows, None if done is None else self._mask.data_ptr())

    def _restart(self, done: torch.Tensor) -> Optional[torch.Tensor]:
        """Masked restart of the envs in `done` from bank rows drawn on the device; returns the rows (-1: not restarted).
        With `reset_states="sample"`: from fresh draws put on the ground in the start kernel; returns None."""
        if self._sample_restarts:
            q, v = self.sc.draw_initial_torch(self._gen, self.n_env, self.torch_device)
            self._q_start.copy_(q)
            self._v_start.copy_(v)
            rows = None
        else:
            q_bank, v_bank = self.reset_states
            rows = torch.randint(0, q_bank.shape[0], (self.n_env,), generator=self._gen, device=self.torch_device)
            torch.index_select(q_bank, 0, rows, out=self._q_start)
            torch.index_select(v_bank, 0, rows, out=self._v_start)
        self._mask.copy_(done)
        self._redraw_disturbance(done)
        self._redraw_sensors(done)
        self._redraw_model(done)
        self._redraw_model_bias(done)
        self.engine.start_device(self._q_start.data_ptr(), self._v_start.data_ptr(), self._mask.data_ptr(),
                                 on_ground=self._sample_restarts)
        if self.compositions is not None:
            self.engine.compositions_device(self._mask.data_ptr())
        self.num_steps.masked_fill_(done, 0)
        return None if rows is None else torch.where(done, rows, torch.full_like(rows, -1))

    # ------------------------------------------------------------------ gym API
    def reset(self, mask: Optional[torch.Tensor] = None) -> Tuple[Dict[str, Any], Dict[str, Any]]:
        """First call (or `mask=None`): every env starts -- from the scenario's initial states the first time, from bank
        rows (or fresh grounded draws) afterwards.  `mask` [n_env] (bool / uint8 tensor): a masked restart of those envs
        the same way."""
        with self._on_batch_stream() as caller:
            info: Dict[str, Any] = {}
            if not self._started:
                self._first_command()
                self._redraw_disturbance(None)
                self._redraw_sensors(None)
                self._redraw_model(None)
                self._redraw_model_bias(None)
                self.engine.start(self.sc.q0, self.sc.v0)
                if self.compositions is not None:
                    self.engine.compositions_device(self._all.data_ptr())
                self.num_steps.zero_()
                self._started = True
            else:
                if mask is None:
                    self._first_command()
                done = torch.ones(self.n_env, dtype=torch.bool, device=self.torch_device) if mask is None else \
                    torch.as_tensor(mask, device=self.torch_device).to(torch.bool)
                rows = self._restart(done)
                if rows is not None:
                    info["reset_rows"] = rows
            obs = self._observation()
            self._hand_over(caller, list(self._leaves(obs)) + list(info.values()))
        return obs, info

    def step(self, action: torch.Tensor):
        """action: [n_env, nmotors] tensor (efforts, or position targets in PD mode).  Returns the gymnasium 5-tuple of
        device tensors; finished envs are restarted before returning (their terminal observation is in
        info["final_observation"], valid where info["_final_observation"])."""
        if not self._started:
            raise core.BadControlFlow("No simulation running. Please call `reset` before `step`.")
        with self._on_batch_stream() as caller:
            # (no record_stream on the batch stream: the caller's stream waits for it on exit, so its later work -- the
            # reuse of `action`'s memory included -- is ordered after the reads below)
            action = torch.as_tensor(action)
            a = action.to(device=self.torch_device, dtype=torch.float64).reshape(self.n_env, -1)
            torch.minimum(torch.maximum(a, self._low), self._high, out=self._action)   # np.clip
            self._apply_action(self._action)
            self.engine.step(self.step_dt)
            obs = self._observation()
            self.num_steps += 1
            status = self._status.clone()
            extra: Dict[str, torch.Tensor] = {}
            if self.compositions is None:
                terminated, truncated = envs.terminated_truncated(obs["states"]["agent"]["q"], status, self.num_steps.double(),
                                                                  self.step_dt, self.simulation_duration_max, self._height_min)
                reward = (~terminated).to(torch.float64)         # SurviveReward
            else:
                reward, terminated, truncated, extra = self._evaluate_compositions()
            done = terminated | truncated
            rows = self._restart(done)                           # enqueued at every step: no host decision
            info = {"status": status, "final_observation": obs, "_final_observation": done, **extra}
            if rows is not None:
                info["reset_rows"] = rows
            obs = self._observation()
            self._hand_over(caller, list(self._leaves(obs)) + list(self._leaves(info["final_observation"])) +
                            [status, done, reward, terminated, truncated] + list(extra.values()) + ([] if rows is None else [rows]))
        return obs, reward, terminated, truncated, info

    def _evaluate_compositions(self):
        """The contact-frame pass and the composition kernel on the batch stream: (reward, terminated, truncated, info
        entries), fresh tensors."""
        eng = self.engine
        if self.compositions.needs_contacts:
            eng.contact_positions_device(self._contacts.data_ptr())
        eng.compositions_device(None, self.num_steps.data_ptr(), self._contacts.data_ptr(), self._comp_reward.data_ptr(),
                                self._comp_done[0].data_ptr(), self._comp_done[1].data_ptr(), self._comp_index.data_ptr(),
                                self._comp_values.data_ptr())
        done, index, values = self._comp_done.clone(), self._comp_index.clone(), self._comp_values.clone()
        extra = {"terminated": index[0], "truncated": index[1]}
        extra.update({name: values[i] for i, name in enumerate(self.compositions.names)})
        return self._comp_reward.clone(), done[0], done[1], extra


class DevicePDControlBatchedEnv(DeviceBatchedEnv):
    """`PDControlBatchedEnv` (MotorSafetyLimit -> PDController -> PDAdapter -> MahonyFilter) with the adapter on the device
    as well: same constructor arguments and bounds (`envs.configure_pd_blocks`), `augment_observation`, `stack`, the
    `MahonyFilter` object form of `mahony` and `body_observer` included, plus those of `DeviceBatchedEnv`."""

    def __init__(self, scenario: scenarios.Scenario, *, kp=None, kd=None, joint_position_margin: float = 0.0,
                 joint_velocity_limit: float = float("inf"), joint_acceleration_limit: Optional[float] = None,
                 safety: Optional[Dict[str, float]] = None, order: int = 1, joint_velocity_deadband: float = 0.0,
                 is_instantaneous: bool = False, mahony=None, training: bool = True,
                 augment_observation: bool = False, stack=None, body_observer=None, **kw):
        kp, kd = envs.pd_gains(scenario, kp, kd)
        self.training = training
        self.augment_observation = augment_observation
        reset_states, torch_device = kw.pop("reset_states", None), kw.pop("torch_device", None)
        with envs.without_plain_pd(scenario):
            envs.BatchedJiminyEnv.__init__(self, scenario, **kw)
        deadband = envs.configure_pd_blocks(self, kp, kd, joint_position_margin, joint_velocity_limit, joint_acceleration_limit,
                                            safety, order, joint_velocity_deadband, mahony, training, body_observer)
        self.engine.set_pd_adapter(order, is_instantaneous, deadband)
        self._setup_stack(stack)
        self._init_device(reset_states, torch_device, kw.get("api_"))

    def _obs_shapes(self) -> Dict[str, Any]:
        return envs.pd_obs_shapes(self, super()._obs_shapes())

    def _plain_observation(self) -> Dict[str, Any]:
        obs = super()._plain_observation()
        obs["states"]["pd_controller"] = self._pd_state[:, :2].clone()      # PDController.get_state (:488-489)
        if self._observers is not None:
            extra = observers.observation(*self._observers, self._mahony_state, self._observer_record,
                                          lambda x: x.clone(memory_format=torch.contiguous_format))
            obs["states"].update(extra["states"])
            obs["features"] = extra["features"]
        elif self._mahony:
            obs["features"] = {"mahony_filter": self._mahony_state[:, :, :4].transpose(1, 2).clone()}   # [n, 4, n_imu]
        if self.augment_observation:
            obs["actions"] = {"pd_controller": self._command.clone()}         # the block's action (pipeline.py:1134-1141)
        return obs

    def _apply_action(self, action: torch.Tensor) -> None:
        self.engine.pd_adapter_device(action.data_ptr(), self.step_dt)

    def _first_command(self) -> None:
        # no simulation running: the adapter's dt is 0, the target accelerations stay 0 (:652-662)
        self.engine.set_command(np.zeros((self.n_env, self.robot.nmotors)))
