"""Device-resident counterparts of `envs.BatchedJiminyEnv` / `envs.PDControlBatchedEnv` for a policy on the same GPU:
`reset()` / `step(action)` take and return torch tensors on the batch's device, and `step` never synchronises with the
host.

What differs from the host envs is only where the work runs:
- the action is clipped on the device and handed to the step kernel (`jb_set_command_device`) or, in PD mode, to the
  device `PDAdapter` kernel (`jb_pd_adapter_device`), which writes the target accelerations in place;
- the observation is read from the batch's device buffers (`jb_device_views`, `jb_state_ptrs`, `jb_device_block_views`):
  fresh tensors per observation, the same nested dict as the host envs;
- termination, truncation and `SurviveReward` are evaluated on the device with the host envs' rule
  (`envs.terminated_truncated`);
- finished envs are restarted by a masked `jb_start_device` that is enqueued at EVERY step with the done mask as a device
  tensor: envs outside the mask leave at the top of the launch, so no host decision depends on device data.

Restart states.  The host env draws a fresh sample of the scenario's initial-state distribution at every restart event
(`scenarios.make`: a perturbed posture with the feet put on the ground by forward kinematics on the host).  Here the
restart rows are drawn on the device, with replacement, from a fixed bank `reset_states=(q [B, nq], v [B, nv])`; the
default bank is one such sample of `n_env` rows.  The bank is validated once on the host.  `info["reset_rows"]` gives the
bank row each env restarted from (-1: not restarted).  This is the one semantic difference from the host env.

Streams.  All work runs on the batch's own stream (`torch.cuda.ExternalStream(engine.stream())`).  On entry it waits
for the caller's current stream; on exit the caller's current stream waits for it.  With the CPU emulation of the
library (`api_` given), device memory is host memory: the env then runs on `torch_device="cpu"`, without streams.
"""
from __future__ import annotations

import contextlib
import ctypes as C
from typing import Any, Dict, Optional, Tuple

import numpy as np
import torch

from . import core, envs, scenarios
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
    Extra arguments: `reset_states` (restart bank, see the module docstring) and `torch_device` (default: cuda:<device>,
    or cpu with the emulated library)."""

    def __init__(self, scenario: scenarios.Scenario, reset_states: Optional[Tuple[np.ndarray, np.ndarray]] = None,
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
        if reset_states is None:
            bank = scenarios.make(self.sc.name, n, seed=seed)
            reset_states = (bank.q0, bank.v0)
        q_bank = np.ascontiguousarray(reset_states[0], dtype=np.float64)
        v_bank = np.ascontiguousarray(reset_states[1], dtype=np.float64)
        validate_reset_states(self.robot, q_bank, v_bank)
        f64 = dict(dtype=torch.float64, device=dev)
        self.reset_states = (torch.as_tensor(q_bank, **f64), torch.as_tensor(v_bank, **f64))
        self._gen = torch.Generator(device=dev)
        self._gen.manual_seed(seed)
        # inputs of the launches, kept alive between steps (every use is ordered on the batch stream)
        nm = max(self.robot.nmotors, 1)
        self._action = torch.zeros((n, nm), **f64)
        self._q_start, self._v_start = torch.zeros((n, self.robot.nq), **f64), torch.zeros((n, self.robot.nv), **f64)
        self._mask = torch.zeros(n, dtype=torch.uint8, device=dev)
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
        self._set_action_bounds()

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

    def _restart(self, done: torch.Tensor) -> torch.Tensor:
        """Masked restart of the envs in `done` from bank rows drawn on the device; returns the rows (-1: not restarted)."""
        q_bank, v_bank = self.reset_states
        rows = torch.randint(0, q_bank.shape[0], (self.n_env,), generator=self._gen, device=self.torch_device)
        torch.index_select(q_bank, 0, rows, out=self._q_start)
        torch.index_select(v_bank, 0, rows, out=self._v_start)
        self._mask.copy_(done)
        self.engine.start_device(self._q_start.data_ptr(), self._v_start.data_ptr(), self._mask.data_ptr())
        self.num_steps.masked_fill_(done, 0)
        return torch.where(done, rows, torch.full_like(rows, -1))

    # ------------------------------------------------------------------ gym API
    def reset(self, mask: Optional[torch.Tensor] = None) -> Tuple[Dict[str, Any], Dict[str, Any]]:
        """First call (or `mask=None`): every env starts -- from the scenario's initial states the first time, from bank
        rows afterwards.  `mask` [n_env] (bool / uint8 tensor): a masked restart of those envs from bank rows."""
        with self._on_batch_stream() as caller:
            info: Dict[str, Any] = {}
            if not self._started:
                self._first_command()
                self.engine.start(self.sc.q0, self.sc.v0)
                self.num_steps.zero_()
                self._started = True
            else:
                if mask is None:
                    self._first_command()
                done = torch.ones(self.n_env, dtype=torch.bool, device=self.torch_device) if mask is None else \
                    torch.as_tensor(mask, device=self.torch_device).to(torch.bool)
                info["reset_rows"] = self._restart(done)
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
            terminated, truncated = envs.terminated_truncated(obs["states"]["agent"]["q"], status, self.num_steps.double(),
                                                              self.step_dt, self.simulation_duration_max, self._height_min)
            reward = (~terminated).to(torch.float64)             # SurviveReward
            done = terminated | truncated
            rows = self._restart(done)                           # enqueued at every step: no host decision
            info = {"status": status, "final_observation": obs, "_final_observation": done, "reset_rows": rows}
            obs = self._observation()
            self._hand_over(caller, list(self._leaves(obs)) + list(self._leaves(info["final_observation"])) +
                            [status, done, rows, reward, terminated, truncated])
        return obs, reward, terminated, truncated, info


class DevicePDControlBatchedEnv(DeviceBatchedEnv):
    """`PDControlBatchedEnv` (MotorSafetyLimit -> PDController -> PDAdapter -> MahonyFilter) with the adapter on the device
    as well: same constructor arguments and bounds (`envs.configure_pd_blocks`), plus those of `DeviceBatchedEnv`."""

    def __init__(self, scenario: scenarios.Scenario, *, kp=None, kd=None, joint_position_margin: float = 0.0,
                 joint_velocity_limit: float = float("inf"), joint_acceleration_limit: Optional[float] = None,
                 safety: Optional[Dict[str, float]] = None, order: int = 1, joint_velocity_deadband: float = 0.0,
                 is_instantaneous: bool = False, mahony: Optional[Tuple[float, float]] = None, training: bool = True, **kw):
        kp, kd = envs.pd_gains(scenario, kp, kd)
        reset_states, torch_device = kw.pop("reset_states", None), kw.pop("torch_device", None)
        with envs.without_plain_pd(scenario):
            envs.BatchedJiminyEnv.__init__(self, scenario, **kw)
        deadband = envs.configure_pd_blocks(self, kp, kd, joint_position_margin, joint_velocity_limit, joint_acceleration_limit,
                                            safety, order, joint_velocity_deadband, mahony, training)
        self.engine.set_pd_adapter(order, is_instantaneous, deadband)
        self._init_device(reset_states, torch_device, kw.get("api_"))

    def _observation(self) -> Dict[str, Any]:
        obs = super()._observation()
        obs["states"]["pd_controller"] = self._pd_state[:, :2].clone()      # PDController.get_state (:488-489)
        if self._mahony:
            obs["features"] = {"mahony_filter": self._mahony_state[:, :, :4].transpose(1, 2).clone()}   # [n, 4, n_imu]
        return obs

    def _apply_action(self, action: torch.Tensor) -> None:
        self.engine.pd_adapter_device(action.data_ptr(), self.step_dt)

    def _first_command(self) -> None:
        # no simulation running: the adapter's dt is 0, the target accelerations stay 0 (:652-662)
        self.engine.set_command(np.zeros((self.n_env, self.robot.nmotors)))
