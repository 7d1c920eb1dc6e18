"""Python host layer over the C ABI of `libjiminy_b200.so` (`include/jiminy_b200.h`).

Mirrors the part of `jiminy_py.core` that sits on the step path (Boost.Python bindings,
`python/jiminy_pywrap/src/engine.cc:587-787` in the reference): `Engine.start / step / stop /
simulate`, `RobotState`, `StepperState`, option dicts -- for one env (`Engine`) and for N lockstep
envs (`BatchedEngine`).  All physics runs in the CUDA library; there is no CPU path here: if the
library or a CUDA device is missing the constructors raise.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Any, Dict, Optional, Sequence, Tuple

import numpy as np

from . import model as M
from ._ctypes_abi import (JbModelDesc, JbOptions, JbSensorLayout, JbStateViews, ModelDescHolder, c_double_p, c_int32_p,
                          c_int64_p, c_uint8_p, dptr, make_options, safety_table)

JB_OK = 0
JB_ERR_INVALID_ARGUMENT, JB_ERR_BAD_CONTROL_FLOW, JB_ERR_RUNTIME, JB_ERR_NOT_IMPLEMENTED, JB_ERR_CUDA = -1, -2, -3, -4, -5
JB_ERR_PEER_TIMEOUT = -6
# stacked observation leaves (jb_set_obs_stack): time, a sensor-type block of the measured row, PDController action and
# state, MahonyFilter quaternions, angular velocity, roll-pitch-yaw and gyro bias, BodyObserver quaternions,
# roll-pitch-yaw and angular velocity
STACK_T, STACK_IMU, STACK_FORCE, STACK_ENCODER, STACK_EFFORT, STACK_CONTACT = 0, 1, 2, 3, 4, 5
STACK_PD_ACTION, STACK_PD_STATE, STACK_MAHONY = 6, 7, 8
STACK_MAHONY_OMEGA, STACK_MAHONY_RPY, STACK_MAHONY_BIAS, STACK_BODY_QUAT, STACK_BODY_RPY, STACK_BODY_OMEGA = 9, 10, 11, 12, 13, 14
# fields of the per-IMU observer record (jb_get_observers): MahonyFilter roll-pitch-yaw, BodyObserver quaternion,
# roll-pitch-yaw, angular velocity, twist angle
OBSV_MAHONY_RPY, OBSV_BODY_QUAT, OBSV_BODY_RPY, OBSV_BODY_OMEGA, OBSV_TWIST, OBSV_N = 0, 3, 7, 10, 13, 14
JB_ENV_OK, JB_ENV_NAN, JB_ENV_ITER_FAILED, JB_ENV_DT_UNDERFLOW = 0, 1, 2, 4
JB_ENV_JOINT_LIMIT, JB_ENV_NOT_STARTED, JB_ENV_CONTACT_FORCE = 8, 16, 32
JB_ENV_BAD_START = 256


class BadControlFlow(RuntimeError):
    """`jiminy::bad_control_flow` (python/jiminy_pywrap/src/module.cc:98-102)."""


class CudaUnavailable(RuntimeError):
    """No CUDA device / runtime failure.  jiminy_b200 never falls back to a CPU implementation."""


class PeerTimeout(RuntimeError):
    """Multi-GPU observation exchange: a rank never signalled its step (JB_ERR_PEER_TIMEOUT)."""


_EXC = {JB_ERR_INVALID_ARGUMENT: ValueError, JB_ERR_BAD_CONTROL_FLOW: BadControlFlow, JB_ERR_RUNTIME: RuntimeError,
        JB_ERR_NOT_IMPLEMENTED: NotImplementedError, JB_ERR_CUDA: CudaUnavailable, JB_ERR_PEER_TIMEOUT: PeerTimeout}

_LIB_NAME = "libjiminy_b200.so"


def library_path() -> str:
    # JB_LIBRARY: development override (A/B builds of the same C ABI)
    return os.environ.get("JB_LIBRARY") or os.path.join(os.path.dirname(os.path.abspath(__file__)), _LIB_NAME)


class Api:
    """Typed view of the C ABI exported by a loaded library (every symbol of include/jiminy_b200.h)."""

    SYMBOLS = ("jb_last_error", "jb_version", "jb_default_options", "jb_batch_create", "jb_batch_destroy",
               "jb_set_options", "jb_start", "jb_set_command", "jb_set_command_device", "jb_step",
               "jb_compute_dynamics", "jb_get_state", "jb_get_efforts", "jb_get_sensors", "jb_sensor_layout",
               "jb_get_extra_terms", "jb_get_status", "jb_get_iters", "jb_device_views", "jb_state_ptrs", "jb_set_model_variants", "jb_envs_per_group", "jb_get_stream",
               "jb_launch_count", "jb_synchronize", "jb_set_joint_springs", "jb_set_pd_controller", "jb_copy_sensors_device", "jb_describe",
               "jb_plan_describe", "jb_stop", "jb_register_impulse_force", "jb_set_impulse_force",
               "jb_register_profile_force", "jb_set_profile_force", "jb_remove_all_forces",
               "jb_peer_obs_create", "jb_peer_obs_connect", "jb_peer_obs_wait", "jb_peer_obs_view", "jb_peer_obs_enable",
               "jb_set_pd_controller_full", "jb_set_mahony_filter", "jb_get_mahony_filter",
               "jb_get_pd_controller_state", "jb_set_pd_controller_state", "jb_get_constraints",
               "jb_get_stepper_state", "jb_set_stepper_state", "jb_get_centroidal",
               "jb_set_sensor_options", "jb_set_seeds", "jb_get_sensor_data",
               "jb_start_device", "jb_start_device_on_ground", "jb_set_pd_adapter", "jb_pd_adapter_device", "jb_device_block_views",
               "jb_set_impulse_force_device", "jb_register_process_force", "jb_set_process_force",
               "jb_set_process_force_device", "jb_enable_per_env_sensor_options", "jb_set_sensor_options_env",
               "jb_set_sensor_options_env_device", "jb_set_seeds_device",
               "jb_enable_per_env_flexibility", "jb_set_flexibility_env", "jb_set_flexibility_env_device",
               "jb_get_flexibility_env", "jb_enable_per_env_model", "jb_set_model_env", "jb_set_model_env_device",
               "jb_get_model_env", "jb_contact_positions_device", "jb_set_compositions", "jb_compositions_device",
               "jb_set_obs_stack", "jb_get_obs_stack", "jb_device_obs_views",
               "jb_set_mahony_filter_full", "jb_set_body_observer", "jb_get_observers", "jb_device_observer_views")

    def __init__(self, cdll: C.CDLL):
        self.dll = L = cdll
        missing = [s for s in self.SYMBOLS if not hasattr(L, s)]
        if missing:
            raise ImportError(f"{L._name} does not export: {missing}")
        vp = C.c_void_p
        L.jb_last_error.restype = C.c_char_p
        L.jb_version.restype = C.c_char_p
        L.jb_default_options.argtypes = [C.POINTER(JbOptions)]
        L.jb_default_options.restype = None
        L.jb_batch_create.argtypes = [C.POINTER(JbModelDesc), C.POINTER(JbOptions), C.c_int32, C.c_int32, C.POINTER(vp)]
        L.jb_batch_destroy.argtypes = [vp]
        L.jb_set_options.argtypes = [vp, C.POINTER(JbOptions)]
        L.jb_start.argtypes = [vp, c_uint8_p, c_double_p, c_double_p]
        L.jb_set_command.argtypes = [vp, c_double_p]
        L.jb_set_command_device.argtypes = [vp, vp]
        L.jb_step.argtypes = [vp, C.c_double]
        L.jb_compute_dynamics.argtypes = [vp] + [c_double_p] * 6
        L.jb_get_state.argtypes = [vp] + [c_double_p] * 4
        L.jb_get_efforts.argtypes = [vp] + [c_double_p] * 4
        L.jb_get_stepper_state.argtypes = [vp, c_double_p, c_double_p]
        L.jb_get_centroidal.argtypes = [vp] + [c_double_p] * 5
        L.jb_set_sensor_options.argtypes = [vp, C.c_int32, C.c_int32, c_double_p, c_double_p, C.c_double, C.c_double, C.c_int32]
        L.jb_set_seeds.argtypes = [vp, C.POINTER(C.c_uint32)]
        L.jb_get_sensor_data.argtypes = [vp, c_double_p]
        L.jb_set_stepper_state.argtypes = [vp] + [c_double_p] * 4 + [c_int64_p, c_int64_p, c_double_p]
        L.jb_get_sensors.argtypes = [vp, c_double_p]
        L.jb_sensor_layout.argtypes = [vp, C.POINTER(JbSensorLayout)]
        L.jb_get_extra_terms.argtypes = [vp] + [c_double_p] * 3
        L.jb_get_status.argtypes = [vp, c_int32_p]
        L.jb_get_iters.argtypes = [vp, c_int64_p, c_int64_p]
        L.jb_device_views.argtypes = [vp, C.POINTER(vp), C.POINTER(vp)]
        L.jb_state_ptrs.argtypes = [vp, C.POINTER(JbStateViews), C.POINTER(JbStateViews)]
        L.jb_set_model_variants.argtypes = [vp, C.c_int32, C.POINTER(JbModelDesc), c_int32_p]
        L.jb_envs_per_group.argtypes = [vp]
        L.jb_get_stream.argtypes = [vp, C.POINTER(vp)]
        L.jb_launch_count.argtypes = [vp]
        L.jb_launch_count.restype = C.c_int64
        L.jb_synchronize.argtypes = [vp]
        L.jb_set_joint_springs.argtypes = [vp, c_double_p, c_double_p]
        L.jb_set_pd_controller.argtypes = [vp, c_double_p, c_double_p]
        L.jb_copy_sensors_device.argtypes = [vp, vp]
        L.jb_describe.argtypes = [vp, C.c_char_p, C.c_int32]
        L.jb_plan_describe.argtypes = [C.POINTER(JbModelDesc), C.c_int32, C.c_char_p, C.c_int32, c_int32_p]
        L.jb_stop.argtypes = [vp]
        L.jb_register_impulse_force.argtypes = [vp, C.c_int32] + [c_double_p] * 4 + [c_int32_p]
        L.jb_set_impulse_force.argtypes = [vp, C.c_int32, c_uint8_p] + [c_double_p] * 3
        L.jb_register_profile_force.argtypes = [vp, C.c_int32, c_double_p, C.c_double, c_int32_p]
        L.jb_set_profile_force.argtypes = [vp, C.c_int32, c_double_p]
        L.jb_remove_all_forces.argtypes = [vp]
        L.jb_set_pd_controller_full.argtypes = [vp] + [c_double_p] * 5
        L.jb_get_pd_controller_state.argtypes = [vp, c_double_p]
        L.jb_get_constraints.argtypes = [vp, c_uint8_p, c_double_p, c_uint8_p, c_double_p]
        L.jb_set_pd_controller_state.argtypes = [vp, c_double_p]
        L.jb_set_mahony_filter.argtypes = [vp, C.c_double, C.c_double]
        L.jb_get_mahony_filter.argtypes = [vp, c_double_p]
        L.jb_peer_obs_create.argtypes = [vp, C.c_int32, C.c_int32, C.c_char_p]
        L.jb_peer_obs_connect.argtypes = [vp, C.c_char_p]
        L.jb_peer_obs_wait.argtypes = [vp]
        L.jb_peer_obs_enable.argtypes = [vp, C.c_int32]
        L.jb_peer_obs_view.argtypes = [vp, C.POINTER(vp)]
        L.jb_start_device.argtypes = [vp, vp, vp, vp]
        L.jb_start_device_on_ground.argtypes = [vp, vp, vp, vp]
        L.jb_set_pd_adapter.argtypes = [vp, C.c_int32, C.c_int32, c_double_p]
        L.jb_pd_adapter_device.argtypes = [vp, vp, C.c_double]
        L.jb_device_block_views.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]
        L.jb_set_impulse_force_device.argtypes = [vp, C.c_int32] + [vp] * 4
        L.jb_register_process_force.argtypes = [vp, C.c_int32, c_double_p, C.c_double, C.c_int32, c_int32_p, c_int32_p,
                                                c_double_p, c_int32_p]
        L.jb_set_process_force.argtypes = [vp, C.c_int32, c_uint8_p, c_double_p, c_double_p]
        L.jb_set_process_force_device.argtypes = [vp, C.c_int32, vp, vp, vp]
        L.jb_enable_per_env_sensor_options.argtypes = [vp, C.c_double]
        L.jb_set_sensor_options_env.argtypes = [vp, c_uint8_p] + [c_double_p] * 4
        L.jb_set_sensor_options_env_device.argtypes = [vp] + [vp] * 5
        L.jb_set_seeds_device.argtypes = [vp, vp, vp]
        L.jb_enable_per_env_flexibility.argtypes = [vp, C.c_int32, c_int32_p]
        L.jb_set_flexibility_env.argtypes = [vp, c_uint8_p, c_double_p]
        L.jb_set_flexibility_env_device.argtypes = [vp, vp, vp]
        L.jb_get_flexibility_env.argtypes = [vp, c_double_p]
        L.jb_enable_per_env_model.argtypes = [vp]
        L.jb_set_model_env.argtypes = [vp, c_uint8_p, c_double_p]
        L.jb_set_model_env_device.argtypes = [vp, vp, vp]
        L.jb_get_model_env.argtypes = [vp, c_double_p]
        L.jb_contact_positions_device.argtypes = [vp, vp]
        L.jb_set_compositions.argtypes = [vp, C.c_int32, C.c_int32, c_int32_p, c_double_p, C.c_int32, c_double_p, c_int32_p,
                                          c_double_p, c_double_p, C.c_int32]
        L.jb_compositions_device.argtypes = [vp] * 9
        L.jb_set_obs_stack.argtypes = [vp, C.c_int32, C.c_int32, c_int32_p, C.c_int32]
        L.jb_get_obs_stack.argtypes = [vp, c_double_p]
        L.jb_device_obs_views.argtypes = [vp, C.POINTER(vp), C.POINTER(vp)]
        L.jb_set_mahony_filter_full.argtypes = [vp, C.c_double, C.c_double, C.c_int32, C.c_int32, C.c_int32]
        L.jb_set_body_observer.argtypes = [vp, C.c_int32, C.c_double, C.c_int32]
        L.jb_get_observers.argtypes = [vp, c_double_p]
        L.jb_device_observer_views.argtypes = [vp, C.POINTER(vp)]

    def check(self, rc: int) -> None:
        if rc != JB_OK:
            msg = (self.dll.jb_last_error() or b"").decode()
            raise _EXC.get(rc, RuntimeError)(msg)


_api: Optional[Api] = None


def api() -> Api:
    """The product library.  Raises ImportError if it has not been built (`__graft_entry__.build()`)."""
    global _api
    if _api is None:
        path = library_path()
        if not os.path.exists(path):
            raise ImportError(f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'`. "
                              "jiminy_b200 has no fallback implementation.")
        _api = Api(C.CDLL(path))
    return _api


def plan_describe(robot: M.RobotTable, lanes: int = 0, api_: Optional[Api] = None):
    """Host-only: how the lane planner lays the robot's tree over the lanes of a warp."""
    a = api_ or api()
    holder = ModelDescHolder(robot)
    buf = C.create_string_buffer(512)
    jl = np.zeros(robot.njoints, dtype=np.int32)
    a.check(a.dll.jb_plan_describe(C.byref(holder.desc), lanes, buf, 512, jl.ctypes.data_as(c_int32_p)))
    return buf.value.decode(), jl


class BatchedEngine:
    """N lockstep copies of one robot stepped by one kernel launch per `step`.

    Per-env semantics are those of `jiminy::Engine` with a zero-order-held command
    (`Engine::start` engine.cc:952, `Engine::step` engine.cc:1724); arrays are env-major.
    """

    def __init__(self, robot: M.RobotTable, options: Dict[str, Any], n_env: int, device: int = 0,
                 api_: Optional[Api] = None):
        self._api = api_ or api()
        self.robot, self.n_env, self.device = robot, int(n_env), int(device)
        self.options = options
        M.validate_options(options)
        self._holder = ModelDescHolder(robot)
        self._opt = make_options(options)
        h = C.c_void_p()
        self._api.check(self._api.dll.jb_batch_create(C.byref(self._holder.desc), C.byref(self._opt), self.n_env,
                                                       self.device, C.byref(h)))
        self._h = h
        self.nq, self.nv, self.nm, self.nj = robot.nq, robot.nv, robot.nmotors, robot.njoints
        lay = JbSensorLayout()
        self._api.check(self._api.dll.jb_sensor_layout(self._h, C.byref(lay)))
        self.sensor_layout, self.width = lay, lay.width
        self._process_knots: Dict[int, int] = {}   # knots of each process force (row width of its tables)

    def close(self) -> None:
        if getattr(self, "_h", None):
            self._api.dll.jb_batch_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def describe(self) -> str:
        buf = C.create_string_buffer(512)
        self._api.check(self._api.dll.jb_describe(self._h, buf, 512))
        return buf.value.decode()

    def set_options(self, options: Dict[str, Any]) -> None:
        M.validate_options(options)
        self.options, self._opt = options, make_options(options)
        self._api.check(self._api.dll.jb_set_options(self._h, C.byref(self._opt)))

    def set_joint_springs(self, stiffness: Optional[Sequence[float]], damping: Optional[Sequence[float]]) -> None:
        if stiffness is None:
            self._api.check(self._api.dll.jb_set_joint_springs(self._h, None, None))
            return
        k = np.ascontiguousarray(stiffness, dtype=np.float64)
        d = np.ascontiguousarray(damping, dtype=np.float64)
        assert k.shape == (self.nv,) and d.shape == (self.nv,)
        self._api.check(self._api.dll.jb_set_joint_springs(self._h, dptr(k), dptr(d)))

    # ---- model randomisation (Model::addBiasedToExtendedModel, model.cc:1166-1236)
    @property
    def envs_per_group(self) -> int:
        """How many consecutive envs share one model variant (the envs of a warp)."""
        return int(self._api.dll.jb_envs_per_group(self._h))

    def set_model_variants(self, robots: Sequence[M.RobotTable], variant_of_group: Sequence[int]) -> None:
        """Give every group of `envs_per_group` consecutive envs one of `robots` -- draws of `model.biased_robot` on the
        robot the batch was built with (same tree, hardware and frames; other inertias / joint placements).  The
        batched form of the per-reset model randomisation of the reference; takes effect at the next `start`."""
        holders = [ModelDescHolder(r) for r in robots]
        descs = (JbModelDesc * len(robots))(*[h.desc for h in holders])
        ngroups = -(-self.n_env // self.envs_per_group)
        vog = np.ascontiguousarray(variant_of_group, dtype=np.int32)
        if vog.shape != (ngroups,):
            raise ValueError(f"variant_of_group must have one entry per group of {self.envs_per_group} envs ({ngroups})")
        self._api.check(self._api.dll.jb_set_model_variants(self._h, len(robots), descs, vog.ctypes.data_as(c_int32_p)))
        self._variants = (list(robots), vog)

    # ---- external forces (Engine.register_impulse_force / register_profile_force / remove_all_forces)
    def stop(self) -> None:
        """`Engine.stop`: every env goes back to "not started" (needed before (un)registering forces)."""
        self._api.check(self._api.dll.jb_stop(self._h))

    def _frame(self, frame) -> Tuple[int, np.ndarray]:
        """A frame name of the robot, or an explicit (parent joint index, translation in the joint frame)."""
        if isinstance(frame, str):
            if frame == "universe":
                raise ValueError("Impossible to apply external forces to the universe itself!")
            if frame not in self.robot.frames:
                raise ValueError(f"Frame '{frame}' does not exist.")
            f = self.robot.frames[frame]
            return int(f.joint), np.ascontiguousarray(f.placement.p, dtype=np.float64)
        joint, p = frame
        return int(joint), np.ascontiguousarray(p, dtype=np.float64)

    def _per_env(self, x, shape) -> np.ndarray:
        return np.ascontiguousarray(np.broadcast_to(np.asarray(x, dtype=np.float64), (self.n_env,) + shape))

    def register_impulse_force(self, frame, t, dt, force) -> int:
        """`force` (world-aligned axes, at the frame origin) applied during [t, t + dt) of each env's own
        clock; `t`, `dt` scalars or [n_env], `force` [6] or [n_env, 6].  Returns the impulse index."""
        joint, p = self._frame(frame)
        t, dt, force = self._per_env(t, ()), self._per_env(dt, ()), self._per_env(force, (6,))
        idx = C.c_int32(-1)
        self._api.check(self._api.dll.jb_register_impulse_force(self._h, joint, dptr(p), dptr(t), dptr(dt), dptr(force),
                                                               C.byref(idx)))
        return int(idx.value)

    def set_impulse_force(self, index: int, t, dt, force, mask: Optional[np.ndarray] = None) -> None:
        t, dt, force = self._per_env(t, ()), self._per_env(dt, ()), self._per_env(force, (6,))
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        self._api.check(self._api.dll.jb_set_impulse_force(
            self._h, int(index), None if m is None else m.ctypes.data_as(c_uint8_p), dptr(t), dptr(dt), dptr(force)))

    def register_profile_force(self, frame, update_period: float = 0.0) -> int:
        """A force whose per-env value is whatever `set_profile_force` last wrote (the batched stand-in for
        the reference's Python force function).  Returns the slot index."""
        joint, p = self._frame(frame)
        slot = C.c_int32(-1)
        self._api.check(self._api.dll.jb_register_profile_force(self._h, joint, dptr(p), float(update_period),
                                                               C.byref(slot)))
        return int(slot.value)

    def set_profile_force(self, slot: int, force) -> None:
        force = self._per_env(force, (6,))
        self._api.check(self._api.dll.jb_set_profile_force(self._h, int(slot), dptr(force)))
        self._api.check(self._api.dll.jb_synchronize(self._h))

    def set_impulse_force_device(self, index: int, t_ptr: int, dt_ptr: int, force_ptr: int,
                                 mask_ptr: Optional[int] = None) -> None:
        """`set_impulse_force` from device buffers (t, dt [n_env], force [n_env, 6] fp64, mask [n_env] uint8 or None = all),
        enqueued on the batch stream with no host synchronisation: keep the buffers alive until the stream has passed the
        call.  A row with a NaN, t < 0 or dt < 1e-10 is not written; its env gets JB_ENV_NOT_STARTED | JB_ENV_BAD_START."""
        self._api.check(self._api.dll.jb_set_impulse_force_device(self._h, int(index), C.c_void_p(mask_ptr or None),
                                                                  C.c_void_p(t_ptr), C.c_void_p(dt_ptr), C.c_void_p(force_ptr)))

    def register_process_force(self, frame, components, n_knots, periods, update_period: float = 0.0) -> int:
        """A force whose wrench component `components[k]` (0..5, world-aligned, at the frame origin) is a periodic
        cubic-Hermite table of `n_knots[k]` knots over `periods[k]` seconds, per env, evaluated at the env's own time at
        every dynamics evaluation (update_period 0) or sampled and held at the multiples of `update_period`.  The tables
        start at zero (`set_process_force`).  Returns the process-force index."""
        joint, p = self._frame(frame)
        comp = np.ascontiguousarray(components, dtype=np.int32)
        nk = np.ascontiguousarray(n_knots, dtype=np.int32)
        per = np.ascontiguousarray(periods, dtype=np.float64)
        if not comp.shape == nk.shape == per.shape or comp.ndim != 1:
            raise ValueError("components, n_knots and periods must be 1-D and of the same length")
        idx = C.c_int32(-1)
        self._api.check(self._api.dll.jb_register_process_force(
            self._h, joint, dptr(p), float(update_period), int(comp.size), comp.ctypes.data_as(c_int32_p),
            nk.ctypes.data_as(c_int32_p), dptr(per), C.byref(idx)))
        self._process_knots[int(idx.value)] = int(nk.sum())
        return int(idx.value)

    def set_process_force(self, index: int, values, grads, mask: Optional[np.ndarray] = None) -> None:
        """Knot values and slopes [n_env, sum(n_knots)] of process force `index` (tables one after the other) for the envs
        of `mask` (None = all); the other rows keep their tables."""
        k = self._process_knots[int(index)]
        values, grads = self._per_env(values, (k,)), self._per_env(grads, (k,))
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        self._api.check(self._api.dll.jb_set_process_force(self._h, int(index), None if m is None else m.ctypes.data_as(c_uint8_p),
                                                           dptr(values), dptr(grads)))

    def set_process_force_device(self, index: int, values_ptr: int, grads_ptr: int, mask_ptr: Optional[int] = None) -> None:
        """`set_process_force` from device buffers (values, grads [n_env, sum(n_knots)] fp64, mask [n_env] uint8 or None),
        enqueued on the batch stream with no host synchronisation."""
        self._api.check(self._api.dll.jb_set_process_force_device(self._h, int(index), C.c_void_p(mask_ptr or None),
                                                                  C.c_void_p(values_ptr), C.c_void_p(grads_ptr)))

    def remove_all_forces(self) -> None:
        self._api.check(self._api.dll.jb_remove_all_forces(self._h))
        self._process_knots.clear()

    def set_pd_controller_full(self, kp, kd, state_lower, state_upper, safety=None) -> None:
        """gym_jiminy's `PDController` block on the device (+ `MotorSafetyLimit` when `safety` = [kp, kd, soft_lower,
        soft_upper(, velocity_limit)], each [nmotors]; the velocity limit defaults to the motors' own): `set_command`
        then uploads target motor accelerations.  `state_lower/upper`:
        [3, nmotors] position / velocity / acceleration bounds of the targets.  `kp=None` disables it."""
        if kp is None:
            self._api.check(self._api.dll.jb_set_pd_controller_full(self._h, None, None, None, None, None))
            return
        nm = self.nm
        kp = np.ascontiguousarray(np.broadcast_to(kp, (nm,)), dtype=np.float64)
        kd = np.ascontiguousarray(np.broadcast_to(kd, (nm,)), dtype=np.float64)
        lo = np.ascontiguousarray(state_lower, dtype=np.float64).reshape(3, nm)
        hi = np.ascontiguousarray(state_upper, dtype=np.float64).reshape(3, nm)
        sf = safety_table(safety, self.robot)
        self._api.check(self._api.dll.jb_set_pd_controller_full(self._h, dptr(kp), dptr(kd), dptr(lo), dptr(hi),
                                                                None if sf is None else dptr(sf)))

    def get_constraints(self):
        """(joint_enabled [n_env, njoints], joint_lambda [n_env, njoints], contact_enabled [n_env, ncontacts],
        contact_lambda [n_env, ncontacts, 4]): `is_enabled` / `lambda_c` of the bound and contact constraints."""
        nc = max(len(self.robot.contact_frame_names), 1)
        je, jl = np.zeros((self.n_env, self.nj), dtype=np.uint8), np.zeros((self.n_env, self.nj))
        ce, cl = np.zeros((self.n_env, nc), dtype=np.uint8), np.zeros((self.n_env, nc, 4))
        self._api.check(self._api.dll.jb_get_constraints(self._h, je.ctypes.data_as(c_uint8_p), dptr(jl), ce.ctypes.data_as(c_uint8_p), dptr(cl)))
        n = len(self.robot.contact_frame_names)
        return je.astype(bool), jl, ce[:, :n].astype(bool), cl[:, :n]

    def get_pd_controller_state(self) -> np.ndarray:
        """Target motor position / velocity / acceleration of the `PDController` block, [n_env, 3, nmotors]."""
        out = np.zeros((self.n_env, 3, self.nm))
        self._api.check(self._api.dll.jb_get_pd_controller_state(self._h, dptr(out)))
        return out

    def set_pd_controller_state(self, state) -> None:
        state = np.ascontiguousarray(state, dtype=np.float64).reshape(self.n_env, 3, self.nm)
        self._api.check(self._api.dll.jb_set_pd_controller_state(self._h, dptr(state)))

    def set_mahony_filter(self, kp: Optional[float] = 1.0, ki: float = 0.1) -> None:
        """gym_jiminy's `MahonyFilter` observer on the device (exact_init, no twist removal); `kp=None` disables it."""
        self._api.check(self._api.dll.jb_set_mahony_filter(self._h, -1.0 if kp is None else float(kp), float(ki)))

    def set_mahony_filter_full(self, kp: Optional[float] = 1.0, ki: float = 0.1, exact_init: bool = True,
                               ignore_twist: bool = False, compute_rpy: bool = False) -> None:
        """`MahonyFilter` with the reference's options: `exact_init=False` starts from the measured accelerometer
        (the true orientation in free fall), `ignore_twist` removes the twist after every iteration, `compute_rpy`
        fills the roll-pitch-yaw of `get_observers`.  `kp=None` disables the filter and the body observer."""
        self._api.check(self._api.dll.jb_set_mahony_filter_full(self._h, -1.0 if kp is None else float(kp), float(ki),
                                                                int(bool(exact_init)), int(bool(ignore_twist)),
                                                                int(bool(compute_rpy))))

    def set_body_observer(self, enable: bool = True, twist_time_constant: Optional[float] = None,
                          compute_rpy: bool = True) -> None:
        """gym_jiminy's `BodyObserver` after the Mahony filter: `twist_time_constant` None keeps the filter's twist, 0
        removes it, > 0 re-estimates it with a leaky integrator.  Only between episodes (BadControlFlow while envs
        run)."""
        tc = float("nan") if twist_time_constant is None else float(twist_time_constant)
        self._api.check(self._api.dll.jb_set_body_observer(self._h, int(bool(enable)), tc, int(bool(compute_rpy))))

    def get_observers(self) -> np.ndarray:
        """[n_env, nimu, OBSV_N]: MahonyFilter roll-pitch-yaw, BodyObserver quaternion, roll-pitch-yaw, angular velocity
        and twist angle (BadControlFlow when the filter runs its default path only)."""
        nimu = self.robot.sensor_layout()["ImuSensor"][2]
        out = np.zeros((self.n_env, nimu, OBSV_N))
        self._api.check(self._api.dll.jb_get_observers(self._h, dptr(out)))
        return out

    def device_observer_views(self) -> int:
        """Device pointer of the observer record [n_env, nimu, OBSV_N]; 0 when there is none."""
        o = C.c_void_p()
        self._api.check(self._api.dll.jb_device_observer_views(self._h, C.byref(o)))
        return o.value or 0

    def get_mahony_filter(self) -> np.ndarray:
        """[n_env, nimu, 10]: quaternion estimate (x, y, z, w), gyro bias estimate, unbiased angular velocity."""
        nimu = self.robot.sensor_layout()["ImuSensor"][2]
        out = np.zeros((self.n_env, nimu, 10))
        self._api.check(self._api.dll.jb_get_mahony_filter(self._h, dptr(out)))
        return out

    # ---- observation stacking (gym_jiminy's StackObservation inside the step kernel; see jiminy_b200.observation_stack)
    def set_obs_stack(self, num_stack: int, skip_frames_ratio: int = -1, leaves: Sequence[int] = ()) -> None:
        """Stacks `num_stack` frames of the leaves `leaves` (STACK_* codes, in frame order) at every observer refresh;
        `num_stack=0` turns it off.  Only between episodes (BadControlFlow while envs run)."""
        ids = np.ascontiguousarray(leaves, dtype=np.int32)
        self._api.check(self._api.dll.jb_set_obs_stack(self._h, int(num_stack), int(skip_frames_ratio),
                                                       ids.ctypes.data_as(c_int32_p), len(ids)))
        # [num_stack, frame width] of the stacked frames, None when off
        self.stack_shape = (int(num_stack), sum(self.stack_leaf_width(k) for k in ids)) if num_stack else None

    def stack_leaf_width(self, leaf: int) -> int:
        """Doubles one frame of leaf `leaf` (a STACK_* code) takes."""
        if leaf == STACK_T:
            return 1
        if STACK_IMU <= leaf <= STACK_CONTACT:
            name = ("ImuSensor", "ForceSensor", "EncoderSensor", "EffortSensor", "ContactSensor")[leaf - STACK_IMU]
            return (6, 6, 2, 1, 3)[leaf - STACK_IMU] * self.robot.sensor_layout()[name][2]
        if leaf == STACK_PD_ACTION:
            return self.nm
        if leaf == STACK_PD_STATE:
            return 2 * self.nm
        return (4 if leaf in (STACK_MAHONY, STACK_BODY_QUAT) else 3) * self.robot.sensor_layout()["ImuSensor"][2]

    def get_obs_stack(self) -> np.ndarray:
        """The stacked frames [n_env, num_stack, frame width], oldest first (BadControlFlow when stacking is off)."""
        if getattr(self, "stack_shape", None) is None:
            raise BadControlFlow("observation stacking is not enabled (set_obs_stack)")
        out = np.zeros((self.n_env,) + self.stack_shape)
        self._api.check(self._api.dll.jb_get_obs_stack(self._h, dptr(out)))
        return out

    def device_obs_views(self) -> Tuple[int, int]:
        """Device pointers (stacked frames [n_env, num_stack, frame width], 0 when stacking is off; command buffer
        [n_env, nmotors])."""
        s, c = C.c_void_p(), C.c_void_p()
        self._api.check(self._api.dll.jb_device_obs_views(self._h, C.byref(s), C.byref(c)))
        return s.value or 0, c.value or 0

    # ---- multi-GPU observation exchange over peer memory (one process per GPU)
    def peer_obs_create(self, world: int, rank: int) -> bytes:
        """Allocates this rank's gathered observation buffer `[world][n_env][width]`; returns its CUDA IPC handle."""
        buf = C.create_string_buffer(64)
        self._api.check(self._api.dll.jb_peer_obs_create(self._h, int(world), int(rank), buf))
        return buf.raw

    def peer_obs_connect(self, handles: Sequence[bytes]) -> None:
        """`handles[r]` = what rank r's `peer_obs_create` returned (exchange them with e.g. all_gather_object).
        From now on every `step` publishes this rank's sensor rows into every rank's buffer from inside the kernel."""
        self._api.check(self._api.dll.jb_peer_obs_connect(self._h, b"".join(bytes(h) for h in handles)))

    def peer_obs_wait(self) -> None:
        """Enqueues (on the batch stream) the wait for every rank's rows of the last step."""
        self._api.check(self._api.dll.jb_peer_obs_wait(self._h))

    def peer_obs_enable(self, on: bool) -> None:
        self._api.check(self._api.dll.jb_peer_obs_enable(self._h, 1 if on else 0))

    def peer_obs_view(self) -> int:
        """Device pointer of the gathered observations `[world][n_env][width]` of the last step."""
        p = C.c_void_p()
        self._api.check(self._api.dll.jb_peer_obs_view(self._h, C.byref(p)))
        return int(p.value)

    def set_pd_controller(self, kp, kd) -> None:
        """Device-side `PDController` block (position targets, zero target velocity); `set_command` then
        uploads targets.  `kp=None` disables it."""
        if kp is None:
            self._api.check(self._api.dll.jb_set_pd_controller(self._h, None, None))
            return
        kp = np.ascontiguousarray(np.broadcast_to(kp, (self.nm,)), dtype=np.float64)
        kd = np.ascontiguousarray(np.broadcast_to(kd, (self.nm,)), dtype=np.float64)
        self._api.check(self._api.dll.jb_set_pd_controller(self._h, dptr(kp), dptr(kd)))

    def start(self, q0, v0, mask=None) -> None:
        q0 = np.ascontiguousarray(np.broadcast_to(q0, (self.n_env, self.nq)), dtype=np.float64)
        v0 = np.ascontiguousarray(np.broadcast_to(v0, (self.n_env, self.nv)), dtype=np.float64)
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        self._api.check(self._api.dll.jb_start(self._h, None if m is None else m.ctypes.data_as(c_uint8_p),
                                               dptr(q0), dptr(v0)))

    def start_device(self, q0_ptr: int, v0_ptr: int, mask_ptr: Optional[int] = None, on_ground: bool = False) -> None:
        """`start` from device buffers (q0 [n_env, nq], v0 [n_env, nv] fp64, mask [n_env] uint8 or None = all), enqueued on
        the batch stream with no host synchronisation: keep the buffers alive until the stream has passed the call.  Rows
        that fail the input checks leave their env not started, with status JB_ENV_NOT_STARTED | JB_ENV_BAD_START.
        `on_ground`: each started env's free-flyer height is first shifted so that its lowest contact frame touches z = 0
        (`robots.ground_base_height` in the kernel, `jb_start_device_on_ground`); the buffers are not written."""
        fn = self._api.dll.jb_start_device_on_ground if on_ground else self._api.dll.jb_start_device
        self._api.check(fn(self._h, C.c_void_p(mask_ptr or None), C.c_void_p(q0_ptr), C.c_void_p(v0_ptr)))

    def set_pd_adapter(self, order: int = 1, is_instantaneous: bool = False, velocity_deadband=None) -> None:
        """Configures the device `PDAdapter` block in front of the `PDController` block (`set_pd_controller_full`)."""
        db = None if velocity_deadband is None else \
            np.ascontiguousarray(np.broadcast_to(np.asarray(velocity_deadband, dtype=np.float64), (self.nm,)))
        self._api.check(self._api.dll.jb_set_pd_adapter(self._h, int(order), 1 if is_instantaneous else 0,
                                                        None if db is None else dptr(db)))

    def pd_adapter_device(self, action_ptr: int, step_dt: float) -> None:
        """Device `PDAdapter` on the action buffer [n_env, nmotors] (fp64, device): the target accelerations of the
        coming env-step go to the command buffer.  Asynchronous, on the batch stream."""
        self._api.check(self._api.dll.jb_pd_adapter_device(self._h, C.c_void_p(action_ptr), float(step_dt)))

    def device_block_views(self) -> Tuple[int, int, int]:
        """Device pointers (status [n_env] int32, PD controller state [n_env, 3, nmotors], Mahony filter state
        [n_env, nimu, 10]); 0 where the block is off."""
        s, p, m = C.c_void_p(), C.c_void_p(), C.c_void_p()
        self._api.check(self._api.dll.jb_device_block_views(self._h, C.byref(s), C.byref(p), C.byref(m)))
        return s.value or 0, p.value or 0, m.value or 0

    def set_command(self, cmd) -> None:
        if not self.nm:
            return
        cmd = np.ascontiguousarray(np.broadcast_to(cmd, (self.n_env, self.nm)), dtype=np.float64)
        self._api.check(self._api.dll.jb_set_command(self._h, dptr(cmd)))
        self._api.check(self._api.dll.jb_synchronize(self._h))  # `cmd` may be a temporary

    def set_command_pinned(self, cmd: np.ndarray) -> None:
        """Asynchronous upload from a caller-owned (ideally pinned) C-contiguous fp64 buffer of shape
        (n_env, nmotors); the buffer must stay alive until the stream has consumed it."""
        assert cmd.dtype == np.float64 and cmd.flags.c_contiguous and cmd.size == self.n_env * max(self.nm, 1)
        if self.nm:
            self._api.check(self._api.dll.jb_set_command(self._h, dptr(cmd)))

    def copy_sensors_to(self, dev_ptr: int) -> None:
        self._api.check(self._api.dll.jb_copy_sensors_device(self._h, C.c_void_p(dev_ptr)))

    def set_command_device(self, dev_ptr: int) -> None:
        self._api.check(self._api.dll.jb_set_command_device(self._h, C.c_void_p(dev_ptr)))

    def step(self, step_dt: float = -1.0) -> None:
        self._api.check(self._api.dll.jb_step(self._h, float(step_dt)))

    def synchronize(self) -> None:
        self._api.check(self._api.dll.jb_synchronize(self._h))

    def get_state(self):
        t = np.zeros(self.n_env)
        q, v, a = np.zeros((self.n_env, self.nq)), np.zeros((self.n_env, self.nv)), np.zeros((self.n_env, self.nv))
        self._api.check(self._api.dll.jb_get_state(self._h, dptr(t), dptr(q), dptr(v), dptr(a)))
        return t, q, v, a

    SENSOR_TYPES = ("ImuSensor", "ForceSensor", "EncoderSensor", "EffortSensor", "ContactSensor")

    def set_sensor_options(self, sensor_type: str, index: int, noise_std=None, bias=None, delay: float = 0.0,
                           jitter: float = 0.0, delay_interpolation_order: int = 1) -> None:
        """`sensor.set_options({"noiseStd", "bias", "delay", "jitter", "delayInterpolationOrder"})` of one sensor
        (abstract_sensor.h:66-100): afterwards `get_sensors` returns measurements, `get_sensor_data` the true values."""
        ns = None if noise_std is None else np.ascontiguousarray(noise_std, dtype=np.float64)
        bs = None if bias is None else np.ascontiguousarray(bias, dtype=np.float64)
        self._api.check(self._api.dll.jb_set_sensor_options(
            self._h, self.SENSOR_TYPES.index(sensor_type), int(index), None if ns is None else dptr(ns),
            None if bs is None else dptr(bs), float(delay), float(jitter), int(delay_interpolation_order)))

    def set_seeds(self, seeds) -> None:
        """One engine seed per env (`stepper.randomSeedSeq = [seed]`): consumed at the next start of each env."""
        s = np.ascontiguousarray(seeds, dtype=np.uint32)
        assert s.shape == (self.n_env,)
        self._api.check(self._api.dll.jb_set_seeds(self._h, s.ctypes.data_as(C.POINTER(C.c_uint32))))

    def set_seeds_device(self, seeds_ptr: int, mask_ptr: Optional[int] = None) -> None:
        """`set_seeds` for the envs of `mask` (None = all) from a device buffer (seeds [n_env] uint32, or int32 with the
        same bits), enqueued on the batch stream with no host synchronisation: the generator start states of those envs
        are derived on the device, bit-identical to the host derivation."""
        self._api.check(self._api.dll.jb_set_seeds_device(self._h, C.c_void_p(mask_ptr or None), C.c_void_p(seeds_ptr)))

    def enable_per_env_sensor_options(self, delay_bound: float) -> None:
        """Per-env options for every sensor (`set_sensor_options_env`), all zero until set, in place of the batch-wide
        `set_sensor_options`.  `delay_bound`: the largest delay + jitter any row may hold (sizes the delay buffer)."""
        self._api.check(self._api.dll.jb_enable_per_env_sensor_options(self._h, float(delay_bound)))

    @property
    def n_sensors(self) -> int:
        """Sensors of the measurement pipeline: the rows of `delay` / `jitter` in `set_sensor_options_env`."""
        return sum(self.robot.sensor_layout()[t][2] for t in self.SENSOR_TYPES)

    def set_sensor_options_env(self, noise_std, bias, delay, jitter, mask: Optional[np.ndarray] = None) -> None:
        """Per-env options of the envs of `mask` (None = all): noise_std, bias [n_env, width] in the columns of the sensor
        matrix, delay, jitter [n_env, n_sensors] in the order Imu, Force, Encoder, Effort, Contact.  They apply from each
        env's next start.  A row with a NaN, a negative delay or jitter, or delay + jitter beyond the bound raises
        ValueError and nothing is written."""
        ns = self.n_sensors
        noise_std, bias = self._per_env(noise_std, (self.width,)), self._per_env(bias, (self.width,))
        delay, jitter = self._per_env(delay, (ns,)), self._per_env(jitter, (ns,))
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        self._api.check(self._api.dll.jb_set_sensor_options_env(
            self._h, None if m is None else m.ctypes.data_as(c_uint8_p), dptr(noise_std), dptr(bias), dptr(delay), dptr(jitter)))

    def set_sensor_options_env_device(self, noise_std_ptr: int, bias_ptr: int, delay_ptr: int, jitter_ptr: int,
                                      mask_ptr: Optional[int] = None) -> None:
        """`set_sensor_options_env` from device buffers of the same layouts (fp64; mask [n_env] uint8 or None), enqueued on
        the batch stream with no host synchronisation.  A rejected row is not written and its env stays
        JB_ENV_NOT_STARTED | JB_ENV_BAD_START through its starts until a valid row for it arrives."""
        self._api.check(self._api.dll.jb_set_sensor_options_env_device(
            self._h, C.c_void_p(mask_ptr or None), C.c_void_p(noise_std_ptr), C.c_void_p(bias_ptr), C.c_void_p(delay_ptr),
            C.c_void_p(jitter_ptr)))

    # ---- per-env flexibility parameters (the walker env's `model` randomisation)
    @property
    def n_flex(self) -> int:
        """Flexibility joints of the robot: the rows of `set_flexibility_env`, in `robot.flexibility_joint_indices` order."""
        return len(self.robot.flexibility_joint_names)

    def enable_per_env_flexibility(self) -> None:
        """Per-env stiffness and damping of every flexibility joint (`set_flexibility_env`), starting from each env's
        model values.  Refused on a robot without flexibility joints and on a second call."""
        j = np.ascontiguousarray(self.robot.flexibility_joint_indices, dtype=np.int32)
        self._api.check(self._api.dll.jb_enable_per_env_flexibility(self._h, len(j), j.ctypes.data_as(c_int32_p)))

    def set_flexibility_env(self, rows, mask: Optional[np.ndarray] = None) -> None:
        """Rows [n_env, n_flex, 6] (stiffness xyz, damping xyz per flexibility) of the envs of `mask` (None = all), applied
        from each env's next start.  A value that is not finite or is negative raises ValueError and nothing is written."""
        rows = self._per_env(rows, (self.n_flex, 6))
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        self._api.check(self._api.dll.jb_set_flexibility_env(self._h, None if m is None else m.ctypes.data_as(c_uint8_p), dptr(rows)))

    def set_flexibility_env_device(self, rows_ptr: int, mask_ptr: Optional[int] = None) -> None:
        """`set_flexibility_env` from a device buffer of the same layout (fp64; mask [n_env] uint8 or None), enqueued on
        the batch stream with no host synchronisation.  A rejected row is not written and its env stays
        JB_ENV_NOT_STARTED | JB_ENV_BAD_START through its starts until a valid row for it arrives."""
        self._api.check(self._api.dll.jb_set_flexibility_env_device(self._h, C.c_void_p(mask_ptr or None), C.c_void_p(rows_ptr)))

    def get_flexibility_env(self) -> np.ndarray:
        """The rows every env runs with (latched at its last start), [n_env, n_flex, 6]."""
        out = np.zeros((self.n_env, self.n_flex, 6))
        self._api.check(self._api.dll.jb_get_flexibility_env(self._h, dptr(out)))
        return out

    # ---- per-env model rows (the body biases of the model options, re-drawn per env)
    MODEL_ROW = 13

    def enable_per_env_model(self) -> None:
        """Per-env model rows (`set_model_env`): every env runs its own inertias and joint-placement translations,
        starting from its model values.  Refused on a second call; `set_model_variants` is refused afterwards."""
        self._api.check(self._api.dll.jb_enable_per_env_model(self._h))

    def set_model_env(self, rows, mask: Optional[np.ndarray] = None) -> None:
        """Rows [n_env, njoints, 13] (per joint: mass, lever xyz, inertia about the centre of mass xx xy yy xz yz zz,
        joint-placement translation xyz; joint 0 ignored) of the envs of `mask` (None = all), applied from each env's
        next start.  A value that is not finite or a mass that is not positive raises ValueError and nothing is
        written."""
        rows = self._per_env(rows, (self.robot.njoints, self.MODEL_ROW))
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        self._api.check(self._api.dll.jb_set_model_env(self._h, None if m is None else m.ctypes.data_as(c_uint8_p), dptr(rows)))

    def set_model_env_device(self, rows_ptr: int, mask_ptr: Optional[int] = None) -> None:
        """`set_model_env` from a device buffer of the same layout (fp64; mask [n_env] uint8 or None), enqueued on the
        batch stream with no host synchronisation.  A rejected row is not written and its env stays
        JB_ENV_NOT_STARTED | JB_ENV_BAD_START through its starts until a valid row for it arrives."""
        self._api.check(self._api.dll.jb_set_model_env_device(self._h, C.c_void_p(mask_ptr or None), C.c_void_p(rows_ptr)))

    def get_model_env(self) -> np.ndarray:
        """The rows every env runs with (latched at its last start), [n_env, njoints, 13]."""
        out = np.zeros((self.n_env, self.robot.njoints, self.MODEL_ROW))
        self._api.check(self._api.dll.jb_get_model_env(self._h, dptr(out)))
        return out

    def model(self, env: int) -> "M.RobotTable":
        """The robot table env `env` runs with: the batch's robot with that env's inertias and joint-placement
        translations (`get_model_env`)."""
        return M.with_body_rows(self.robot, self.get_model_env()[env])

    # ---- reward and termination compositions (jiminy_b200.compositions)
    def contact_positions_device(self, out_ptr: int) -> None:
        """Enqueues the world position of every contact frame of every env, from the accepted state and each env's own
        model, into the device buffer `out_ptr` [n_env, ncontacts, 3] (fp64).  Not started / NaN envs read NaN."""
        self._api.check(self._api.dll.jb_contact_positions_device(self._h, C.c_void_p(out_ptr)))

    def set_compositions(self, node_int, node_dbl, n_reward: int, weights, motor_int, motor_dbl, env, training: bool) -> None:
        """Uploads a composition spec (`compositions.Spec` gives the arrays; layout in include/jiminy_b200.h) and empties
        every env's power stacks.  A malformed spec raises ValueError and nothing is uploaded."""
        ni, nd = np.ascontiguousarray(node_int, dtype=np.int32), np.ascontiguousarray(node_dbl, dtype=np.float64)
        w = np.ascontiguousarray(weights, dtype=np.float64)
        mi, md = np.ascontiguousarray(motor_int, dtype=np.int32), np.ascontiguousarray(motor_dbl, dtype=np.float64)
        e = np.ascontiguousarray(env, dtype=np.float64)
        self._api.check(self._api.dll.jb_set_compositions(
            self._h, len(ni), n_reward, ni.ctypes.data_as(c_int32_p), dptr(nd), len(w), dptr(w) if len(w) else None,
            mi.ctypes.data_as(c_int32_p) if len(mi) else None, dptr(md) if len(md) else None, dptr(e), int(bool(training))))

    def compositions_device(self, restart_mask_ptr: Optional[int] = None, num_steps_ptr: int = 0, contact_ptr: int = 0,
                            reward_ptr: int = 0, terminated_ptr: int = 0, truncated_ptr: int = 0, index_ptr: int = 0,
                            values_ptr: int = 0) -> None:
        """Enqueues one launch of the composition kernel (see include/jiminy_b200.h): the evaluation after an env-step,
        or, with `restart_mask_ptr`, the reseeding of the power stacks of the envs that have just (re)started."""
        ptrs = (restart_mask_ptr, num_steps_ptr, contact_ptr, reward_ptr, terminated_ptr, truncated_ptr, index_ptr, values_ptr)
        self._api.check(self._api.dll.jb_compositions_device(self._h, *(C.c_void_p(p or None) for p in ptrs)))

    def get_sensor_data(self) -> np.ndarray:
        out = np.zeros((self.n_env, max(self.width, 1)))
        self._api.check(self._api.dll.jb_get_sensor_data(self._h, dptr(out)))
        return out[:, :self.width]

    def get_centroidal(self):
        """`pinocchio_data.{Ycrb, com, vcom, hg, dhg}` after the last step: (ycrb [n_env, njoints, 10], com [n_env, njoints, 3],
        vcom [n_env, njoints, 3], hg [n_env, 6], dhg [n_env, 6])."""
        n, nj = self.n_env, self.robot.njoints
        y, c, vc, hg, dhg = np.zeros((n, nj, 10)), np.zeros((n, nj, 3)), np.zeros((n, nj, 3)), np.zeros((n, 6)), np.zeros((n, 6))
        self._api.check(self._api.dll.jb_get_centroidal(self._h, dptr(y), dptr(c), dptr(vc), dptr(hg), dptr(dhg)))
        return y, c, vc, hg, dhg

    def get_stepper_state(self):
        """(sched [n_env, 6] = t, dt, dtLargest, dtLargestPrev, tError, tPrev; command held since the last controller update)."""
        sched, cmd = np.zeros((self.n_env, 6)), np.zeros((self.n_env, max(self.nm, 1)))
        self._api.check(self._api.dll.jb_get_stepper_state(self._h, dptr(sched), dptr(cmd)))
        return sched, cmd[:, :self.nm]

    def set_stepper_state(self, sched=None, q=None, v=None, a=None, iters=None, iters_failed=None, command_held=None) -> None:
        """Checkpoint restore: overwrites the given parts of the running state of every env."""
        def arr(x, shape, dtype=np.float64):
            if x is None:
                return None
            x = np.ascontiguousarray(x, dtype=dtype)
            assert x.shape == shape, (x.shape, shape)
            return x
        n = self.n_env
        keep = [arr(sched, (n, 6)), arr(q, (n, self.nq)), arr(v, (n, self.nv)), arr(a, (n, self.nv)),
                arr(iters, (n,), np.int64), arr(iters_failed, (n,), np.int64), arr(command_held, (n, self.nm))]
        ptr = [None if x is None else (x.ctypes.data_as(c_int64_p) if x.dtype == np.int64 else dptr(x)) for x in keep]
        self._api.check(self._api.dll.jb_set_stepper_state(self._h, *ptr))

    def get_efforts(self):
        u, um = np.zeros((self.n_env, self.nv)), np.zeros((self.n_env, max(self.nm, 1)))
        cmd, fext = np.zeros((self.n_env, max(self.nm, 1))), np.zeros((self.n_env, self.nj, 6))
        self._api.check(self._api.dll.jb_get_efforts(self._h, dptr(u), dptr(um), dptr(cmd), dptr(fext)))
        return u, um[:, :self.nm], cmd[:, :self.nm], fext

    def get_sensors(self, out: Optional[np.ndarray] = None) -> np.ndarray:
        if out is None:
            out = np.zeros((self.n_env, max(self.width, 1)))
        self._api.check(self._api.dll.jb_get_sensors(self._h, dptr(out)))
        return out[:, :self.width]

    def get_extra_terms(self):
        """(energy [n, 2] = kinetic, potential; joint accelerations [n, njoints, 6]; joint wrenches [n, njoints, 6])
        of the accepted state: what `computeExtraTerms` leaves in `pinocchio_data` (engine.cc:800-905)."""
        e = np.zeros((self.n_env, 2))
        ja, jf = np.zeros((self.n_env, self.nj, 6)), np.zeros((self.n_env, self.nj, 6))
        self._api.check(self._api.dll.jb_get_extra_terms(self._h, dptr(e), dptr(ja), dptr(jf)))
        return e, ja, jf

    def get_status(self) -> np.ndarray:
        s = np.zeros(self.n_env, dtype=np.int32)
        self._api.check(self._api.dll.jb_get_status(self._h, s.ctypes.data_as(c_int32_p)))
        return s

    def get_iters(self):
        it, itf = np.zeros(self.n_env, dtype=np.int64), np.zeros(self.n_env, dtype=np.int64)
        self._api.check(self._api.dll.jb_get_iters(self._h, it.ctypes.data_as(c_int64_p), itf.ctypes.data_as(c_int64_p)))
        return it, itf

    def compute_dynamics(self, q, v, cmd=None):
        q = np.ascontiguousarray(np.broadcast_to(q, (self.n_env, self.nq)), dtype=np.float64)
        v = np.ascontiguousarray(np.broadcast_to(v, (self.n_env, self.nv)), dtype=np.float64)
        cmd = np.zeros((self.n_env, max(self.nm, 1))) if cmd is None else \
            np.ascontiguousarray(np.broadcast_to(cmd, (self.n_env, max(self.nm, 1))), dtype=np.float64)
        a, fext, u = np.zeros((self.n_env, self.nv)), np.zeros((self.n_env, self.nj, 6)), np.zeros((self.n_env, self.nv))
        self._api.check(self._api.dll.jb_compute_dynamics(self._h, dptr(q), dptr(v), dptr(cmd), dptr(a), dptr(fext), dptr(u)))
        return a, fext, u

    def device_views(self):
        s, qv = C.c_void_p(), C.c_void_p()
        self._api.check(self._api.dll.jb_device_views(self._h, C.byref(s), C.byref(qv)))
        return s.value, qv.value

    def state_views(self) -> Dict[str, np.ndarray]:
        """Zero-copy views of the state (`jb_state_ptrs`): numpy arrays over pinned host memory that every `start` /
        `step` refreshes behind the kernel -- the batched counterpart of the array views the reference hands out for
        `stepper_state.q`, `robot_state.v`, `robot.sensor_measurements` (functors.h:57-68).  The arrays are created
        once and keep their address; read them after `synchronize()` (or any getter).  Keys: t [n], q [n, nq],
        v [n, nv], a [n, nv], sensors [n, width]; treat them as read-only."""
        if getattr(self, "_views", None) is None:
            hv = JbStateViews()
            self._api.check(self._api.dll.jb_state_ptrs(self._h, C.byref(hv), None))
            n = self.n_env
            qv = np.ctypeslib.as_array(hv.qv, shape=(n, self.nq + self.nv))
            self._views = {
                "t": np.ctypeslib.as_array(hv.t, shape=(n,)),
                "q": qv[:, :self.nq], "v": qv[:, self.nq:],
                "a": np.ctypeslib.as_array(hv.a, shape=(n, max(self.nv, 1)))[:, :self.nv],
                "sensors": np.ctypeslib.as_array(hv.sensors, shape=(n, max(self.width, 1)))[:, :self.width],
            }
        return self._views

    def device_state_ptrs(self) -> Dict[str, int]:
        """Device pointers of `jb_state_ptrs`: t [n_env], qv [n_env, nq + nv], sensors [n_env, width] (env-major)."""
        dv = JbStateViews()
        self._api.check(self._api.dll.jb_state_ptrs(self._h, None, C.byref(dv)))
        return {"t": C.cast(dv.t, C.c_void_p).value or 0, "qv": C.cast(dv.qv, C.c_void_p).value or 0,
                "sensors": C.cast(dv.sensors, C.c_void_p).value or 0}

    def stream(self) -> int:
        s = C.c_void_p()
        self._api.check(self._api.dll.jb_get_stream(self._h, C.byref(s)))
        return s.value or 0

    def launch_count(self) -> int:
        return int(self._api.dll.jb_launch_count(self._h))

    def simulate(self, t_end: float, q0, v0, log: bool = True):
        """`Engine::simulate` (engine.cc:1614-1699) for every env; returns logged (t, q, v, a) of env 0..N-1."""
        self.start(q0, v0)
        st = self._opt
        period = min([p for p in (st.sensors_update_period, st.controller_update_period) if p > 2.3e-16], default=np.inf)
        ts, qs, vs, as_ = [], [], [], []

        def snap():
            t, q, v, a = self.get_state()
            ts.append(t.copy()); qs.append(q.copy()); vs.append(v.copy()); as_.append(a.copy())
        if log:
            snap()
        t = 0.0
        while t_end - t >= 1e-6:
            h = min(period if np.isfinite(period) else st.dt_max, t_end - t)
            self.step(h)
            t = float(self.get_state()[0][0])
            if log:
                snap()
        return np.array(ts), np.array(qs), np.array(vs), np.array(as_)


# ------------------------------------------------------------------------------------------------
# Single-env facade with the reference's names (python/jiminy_pywrap/src/engine.cc:587-787)
# ------------------------------------------------------------------------------------------------
class RobotState:
    """`jiminy.RobotState` (pywrap engine.cc:175-187): stable numpy buffers refreshed in place after
    every `start` / `step`, as `BaseJiminyEnv` expects (generic.py:688-690)."""

    def __init__(self, nq: int, nv: int, nm: int, nj: int):
        self.q, self.v, self.a = np.zeros(nq), np.zeros(nv), np.zeros(nv)
        self.command, self.u, self.u_motor = np.zeros(nm), np.zeros(nv), np.zeros(nm)
        self.f_external = np.zeros((nj, 6))


class StepperState:
    """`jiminy.StepperState` (pywrap engine.cc:134-143)."""

    def __init__(self, nq: int, nv: int):
        self.iter, self.iter_failed, self.t, self.dt = 0, 0, 0.0, 0.0
        self.q, self.v, self.a = np.zeros(nq), np.zeros(nv), np.zeros(nv)


class FunctionalController:
    """`jiminy.FunctionalController(compute_command, internal_dynamics)` (controller_functor.h:27-80).
    `compute_command(t, q, v, sensor_measurements, command)` is evaluated on the host at every
    controller breakpoint and held in between (discrete controllers only)."""

    def __init__(self, compute_command=None, internal_dynamics=None):
        if internal_dynamics is not None:
            raise NotImplementedError("Python `internal_dynamics` callbacks cannot run inside the device step; "
                                      "use `Engine.set_joint_springs` for the linear case.")
        self.compute_command = compute_command


class Engine:
    """One-robot, one-env engine with the surface `jiminy_py.simulator.Simulator` / `BaseJiminyEnv` use:
    `add_robot`, `get_options / set_options`, `start`, `step`, `stop`, `simulate`, `robot_states`,
    `stepper_state`, `is_simulation_running`.  The physics runs on the GPU (a batch of one env); a
    Python controller is called back on the host once per controller period, like the reference
    does through `FunctionalController` (engine.cc:1920-1940)."""

    def __init__(self, device: int = 0, api_: Optional[Api] = None):
        self._device, self._api_ = device, api_
        self._options = M.default_engine_options()
        self._options["contacts"]["model"] = "spring_damper"
        self.robots: list = []
        self.robot_states: list = []
        self.stepper_state: Optional[StepperState] = None
        self.is_simulation_running = False
        self._batch: Optional[BatchedEngine] = None
        self._controller: Optional[FunctionalController] = None
        self._springs = None
        self._impulse_forces: list = []
        self._profile_forces: list = []       # [frame, function, update period, device slot]
        self._forces_dirty = False
        self._recorder = None

    # -- configuration
    def add_robot(self, robot: M.RobotTable, controller: Optional[FunctionalController] = None) -> None:
        if self.robots:
            raise NotImplementedError("Multi-robot engines are outside the accelerated path.")
        if isinstance(robot, M.Robot):       # the engine simulates the extended model (flexibilities, biases, backlash)
            robot = robot.extended
        self.robots.append(robot)
        self._controller = controller
        self.robot_states = [RobotState(robot.nq, robot.nv, robot.nmotors, robot.njoints)]
        self.stepper_state = StepperState(robot.nq, robot.nv)

    def get_options(self) -> Dict[str, Any]:
        import copy
        return copy.deepcopy(self._options)

    def set_options(self, options: Dict[str, Any]) -> None:
        if self.is_simulation_running:
            raise BadControlFlow("Please stop the simulation before updating the options.")
        M.validate_options(options)
        self._options = options
        self._batch = None

    def set_joint_springs(self, stiffness, damping) -> None:
        self._springs = (np.asarray(stiffness, dtype=np.float64), np.asarray(damping, dtype=np.float64))

    # -- external forces (python/jiminy_pywrap/src/engine.cc:651-657, :761)
    def register_impulse_force(self, robot_name: str, frame_name: str, t: float, dt: float, force) -> None:
        if self.is_simulation_running:
            raise BadControlFlow("Simulation already running. Please stop it before registering new forces.")
        if dt < 1e-10:
            raise ValueError("Force duration cannot be smaller than 1e-10s.")
        if t < 0.0:
            raise ValueError("Force application time must be positive.")
        if frame_name == "universe":
            raise ValueError("Impossible to apply external forces to the universe itself!")
        if not self.robots or frame_name not in self.robots[0].frames:
            raise ValueError(f"Frame '{frame_name}' does not exist.")
        self._impulse_forces.append((frame_name, float(t), float(dt), np.asarray(force, dtype=np.float64).copy()))
        self._forces_dirty = True

    def register_profile_force(self, robot_name: str, frame_name: str, force_func, update_period: float = 0.0) -> None:
        """`Engine.register_profile_force` (pywrap engine.cc:655; Engine::registerProfileForce, engine.cc:2518-2567) for a
        force function sampled at a finite `update_period`: `force_func(t, q, v, out)` is called on the host at every
        multiple of the period -- which is an integration breakpoint, as in the reference -- and its value held in
        between.  A time-continuous function (`update_period = 0`) would have to run inside the device integrator."""
        if self.is_simulation_running:
            raise BadControlFlow("Simulation already running. Please stop it before registering new forces.")
        if not (update_period > 1e-10):
            raise NotImplementedError("A time-continuous Python force function cannot be called from inside the device-side "
                                      "integrator: give it an update period, or use BatchedEngine.set_profile_force.")
        if frame_name == "universe":
            raise ValueError("Impossible to apply external forces to the universe itself!")
        if not self.robots or frame_name not in self.robots[0].frames:
            raise ValueError(f"Frame '{frame_name}' does not exist.")
        self._profile_forces.append([frame_name, force_func, float(update_period), -1])
        self._forces_dirty = True

    def remove_all_forces(self) -> None:
        if self.is_simulation_running:
            raise BadControlFlow("Simulation already running. Please stop it before removing forces.")
        self._impulse_forces.clear()
        self._profile_forces.clear()
        self._forces_dirty = True

    @property
    def impulse_forces(self) -> list:
        return list(self._impulse_forces)

    # -- life cycle
    def _refresh(self) -> None:
        b, rs, ss = self._batch, self.robot_states[0], self.stepper_state
        t, q, v, a = b.get_state()
        u, um, cmd, fext = b.get_efforts()
        for dst, src in ((rs.q, q[0]), (rs.v, v[0]), (rs.a, a[0]), (rs.u, u[0]), (rs.u_motor, um[0]),
                         (rs.f_external, fext[0]), (ss.q, q[0]), (ss.v, v[0]), (ss.a, a[0])):
            np.copyto(dst, src)
        ss.t = float(t[0])
        it, itf = b.get_iters()
        ss.iter, ss.iter_failed = int(it[0]), int(itf[0])
        self._sensors = b.get_sensors()[0].copy()

    def _call_controller(self) -> None:
        if self._controller is None or self._controller.compute_command is None:
            return
        rs = self.robot_states[0]
        rs.command[:] = 0.0
        self._controller.compute_command(self.stepper_state.t, rs.q, rs.v, self._sensors, rs.command)
        self._batch.set_command(rs.command[None, :])

    def start(self, q_init, v_init, a_init=None, is_state_theoretical: bool = False) -> None:
        if not self.robots:
            raise BadControlFlow("No robot to simulate. Please add one before starting a simulation.")
        if self.is_simulation_running:
            raise BadControlFlow("A simulation is already running. Please stop it before starting a new one.")
        robot = self.robots[0]
        if self._controller is not None and self._controller.compute_command is not None and \
                self._options["stepper"]["controllerUpdatePeriod"] <= 0.0:
            raise NotImplementedError("A Python controller needs a discrete controllerUpdatePeriod: it cannot be "
                                      "called from inside the device-side integrator.")
        if self._batch is None:
            self._batch = BatchedEngine(robot, self._options, 1, device=self._device, api_=self._api_)
            if self._springs is not None:
                self._batch.set_joint_springs(*self._springs)
            self._forces_dirty = bool(self._impulse_forces or self._profile_forces)
        if self._forces_dirty:
            self._batch.stop()
            self._batch.remove_all_forces()
            for frame_name, t, dt, force in self._impulse_forces:
                self._batch.register_impulse_force(frame_name, t, dt, force)
            for pf in self._profile_forces:
                pf[3] = self._batch.register_profile_force(pf[0], pf[2])
            self._forces_dirty = False
        q0 = np.asarray(q_init, dtype=np.float64).reshape(1, robot.nq)
        v0 = np.asarray(v_init, dtype=np.float64).reshape(1, robot.nv)
        self._batch.set_command(np.zeros((1, max(robot.nmotors, 1))))
        for pf in self._profile_forces:      # the forces at t = 0 take part in the initial acceleration
            out = np.zeros(6)
            pf[1](0.0, q0[0], v0[0], out)
            self._batch.set_profile_force(pf[3], out[None, :])
        self._batch.start(q0, v0)
        self._refresh()
        if self._controller is not None and self._controller.compute_command is not None:
            # the command participates in the initial acceleration (INIT_ITERATIONS loop, engine.cc:1400-1467)
            self._call_controller()
            self._batch.start(q0, v0)
            self._refresh()
        st = int(self._batch.get_status()[0])
        if st & JB_ENV_CONTACT_FORCE:
            raise ValueError("The initial force exceeds 1e5 for at least one contact point, which is forbidden for "
                             "the sake of numerical stability. Please update the initial state.")
        self.is_simulation_running = True
        # telemetry (Engine::start registers the variables and logs the initial state, engine.cc:1495-1527, :1550)
        from .telemetry import TelemetryRecorder
        self._recorder = TelemetryRecorder(robot, self._options)
        self._log_snapshot()

    def _log_snapshot(self) -> None:
        rs, rec = self.robot_states[0], self._recorder
        keys = {k for k, _ in rec._groups}
        energy = float(self._batch.get_extra_terms()[0][0].sum()) if "energy" in keys else None
        rec.append(self.stepper_state.t, rs.q, rs.v, rs.a, sensors=self._sensors if "sensors" in keys else None,
                   u=rs.u, command=rs.command, energy=energy)

    @property
    def log_data(self) -> dict:
        """`Engine.log_data` (pywrap engine.cc:776): constants and variables of the current / last simulation."""
        if self._recorder is None:
            raise BadControlFlow("No simulation has been started: there is no log to read.")
        return self._recorder.log_data

    def write_log(self, fullpath: str, format: str = "binary") -> None:
        """`Engine.write_log` (engine.cc:3975-4060), binary format (`TelemetryRecorder::writeLog`)."""
        if format != "binary":
            raise NotImplementedError("Only the 'binary' log format is written (the hdf5 one needs h5py).")
        if self._recorder is None or not self._recorder._times:
            raise BadControlFlow("No data available. Please start a simulation before writing log.")
        self._recorder.write_log(fullpath)

    def step(self, step_dt: float = -1.0) -> None:
        if not self.is_simulation_running:
            raise BadControlFlow("No simulation running. Please start one before using step method.")
        st = self._options["stepper"]
        cp = float(st["controllerUpdatePeriod"])
        if step_dt < 2.3e-16:
            step_dt = cp if cp > 0 else (st["sensorsUpdatePeriod"] if st["sensorsUpdatePeriod"] > 0 else st["dtMax"])
        has_cb = self._controller is not None and self._controller.compute_command is not None
        t_end = self.stepper_state.t + step_dt
        while t_end - self.stepper_state.t >= 1e-10:
            h = t_end - self.stepper_state.t
            t = self.stepper_state.t
            if has_cb:
                # stop at every controller breakpoint to call the Python controller back
                nxt = (np.floor(t / cp + 1e-9) + 1.0) * cp
                if abs(t / cp - round(t / cp)) < 1e-9:
                    self._call_controller()
                h = min(h, nxt - t)
            for frame_name, func, period, slot in self._profile_forces:
                # ... and at every update of a sampled force function
                if abs(t / period - round(t / period)) < 1e-9:
                    out = np.zeros(6)
                    func(t, self.robot_states[0].q, self.robot_states[0].v, out)
                    self._batch.set_profile_force(slot, out[None, :])
                h = min(h, (np.floor(t / period + 1e-9) + 1.0) * period - t)
            self._batch.step(h)
            self._refresh()
            status = int(self._batch.get_status()[0])
            if status & JB_ENV_NAN:
                raise RuntimeError("Low-level ode solver failed. Consider increasing stepper accuracy.")
            if status & JB_ENV_ITER_FAILED:
                raise RuntimeError("Too many successive iteration failures. Probably something is wrong with the "
                                   "physics. Aborting integration.")
            if status & JB_ENV_DT_UNDERFLOW:
                raise RuntimeError("The internal time step is getting too small. Impossible to integrate physics "
                                   "further in time. Aborting integration.")
            self._log_snapshot()      # one line per engine step (telemetry.logInternalStepperSteps = false)

    def stop(self) -> None:
        self.is_simulation_running = False

    def reset(self, reset_random_generator: bool = False, remove_all_forces: bool = False) -> None:
        self.stop()
        if remove_all_forces:
            self.remove_all_forces()

    def simulate(self, t_end: float, q_init, v_init, a_init=None, is_state_theoretical: bool = False,
                 callback=None) -> None:
        """`Engine::simulate` (engine.cc:1614-1699)."""
        self.reset()
        self.start(q_init, v_init)
        st = self._options["stepper"]
        periods = [p for p in (st["sensorsUpdatePeriod"], st["controllerUpdatePeriod"]) if p > 0]
        h = min(periods) if periods else st["dtMax"]
        while t_end - self.stepper_state.t >= 1e-6:
            if callback is not None and not callback():
                break
            self.step(min(h, t_end - self.stepper_state.t))
        self.stop()

    @property
    def sensor_measurements(self) -> np.ndarray:
        return self._sensors
