"""The BASELINE.json configs made concrete (SURVEY.md 8d): robot, engine options, initial-state
distribution, controller and per-step action distribution.  Shared by bench.py, the parity tests
and `__graft_entry__.smoke()` so that the GPU path, the oracle and the CPU baseline all run the
very same synthetic workload.

Legged robots are driven through the PD controller block of the reference's own gym pipelines
(`ANYmalPDControlJiminyEnv`, python/gym_jiminy/envs/gym_jiminy/envs/anymal.py:27-31,:82-96;
`AtlasPDControlJiminyEnv`, atlas.py:45-75) with per-step random position targets around a standing
posture: with raw random torques the spring-damper contact model (k = 4e6 N/m) and fixed-step RK4
leave the well-posed regime within a few hundred milliseconds (joints cross their bounds, which
the reference would hand to its constraint solver -- a later scope row), so the throughput of a
collapsing robot would not be a meaningful number.
"""
from __future__ import annotations

import copy
import json
import os
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

from . import robots as R
from .model import RobotTable

# PD gains of the reference envs, keyed by motor-name suffix (atlas.py:45-75)
_ATLAS_KP = {"back_bkz": 5000.0, "back_bky": 8000.0, "back_bkx": 5000.0,
             "arm_shz": 500.0, "arm_shx": 100.0, "arm_ely": 200.0, "arm_elx": 500.0, "arm_wry": 10.0,
             "arm_wrx": 100.0, "arm_wry2": 10.0, "neck_ry": 100.0,
             "leg_hpz": 5000.0, "leg_hpx": 5000.0, "leg_hpy": 8000.0, "leg_kny": 4000.0, "leg_aky": 8000.0,
             "leg_akx": 5000.0}
_ATLAS_KD = {"back_bkz": 0.01, "back_bky": 0.015, "back_bkx": 0.02,
             "arm_shz": 0.01, "arm_shx": 0.01, "arm_ely": 0.01, "arm_elx": 0.02, "arm_wry": 0.01,
             "arm_wrx": 0.02, "arm_wry2": 0.02, "neck_ry": 0.01,
             "leg_hpz": 0.01, "leg_hpx": 0.02, "leg_hpy": 0.02, "leg_kny": 0.01, "leg_aky": 0.025,
             "leg_akx": 0.01}


def _gain(table, motor_name: str) -> float:
    for key in sorted(table, key=len, reverse=True):
        if motor_name.endswith(key):
            return table[key]
    raise KeyError(motor_name)


@dataclass
class Scenario:
    name: str
    robot: RobotTable
    options: dict
    n_env: int
    step_dt: float
    q0: np.ndarray
    v0: np.ndarray
    kp: Optional[np.ndarray]          # None: the action is the motor effort itself
    kd: Optional[np.ndarray]
    target0: np.ndarray               # action held during start()
    action_noise: float
    seed: int
    description: str = ""
    _motor_q: np.ndarray = field(default_factory=lambda: np.zeros(0, dtype=np.int64))
    torque_amplitude: float = 0.0     # > 0: raw effort actions U(-amplitude, amplitude) (SURVEY.md 8d config 3 as written)
    flagged_fraction: float = 0.0     # PD mode: this share of the envs drives its hip-abduction targets beyond the joint bounds
    rigid_robot: Optional[RobotTable] = None   # the model without flexibility joints ("anymal_flexible")
    _torch_tables: dict = field(default_factory=dict, repr=False)

    def draw_initial_torch(self, gen, n: int, device):
        """`n` rows (q [n, nq], v [n, nv], fp64 tensors on `device`) of the initial-state distribution of `make`, drawn
        with the torch generator `gen`, BEFORE the feet are put on the ground (`jb_start_device_on_ground` does that on the
        device).  The free-flyer keeps the posture's base row."""
        import torch
        dev = torch.device(device)
        f64 = dict(dtype=torch.float64, device=dev)
        name = "anymal" if self.name == "anymal_flexible" else self.name
        if name == "cartpole":
            x = torch.rand((n, 4), generator=gen, **f64) * (2 * CARTPOLE_HALF_WIDTH) - CARTPOLE_HALF_WIDTH
            return torch.stack([x[:, 0], torch.cos(x[:, 1]), torch.sin(x[:, 1])], dim=1), x[:, 2:4].clone()
        if name == "double_pendulum":
            return torch.tensor(DOUBLE_PENDULUM_Q0, **f64).expand(n, 2).clone(), torch.zeros((n, 2), **f64)
        if name not in ("anymal", "atlas"):
            raise KeyError(self.name)
        rigid = self.rigid_robot if self.rigid_robot is not None else self.robot
        key = str(dev)
        if key not in self._torch_tables:
            qs = standing_start(name, rigid)
            t = {"qs": torch.as_tensor(qs, **f64), "lo": torch.as_tensor(rigid.q_lower[7:], **f64),
                 "hi": torch.as_tensor(rigid.q_upper[7:], **f64)}
            if self.rigid_robot is not None:
                # model.extended_state_from_theoretical: every rigid coordinate copied by joint name, the flexibility
                # joints at the neutral (identity) quaternion
                from .model import JOINT_NQ
                src, dst = [], []
                for j in range(1, rigid.njoints):
                    k = self.robot.joint_index(rigid.joint_names[j])
                    nqj = JOINT_NQ[int(rigid.joint_type[j])]
                    src += range(rigid.idx_q[j], rigid.idx_q[j] + nqj)
                    dst += range(self.robot.idx_q[k], self.robot.idx_q[k] + nqj)
                t["src"] = torch.as_tensor(src, dtype=torch.int64, device=dev)
                t["dst"] = torch.as_tensor(dst, dtype=torch.int64, device=dev)
                t["neutral"] = torch.as_tensor(self.robot.neutral(), **f64)
            self._torch_tables[key] = t
        t = self._torch_tables[key]
        # U(-w, w) as numpy's Generator.uniform draws it: low + (high - low) * U[0, 1)
        pert = torch.rand((n, rigid.nq - 7), generator=gen, **f64) * (2 * JOINT_PERTURBATION) - JOINT_PERTURBATION
        q = t["qs"].expand(n, rigid.nq).clone()
        q[:, 7:] = torch.minimum(torch.maximum(q[:, 7:] + pert, t["lo"]), t["hi"])
        if self.rigid_robot is not None:
            qe = t["neutral"].expand(n, self.robot.nq).clone()
            qe[:, t["dst"]] = q[:, t["src"]]
            q = qe
        return q, torch.zeros((n, self.robot.nv), **f64)

    def sample_targets(self, k: int) -> np.ndarray:
        """Action of env-step k, reproducible: position targets (PD mode) or efforts."""
        rng = np.random.default_rng([self.seed, 7919, k])
        if self.name == "cartpole":
            # per env random element of {-limit, 0, +limit} (cartpole.py:139-147)
            lim = self.robot.motors[0].effort_limit
            return rng.integers(-1, 2, size=(self.n_env, 1)).astype(np.float64) * lim
        if self.torque_amplitude > 0.0:
            return rng.uniform(-self.torque_amplitude, self.torque_amplitude, size=(self.n_env, max(self.robot.nmotors, 1)))
        if self.kp is None:
            return np.zeros((self.n_env, max(self.robot.nmotors, 1)))
        act = self.target0 + rng.uniform(-self.action_noise, self.action_noise, size=self.target0.shape)
        if self.flagged_fraction > 0.0:
            # every (1/fraction)-th env pushes its hip-abduction joints through their position bounds: those envs leave
            # the hot path and are stepped by the full body with their joint-bound constraints (spread over the warps)
            stride = max(1, int(round(1.0 / self.flagged_fraction)))
            haa = [k for k, m in enumerate(self.robot.motors) if "HAA" in m.name.upper() or "shx" in m.name]
            for j in haa:
                act[::stride, j] = self.robot.q_upper[self._motor_q[j]] + 0.3
        return act

    def algorithmic_bytes_per_env_step(self) -> int:
        """SURVEY.md 8d: compulsory HBM traffic of one env-step: read (q, v, a, command), write
        (q, v, a, sensor row, t)."""
        r = self.robot
        w = r.sensor_layout()["width"][0]
        return 8 * ((r.nq + 2 * r.nv + r.nmotors) + (r.nq + 2 * r.nv + w + 1))


# The initial-state distribution of the legged scenarios (read by `make` and `Scenario.draw_initial_torch`): the standing
# posture kept JOINT_MARGIN rad inside the joint bounds, plus U(-JOINT_PERTURBATION, JOINT_PERTURBATION) rad on every
# joint, clipped to the bounds, zero velocity, then the feet put on the ground.
JOINT_MARGIN = 0.25
JOINT_PERTURBATION = 0.05
# cartpole: x, theta, dx, dtheta ~ U(-w, w) (cartpole.py:184-199); double pendulum: q0 (double_pendulum.cc:123-126)
CARTPOLE_HALF_WIDTH = 0.05
DOUBLE_PENDULUM_Q0 = (0.0, 0.1)


def standing_start(name: str, robot: RobotTable) -> np.ndarray:
    """The standing posture kept JOINT_MARGIN inside the joint bounds (Atlas' neutral arm pose sits exactly on some of
    them): a joint leaving its bounds switches the env to the (slower) constraint path."""
    qs = standing_posture(name, robot)
    qs[7:] = np.clip(qs[7:], robot.q_lower[7:] + JOINT_MARGIN, robot.q_upper[7:] - JOINT_MARGIN)
    return qs


def standing_posture(name: str, robot: RobotTable) -> np.ndarray:
    q = robot.neutral()
    if name == "anymal":
        # crouched "X" stance: front knees bend backward, hind knees forward (feet stay under the hips)
        for leg, s in (("LF", 1.0), ("RF", 1.0), ("LH", -1.0), ("RH", -1.0)):
            q[robot.idx_q[robot.joint_index(leg + "_HFE")]] = 0.4 * s
            q[robot.idx_q[robot.joint_index(leg + "_KFE")]] = -0.8 * s
    elif name == "atlas":
        with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "robots", "atlas.json")) as fh:
            q = np.array(json.load(fh)["meta"]["neutral"])  # AtlasJiminyEnv._neutral (atlas.py:147-166)
        # slightly bent knees, torso kept upright and feet flat (hip + knee + ankle pitch = 0): the
        # reference neutral has the knees exactly on their lower bound
        for side in ("l", "r"):
            q[robot.idx_q[robot.joint_index(f"{side}_leg_kny")]] = 0.3
            q[robot.idx_q[robot.joint_index(f"{side}_leg_hpy")]] = -0.15
            q[robot.idx_q[robot.joint_index(f"{side}_leg_aky")]] = -0.15
    return q


# flexibilities of the "anymal_flexible" scenario (`modelOptions["dynamics"]["flexibilityConfig"]` of the reference)
FLEXIBLE_ANYMAL_CONFIG = [dict(frameName=jn, stiffness=[5e3, 4e3, 6e3], damping=[20.0, 30.0, 25.0], inertia=[0.05, 0.04, 0.06])
                          for jn in ("LF_HFE", "RF_KFE", "LH_HAA", "RH_HFE")]


def make(name: str, n_env: int, seed: int = 0, dt_max: Optional[float] = None, solver: Optional[str] = None,
         contact_model: Optional[str] = None, action: str = "pd", flagged_fraction: float = 0.0) -> Scenario:
    if name == "anymal_flexible":
        # the ANYmal scenario with `dynamics.enableFlexibility`: a flexibility joint in front of a joint of every leg
        # (Model::addFlexibilityJointsToExtendedModel), undeformed at the start
        from . import model as M
        sc = make("anymal", n_env, seed=seed, dt_max=dt_max, solver=solver, contact_model=contact_model, action=action,
                  flagged_fraction=flagged_fraction)
        rigid = sc.robot
        sc.robot = M.add_flexibility_joints(rigid, FLEXIBLE_ANYMAL_CONFIG)
        sc.q0, sc.v0 = M.extended_state_from_theoretical(sc.robot, rigid, sc.q0, sc.v0)
        sc._motor_q = np.array([sc.robot.idx_q[m.joint] for m in sc.robot.motors])
        sc.rigid_robot = rigid
        sc.name, sc.description = name, sc.description.replace("anymal:", "anymal with 4 flexibility joints:")
        return sc
    robot, base = R.load_robot(name)
    opt = R.baseline_options(name, copy.deepcopy(base))
    if dt_max is not None:
        opt["stepper"]["dtMax"] = dt_max
    if solver is not None:
        opt["stepper"]["odeSolver"] = solver
    if contact_model is not None:
        opt["contacts"]["model"] = contact_model
    rng = np.random.default_rng([seed, 104729])
    nm = max(robot.nmotors, 1)
    if name in ("anymal", "atlas"):
        qs = standing_start(name, robot)
        q0 = np.tile(qs, (n_env, 1))
        # per-env joint perturbation, feet on the ground
        pert = rng.uniform(-JOINT_PERTURBATION, JOINT_PERTURBATION, size=(n_env, robot.nq - 7))
        q0[:, 7:] = np.clip(q0[:, 7:] + pert, robot.q_lower[7:], robot.q_upper[7:])
        for i in range(n_env):
            q0[i] = R.ground_base_height(robot, q0[i])
        v0 = np.zeros((n_env, robot.nv))
        mq = np.array([robot.idx_q[m.joint] for m in robot.motors])
        if name == "anymal":
            kp = np.full(robot.nmotors, 1500.0)   # anymal.py:27-31
            kd = np.full(robot.nmotors, 0.01)
        else:
            kp = np.array([_gain(_ATLAS_KP, m.name) for m in robot.motors])
            kd = np.array([_gain(_ATLAS_KD, m.name) for m in robot.motors])
        target0 = np.tile(qs[mq], (n_env, 1))
        if action == "torque":
            # SURVEY.md 8(d) config 3 as written: raw effort actions U(-20, 20) Nm, zero-order held over the env-step
            return Scenario(name, robot, opt, n_env, 0.04, q0, v0, None, None, np.zeros((n_env, robot.nmotors)), 0.0, seed,
                            f"{name}: raw torque actions U(-20, 20) Nm per env-step, {opt['stepper']['odeSolver']} "
                            f"dtMax={opt['stepper']['dtMax']}, contacts.model={opt['contacts']['model']}", _motor_q=mq,
                            torque_amplitude=20.0)
        return Scenario(name, robot, opt, n_env, 0.04, q0, v0, kp, kd, target0, 0.02, seed,
                        f"{name}: PD standing (reference gains), targets = posture + U(-0.02, 0.02) rad per env-step, "
                        f"{opt['stepper']['odeSolver']} dtMax={opt['stepper']['dtMax']}, " +
                        (f"spring-damper contact k={opt['contacts']['stiffness']:g} c={opt['contacts']['damping']:g} "
                         if opt["contacts"]["model"] == "spring_damper" else "constraint contact (PGS) ") +
                        f"mu={opt['contacts']['friction']:g}" +
                        (f"; {flagged_fraction:g} of the envs driven through their hip joint bounds" if flagged_fraction > 0 else ""),
                        _motor_q=mq, flagged_fraction=flagged_fraction)
    if name == "cartpole":
        # x, theta, dx, dtheta ~ U(-w, w); q = (x, cos, sin)
        x = rng.uniform(-CARTPOLE_HALF_WIDTH, CARTPOLE_HALF_WIDTH, size=(n_env, 4))
        q0 = np.stack([x[:, 0], np.cos(x[:, 1]), np.sin(x[:, 1])], axis=1)
        v0 = x[:, 2:4].copy()
        return Scenario(name, robot, opt, n_env, 0.02, q0, v0, None, None, np.zeros((n_env, nm)), 0.0, seed,
                        "cartpole: euler_explicit dt=0.02, continuous controller, force in {-10, 0, 10} N per step")
    if name == "double_pendulum":
        q0 = np.tile(np.array(DOUBLE_PENDULUM_Q0), (n_env, 1))
        v0 = np.zeros((n_env, 2))
        opt["stepper"]["sensorsUpdatePeriod"] = 0.0
        opt["stepper"]["controllerUpdatePeriod"] = 0.0
        return Scenario(name, robot, opt, n_env, opt["stepper"]["dtMax"], q0, v0, None, None, np.zeros((n_env, nm)),
                        0.0, seed, "double pendulum: runge_kutta_4 dtMax=1e-3, zero torque, q0=(0, 0.1)")
    raise KeyError(name)
