"""The walker env's model randomisation (gym_jiminy `WalkerJiminyEnv._setup`, common/envs/locomotion.py:288-296): new
stiffness and damping of every flexibility joint for the envs that (re)start.

With r = std_ratio["model"], per flexibility joint and restart:
- stiffness k = k0 + FLEX_STIFFNESS_SCALE r u_k, damping d = d0 + FLEX_DAMPING_SCALE r u_d;
- u_k and u_d are independent U(-1, 1) draws, one of each per flexibility, shared by its three axes (the reference's
  `sample(scale=r)` without a shape is one scalar);
- k0 and d0 are the robot's nominal values (`robot.flexibility`).

The reference adds the draw to the values it reads back from the robot, which it never restores: its parameters take a
random walk across episodes until one goes negative and `Model::setOptions` raises (model.cc:1620-1626).  Here every
restart draws around the nominal values instead, and a ratio whose draws could go negative is refused at construction.
Draws come from numpy's stream on the host (`draw_numpy`) or a torch generator on the device (`draw_torch`).
On a robot without flexibility joints a positive ratio raises NotImplementedError, as every unsupported `std_ratio` key
does (the reference's `model` randomisation does nothing there).

The body biases of the robot options (`ModelBiasRandomisation`, the envs' `model_bias_std`) are drawn per env at every
restart around the nominal model, with the transformation of `model.biased_robot`.  The host envs and the device envs'
restart bank keep grounding their restart states on the nominal model; only the in-kernel grounding of the device envs'
`reset_states="sample"` puts each env on the ground of its own biased model.
"""
from __future__ import annotations

from typing import Optional

import numpy as np

from . import model as M

FLEX_STIFFNESS_SCALE = 1000.0
FLEX_DAMPING_SCALE = 10.0


class WalkerModelRandomisation:
    """Nominal rows [n_flex, 6] (stiffness xyz, damping xyz, flexibilities in `robot.flexibility_joint_indices` order) and
    the draw around them for ratio r.  A draw is an array [n, n_flex, 6]."""

    def __init__(self, robot, ratio: float):
        self.ratio = float(ratio)
        if not self.ratio >= 0.0:
            raise ValueError("std_ratio['model'] must be positive")
        if not robot.is_flexibility_enabled:
            raise ValueError("the robot has no flexibility joint: there is no model parameter to randomise")
        self.nominal = np.ascontiguousarray(np.asarray(robot.flexibility, dtype=np.float64)[robot.flexibility_joint_indices])
        self.n_flex = len(self.nominal)
        self.stiffness_half_width = FLEX_STIFFNESS_SCALE * self.ratio
        self.damping_half_width = FLEX_DAMPING_SCALE * self.ratio
        if self.stiffness_half_width > self.nominal[:, :3].min() or self.damping_half_width > self.nominal[:, 3:].min():
            raise ValueError(f"std_ratio['model'] = {self.ratio} can draw a negative flexibility stiffness or damping: it must "
                             f"be at most {min(self.nominal[:, :3].min() / FLEX_STIFFNESS_SCALE, self.nominal[:, 3:].min() / FLEX_DAMPING_SCALE)}")
        # per column of a row: the half width of its draw (stiffness xyz, then damping xyz)
        self.half_width = np.repeat([self.stiffness_half_width, self.damping_half_width], 3)
        self._torch = {}     # nominal rows and half widths as tensors, per device (uploaded once: a copy would synchronise)

    def register(self, engine) -> None:
        """Per-env flexibility rows, starting from the model's values."""
        engine.enable_per_env_flexibility()

    # ------------------------------------------------------------------ sampling
    def draw_numpy(self, rng: np.random.Generator, n: int) -> np.ndarray:
        u = rng.uniform(-1.0, 1.0, (n, self.n_flex, 2))
        return self.nominal + np.repeat(u, 3, axis=2) * self.half_width

    def draw_torch(self, gen, n: int, device):
        """The same distribution with a torch generator on `device` (fp64, contiguous)."""
        import torch
        f64 = dict(dtype=torch.float64, device=device)
        if str(device) not in self._torch:
            self._torch[str(device)] = tuple(torch.as_tensor(x, **f64) for x in (self.nominal, self.half_width))
        nominal, hw = self._torch[str(device)]
        u = torch.rand((n, self.n_flex, 2), generator=gen, **f64) * 2.0 - 1.0
        return nominal + u.repeat_interleave(3, dim=2) * hw

    # ------------------------------------------------------------------ writing rows
    def apply_host(self, engine, rows: np.ndarray, mask: Optional[np.ndarray] = None) -> None:
        """Host setter: the rows of `mask` (None = all), for the envs' next start."""
        engine.set_flexibility_env(rows, mask=mask)

    def apply_device(self, engine, rows, mask_ptr: Optional[int] = None) -> None:
        """Device setter, enqueued on the batch stream: the rows of the device mask (uint8 [n_env], None = all) of a
        contiguous torch tensor that stays alive until the stream has passed it."""
        engine.set_flexibility_env_device(rows.data_ptr(), mask_ptr)


def from_std_ratio(robot, std_ratio: Optional[dict]) -> Optional[WalkerModelRandomisation]:
    """The model randomisation of an env's `std_ratio`: {"model": r} with r > 0, else none.  Needs a robot with flexibility
    joints (NotImplementedError otherwise).  The other keys are checked by `disturbance.from_std_ratio`."""
    r = float((std_ratio or {}).get("model", 0.0))
    if not r >= 0.0:
        raise ValueError("std_ratio['model'] must be positive")
    if r == 0.0:
        return None
    if not robot.is_flexibility_enabled:
        raise NotImplementedError("std_ratio key 'model' is supported by the batched envs on robots with flexibility joints "
                                  "only (per-env stiffness and damping of the flexibilities)")
    return WalkerModelRandomisation(robot, r)


# ---------------------------------------------------------------------------------------------- body biases
BIAS_OPTIONS = ("massBodiesBiasStd", "centerOfMassPositionBodiesBiasStd", "inertiaBodiesBiasStd",
                "relativePositionBodiesBiasStd")
_BIAS_ARGS = dict(zip(BIAS_OPTIONS, ("mass_std", "com_std", "inertia_std", "relative_position_std")))


def _checked_bias_std(std: Optional[dict]) -> dict:
    std = dict(std or {})
    unknown = set(std) - set(BIAS_OPTIONS)
    if unknown:
        raise ValueError(f"unknown model bias option(s) {sorted(unknown)}: expected {list(BIAS_OPTIONS)}")
    for k, v in std.items():
        if not float(v) >= 0.0:
            raise ValueError(f"{k} must be positive")
    return std


class ModelBiasRandomisation:
    """Per-env body biases: the draw of `Model::addBiasedToExtendedModel` (core/src/robot/model.cc:1166-1236), which the
    reference repeats at every reset (`Model::reset`, model.cc:398-416), for the envs that (re)start.

    `std` holds the standard deviations under the reference's robot option names (`BIAS_OPTIONS`; missing keys are 0).
    Every draw is taken around the nominal table with `model.bias_bodies` -- the transformation of `model.biased_robot` --
    on the mechanical joints; the free-flyer and flexibility rows keep their nominal values.  A draw is an array
    [n, njoints, 13] in the layout of `BatchedEngine.set_model_env` (`model.body_rows`).  The normals are single
    precision like the reference's; they come from numpy's stream on the host (`draw_numpy`, which reproduces
    `biased_robot` for the same generator) or a torch generator on the device (`draw_torch`), not from jiminy's PCG32.
    The eigen-decompositions of the nominal inertias are taken once here, so the torch draw runs no `linalg` call and
    never synchronises.  Robots with backlash joints are refused: the reference biases the model before it inserts them,
    so a biased body may sit on another row of the extended table."""

    def __init__(self, robot, std: Optional[dict]):
        std = _checked_bias_std(std)
        if any(n.endswith(M.BACKLASH_JOINT_SUFFIX) for n in robot.joint_names) or any(m.backlash >= M.EPS for m in robot.motors):
            raise NotImplementedError("per-env body biases of a model with backlash joints")
        self.stds = {_BIAS_ARGS[k]: float(std.get(k, 0.0)) for k in BIAS_OPTIONS}
        self.nominal = M.body_rows(robot)
        self.joints = M.bias_joints(robot)
        self.n_normals = M.bias_normals(**self.stds)
        self.eig = M.inertia_eig(self.nominal[self.joints, :10])     # (moments [J, 3], axes [J, 3, 3])
        self._torch = {}     # nominal rows and eigen-decompositions as tensors, per device (uploaded once)

    @property
    def active(self) -> bool:
        """Does a draw change anything (some standard deviation above machine epsilon)?"""
        return self.n_normals > 0

    def register(self, engine) -> None:
        """Per-env model rows, starting from the model's values."""
        engine.enable_per_env_model()

    # ------------------------------------------------------------------ sampling
    def rows_from_normals(self, z: np.ndarray) -> np.ndarray:
        """Rows [n, njoints, 13] from single-precision standard normals z [n, len(joints), n_normals]."""
        rows = np.repeat(self.nominal[None], z.shape[0], axis=0)
        rows[:, self.joints, :10], rows[:, self.joints, 10:] = M.bias_bodies(
            self.nominal[self.joints, :10], self.nominal[self.joints, 10:], z, self.eig, **self.stds)
        return rows

    def draw_numpy(self, rng: np.random.Generator, n: int) -> np.ndarray:
        """n rows; with n = 1 the draw `model.biased_robot` makes from the same generator."""
        return self.rows_from_normals(rng.standard_normal((n, len(self.joints), self.n_normals), dtype=np.float32))

    def rows_from_normals_torch(self, z):
        """`rows_from_normals` with torch, on z's device (z: float32 [n, len(joints), n_normals]); fp64, contiguous."""
        import torch
        dev = z.device
        f64 = dict(dtype=torch.float64, device=dev)
        if str(dev) not in self._torch:
            self._torch[str(dev)] = (torch.as_tensor(self.nominal, **f64), torch.as_tensor(self.joints, dtype=torch.long, device=dev),
                                     torch.as_tensor(self.eig[0], **f64), torch.as_tensor(self.eig[1], **f64))
        nominal, joints, moments, axes = self._torch[str(dev)]
        n = z.shape[0]
        x = nominal[joints].unsqueeze(0).repeat(n, 1, 1)
        k = 0

        def normal(m, mean, std):
            nonlocal k
            # single precision like numpy's float32(mean) + float32(std) * z: the scalars enter the float32 ops as float32
            g = (z[..., k:k + m] * float(np.float32(std)) + float(np.float32(mean))).to(torch.float64)
            k += m
            return g
        s = self.stds
        if s["com_std"] > M.BIAS_EPS:
            x[..., 1:4] = x[..., 1:4] * normal(3, 1.0, s["com_std"])
        if s["mass_std"] > M.BIAS_EPS:
            m = x[..., 0]
            x[..., 0] = torch.maximum(m * normal(1, 1.0, s["mass_std"])[..., 0], torch.clamp(m, max=1.0e-3))
        if s["inertia_std"] > M.BIAS_EPS:
            w = normal(3, 0.0, s["inertia_std"])
            th = torch.sqrt((w * w).sum(-1))[..., None, None]
            zero = torch.zeros_like(w[..., 0])
            K = torch.stack([zero, -w[..., 2], w[..., 1], w[..., 2], zero, -w[..., 0], -w[..., 1], w[..., 0], zero], -1).reshape(w.shape[:-1] + (3, 3))
            eye = torch.eye(3, **f64)
            small = th < 1e-12
            ths = torch.where(small, torch.ones_like(th), th)
            R = eye + torch.where(small, K, torch.sin(ths) / ths * K + (1.0 - torch.cos(ths)) / (ths * ths) * (K @ K))
            ax = axes @ R
            mo = moments * normal(3, 1.0, s["inertia_std"])
            I = (ax * mo[..., None, :]) @ ax.transpose(-1, -2)
            x[..., 4:10] = torch.stack([I[..., 0, 0], I[..., 0, 1], I[..., 1, 1], I[..., 0, 2], I[..., 1, 2], I[..., 2, 2]], -1)
        if s["relative_position_std"] > M.BIAS_EPS:
            x[..., 10:13] = x[..., 10:13] * normal(3, 1.0, s["relative_position_std"])
        rows = nominal.unsqueeze(0).repeat(n, 1, 1)
        rows[:, joints] = x
        return rows.contiguous()

    def draw_torch(self, gen, n: int, device):
        """The same distribution with a torch generator on `device` (fp64, contiguous)."""
        import torch
        z = torch.randn((n, len(self.joints), self.n_normals), generator=gen, dtype=torch.float32, device=device)
        return self.rows_from_normals_torch(z)

    # ------------------------------------------------------------------ writing rows
    def apply_host(self, engine, rows: np.ndarray, mask: Optional[np.ndarray] = None) -> None:
        """Host setter: the rows of `mask` (None = all), for the envs' next start."""
        engine.set_model_env(rows, mask=mask)

    def apply_device(self, engine, rows, mask_ptr: Optional[int] = None) -> None:
        """Device setter, enqueued on the batch stream: the rows of the device mask (uint8 [n_env], None = all) of a
        contiguous torch tensor that stays alive until the stream has passed it."""
        engine.set_model_env_device(rows.data_ptr(), mask_ptr)


def from_model_bias_std(robot, model_bias_std: Optional[dict]) -> Optional[ModelBiasRandomisation]:
    """The body-bias randomisation of an env's `model_bias_std`: None, {} or all standard deviations zero give none."""
    std = _checked_bias_std(model_bias_std)
    if all(float(v) <= M.BIAS_EPS for v in std.values()):
        return None
    return ModelBiasRandomisation(robot, std)
