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
The only model parameters randomised per env are the flexibilities': on a robot without flexibility joints a positive
ratio raises NotImplementedError, as every unsupported `std_ratio` key does (the reference's `model` randomisation does
nothing there, but the per-reset model biases of such a robot are not drawn per env by the batched envs either).
"""
from __future__ import annotations

from typing import Optional

import numpy as np

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
