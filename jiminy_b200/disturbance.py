"""The walker env's disturbance forces (gym_jiminy `WalkerJiminyEnv._setup`, common/envs/locomotion.py:298-330, and
`_force_external_profile`, :340-359), re-drawn for the restarted envs of a batch.

On the root body frame (the first body frame whose parent joint is 1), in world-aligned axes at the frame origin:
- one impulse per `t_ref in arange(0, simulation_duration_max, 2)[1:]`, at t_ref + U(-0.25, 0.25), lasting 10 ms, of
  wrench (|F| n, 0, 0, 0, 0) with n = N(0, I2) / |.| and |F| = U(0, 1000 r);
- the profile r 50 (f0(t), f1(t), 0, 0, 0, 0) evaluated at every dynamics evaluation, with f0, f1 periodic Gaussian
  processes of wavelength 0.2 s and 1 s over a 1 s period (PeriodicGaussianProcess, core/include/jiminy/core/utilities/
  random.h:317-387, core/src/utilities/random.cc:318-458), r = std_ratio["disturbance"].

The profile runs on the device as a process force (`BatchedEngine.register_process_force`): each process is a table of
knot values and slopes per env, and the gain r 50 is folded into the tables (the cubic Hermite interpolation is linear
in them).  Draws come from numpy's stream on the host (`draw_numpy`) or from a torch generator on the device
(`draw_torch`); neither reproduces the reference's own generator (float32 normals of jiminy's PCG32).
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import numpy as np

F_IMPULSE_DT = 10.0e-3
F_IMPULSE_PERIOD = 2.0
F_IMPULSE_DELTA = 0.25
F_IMPULSE_SCALE = 1000.0
F_PROFILE_SCALE = 50.0
F_PROFILE_WAVELENGTH = 0.2
F_PROFILE_PERIOD = 1.0
COV_REGULARIZATION = 1e-9          # diagonal added before the Toeplitz Cholesky (random.h:361-370)


def root_body_frame(robot) -> str:
    """Name of the first BODY frame whose parent joint is 1 (`base` on ANYmal, `pelvis` on Atlas)."""
    for name, f in robot.frames.items():
        if f.kind == "body" and f.joint == 1:
            return name
    raise RuntimeError("There is an issue with the robot model. Impossible to determine the root joint.")


class PeriodicGaussianProcess:
    """Knots, covariance factor and evaluator of one periodic Gaussian process, restated in numpy.

    n = ceil(P / (0.1 lambda)) knots spaced delta = P / n; covariance first row c_i = exp(-2 (sin(pi i / n) / lambda)^2)
    with COV_REGULARIZATION on the diagonal, L its Cholesky factor; a draw z ~ N(0, I_n) gives the knot values L z and
    slopes G z with G = J L^-T, J_ij = -2 pi / (P lambda^2) sin(2 pi (i - j) / n) exp(-2 (sin(pi (i - j) / n) / lambda)^2)."""

    def __init__(self, wavelength: float, period: float):
        self.wavelength, self.period = float(wavelength), float(period)
        self.n = int(math.ceil(self.period / (0.1 * self.wavelength)))
        self.delta = self.period / self.n
        i = np.arange(self.n)
        d = i[:, None] - i[None, :]
        self.cov = np.exp(-2.0 * (np.sin(np.pi / self.n * d) / self.wavelength) ** 2) + COV_REGULARIZATION * np.eye(self.n)
        self.L = np.linalg.cholesky(self.cov)
        self.J = (-2.0 * np.pi / self.period / self.wavelength ** 2 * np.sin(2.0 * np.pi / self.n * d) *
                  np.exp(-2.0 * (np.sin(np.pi / self.n * d) / self.wavelength) ** 2))
        self.G = np.linalg.solve(self.L, self.J.T).T          # J L^-T

    def evaluate(self, values: np.ndarray, grads: np.ndarray, t) -> np.ndarray:
        """The table (values, grads [..., n]) at times t (broadcast against the leading axes):
        PeriodicTabularProcess::operator() (random.cc:336-400)."""
        t = np.asarray(t, dtype=np.float64)
        x = np.fmod(t, self.period)
        x = np.where(x < 0.0, x + self.period, x)
        quot = x / self.delta
        il = np.minimum(np.floor(quot).astype(np.int64), self.n - 1)
        ir = np.where(il + 1 == self.n, 0, il + 1)
        ratio = quot - il
        take = lambda a, k: np.take_along_axis(a, k[..., None], axis=-1)[..., 0]   # noqa: E731
        yl, yr, gl, gr = take(values, il), take(values, ir), take(grads, il), take(grads, ir)
        dy = yr - yl
        a = gl * self.delta - dy
        b = -gr * self.delta + dy
        return yl + ratio * ((1.0 - ratio) * ((1.0 - ratio) * a + ratio * b) + dy)


class WalkerDisturbance:
    """The impulse schedule and the profile of one batch: `register` puts them on an engine, `draw_numpy` / `draw_torch`
    sample rows, `apply_host` / `apply_device` write the rows of a mask through the engine's setters.

    A draw is a dict: t, dt [n_imp, n_env], wrench [n_imp, n_env, 6], values, grads [n_env, sum of knots] (f0's knots,
    then f1's), with the gain r 50 folded into values and grads."""

    def __init__(self, robot, ratio: float, simulation_duration_max: float = 20.0):
        if not ratio > 0.0:
            raise ValueError("the disturbance ratio must be positive")
        self.ratio = float(ratio)
        self.frame = root_body_frame(robot)
        self.t_ref = np.arange(0.0, simulation_duration_max, F_IMPULSE_PERIOD)[1:]
        self.processes = (PeriodicGaussianProcess(F_PROFILE_WAVELENGTH, F_PROFILE_PERIOD),
                          PeriodicGaussianProcess(F_PROFILE_PERIOD, F_PROFILE_PERIOD))
        self.gain = self.ratio * F_PROFILE_SCALE
        self.n_knots = [p.n for p in self.processes]
        self.impulses: list = []
        self.process: Optional[int] = None
        self._torch: Dict[str, object] = {}

    @property
    def n_impulses(self) -> int:
        return len(self.t_ref)

    def register(self, engine) -> None:
        """Registers the impulses (zero wrench until the first draw) and the profile on `engine` (no env running)."""
        n = engine.n_env
        self.impulses = [engine.register_impulse_force(self.frame, np.full(n, t), np.full(n, F_IMPULSE_DT), np.zeros(6))
                         for t in self.t_ref]
        self.process = engine.register_process_force(self.frame, [0, 1], self.n_knots,
                                                     [p.period for p in self.processes], 0.0)

    def profile(self, draw: Dict[str, np.ndarray], t) -> np.ndarray:
        """The profile wrench's (Fx, Fy) [..., 2] of the drawn rows at times t, with the numpy evaluator."""
        out, k0 = [], 0
        for p in self.processes:
            v, g = np.asarray(draw["values"])[:, k0:k0 + p.n], np.asarray(draw["grads"])[:, k0:k0 + p.n]
            out.append(p.evaluate(v, g, t))
            k0 += p.n
        return np.stack(out, axis=-1)

    # ------------------------------------------------------------------ sampling
    def draw_numpy(self, rng: np.random.Generator, n: int) -> Dict[str, np.ndarray]:
        m = self.n_impulses
        t = self.t_ref[:, None] + rng.uniform(-F_IMPULSE_DELTA, F_IMPULSE_DELTA, (m, n))
        f_xy = rng.normal(size=(m, n, 2))
        f_xy /= np.linalg.norm(f_xy, axis=-1, keepdims=True)
        f_xy *= rng.uniform(0.0, self.ratio * F_IMPULSE_SCALE, (m, n, 1))
        wrench = np.zeros((m, n, 6))
        wrench[..., :2] = f_xy
        values, grads = [], []
        for p in self.processes:
            z = rng.normal(size=(n, p.n))
            values.append(self.gain * (z @ p.L.T))
            grads.append(self.gain * (z @ p.G.T))
        return dict(t=t, dt=np.full((m, n), F_IMPULSE_DT), wrench=wrench,
                    values=np.ascontiguousarray(np.concatenate(values, axis=1)),
                    grads=np.ascontiguousarray(np.concatenate(grads, axis=1)))

    def _torch_tables(self, device):
        import torch
        key = str(device)
        if key not in self._torch:
            f64 = dict(dtype=torch.float64, device=device)
            self._torch[key] = ([torch.as_tensor(self.gain * p.L.T, **f64) for p in self.processes],
                                [torch.as_tensor(self.gain * p.G.T, **f64) for p in self.processes],
                                torch.as_tensor(self.t_ref[:, None], **f64))
        return self._torch[key]

    def draw_torch(self, gen, n: int, device) -> Dict[str, object]:
        """The same distribution drawn with the torch generator `gen` on `device`: values = z (gain L)^T and
        grads = z (gain G)^T as batched matmuls."""
        import torch
        LT, GT, t_ref = self._torch_tables(device)
        f64 = dict(dtype=torch.float64, device=device)
        m = self.n_impulses
        t = t_ref + (torch.rand((m, n), generator=gen, **f64) * (2.0 * F_IMPULSE_DELTA) - F_IMPULSE_DELTA)
        f_xy = torch.randn((m, n, 2), generator=gen, **f64)
        f_xy = f_xy / torch.linalg.vector_norm(f_xy, dim=-1, keepdim=True)
        f_xy = f_xy * (torch.rand((m, n, 1), generator=gen, **f64) * (self.ratio * F_IMPULSE_SCALE))
        wrench = torch.zeros((m, n, 6), **f64)
        wrench[..., :2] = f_xy
        z = [torch.randn((n, p.n), generator=gen, **f64) for p in self.processes]
        values = torch.cat([zi @ a for zi, a in zip(z, LT)], dim=1)
        grads = torch.cat([zi @ a for zi, a in zip(z, GT)], dim=1)
        return dict(t=t, dt=torch.full((m, n), F_IMPULSE_DT, **f64), wrench=wrench, values=values, grads=grads)

    # ------------------------------------------------------------------ writing rows
    def apply_host(self, engine, draw: Dict[str, np.ndarray], mask: Optional[np.ndarray] = None) -> None:
        """Host setters: the rows of `mask` (None = all) of a numpy draw."""
        for k, idx in enumerate(self.impulses):
            engine.set_impulse_force(idx, draw["t"][k], draw["dt"][k], draw["wrench"][k], mask=mask)
        engine.set_process_force(self.process, draw["values"], draw["grads"], mask=mask)

    def apply_device(self, engine, draw: Dict[str, object], mask_ptr: Optional[int] = None) -> None:
        """Device setters, enqueued on the batch stream: the rows of the device mask (uint8 [n_env], None = all) of a
        torch draw whose tensors are contiguous and stay alive until the stream has passed them."""
        t, dt, w = draw["t"], draw["dt"], draw["wrench"]
        for k, idx in enumerate(self.impulses):
            engine.set_impulse_force_device(idx, t[k].data_ptr(), dt[k].data_ptr(), w[k].data_ptr(), mask_ptr)
        engine.set_process_force_device(self.process, draw["values"].data_ptr(), draw["grads"].data_ptr(), mask_ptr)


def from_std_ratio(robot, std_ratio: Optional[dict], simulation_duration_max: float) -> Optional[WalkerDisturbance]:
    """The disturbance an env's `std_ratio` asks for: None or {} -> none, {"disturbance": r} -> the walker disturbance
    (none when r == 0 or absent).  "sensors" is `sensor_randomisation.from_std_ratio`'s and "model"
    `model_randomisation.from_std_ratio`'s; the other keys of the reference (ground, flexibility) are not implemented."""
    if not std_ratio:
        return None
    other = sorted(set(std_ratio) - {"disturbance", "sensors", "model"})
    if other:
        raise NotImplementedError(f"std_ratio keys not supported by the batched envs: {other} (only 'disturbance', 'sensors' and 'model')")
    r = float(std_ratio.get("disturbance", 0.0))
    if r < 0.0:
        raise ValueError("std_ratio['disturbance'] must be positive")
    return WalkerDisturbance(robot, r, simulation_duration_max) if r > 0.0 else None
