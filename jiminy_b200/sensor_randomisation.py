"""The walker env's sensor randomisation (gym_jiminy `WalkerJiminyEnv._setup`, common/envs/locomotion.py:40-60, :264-286):
new noise, bias, delay and jitter for every sensor of the envs that (re)start, and a fresh engine seed for their sensor
generators.

Per sensor of class `cls`, with r = std_ratio["sensors"]:
- `delay`, `jitter`: each U(0, r D[cls]), D = 3 ms for EncoderSensor and 0 for every other class (SENSOR_DELAY_SCALE);
- `bias`: per field U(-r B, r B) with B = SENSOR_BIAS_SCALE[cls];
- `noiseStd`: per field U(-r S, r S) with S = SENSOR_NOISE_SCALE[cls].

The reference's block cannot run as written in v1.8.12, so this follows its evident intent:
- it loops over `("bias", SENSOR_BIAS_SCALE), ("noiseStd", SENSOR_NOISE_SCALE)` and uses each tuple as a dict key
  (`TypeError: unhashable type`); here `bias` takes SENSOR_BIAS_SCALE and `noiseStd` SENSOR_NOISE_SCALE;
- its IMU scale arrays have 9 entries for the 6 fields of `ImuSensor` (basic_sensors.cc:66-67), so no draw of shape (6,)
  can broadcast them; here the last six apply, gyroscope then accelerometer: noise (0.01, 0.01, 0.01, 0.2, 0.2, 0.2),
  bias (0.02, 0.02, 0.02, 0, 0, 0);
- `noiseStd` keeps the sign it is drawn with: the reference multiplies a float normal by it, so the sign does not change
  the distribution (the device and the oracle do the same);
- `delayInterpolationOrder` stays at its default, 1.

The delay buffer is sized once for `delay_bound = 2 r max(D)`, which no draw reaches.  Every restart also draws a new
32-bit engine seed (`stepper.randomSeedSeq`): the env's sensor generators then run a new, independent stream each
episode, as the reference's `engine.reset(False, ...)` gives (engine.cc:726-763), through the same seeding chain
(`jb_set_seeds`).  Draws come from numpy's stream on the host (`draw_numpy`) or a torch generator on the device
(`draw_torch`): the distribution is the reference's, the bits are not jiminy's PCG32 stream.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np

SENSOR_TYPES = ("ImuSensor", "ForceSensor", "EncoderSensor", "EffortSensor", "ContactSensor")
SENSOR_DELAY_SCALE = {"EncoderSensor": 3.0e-3, "EffortSensor": 0.0, "ContactSensor": 0.0, "ForceSensor": 0.0, "ImuSensor": 0.0}
SENSOR_NOISE_SCALE = {"EncoderSensor": (0.0, 0.02), "EffortSensor": (10.0,), "ContactSensor": (2.0, 2.0, 2.0),
                      "ForceSensor": (2.0, 2.0, 2.0, 10.0, 10.0, 10.0), "ImuSensor": (0.01, 0.01, 0.01, 0.2, 0.2, 0.2)}
SENSOR_BIAS_SCALE = {"EncoderSensor": (0.0, 0.0), "EffortSensor": (0.0,), "ContactSensor": (4.0, 4.0, 4.0),
                     "ForceSensor": (4.0, 4.0, 4.0, 20.0, 20.0, 20.0), "ImuSensor": (0.02, 0.02, 0.02, 0.0, 0.0, 0.0)}


class WalkerSensorRandomisation:
    """Scales of every column of the sensor matrix and of every sensor, for ratio r.  `engine_or_layout`: a
    `BatchedEngine` or a `RobotTable.sensor_layout()` dict.  A draw is a dict of `noise_std`, `bias` [n, width],
    `delay`, `jitter` [n, n_sensors] (sensor order Imu, Force, Encoder, Effort, Contact) and `seed` [n]."""

    def __init__(self, engine_or_layout, ratio: float):
        layout = engine_or_layout.robot.sensor_layout() if hasattr(engine_or_layout, "robot") else engine_or_layout
        self.ratio = float(ratio)
        self.width = int(layout["width"][0])
        self.noise_scale, self.bias_scale, delay = np.zeros(self.width), np.zeros(self.width), []
        for t in SENSOR_TYPES:
            off, nf, ns = layout[t]
            for f in range(nf):
                self.noise_scale[off + f * ns:off + (f + 1) * ns] = self.ratio * SENSOR_NOISE_SCALE[t][f]
                self.bias_scale[off + f * ns:off + (f + 1) * ns] = self.ratio * SENSOR_BIAS_SCALE[t][f]
            delay += [self.ratio * SENSOR_DELAY_SCALE[t]] * ns
        self.delay_scale = np.asarray(delay, dtype=np.float64)
        self.n_sensors = len(delay)
        self.delay_bound = 2.0 * self.ratio * max(SENSOR_DELAY_SCALE.values())
        self._torch: Dict[str, tuple] = {}     # the scales as tensors, per device (uploaded once: a copy would synchronise)

    def register(self, engine) -> None:
        """Per-env options for every sensor, the delay buffer sized for `delay_bound`."""
        engine.enable_per_env_sensor_options(self.delay_bound)

    # ------------------------------------------------------------------ sampling
    def draw_numpy(self, rng: np.random.Generator, n: int) -> Dict[str, np.ndarray]:
        return dict(noise_std=rng.uniform(-1.0, 1.0, (n, self.width)) * self.noise_scale,
                    bias=rng.uniform(-1.0, 1.0, (n, self.width)) * self.bias_scale,
                    delay=rng.uniform(0.0, 1.0, (n, self.n_sensors)) * self.delay_scale,
                    jitter=rng.uniform(0.0, 1.0, (n, self.n_sensors)) * self.delay_scale,
                    seed=rng.integers(0, 2 ** 32, n, dtype=np.uint32))

    def draw_torch(self, gen, n: int, device) -> Dict[str, object]:
        """The same distribution with a torch generator on `device`; `seed` holds the 32 bits as int32."""
        import torch
        f64 = dict(dtype=torch.float64, device=device)
        if str(device) not in self._torch:
            self._torch[str(device)] = tuple(torch.as_tensor(x, **f64) for x in (self.noise_scale, self.bias_scale, self.delay_scale))
        ns, bs, ds = self._torch[str(device)]
        return dict(noise_std=(torch.rand((n, self.width), generator=gen, **f64) * 2.0 - 1.0) * ns,
                    bias=(torch.rand((n, self.width), generator=gen, **f64) * 2.0 - 1.0) * bs,
                    delay=torch.rand((n, self.n_sensors), generator=gen, **f64) * ds,
                    jitter=torch.rand((n, self.n_sensors), generator=gen, **f64) * ds,
                    seed=torch.randint(-2 ** 31, 2 ** 31, (n,), generator=gen, dtype=torch.int32, device=device))

    # ------------------------------------------------------------------ writing rows
    def apply_host(self, engine, draw: Dict[str, np.ndarray], mask: Optional[np.ndarray] = None) -> None:
        """Host setters: options of the rows of `mask` (None = all) and the seeds, for the envs' next start.  The seeds
        of every env are written; a start re-derives the generators of the started envs only."""
        engine.set_sensor_options_env(draw["noise_std"], draw["bias"], draw["delay"], draw["jitter"], mask=mask)
        engine.set_seeds(np.asarray(draw["seed"]).astype(np.uint32))

    def apply_device(self, engine, draw: Dict[str, object], mask_ptr: Optional[int] = None) -> None:
        """Device setters, enqueued on the batch stream: the rows of the device mask (uint8 [n_env], None = all) of a
        torch draw whose tensors are contiguous and stay alive until the stream has passed them."""
        engine.set_sensor_options_env_device(draw["noise_std"].data_ptr(), draw["bias"].data_ptr(), draw["delay"].data_ptr(),
                                             draw["jitter"].data_ptr(), mask_ptr)
        engine.set_seeds_device(draw["seed"].data_ptr(), mask_ptr)


def from_std_ratio(engine_or_layout, std_ratio: Optional[dict]) -> Optional[WalkerSensorRandomisation]:
    """The sensor randomisation of an env's `std_ratio`: {"sensors": r} with r > 0, else none.  The other keys are
    checked by `disturbance.from_std_ratio`."""
    r = float((std_ratio or {}).get("sensors", 0.0))
    if not r >= 0.0:
        raise ValueError("std_ratio['sensors'] must be positive")
    return WalkerSensorRandomisation(engine_or_layout, r) if r > 0.0 else None
