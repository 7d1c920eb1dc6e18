"""Walker sensor randomisation: per-env sensor options latched at every start (`jb_enable_per_env_sensor_options`,
`jb_set_sensor_options_env(_device)`), generator seeds from device buffers (`jb_set_seeds_device`), the samplers of
`jiminy_b200.sensor_randomisation` and the envs' `std_ratio={"sensors": r}`.

Every kernel scenario is a function of `api`: the CPU suite runs it on the emulated library (device memory is host
memory, torch tensors on the CPU), the `-m gpu` variants on the device with `api=None`.  The oracle holds one engine per
env, so each env is compared with a one-env oracle batch configured with that env's options and seed."""
import numpy as np
import pytest
import torch

from jiminy_b200 import core, envs, scenarios
from jiminy_b200.core import BatchedEngine
from jiminy_b200.sensor_randomisation import SENSOR_TYPES, WalkerSensorRandomisation, from_std_ratio
from jiminy_b200.torch_envs import DeviceBatchedEnv, DevicePDControlBatchedEnv

from emul import emul_api
from oracle.oracle import OracleBatch

BAD = core.JB_ENV_NOT_STARTED | core.JB_ENV_BAD_START
TOL = 1e-9          # tests/sensor_pipeline_common.py: atol = 1e3 TOL max(1, |true values|)


@pytest.fixture(scope="module")
def api():
    return emul_api()


def _dev(api, x, dtype=torch.float64):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype, device="cpu" if api is not None else "cuda").contiguous()


def _np(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _sync(api):
    if api is None:
        torch.cuda.synchronize()


def _seeds_i32(seeds):
    return np.asarray(seeds, dtype=np.uint32).view(np.int32)


# ---------------------------------------------------------------------------------------------- sampler
def _check_sampler(s: WalkerSensorRandomisation, lay, draw, n):
    noise, bias, delay, jitter, seed = (_np(draw[k]) for k in ("noise_std", "bias", "delay", "jitter", "seed"))
    assert noise.shape == bias.shape == (n, s.width) and delay.shape == jitter.shape == (n, s.n_sensors) and seed.shape == (n,)
    # U(-a, a) per column: z = x / a has mean 0, E z^2 = 1/3, var z = 1/3, var z^2 = 4/45
    for x, scale in ((noise, s.noise_scale), (bias, s.bias_scale)):
        on = scale > 0
        assert (np.abs(x) <= scale).all() and (x[:, ~on] == 0).all()
        z = x[:, on] / scale[on]
        assert (np.abs(z.mean(0)) <= 6 * np.sqrt(1 / 3 / n)).all()
        assert (np.abs((z ** 2).mean(0) - 1 / 3) <= 6 * np.sqrt(4 / 45 / n)).all()
    # U(0, r 3 ms) on the encoders, exactly 0 elsewhere: mean 1/2, var 1/12
    enc = np.zeros(s.n_sensors, bool)
    k0 = sum(lay[t][2] for t in SENSOR_TYPES[:2])
    enc[k0:k0 + lay["EncoderSensor"][2]] = True
    np.testing.assert_array_equal(s.delay_scale > 0, enc)
    for x in (delay, jitter):
        assert (x[:, ~enc] == 0).all()
        z = x[:, enc] / (s.ratio * 3e-3)
        assert (z >= 0).all() and (z < 1).all()
        assert (np.abs(z.mean(0) - 0.5) <= 6 * np.sqrt(1 / 12 / n)).all()
        assert (np.abs((z ** 2).mean(0) - 1 / 3) <= 6 * np.sqrt(4 / 45 / n)).all()
    assert (delay + jitter <= s.delay_bound).all()
    # the IMU takes the last six entries of the reference's nine: gyroscope, then accelerometer
    off, nf, ni = lay["ImuSensor"]
    np.testing.assert_array_equal(s.noise_scale[off:off + nf * ni:ni], s.ratio * np.array([0.01, 0.01, 0.01, 0.2, 0.2, 0.2]))
    np.testing.assert_array_equal(s.bias_scale[off:off + nf * ni:ni], s.ratio * np.array([0.02, 0.02, 0.02, 0.0, 0.0, 0.0]))
    # seeds: every one of the 32 bits varies, each set about half the time
    u = seed.astype(np.int64) & 0xFFFFFFFF
    bits = (u[:, None] >> np.arange(32)) & 1
    assert (np.abs(bits.mean(0) - 0.5) <= 6 * np.sqrt(0.25 / n)).all()


def _sampler_case(kind, device="cpu"):
    lay = scenarios.make("anymal", 1, seed=0).robot.sensor_layout()
    s = WalkerSensorRandomisation(lay, 0.8)
    n = 2 ** 15
    if kind == "numpy":
        draw = s.draw_numpy(np.random.default_rng(3), n)
    else:
        gen = torch.Generator(device=device)
        gen.manual_seed(4)
        draw = s.draw_torch(gen, n, device)
        assert draw["seed"].dtype == torch.int32
    _check_sampler(s, lay, draw, n)


@pytest.mark.parametrize("kind", ["numpy", "torch"])
def test_sampler_statistics(kind):
    _sampler_case(kind)


def test_std_ratio_sensors(api):
    lay = scenarios.make("anymal", 1).robot.sensor_layout()
    assert from_std_ratio(lay, None) is None and from_std_ratio(lay, {"sensors": 0.0}) is None
    assert from_std_ratio(lay, {"disturbance": 1.0}) is None
    assert from_std_ratio(lay, {"sensors": 0.5}).delay_bound == 2 * 0.5 * 3e-3
    with pytest.raises(ValueError):
        from_std_ratio(lay, {"sensors": -1.0})
    # r == 0 registers nothing; ground / model / flexibility stay unsupported; a continuous sensor period is refused
    env = envs.BatchedJiminyEnv(scenarios.make("anymal", 2, seed=1), api_=api, std_ratio={"sensors": 0.0})
    assert env.sensor_randomisation is None
    for key in ("ground", "model", "flexibility"):
        with pytest.raises(NotImplementedError, match=key):
            envs.BatchedJiminyEnv(scenarios.make("anymal", 2, seed=1), api_=api, std_ratio={"sensors": 1.0, key: 0.5})
    sc = scenarios.make("anymal", 2, seed=1)
    sc.options["stepper"]["sensorsUpdatePeriod"] = 0.0
    with pytest.raises(NotImplementedError, match="sensorsUpdatePeriod"):
        envs.BatchedJiminyEnv(sc, api_=api, std_ratio={"sensors": 1.0})


# ---------------------------------------------------------------------------------------------- engine helpers
def _engine(api, sc, rows=None, seeds=None, bound=6e-3):
    eng = BatchedEngine(sc.robot, sc.options, sc.n_env, api_=api)
    eng.set_pd_controller(sc.kp, sc.kd)
    eng.enable_per_env_sensor_options(bound)
    if rows is not None:
        eng.set_sensor_options_env(rows["noise_std"], rows["bias"], rows["delay"], rows["jitter"])
    if seeds is not None:
        eng.set_seeds(seeds)
    eng.set_command(sc.target0)
    return eng


def _configure_oracle(o, lay, rows, i, seed):
    col = 0
    for t in SENSOR_TYPES:
        off, nf, ns = lay[t]
        for k in range(ns):
            cols = off + np.arange(nf) * ns + k
            o.set_sensor_options(t, k, noise_std=rows["noise_std"][i, cols], bias=rows["bias"][i, cols],
                                 delay=float(rows["delay"][i, col]), jitter=float(rows["jitter"][i, col]), delay_interpolation_order=1)
            col += 1
    o.set_seeds(np.array([seed], dtype=np.uint32))


def _rows(s, rng, n):
    d = s.draw_numpy(rng, n)
    return {k: v for k, v in d.items() if k != "seed"}, d["seed"]


def _compare_oracles(eng, orcs):
    m1, d1 = eng.get_sensors(), eng.get_sensor_data()
    m0 = np.concatenate([o.get_sensors() for o in orcs])
    d0 = np.concatenate([o.get_sensor_data() for o in orcs])
    scale = max(1.0, np.abs(d0).max())
    np.testing.assert_allclose(d1, d0, rtol=0, atol=1e3 * TOL * scale)
    np.testing.assert_allclose(m1 - d1, m0 - d0, rtol=0, atol=1e3 * TOL * scale)
    np.testing.assert_array_equal(eng.get_iters()[0], np.concatenate([o.get_iters()[0] for o in orcs]))
    np.testing.assert_array_equal(eng.get_status(), np.concatenate([o.get_status() for o in orcs]))
    return m1 - d1


# ---------------------------------------------------------------------------------------------- per-env options vs oracle
def per_env_oracle(api, solver):
    """5 ANYmal envs, each with its own options and seed: env 0 all zero, env 1 with delay + jitter at the bound on every
    sensor, the others drawn with r = 1.  With RK4, envs 0 and 4 drive a hip through its bound and are handed to the full
    body.  After the first env-step envs 1 and 3 restart with new rows and seeds.  Explicit Euler's 1 ms steps on the stiff
    ground diverge after a few env-steps on this scenario (the oracle's as well), so it runs two env-steps and no env
    at the bound."""
    n = 5
    flagged = solver == "runge_kutta_4"
    sc = scenarios.make("anymal", n, seed=21, flagged_fraction=0.25 if flagged else 0.0, solver=solver)
    lay = sc.robot.sensor_layout()
    s = WalkerSensorRandomisation(lay, 1.0)
    rng = np.random.default_rng(22)
    rows, seeds = _rows(s, rng, n)
    for k in rows:
        rows[k][0] = 0.0
    rows["delay"][1] = rows["jitter"][1] = s.delay_bound / 2
    seeds[:2] = (0, 2 ** 32 - 1)
    eng = _engine(api, sc, rows, seeds, s.delay_bound)
    orcs = []
    for i in range(n):
        o = OracleBatch(sc.robot, sc.options, 1)
        o.set_pd_controller(sc.kp, sc.kd)
        _configure_oracle(o, lay, rows, i, seeds[i])
        o.set_command(sc.target0[i:i + 1])
        orcs.append(o)
    eng.start(sc.q0, sc.v0)
    for i, o in enumerate(orcs):
        assert not o.start(sc.q0[i:i + 1], sc.v0[i:i + 1]).any()
    _compare_oracles(eng, orcs)
    mask = np.array([0, 1, 0, 1, 0], np.uint8)
    for k in range(4 if flagged else 2):
        act = sc.sample_targets(k)
        eng.set_command(act)
        eng.step(sc.step_dt)
        for i, o in enumerate(orcs):
            o.set_command(act[i:i + 1])
            assert not o.step(sc.step_dt).any()
        noise = _compare_oracles(eng, orcs)
        if k == 0:
            new, new_seeds = _rows(s, rng, n)
            eng.set_sensor_options_env(new["noise_std"], new["bias"], new["delay"], new["jitter"], mask=mask)
            seeds = np.where(mask.astype(bool), new_seeds, seeds)
            eng.set_seeds(seeds)
            eng.start(sc.q0, sc.v0, mask=mask)
            for i in np.flatnonzero(mask):
                _configure_oracle(orcs[i], lay, new, i, seeds[i])
                assert not orcs[i].start(sc.q0[i:i + 1], sc.v0[i:i + 1]).any()
            _compare_oracles(eng, orcs)
    # the options did something, the zero env measures its true values, the flagged envs left the hot path
    assert np.abs(noise[2:]).max() > 1e-3
    assert np.abs(noise[0]).max() < 1e3 * TOL * max(1.0, np.abs(eng.get_sensor_data()).max())
    if flagged:
        assert (eng.get_status()[[0, 4]] & core.JB_ENV_JOINT_LIMIT).all()


@pytest.mark.parametrize("solver", ["runge_kutta_4", "euler_explicit"])
def test_per_env_options_match_oracle(api, solver, monkeypatch):
    monkeypatch.setenv("JB_NO_FAST_BOUNDS", "1")
    per_env_oracle(api, solver)


# ---------------------------------------------------------------------------------------------- uniform rows, latch
def uniform_rows(api):
    """Per-env rows that all equal one set of options give the bits of the batch-wide path."""
    n = 3
    sc = scenarios.make("anymal", n, seed=5)
    lay = sc.robot.sensor_layout()
    s = WalkerSensorRandomisation(lay, 1.0)
    one, _ = _rows(s, np.random.default_rng(6), 1)
    rows = {k: np.repeat(v, n, axis=0) for k, v in one.items()}
    seeds = np.array([3, 77, 2 ** 31], np.uint32)
    a = _engine(api, sc, rows, seeds, s.delay_bound)
    b = BatchedEngine(sc.robot, sc.options, n, api_=api)
    b.set_pd_controller(sc.kp, sc.kd)
    o = OracleBatch(sc.robot, sc.options, 1)      # (only to reuse the per-sensor unpacking)
    calls = []
    o.set_sensor_options = lambda *args, **kw: calls.append((args, kw))
    o.set_seeds = lambda x: None
    _configure_oracle(o, lay, rows, 0, 0)
    for args, kw in calls:
        b.set_sensor_options(*args, **kw)
    b.set_seeds(seeds)
    b.set_command(sc.target0)
    for e in (a, b):
        e.start(sc.q0, sc.v0)
    for k in range(2):
        act = sc.sample_targets(k)
        for e in (a, b):
            e.set_command(act)
            e.step(sc.step_dt)
        np.testing.assert_array_equal(a.get_sensors(), b.get_sensors())
        np.testing.assert_array_equal(a.get_sensor_data(), b.get_sensor_data())
    # the batch-wide setter is refused in per-env mode
    with pytest.raises(core.BadControlFlow):
        a.stop()
        a.set_sensor_options("ImuSensor", 0, noise_std=[0.1] * 6)


def test_uniform_rows_equal_batch_wide(api):
    uniform_rows(api)


def latch(api):
    """A row written to a running env changes nothing until that env's next start; a masked restart changes only it."""
    n = 4
    sc = scenarios.make("anymal", n, seed=7)
    s = WalkerSensorRandomisation(sc.robot.sensor_layout(), 1.0)
    rows, seeds = _rows(s, np.random.default_rng(8), n)
    a, b = _engine(api, sc, rows, seeds, s.delay_bound), _engine(api, sc, rows, seeds, s.delay_bound)
    for e in (a, b):
        e.start(sc.q0, sc.v0)
    big = {k: v.copy() for k, v in rows.items()}
    big["bias"][2] += 100.0
    mask = np.array([0, 0, 1, 0], np.uint8)
    b.set_sensor_options_env(big["noise_std"], big["bias"], big["delay"], big["jitter"], mask=mask)
    for k in range(2):
        act = sc.sample_targets(k)
        for e in (a, b):
            e.set_command(act)
            e.step(sc.step_dt)
        np.testing.assert_array_equal(a.get_sensors(), b.get_sensors())
    for e in (a, b):
        e.start(sc.q0, sc.v0, mask=mask)
    ma, mb = a.get_sensors(), b.get_sensors()
    keep = ~mask.astype(bool)
    np.testing.assert_array_equal(ma[keep], mb[keep])
    np.testing.assert_allclose(mb[2] - ma[2], 100.0, rtol=0, atol=1e-9)


def test_latch(api):
    latch(api)


# ---------------------------------------------------------------------------------------------- setters
def setters(api):
    n = 4
    sc = scenarios.make("anymal", n, seed=9)
    s = WalkerSensorRandomisation(sc.robot.sensor_layout(), 1.0)
    rng = np.random.default_rng(10)
    rows, seeds = _rows(s, rng, n)
    new, _ = _rows(s, rng, n)
    mask = np.array([1, 0, 1, 0], np.uint8)
    a, b = _engine(api, sc, rows, seeds, s.delay_bound), _engine(api, sc, rows, seeds, s.delay_bound)
    a.set_sensor_options_env(new["noise_std"], new["bias"], new["delay"], new["jitter"], mask=mask)
    dv = {k: _dev(api, v) for k, v in new.items()}
    m = _dev(api, mask, torch.uint8)
    b.set_sensor_options_env_device(dv["noise_std"].data_ptr(), dv["bias"].data_ptr(), dv["delay"].data_ptr(),
                                    dv["jitter"].data_ptr(), m.data_ptr())
    for e in (a, b):
        e.start(sc.q0, sc.v0)
        e.set_command(sc.sample_targets(0))
        e.step(sc.step_dt)
    _sync(api)
    np.testing.assert_array_equal(a.get_sensors(), b.get_sensors())
    # host form: a bad row raises naming its env, and nothing is written
    a.stop()
    for key, val, what in (("noise_std", np.nan, "NaN"), ("delay", -1e-3, "positive"), ("jitter", 1.5 * s.delay_bound, "bound")):
        bad = {k: v.copy() for k, v in rows.items()}
        bad[key][3, -1 if key != "noise_std" else 0] = val
        with pytest.raises(ValueError, match=f"{what}.*env 3"):
            a.set_sensor_options_env(bad["noise_std"], bad["bias"], bad["delay"], bad["jitter"])
    # device form: the bad row is not written, its env stays not started through the next starts until a valid row
    bad = {k: v.copy() for k, v in new.items()}
    bad["delay"][1, 0] = np.nan
    dv = {k: _dev(api, v) for k, v in bad.items()}
    b.set_sensor_options_env_device(dv["noise_std"].data_ptr(), dv["bias"].data_ptr(), dv["delay"].data_ptr(), dv["jitter"].data_ptr())
    q0, v0 = _dev(api, sc.q0), _dev(api, sc.v0)
    b.start_device(q0.data_ptr(), v0.data_ptr())
    _sync(api)
    np.testing.assert_array_equal(b.get_status(), [0, BAD, 0, 0])
    one = _dev(api, [0, 1, 0, 0], torch.uint8)
    b.start_device(q0.data_ptr(), v0.data_ptr(), one.data_ptr())
    _sync(api)
    np.testing.assert_array_equal(b.get_status(), [0, BAD, 0, 0])
    dv = {k: _dev(api, v) for k, v in new.items()}
    b.set_sensor_options_env_device(dv["noise_std"].data_ptr(), dv["bias"].data_ptr(), dv["delay"].data_ptr(),
                                    dv["jitter"].data_ptr(), one.data_ptr())
    b.start_device(q0.data_ptr(), v0.data_ptr(), one.data_ptr())
    _sync(api)
    np.testing.assert_array_equal(b.get_status(), [0, 0, 0, 0])


def test_setters(api):
    setters(api)


# ---------------------------------------------------------------------------------------------- seeds
def seeds_device(api):
    n = 5
    sc = scenarios.make("anymal", n, seed=11)
    s = WalkerSensorRandomisation(sc.robot.sensor_layout(), 1.0)
    rows, _ = _rows(s, np.random.default_rng(12), n)
    rows["noise_std"][:] = 0.1           # noise on every field of every sensor
    seeds = np.array([0, 2 ** 32 - 1, 12345, 2 ** 31, 7], np.uint32)
    host, dev = _engine(api, sc, rows, seeds, s.delay_bound), _engine(api, sc, rows, None, s.delay_bound)
    sd = _dev(api, _seeds_i32(seeds), torch.int32)
    dev.set_seeds_device(sd.data_ptr())
    # the masked form leaves the other envs with the start states of their host seeds
    part = _engine(api, sc, rows, seeds, s.delay_bound)
    other = np.array([5, 6, 7, 8, 9], np.uint32)
    mask = np.array([0, 1, 0, 1, 0], np.uint8)
    ref = _engine(api, sc, rows, np.where(mask.astype(bool), other, seeds), s.delay_bound)
    od, md = _dev(api, _seeds_i32(other), torch.int32), _dev(api, mask, torch.uint8)
    part.set_seeds_device(od.data_ptr(), md.data_ptr())
    engines = (host, dev, part, ref)
    for e in engines:
        e.start(sc.q0, sc.v0)
    for k in range(2):
        act = sc.sample_targets(k)
        for e in engines:
            e.set_command(act)
            e.step(sc.step_dt)
        _sync(api)
        np.testing.assert_array_equal(host.get_sensors(), dev.get_sensors())
        np.testing.assert_array_equal(part.get_sensors(), ref.get_sensors())
    # a later host start of a masked env keeps the device-written states (the host's copy of the seeds is stale)
    for e in (part, ref):
        e.start(sc.q0, sc.v0, mask=mask)
    np.testing.assert_array_equal(part.get_sensors(), ref.get_sensors())
    # the same env restarted with the same seed measures the same noise, with another seed different noise
    one = np.array([1, 0, 0, 0, 0], np.uint8)
    m1 = _dev(api, one, torch.uint8)
    q0, v0 = _dev(api, sc.q0), _dev(api, sc.v0)
    noise = []
    for seed in (42, 42, 43):
        x = _dev(api, _seeds_i32(np.full(n, seed, np.uint32)), torch.int32)
        dev.set_seeds_device(x.data_ptr(), m1.data_ptr())
        dev.start_device(q0.data_ptr(), v0.data_ptr(), m1.data_ptr())
        _sync(api)
        noise.append((dev.get_sensors() - dev.get_sensor_data())[0])
    np.testing.assert_array_equal(noise[0], noise[1])
    assert np.abs(noise[0] - noise[2]).max() > 1e-3


def test_seeds_device(api):
    seeds_device(api)


# ---------------------------------------------------------------------------------------------- device env vs host shadow
def env_shadow(api, std_ratio, pd=False, n_steps=5):
    """The device env against a host env that replays the device's rows (`sensor_rows`, `disturbance_rows`) and restart
    rows through the host setters: bit-equal observations, measurements included, through restarts."""
    n = 5
    kw = dict(simulation_duration_max=4.1, api_=api, std_ratio=std_ratio)
    if pd:
        kw["mahony"] = (1.0, 0.1)
    dev = (DevicePDControlBatchedEnv if pd else DeviceBatchedEnv)(scenarios.make("anymal", n, seed=9), **kw)
    shadow = (envs.PDControlBatchedEnv if pd else envs.BatchedJiminyEnv)(scenarios.make("anymal", n, seed=9), **kw)
    bank_q, bank_v = (_np(x) for x in dev.reset_states)

    def replay(rows):
        snap = {k: _np(v).copy() for k, v in dev.sensor_rows.items()}
        snap["seed"] = snap["seed"].astype(np.uint32)
        shadow._redraw_sensors = lambda mask: shadow.sensor_randomisation.apply_host(shadow.engine, snap, mask)
        if dev.disturbance is not None:
            dsnap = {k: _np(v).copy() for k, v in dev.disturbance_rows.items()}
            shadow._redraw_disturbance = lambda mask: shadow.disturbance.apply_host(shadow.engine, dsnap, mask)
        shadow._sample_state = lambda m: (bank_q[np.maximum(rows, 0)], bank_v[np.maximum(rows, 0)])

    def same(o_d, o_s):
        np.testing.assert_array_equal(_np(o_d["states"]["agent"]["q"]), o_s["states"]["agent"]["q"])
        for name, x in o_s["measurements"].items():
            np.testing.assert_array_equal(_np(o_d["measurements"][name]), x)
        if pd:
            np.testing.assert_array_equal(_np(o_d["features"]["mahony_filter"]), o_s["features"]["mahony_filter"])

    o_d, _ = dev.reset()
    replay(np.zeros(n, np.int64))
    o_s, _ = shadow.reset()
    same(o_d, o_s)
    rng = np.random.default_rng(11)
    for k in range(n_steps):
        act = np.zeros((n, sc_nm(shadow))) if pd else shadow.sc.sample_targets(k)
        o_d, _, _, _, info = dev.step(_dev(api, act))
        replay(_np(info["reset_rows"]))
        o_s, _, _, _, info_s = shadow.step(act)
        same(o_d, o_s)
        np.testing.assert_array_equal(_np(info["status"]), info_s["status"])
        if k % 2 == 0:
            mask = (rng.uniform(size=n) < 0.5).astype(np.uint8)
            o_d, info = dev.reset(mask=_dev(api, mask, torch.uint8))
            replay(_np(info["reset_rows"]))
            o_s, _ = shadow.reset(mask=mask)
            same(o_d, o_s)
    meas = np.concatenate([x.reshape(n, -1) for x in o_s["measurements"].values()], axis=1)
    assert np.abs(meas).max() > 0
    for e in (dev, shadow):
        e.close()


def sc_nm(env):
    return env.robot.nmotors


@pytest.mark.parametrize("case", ["sensors", "sensors+disturbance", "pd"])
def test_device_env_matches_shadow(api, case):
    ratio = {"sensors": 1.0, "disturbance": 1.0} if case == "sensors+disturbance" else {"sensors": 1.0}
    env_shadow(api, ratio, pd=case == "pd")


# ---------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_gpu_sampler_statistics_torch():
    _sampler_case("torch", "cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("solver", ["runge_kutta_4", "euler_explicit"])
def test_gpu_per_env_options_match_oracle(solver, monkeypatch):
    monkeypatch.setenv("JB_NO_FAST_BOUNDS", "1")
    per_env_oracle(None, solver)


@pytest.mark.gpu
def test_gpu_uniform_rows_equal_batch_wide():
    uniform_rows(None)


@pytest.mark.gpu
def test_gpu_latch():
    latch(None)


@pytest.mark.gpu
def test_gpu_setters():
    setters(None)


@pytest.mark.gpu
def test_gpu_seeds_device():
    seeds_device(None)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["sensors", "sensors+disturbance", "pd"])
def test_gpu_device_env_matches_shadow(case):
    ratio = {"sensors": 1.0, "disturbance": 1.0} if case == "sensors+disturbance" else {"sensors": 1.0}
    env_shadow(None, ratio, pd=case == "pd")


@pytest.mark.gpu
def test_gpu_sensors_step_never_synchronises():
    n = 256
    env = DeviceBatchedEnv(scenarios.make("anymal", n, seed=0), simulation_duration_max=4.1, std_ratio={"sensors": 1.0})
    env.reset()
    acts = [torch.as_tensor(env.sc.sample_targets(k), device="cuda") for k in range(4)]
    env.step(acts.pop())                  # first use of the draw's kernels on this stream
    torch.cuda.synchronize()
    with torch.cuda.stream(env._stream):
        torch.cuda._sleep(int(0.5 * 2e9))
    pending = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for a in acts:
            env.step(a)
            pending.append(not env._stream.query())
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    env.close()
    assert all(pending), pending
