"""Walker disturbances: the periodic Gaussian process restated in numpy (`jiminy_b200.disturbance`), process forces
evaluated at every dynamics evaluation (`jb_register_process_force` / `jb_set_process_force(_device)`), the masked impulse
setter from device rows (`jb_set_impulse_force_device`) and the envs' `std_ratio={"disturbance": r}`.

Every kernel scenario is a function of `api`: the CPU suite runs it on the emulated library (device memory is host
memory, torch tensors on the CPU), the `-m gpu` variants on the device with `api=None`."""
import os

import numpy as np
import pytest
import torch

from jiminy_b200 import core, envs, scenarios
from jiminy_b200 import model as M
from jiminy_b200.core import BatchedEngine
from jiminy_b200.disturbance import (F_IMPULSE_DELTA, F_IMPULSE_DT, F_IMPULSE_SCALE, PeriodicGaussianProcess,
                                     WalkerDisturbance, from_std_ratio, root_body_frame)
from jiminy_b200.torch_envs import DeviceBatchedEnv

from emul import emul_api
from oracle.oracle import OracleBatch
from parity_common import compare

DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data")
BAD = core.JB_ENV_NOT_STARTED | core.JB_ENV_BAD_START


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


def _draw(p, rng, n=1):
    z = rng.normal(size=(n, p.n))
    return z @ p.L.T, z @ p.G.T


# ---------------------------------------------------------------------------------------------- the process (numpy)
@pytest.mark.parametrize("wavelength", [0.2, 1.0])
def test_process_closed_forms(wavelength):
    p = PeriodicGaussianProcess(wavelength, 1.0)
    assert p.n == {0.2: 50, 1.0: 10}[wavelength]
    y, g = _draw(p, np.random.default_rng(1))
    knots = np.arange(p.n) * p.delta
    np.testing.assert_allclose(p.evaluate(y, g, knots), y[0], rtol=0, atol=1e-14)
    # slope at the knots, and value and slope continuous across every knot and across the period wrap
    h = 1e-6
    left = (p.evaluate(y, g, knots) - p.evaluate(y, g, knots - h)) / h
    right = (p.evaluate(y, g, knots + h) - p.evaluate(y, g, knots)) / h
    scale = np.abs(g).max()
    np.testing.assert_allclose(left, g[0], rtol=0, atol=1e-4 * scale)
    np.testing.assert_allclose(right, g[0], rtol=0, atol=1e-4 * scale)
    np.testing.assert_allclose(p.evaluate(y, g, knots - 1e-12), p.evaluate(y, g, knots + 1e-12), rtol=0, atol=1e-10 * scale)
    # periodic, negative times included
    t = np.random.default_rng(2).uniform(-3.0, 3.0, 200)
    for k in (-3, -1, 1, 4):
        np.testing.assert_allclose(p.evaluate(y, g, t + k * p.period), p.evaluate(y, g, t), rtol=0, atol=1e-12)


@pytest.mark.parametrize("wavelength", [0.2, 1.0])
def test_process_table_identity(wavelength):
    """grads = K'(t*, t*) K^-1 values for any draw (K regularised): checks G = J L^-T without statistics."""
    p = PeriodicGaussianProcess(wavelength, 1.0)
    y, g = _draw(p, np.random.default_rng(3), 8)
    expect = (p.J @ np.linalg.solve(p.cov, y.T)).T
    np.testing.assert_allclose(g, expect, rtol=0, atol=1e-9 * np.abs(expect).max())


def _check_statistics(d: WalkerDisturbance, draw, n):
    """Empirical covariance of the knot values against the regularised Toeplitz matrix, each entry within 6 standard
    errors (var of x_i x_j = C_ii C_jj + C_ij^2 for a centred Gaussian), and the impulse schedule of every row."""
    values = _np(draw["values"]) / d.gain
    k0 = 0
    for p in d.processes:
        x = values[:, k0:k0 + p.n]
        k0 += p.n
        emp = x.T @ x / n
        se = np.sqrt((np.outer(np.diag(p.cov), np.diag(p.cov)) + p.cov ** 2) / n)
        assert (np.abs(emp - p.cov) <= 6.0 * se).all(), np.abs((emp - p.cov) / se).max()
    t, dt, w = _np(draw["t"]), _np(draw["dt"]), _np(draw["wrench"])
    assert t.shape == (9, n) and dt.shape == (9, n) and w.shape == (9, n, 6)
    assert (np.abs(t - d.t_ref[:, None]) <= F_IMPULSE_DELTA).all()
    assert (dt == F_IMPULSE_DT).all()
    f = np.linalg.norm(w[..., :2], axis=-1)
    assert (f <= d.ratio * F_IMPULSE_SCALE).all() and f.max() > 0.99 * d.ratio * F_IMPULSE_SCALE
    assert (w[..., 2:] == 0.0).all()
    # the direction is a unit vector: |F| is uniform on [0, 1000 r] (mean 500 r)
    assert abs(f.mean() / (d.ratio * F_IMPULSE_SCALE) - 0.5) < 0.01


def test_sampler_statistics_numpy():
    sc = scenarios.make("anymal", 1, seed=0)
    d = WalkerDisturbance(sc.robot, 0.7)
    n = 2 ** 15
    _check_statistics(d, d.draw_numpy(np.random.default_rng(4), n), n)


def test_sampler_statistics_torch():
    sc = scenarios.make("anymal", 1, seed=0)
    d = WalkerDisturbance(sc.robot, 0.7)
    n = 2 ** 15
    gen = torch.Generator(device="cpu")
    gen.manual_seed(5)
    _check_statistics(d, d.draw_torch(gen, n, "cpu"), n)


def test_root_body_frame_and_std_ratio():
    assert root_body_frame(scenarios.make("anymal", 1).robot) == "base"
    assert root_body_frame(scenarios.make("atlas", 1).robot) == "pelvis"
    rob = scenarios.make("anymal", 1).robot
    assert from_std_ratio(rob, None, 20.0) is None and from_std_ratio(rob, {}, 20.0) is None
    assert len(from_std_ratio(rob, {"disturbance": 1.0}, 20.0).t_ref) == 9
    with pytest.raises(NotImplementedError, match="ground"):
        from_std_ratio(rob, {"disturbance": 1.0, "ground": 0.5}, 20.0)


# ---------------------------------------------------------------------------------------------- stage-time evaluation
def point_mass_momentum(api, solver):
    """Unit point mass, gravity off, only a process force on its root body.  RK4 steps of 1 ms on a grid that holds every
    knot (delta = 20 ms): the momentum change over each 20 ms interval is the closed-form integral of the cubic Hermite
    spline, delta (y0 + y1) / 2 + delta^2 (g0 - g1) / 12, because Simpson's rule (what RK4 is for a force of t alone) is
    exact on cubics.  Only the scheduler's first 1 us step and the rest of the first millisecond differ from the grid, and
    neither straddles a knot; a step of length h that did straddle one would add Simpson's error for the jump J of f''
    there, at most h^3 |J| / 48 (here h = 1 ms and |J| <= 12 max|g| / delta + 12 max|y| / delta^2).  Explicit Euler
    gives the left Riemann sum over the same grid (each step starts from the re-evaluation at t that the controller update
    of every millisecond triggers).  Dormand-Prince's weights integrate quartics exactly, so its adaptive steps, which the
    1 ms breakpoints keep off the knots, give the closed form as well.  A value held per step, or per scheduler iteration,
    misses by orders of magnitude.

    An impulse along z registered AFTER the process force, on the same frame, must still act: dv_z = F_z dt over the
    env-step that holds it (it may not share the slot the process force overwrites before every evaluation)."""
    r = M.build_robot_table(os.path.join(DATA, "point_mass.urdf"), True)
    opt = M.default_engine_options()
    opt["world"]["gravity"] = [0.0] * 6
    opt["stepper"].update(odeSolver=solver, dtMax=1e-3, sensorsUpdatePeriod=1e-3, controllerUpdatePeriod=1e-3)
    n = 3
    eng = BatchedEngine(r, opt, n, api_=api)
    p = PeriodicGaussianProcess(0.2, 1.0)
    q = PeriodicGaussianProcess(1.0, 1.0)
    rng = np.random.default_rng(6)
    (yp, gp), (yq, gq) = _draw(p, rng, n), _draw(q, rng, n)
    yp, gp, yq, gq = 50 * yp, 50 * gp, 30 * yq, 30 * gq
    slot = eng.register_process_force(root_body_frame(r), [1, 0], [p.n, q.n], [1.0, 1.0])
    fz = np.zeros((n, 6))
    fz[:, 2] = rng.uniform(5.0, 10.0, n)
    eng.register_impulse_force(root_body_frame(r), 0.05, 0.01, fz)
    assert "evaluated at every dynamics evaluation" in eng.describe()
    eng.set_process_force(slot, np.c_[yp, yq], np.c_[gp, gq])
    eng.start(np.tile(r.neutral(), (n, 1)), np.zeros((n, 6)))
    v_prev = np.zeros((n, 6))
    for k in range(10):
        eng.step(p.delta)
        t, _, v, _ = eng.get_state()
        np.testing.assert_allclose(t, (k + 1) * p.delta, rtol=0, atol=1e-15)
        if solver != "euler_explicit":
            dp = p.delta * (yp[:, k] + yp[:, k + 1]) / 2 + p.delta ** 2 * (gp[:, k] - gp[:, k + 1]) / 12
            tq = np.linspace(k * p.delta, (k + 1) * p.delta, 3)
            fq = q.evaluate(yq[:, None, :], gq[:, None, :], tq[None, :])
            # f1's knots are 100 ms apart: inside them it is one cubic, which Simpson's rule on [k delta, (k+1) delta] integrates exactly
            dq = p.delta / 6 * (fq[:, 0] + 4 * fq[:, 1] + fq[:, 2])
        else:
            grid = np.r_[k * p.delta + (1e-6 if k == 0 else 0.0), k * p.delta + np.arange(1, 20) * 1e-3]
            grid = np.r_[k * p.delta, grid] if k == 0 else grid
            ends = np.r_[grid[1:], (k + 1) * p.delta]
            w = ends - grid
            dp = (p.evaluate(yp[:, None, :], gp[:, None, :], grid[None, :]) * w).sum(axis=1)
            dq = (q.evaluate(yq[:, None, :], gq[:, None, :], grid[None, :]) * w).sum(axis=1)
        scale = max(np.abs(yp).max(), np.abs(yq).max()) * p.delta
        np.testing.assert_allclose(v[:, 1] - v_prev[:, 1], dp, rtol=0, atol=1e-12 * scale)
        np.testing.assert_allclose(v[:, 0] - v_prev[:, 0], dq, rtol=0, atol=1e-12 * scale)
        np.testing.assert_allclose(v[:, 2] - v_prev[:, 2], fz[:, 2] * 0.01 if k == 2 else 0.0, rtol=0, atol=1e-14 * scale)
        np.testing.assert_allclose(v[:, 3:], 0.0, rtol=0, atol=1e-15 * scale)   # rounding of the sweeps only
        v_prev = v


@pytest.mark.parametrize("solver", ["runge_kutta_4", "euler_explicit", "runge_kutta_dopri"])
def test_point_mass_momentum_closed_form(api, solver):
    point_mass_momentum(api, solver)


# ---------------------------------------------------------------------------------------------- against the oracle
def oracle_scenario(api, robot="anymal", solver="runge_kutta_4", contact_model=None, n_steps=4, tol=1e-9):
    """The full walker disturbance (r = 1) with the profile sampled once per env-step (update period = the env-step): the
    oracle's held profile force, fed with the numpy evaluator at the step times, then applies the same wrench.  The
    first impulse of every env is moved into the run so that a step crosses it."""
    n = 6
    sc = scenarios.make(robot, n, seed=3, solver=solver, contact_model=contact_model)
    eng = BatchedEngine(sc.robot, sc.options, n, api_=api)
    orc = OracleBatch(sc.robot, sc.options, n)
    if sc.kp is not None:
        for x in (eng, orc):
            x.set_pd_controller(sc.kp, sc.kd)
    d = WalkerDisturbance(sc.robot, 1.0)
    draw = d.draw_numpy(np.random.default_rng(7), n)
    draw["t"][0] = np.random.default_rng(8).uniform(0.01, sc.step_dt * (n_steps - 1), n)
    fr = sc.robot.frames[d.frame]
    for k in range(d.n_impulses):
        a = eng.register_impulse_force(d.frame, draw["t"][k], draw["dt"][k], draw["wrench"][k])
        b = orc.register_impulse_force(fr.joint, fr.placement.p, draw["t"][k], draw["dt"][k], draw["wrench"][k])
        assert a == b
    slot = eng.register_process_force(d.frame, [0, 1], d.n_knots, [1.0, 1.0], sc.step_dt)
    oslot = orc.register_profile_force(fr.joint, fr.placement.p, sc.step_dt)
    eng.set_process_force(slot, draw["values"], draw["grads"])
    for x in (eng, orc):
        x.set_command(sc.target0)
    eng.start(sc.q0, sc.v0)
    assert not orc.start(sc.q0, sc.v0).any()
    for k in range(n_steps):
        w = np.zeros((n, 6))
        w[:, :2] = d.profile(draw, np.full(n, k * sc.step_dt))
        orc.set_profile_force(oslot, w)
        act = sc.sample_targets(k)
        for x in (eng, orc):
            x.set_command(act)
        eng.step(sc.step_dt)
        assert not orc.step(sc.step_dt, parallel=True).any()
        compare(eng, orc, tol, 100 * tol)


# explicit Euler at 1 ms on the 4e6 N/m ground amplifies rounding-level differences step after step (by 1e4 per env-step
# in this scenario, with or without the profile): two env-steps, the second crossing the moved impulse
ORACLE_CASES = {"anymal_rk4": dict(), "anymal_euler": dict(solver="euler_explicit", n_steps=2, tol=1e-7),
                "anymal_dopri": dict(solver="runge_kutta_dopri"), "anymal_rk4_constraint": dict(contact_model="constraint"),
                "atlas_constraint": dict(robot="atlas", contact_model="constraint", n_steps=3)}


@pytest.mark.parametrize("case", sorted(ORACLE_CASES))
def test_disturbance_matches_oracle(api, case):
    oracle_scenario(api, **ORACLE_CASES[case])


def oracle_start_scenario(api, robot="anymal", contact_model=None):
    """The process force with update period 0 in the evaluations of `jb_start` (all at t = 0: the contact-force guard and,
    with `constraint` contacts, the INIT_ITERATIONS fixed point) against the oracle's continuous profile force holding the
    numpy evaluator's value at t = 0: state, accelerations, sensors, external wrenches per joint and extra terms."""
    n = 6
    sc = scenarios.make(robot, n, seed=5, contact_model=contact_model)
    eng = BatchedEngine(sc.robot, sc.options, n, api_=api)
    orc = OracleBatch(sc.robot, sc.options, n)
    if sc.kp is not None:
        for x in (eng, orc):
            x.set_pd_controller(sc.kp, sc.kd)
    d = WalkerDisturbance(sc.robot, 1.0)
    draw = d.draw_numpy(np.random.default_rng(12), n)
    d.register(eng)
    d.apply_host(eng, draw)
    fr = sc.robot.frames[d.frame]
    oslot = orc.register_profile_force(fr.joint, fr.placement.p, 0.0)
    w = np.zeros((n, 6))
    w[:, :2] = d.profile(draw, np.zeros(n))
    orc.set_profile_force(oslot, w)
    for x in (eng, orc):
        x.set_command(sc.target0)
    eng.start(sc.q0, sc.v0)
    assert not orc.start(sc.q0, sc.v0).any()
    compare(eng, orc, 1e-13, 1e-10)
    f0 = orc.get_efforts()[3]
    np.testing.assert_allclose(eng.get_efforts()[3], f0, rtol=0, atol=1e-9 * max(1.0, np.abs(f0).max()))
    assert np.abs(w).max() > 1.0       # the profile is not negligible at t = 0


START_CASES = {"anymal": dict(), "anymal_constraint": dict(contact_model="constraint"),
               "atlas_constraint": dict(robot="atlas", contact_model="constraint")}


@pytest.mark.parametrize("case", sorted(START_CASES))
def test_disturbance_start_matches_oracle(api, case):
    oracle_start_scenario(api, **START_CASES[case])


# ---------------------------------------------------------------------------------------------- device setters
def impulse_device_setter(api):
    """jb_set_impulse_force_device is bit-equal to jb_set_impulse_force on subset masks; a NaN, negative t or too short
    dt flags only its own env."""
    n = 5
    sc = scenarios.make("anymal", n, seed=2)
    engs = [BatchedEngine(sc.robot, sc.options, n, api_=api) for _ in range(2)]
    d = WalkerDisturbance(sc.robot, 1.0)
    rng = np.random.default_rng(9)
    draws = [d.draw_numpy(rng, n) for _ in range(3)]
    for dr in draws:
        dr["t"][0] = rng.uniform(0.0, 0.1, n)
    for e in engs:
        d.register(e)
        d.apply_host(e, draws[0])
        e.set_pd_controller(sc.kp, sc.kd)
        e.set_command(sc.target0)
        e.start(sc.q0, sc.v0)
    host, dev = engs
    keep = []
    for dr, mask in ((draws[1], np.array([1, 0, 1, 1, 0], np.uint8)), (draws[2], np.array([0, 1, 0, 0, 1], np.uint8))):
        tens = {k: _dev(api, v) for k, v in dr.items()}
        m = _dev(api, mask, torch.uint8)
        d.apply_host(host, dr, mask)
        d.apply_device(dev, tens, m.data_ptr())
        keep.append((tens, m))
        _sync(api)
        for e in engs:
            e.step(sc.step_dt)
        for a, b in zip(dev.get_state(), host.get_state()):
            np.testing.assert_array_equal(a, b)
        np.testing.assert_array_equal(dev.get_status(), host.get_status())
    # bad rows
    t, dt, w = draws[1]["t"][0].copy(), draws[1]["dt"][0].copy(), draws[1]["wrench"][0].copy()
    t[1], t[2], dt[3] = np.nan, -1e-3, 1e-11
    args = [_dev(api, x) for x in (t, dt, w)]
    dev.set_impulse_force_device(0, *(x.data_ptr() for x in args))
    _sync(api)
    st = dev.get_status()
    np.testing.assert_array_equal(st[[1, 2, 3]], BAD)
    assert not (st[[0, 4]] & BAD).any()
    host.set_impulse_force(0, t[[0]].repeat(n), dt[[0]].repeat(n), w, mask=np.array([1, 0, 0, 0, 1], np.uint8))
    # the env-step still advances the good envs exactly like the host-set ones
    t4 = np.r_[t[0], t[0], t[0], t[0], t[4]]
    host.set_impulse_force(0, t4, dt[[0]].repeat(n), w, mask=np.array([0, 0, 0, 0, 1], np.uint8))
    for e in engs:
        e.step(sc.step_dt)
    np.testing.assert_array_equal(dev.get_state()[1][[0, 4]], host.get_state()[1][[0, 4]])


def test_impulse_device_setter(api):
    impulse_device_setter(api)


def process_masked_setters(api):
    """Rows outside the mask keep their tables, for the host and the device setter alike: an engine rewritten by masked
    setters steps bit-equal to one given the merged rows in one call."""
    n = 5
    sc = scenarios.make("anymal", n, seed=4)
    d = WalkerDisturbance(sc.robot, 1.0)
    rng = np.random.default_rng(10)
    a, b = d.draw_numpy(rng, n), d.draw_numpy(rng, n)
    mask = np.array([0, 1, 1, 0, 1], np.uint8)
    merged = {k: np.where(mask.astype(bool).reshape((1, -1) + (1,) * (a[k].ndim - 2)) if a[k].shape[0] != n
                          else mask.astype(bool)[:, None], b[k], a[k]) for k in a}
    engs = [BatchedEngine(sc.robot, sc.options, n, api_=api) for _ in range(3)]
    for e in engs:
        d.register(e)
        e.set_pd_controller(sc.kp, sc.kd)
        e.set_command(sc.target0)
    ref, host, dev = engs
    d.apply_host(ref, merged)
    d.apply_host(host, a)
    d.apply_host(host, b, mask)
    d.apply_host(dev, a)
    tens, m = {k: _dev(api, v) for k, v in b.items()}, _dev(api, mask, torch.uint8)
    d.apply_device(dev, tens, m.data_ptr())
    _sync(api)
    for e in engs:
        e.start(sc.q0, sc.v0)
        for k in range(2):
            e.step(sc.step_dt)
    for e in (host, dev):
        for x, y in zip(e.get_state(), ref.get_state()):
            np.testing.assert_array_equal(x, y)


def test_process_masked_setters(api):
    process_masked_setters(api)


# ---------------------------------------------------------------------------------------------- envs
def env_shadow(api, n_steps=5):
    """The device env with {"disturbance": 1} against a host env that replays the device's rows (`disturbance_rows`) and
    restart rows through the host setters: bit-equal throughout, restarts included.  With std_ratio None nothing is
    registered."""
    n = 5
    kw = dict(simulation_duration_max=4.1, api_=api, std_ratio={"disturbance": 1.0})
    dev = DeviceBatchedEnv(scenarios.make("anymal", n, seed=9), **kw)
    shadow = envs.BatchedJiminyEnv(scenarios.make("anymal", n, seed=9), **kw)
    assert envs.BatchedJiminyEnv(scenarios.make("anymal", n, seed=9), api_=api).disturbance is None
    assert len(dev.disturbance.impulses) == 2 and "process force 0" in dev.engine.describe()
    bank_q, bank_v = (_np(x) for x in dev.reset_states)

    def replay(rows):
        snap = {k: _np(v).copy() for k, v in dev.disturbance_rows.items()}
        shadow._redraw_disturbance = lambda mask: shadow.disturbance.apply_host(shadow.engine, snap, mask)
        shadow._sample_state = lambda m: (bank_q[np.maximum(rows, 0)], bank_v[np.maximum(rows, 0)])

    dev.reset()
    replay(np.zeros(n, np.int64))
    shadow.reset()
    rng = np.random.default_rng(11)
    for k in range(n_steps):
        act = shadow.sc.sample_targets(k)
        o_d, r_d, te_d, tr_d, info = dev.step(_dev(api, act))
        rows = _np(info["reset_rows"])
        replay(rows)
        o_s, r_s, te_s, tr_s, info_s = shadow.step(act)
        np.testing.assert_array_equal(_np(o_d["states"]["agent"]["q"]), o_s["states"]["agent"]["q"])
        np.testing.assert_array_equal(_np(o_d["measurements"]["ImuSensor"]), o_s["measurements"]["ImuSensor"])
        np.testing.assert_array_equal(_np(info["status"]), info_s["status"])
        if k % 2 == 0:
            mask = (rng.uniform(size=n) < 0.5).astype(np.uint8)
            o_d, info = dev.reset(mask=_dev(api, mask, torch.uint8))
            replay(_np(info["reset_rows"]))
            o_s, _ = shadow.reset(mask=mask)
            np.testing.assert_array_equal(_np(o_d["states"]["agent"]["v"]), o_s["states"]["agent"]["v"])
    for e in (dev, shadow):
        e.close()


def test_device_env_disturbance_matches_shadow(api):
    env_shadow(api)


# ---------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("solver", ["runge_kutta_4", "euler_explicit", "runge_kutta_dopri"])
def test_gpu_point_mass_momentum_closed_form(solver):
    point_mass_momentum(None, solver)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(ORACLE_CASES))
def test_gpu_disturbance_matches_oracle(case):
    oracle_scenario(None, **ORACLE_CASES[case])


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(START_CASES))
def test_gpu_disturbance_start_matches_oracle(case):
    oracle_start_scenario(None, **START_CASES[case])


@pytest.mark.gpu
def test_gpu_impulse_device_setter():
    impulse_device_setter(None)


@pytest.mark.gpu
def test_gpu_process_masked_setters():
    process_masked_setters(None)


@pytest.mark.gpu
def test_gpu_sampler_statistics_torch():
    sc = scenarios.make("anymal", 1, seed=0)
    d = WalkerDisturbance(sc.robot, 0.7)
    n = 2 ** 15
    gen = torch.Generator(device="cuda")
    gen.manual_seed(5)
    _check_statistics(d, d.draw_torch(gen, n, "cuda"), n)


@pytest.mark.gpu
def test_gpu_device_env_disturbance_matches_shadow():
    env_shadow(None)


@pytest.mark.gpu
def test_gpu_disturbance_step_never_synchronises():
    n = 256
    env = DeviceBatchedEnv(scenarios.make("anymal", n, seed=0), simulation_duration_max=4.1, std_ratio={"disturbance": 1.0})
    assert len(env.disturbance.impulses) == 2            # the impulse setter is enqueued at every step
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
