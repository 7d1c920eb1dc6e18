"""Per-env body biases: the transformation shared by `model.biased_robot` and `ModelBiasRandomisation`, per-env model rows
latched at every start (`jb_enable_per_env_model`, `jb_set_model_env(_device)`, `jb_get_model_env`) in the
`env_step_kernel_model*` instances, and the envs' `model_bias_std`.

Every kernel scenario is a function of `api`: the CPU suite runs it on the emulated library (device memory is host
memory, torch tensors on the CPU), the `-m gpu` variants on the device with `api=None`.  The oracle has one model per
batch, so each env is compared with a one-env oracle batch built on that env's own table."""
import numpy as np
import pytest
import torch

from jiminy_b200 import core, envs, robots, scenarios
from jiminy_b200 import model as M
from jiminy_b200.core import BatchedEngine
from jiminy_b200.disturbance import WalkerDisturbance
from jiminy_b200.model_randomisation import (BIAS_OPTIONS, ModelBiasRandomisation, WalkerModelRandomisation,
                                             from_model_bias_std)
from jiminy_b200.torch_envs import DeviceBatchedEnv, DevicePDControlBatchedEnv

from emul import emul_api
from oracle.oracle import OracleBatch

BAD = core.JB_ENV_NOT_STARTED | core.JB_ENV_BAD_START
STD = dict(zip(BIAS_OPTIONS, (0.1, 0.05, 0.1, 0.03)))


@pytest.fixture(scope="module")
def api():
    return emul_api()


def _dev(api, x, dtype=torch.float64):
    return torch.tensor(np.ascontiguousarray(x), dtype=dtype, device="cpu" if api is not None else "cuda")


def _np(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _sync(api):
    if api is None:
        torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- transformation
@pytest.mark.parametrize("name", ["anymal", "atlas", "anymal_flexible"])
def test_numpy_draw_is_biased_robot(name):
    """Fed `biased_robot`'s generator stream, the randomiser reproduces its table bit for bit; the torch transformation of
    the same normals agrees to 1e-15 relative."""
    robot = scenarios.make(name, 1).robot
    for std in (STD, {"massBodiesBiasStd": 0.2}, {"inertiaBodiesBiasStd": 0.3, "relativePositionBodiesBiasStd": 0.1}):
        s = ModelBiasRandomisation(robot, std)
        kw = {a: std.get(k, 0.0) for k, a in zip(BIAS_OPTIONS, ("mass_std", "com_std", "inertia_std", "relative_position_std"))}
        for seed in range(3):
            ref = M.biased_robot(robot, np.random.default_rng(seed), **kw)
            np.testing.assert_array_equal(s.draw_numpy(np.random.default_rng(seed), 1)[0], M.body_rows(ref))
        z = np.random.default_rng(7).standard_normal((64, len(s.joints), s.n_normals), dtype=np.float32)
        x, y = s.rows_from_normals(z), _np(s.rows_from_normals_torch(torch.from_numpy(z)))
        # relative to the size of each quantity: mass, lever, rotational inertia, translation
        scale = np.concatenate([np.repeat(np.abs(x[..., a:b]).max(-1, keepdims=True), b - a, -1)
                                for a, b in ((0, 1), (1, 4), (4, 10), (10, 13))], -1)
        assert (np.abs(y - x) <= 1e-15 * scale).all()


def test_untouched_rows_and_refusals():
    flex = scenarios.make("anymal_flexible", 1).robot
    s = ModelBiasRandomisation(flex, STD)
    rows = s.draw_numpy(np.random.default_rng(1), 8)
    keep = [j for j in range(flex.njoints) if j not in s.joints]
    assert 1 in keep and all(j in keep for j in flex.flexibility_joint_indices)
    np.testing.assert_array_equal(rows[:, keep], np.broadcast_to(s.nominal[keep], (8, len(keep), 13)))
    assert (rows[:, s.joints] != s.nominal[s.joints]).all(axis=(0, 2)).any()
    with pytest.raises(ValueError):
        ModelBiasRandomisation(flex, {"massBodiesBiasStd": -0.1})
    with pytest.raises(ValueError):
        ModelBiasRandomisation(flex, {"massBodyBiasStd": 0.1})
    assert from_model_bias_std(flex, None) is None and from_model_bias_std(flex, {}) is None
    assert from_model_bias_std(flex, {k: 0.0 for k in BIAS_OPTIONS}) is None
    rigid = scenarios.make("anymal", 1).robot
    for m in rigid.motors:
        m.backlash = 0.01
    with pytest.raises(NotImplementedError, match="backlash"):
        ModelBiasRandomisation(M.add_backlash_joints(rigid), STD)


def _moments(rows, s):
    """Mass, lever, translation and principal moments of every biased joint against their closed forms (6 standard
    errors): E[m] = m0 (the 1 g floor is never reached at these deviations), E[c] = c0, E[p] = p0, E[x^2] = x0^2 (1 + s^2),
    principal moments mean I0 (as a set: sorted), and the determinant of I over that of I0 mean prod(1 + ...) = 1."""
    n = rows.shape[0]
    sm, sc, si, sp = (STD[k] for k in BIAS_OPTIONS)
    for i, j in enumerate(s.joints):
        x0 = s.nominal[j]
        for col, sd in [(0, sm)] + [(c, sc) for c in (1, 2, 3)] + [(c, sp) for c in (10, 11, 12)]:
            x = rows[:, j, col]
            if x0[col] == 0.0:
                np.testing.assert_array_equal(x, 0.0)
                continue
            assert abs(x.mean() - x0[col]) <= 6 * abs(x0[col]) * sd / np.sqrt(n)
            # second moment: x0^2 (1 + sd^2), variance of x^2 = x0^4 (2 sd^2 (2 + sd^2))
            assert abs((x ** 2).mean() - x0[col] ** 2 * (1 + sd ** 2)) <= 6 * x0[col] ** 2 * np.sqrt(2 * sd ** 2 * (2 + sd ** 2) / n)
        # principal moments: the eigenvalues of the biased inertia are the nominal ones times N(1, si)
        I = rows[:, j, 4:10]
        full = np.stack([I[:, [0, 1, 3]], I[:, [1, 2, 4]], I[:, [3, 4, 5]]], 1)
        ev = np.linalg.eigvalsh(full)
        tr = ev.sum(1)
        t0 = s.eig[0][i].sum()
        assert abs(tr.mean() - t0) <= 6 * si * np.sqrt((s.eig[0][i] ** 2).sum() / n)
        assert abs(np.prod(ev, 1).mean() - np.prod(s.eig[0][i])) <= 6 * abs(np.prod(s.eig[0][i])) * np.sqrt(((1 + si ** 2) ** 3 - 1) / n)


def _stats_case(kind, device="cpu"):
    robot = scenarios.make("anymal", 1).robot
    s = ModelBiasRandomisation(robot, STD)
    n = 2 ** 15
    if kind == "numpy":
        rows = s.draw_numpy(np.random.default_rng(3), n)
    else:
        gen = torch.Generator(device=device)
        gen.manual_seed(4)
        rows = _np(s.draw_torch(gen, n, device))
    assert rows.shape == (n, robot.njoints, 13)
    _moments(rows, s)


@pytest.mark.parametrize("kind", ["numpy", "torch"])
def test_sampler_statistics(kind):
    _stats_case(kind)


# ---------------------------------------------------------------------------------------------- engines
def _scenario(case, n):
    name = {"atlas": "atlas", "flex": "anymal_flexible"}.get(case, "anymal")
    solver = {"euler": "euler_explicit", "dopri": "runge_kutta_dopri"}.get(case)
    return scenarios.make(name, n, seed=5, solver=solver, contact_model="constraint" if case == "constraint" else None)


def _engine(api, monkeypatch, sc, case, per_env, rows=None):
    monkeypatch.setenv("JB_NO_FAST_KERNEL", "1" if case == "dopri" else "0")
    eng = BatchedEngine(sc.robot, sc.options, sc.n_env, api_=api)
    eng.set_pd_controller(sc.kp, sc.kd)
    eng.set_command(sc.target0)
    if case == "walker":
        d = WalkerDisturbance(sc.robot, 1.0)
        d.register(eng)
        draw = d.draw_numpy(np.random.default_rng(5), sc.n_env)
        draw["t"][0] = np.random.default_rng(6).uniform(0.005, sc.step_dt - 0.005, sc.n_env)
        d.apply_host(eng, draw)
    if case == "flex":
        f = WalkerModelRandomisation(sc.robot, 1.0)
        f.register(eng)
        f.apply_host(eng, f.draw_numpy(np.random.default_rng(8), sc.n_env))
    if per_env:
        eng.enable_per_env_model()
        assert "per-env model rows" in eng.describe()
        if rows is not None:
            eng.set_model_env(rows)
    return eng


def _outputs(eng):
    _, q, v, a = eng.get_state()
    return [q, v, a, eng.get_sensors(), *eng.get_efforts(), *eng.get_extra_terms(), *eng.get_centroidal(), eng.get_status()]


IDENTITY_CASES = ["rk4", "euler", "walker", "constraint", "dopri", "atlas", "flex"]


def identity(api, monkeypatch, case, n_steps=2):
    """Per-env rows equal to the model's values: the bits of the same batch without per-env rows, through env-steps, a
    masked restart and jb_compute_dynamics."""
    n = 3
    sc = _scenario(case, n)
    a = _engine(api, monkeypatch, sc, case, False)
    b = _engine(api, monkeypatch, sc, case, True)
    nominal = b.get_model_env()
    np.testing.assert_array_equal(nominal, np.broadcast_to(M.body_rows(sc.robot), nominal.shape))
    b.set_model_env(nominal)
    mask = np.array([0, 1, 0], np.uint8)
    for e in (a, b):
        e.start(sc.q0, sc.v0)
    for x, y in zip(_outputs(a), _outputs(b)):
        np.testing.assert_array_equal(x, y)
    for k in range(n_steps):
        act = sc.sample_targets(k)
        for e in (a, b):
            e.set_command(act)
            e.step(sc.step_dt)
            if k == 0:
                e.start(sc.q0[::-1].copy(), sc.v0, mask=mask)
        for x, y in zip(_outputs(a), _outputs(b)):
            np.testing.assert_array_equal(x, y)
    q, v = a.get_state()[1:3]
    for x, y in zip(a.compute_dynamics(q, v, sc.target0), b.compute_dynamics(q, v, sc.target0)):
        np.testing.assert_array_equal(x, y)
    for e in (a, b):
        e.close()


@pytest.mark.parametrize("case", IDENTITY_CASES)
def test_identity(api, monkeypatch, case):
    identity(api, monkeypatch, case, n_steps=1 if case in ("constraint", "atlas") else 2)


def _compare(eng, orcs, tol_state, tol_sens):
    t1, q1, v1, a1 = eng.get_state()
    got = [np.concatenate([o.get_state()[i] for o in orcs]) for i in range(4)]
    for x, y, tol in ((t1, got[0], 1e-15), (q1, got[1], tol_state), (v1, got[2], tol_state), (a1, got[3], tol_sens)):
        np.testing.assert_allclose(x, y, rtol=0, atol=tol * max(1.0, np.abs(y).max()))
    s0 = np.concatenate([o.get_sensors() for o in orcs])
    np.testing.assert_allclose(eng.get_sensors(), s0, rtol=0, atol=tol_sens * max(1.0, np.abs(s0).max()))
    np.testing.assert_array_equal(eng.get_status(), np.concatenate([o.get_status() for o in orcs]))


PARITY_CASES = ["rk4_bounds", "constraint", "atlas", "flex"]


def parity(api, monkeypatch, case, n_env=5, n_steps=2, tol_state=1e-9, tol_sens=1e-7):
    """Distinct biased rows per env against one-env oracles built on each env's table; after the first env-step envs 1 and
    3 restart with new rows.  rk4_bounds: half the envs start pushed through a hip bound, so the hot path hands them over
    to the full body."""
    sc = _scenario({"rk4_bounds": "rk4"}.get(case, case), n_env)
    if case == "rk4_bounds":
        sc = scenarios.make("anymal", n_env, seed=21, flagged_fraction=0.25)
    s = ModelBiasRandomisation(sc.robot, STD)
    rng = np.random.default_rng(12)
    rows = s.draw_numpy(rng, n_env)
    eng = _engine(api, monkeypatch, sc, "flex" if case == "flex" else case, True, rows)
    # (the flexibility rows _engine wrote, latched by the first start)
    flex_rows = WalkerModelRandomisation(sc.robot, 1.0).draw_numpy(np.random.default_rng(8), n_env) if case == "flex" else None

    def robot_of(i):
        r = M.with_body_rows(sc.robot, rows[i])
        if flex_rows is not None:
            r.flexibility = np.array(r.flexibility, copy=True)
            r.flexibility[sc.robot.flexibility_joint_indices] = flex_rows[i]
        return r

    def oracle(i, cmd, q0, v0):
        o = OracleBatch(robot_of(i), sc.options, 1)
        o.set_pd_controller(sc.kp, sc.kd)
        o.set_command(cmd[i:i + 1])
        assert not o.start(q0[i:i + 1], v0[i:i + 1]).any()
        return o

    # each env starts on the ground of its own model (translation biases move the feet)
    q0 = lambda: np.array([robots.ground_base_height(robot_of(i), sc.q0[i]) for i in range(n_env)])
    q0s = q0()
    eng.start(q0s, sc.v0)
    np.testing.assert_array_equal(eng.get_model_env(), np.where(np.arange(sc.robot.njoints)[None, :, None] == 0, 0.0, rows))
    for i in range(n_env):
        np.testing.assert_array_equal(eng.model(i).inertia[1:], robot_of(i).inertia[1:])
    orcs = [oracle(i, sc.target0, q0s, sc.v0) for i in range(n_env)]
    _compare(eng, orcs, 1e-13, 1e-11)
    mask = np.zeros(n_env, np.uint8)
    mask[[1, 3]] = 1
    for k in range(n_steps):
        act = sc.sample_targets(k)
        eng.set_command(act)
        eng.step(sc.step_dt)
        for i, o in enumerate(orcs):
            o.set_command(act[i:i + 1])
            assert not o.step(sc.step_dt).any()
        _compare(eng, orcs, tol_state, tol_sens)
        if k == 0:
            new = s.draw_numpy(rng, n_env)
            eng.set_model_env(new, mask)
            rows = np.where(mask.astype(bool)[:, None, None], new, rows)
            q0s = q0()
            eng.start(q0s, sc.v0, mask=mask)
            for i in np.flatnonzero(mask):
                orcs[i] = oracle(i, act, q0s, sc.v0)
            _compare(eng, orcs, tol_state, tol_sens)
    eng.close()


@pytest.mark.parametrize("case", PARITY_CASES)
def test_parity_with_oracle(api, monkeypatch, case):
    parity(api, monkeypatch, case, n_steps=2 if case in ("rk4_bounds", "flex") else 1)


def latch_and_setters(api, monkeypatch):
    """A row written to a running env changes nothing until its next start; host rejects raise and write nothing; a device
    reject flags only its env, independently of the sensor and flexibility flags, and a later good row revives it."""
    n = 4
    sc = _scenario("flex", n)
    a = _engine(api, monkeypatch, sc, "flex", True)
    b = _engine(api, monkeypatch, sc, "flex", True)
    for e in (a, b):
        e.enable_per_env_sensor_options(0.01)              # all-zero options: the sensors' own flag, nothing else
        e.start(sc.q0, sc.v0)
    nominal = a.get_model_env()
    new = ModelBiasRandomisation(sc.robot, STD).draw_numpy(np.random.default_rng(2), n)
    a.set_model_env(new)
    for k in range(2):
        for e in (a, b):
            e.set_command(sc.sample_targets(k))
            e.step(sc.step_dt)
        for x, y in zip(_outputs(a), _outputs(b)):
            np.testing.assert_array_equal(x, y)
    np.testing.assert_array_equal(a.get_model_env(), nominal)
    mask = np.array([0, 0, 1, 0], np.uint8)
    a.start(sc.q0, sc.v0, mask=mask)
    got = a.get_model_env()
    np.testing.assert_array_equal(got[2, 1:], new[2, 1:])
    np.testing.assert_array_equal(got[[0, 1, 3]], nominal[[0, 1, 3]])
    # host rejects: nothing written, the env named
    for bad in (np.nan, np.inf, -1.0, 0.0):
        rows = new.copy()
        col = 0 if bad in (-1.0, 0.0) else 7
        rows[1, 2, col] = bad
        with pytest.raises(ValueError, match="env 1"):
            a.set_model_env(rows)
    a.start(sc.q0, sc.v0)
    np.testing.assert_array_equal(a.get_model_env()[:, 1:], new[:, 1:])       # the pending rows before the rejects
    assert not a.get_status().any()
    # a flexibility joint is massless in the model: 0 stays accepted there, the free-flyer row may be written
    fj = sc.robot.flexibility_joint_indices[0]
    ok = nominal.copy()
    ok[:, fj, 0] = 0.0
    ok[:, 1, 0] *= 1.1
    a.set_model_env(ok)
    # device rejects: only that env, independent of the flexibility flag
    rows = ok.copy()
    rows[3, 4, 0] = -2.0
    rd = _dev(api, rows)
    a.set_model_env_device(rd.data_ptr())
    _sync(api)
    a.start(sc.q0, sc.v0)
    st = a.get_status()
    assert st[3] == BAD and not st[:3].any()
    fd = _dev(api, a.get_flexibility_env())
    a.set_flexibility_env_device(fd.data_ptr())           # a valid flexibility row does not clear the model flag
    w, ns = a.width, a.n_sensors
    sens = [_dev(api, np.zeros((n, w))), _dev(api, np.zeros((n, w))), _dev(api, np.zeros((n, ns))), _dev(api, np.zeros((n, ns)))]
    a.set_sensor_options_env_device(*(x.data_ptr() for x in sens))   # nor does a valid sensor row
    _sync(api)
    a.start(sc.q0, sc.v0)
    st = a.get_status()
    assert st[3] == BAD and not st[:3].any()
    # a sensor reject on env 1: the model rows neither clear it nor are taken by its refused starts
    bad_sens = [x.clone() for x in sens]
    bad_sens[2][1, 0] = -1.0
    a.set_sensor_options_env_device(*(x.data_ptr() for x in bad_sens))
    m = _dev(api, np.array([0, 1, 0, 1], np.uint8), torch.uint8)
    good = _dev(api, ok)
    a.set_model_env_device(good.data_ptr(), m.data_ptr())
    _sync(api)
    before = a.get_model_env()
    a.start(sc.q0, sc.v0)
    st = a.get_status()
    assert st[1] == BAD and not st[[0, 2, 3]].any()
    np.testing.assert_array_equal(a.get_model_env()[1], before[1])
    np.testing.assert_array_equal(a.get_model_env()[3, 1:], ok[3, 1:])
    a.set_sensor_options_env_device(*(x.data_ptr() for x in sens))
    _sync(api)
    a.start(sc.q0, sc.v0)
    assert not a.get_status().any()
    np.testing.assert_array_equal(a.get_model_env()[:, 1:], ok[:, 1:])
    for e in (a, b):
        e.close()


def test_latch_and_setters(api, monkeypatch):
    latch_and_setters(api, monkeypatch)


def test_enable_and_variants(api):
    n = 20
    sc = scenarios.make("anymal", n, seed=1)
    eng = BatchedEngine(sc.robot, sc.options, n, api_=api)
    rng = np.random.default_rng(3)
    variants = [M.biased_robot(sc.robot, rng, mass_std=0.1, relative_position_std=0.05) for _ in range(2)]
    vog = np.arange(-(-n // eng.envs_per_group), dtype=np.int32) % 2
    eng.set_model_variants(variants, vog)
    eng.enable_per_env_model()
    rows = eng.get_model_env()
    for e in range(n):
        np.testing.assert_array_equal(rows[e], M.body_rows(variants[vog[e // eng.envs_per_group]]))
    with pytest.raises(core.BadControlFlow):
        eng.set_model_variants(variants, vog)
    with pytest.raises(ValueError):
        eng.enable_per_env_model()
    eng.close()


def grounding(api):
    """jb_start_device_on_ground with translation biases: each env's lowest contact frame at z = 0 (1e-14 m) against
    `robots.ground_base_height` on the env's own table."""
    n = 12
    sc = scenarios.make("anymal", n, seed=5)
    s = ModelBiasRandomisation(sc.robot, {"relativePositionBodiesBiasStd": 0.1, "massBodiesBiasStd": 0.1})
    rows = s.draw_numpy(np.random.default_rng(4), n)
    eng = BatchedEngine(sc.robot, sc.options, n, api_=api)
    eng.enable_per_env_model()
    eng.set_model_env(rows)
    q = sc.q0.copy()
    q[:, 2] += np.random.default_rng(5).uniform(-0.2, 0.2, n)
    qd, vd = _dev(api, q), _dev(api, sc.v0)
    eng.start_device(qd.data_ptr(), vd.data_ptr(), on_ground=True)
    _sync(api)
    assert not eng.get_status().any()
    q1 = eng.get_state()[1]
    expect = np.array([robots.ground_base_height(M.with_body_rows(sc.robot, rows[e]), q[e])[2] for e in range(n)])
    nominal = np.array([robots.ground_base_height(sc.robot, q[e])[2] for e in range(n)])
    np.testing.assert_allclose(q1[:, 2], expect, rtol=0, atol=1e-14)
    assert np.abs(expect - nominal).max() > 1e-3
    eng.close()


def test_grounding(api):
    grounding(api)


# ---------------------------------------------------------------------------------------------- envs
def test_envs_accept_model_bias_std(api):
    for cls in (envs.BatchedJiminyEnv, envs.PDControlBatchedEnv, DeviceBatchedEnv, DevicePDControlBatchedEnv):
        env = cls(scenarios.make("anymal", 2, seed=1), api_=api, model_bias_std=STD)
        assert env.model_bias is not None and "per-env model rows" in env.engine.describe()
        env.reset()
        assert _np(env.model_bias_rows).shape == (2, env.robot.njoints, 13)
        env.close()
    for std in (None, {}, {k: 0.0 for k in BIAS_OPTIONS}):
        env = envs.BatchedJiminyEnv(scenarios.make("anymal", 2, seed=1), api_=api, model_bias_std=std)
        assert env.model_bias is None and "per-env model rows" not in env.engine.describe()
        env.close()


def env_shadow(api, std_ratio, pd=False, n_steps=6, reset_states="sample"):
    """The device env against a host env that replays the device's model rows (and placed states, and the other
    randomisations' rows) through the host setters: bit-equal throughout; the rows every env runs with are
    `env.model_bias_rows`."""
    n = 4
    kw = dict(simulation_duration_max=0.12, api_=api, std_ratio=std_ratio, model_bias_std=STD)
    if pd:
        kw["mahony"] = (1.0, 0.1)
    name = "anymal_flexible" if std_ratio else "anymal"
    dev = (DevicePDControlBatchedEnv if pd else DeviceBatchedEnv)(scenarios.make(name, n, seed=9), reset_states=reset_states, **kw)
    shadow = (envs.PDControlBatchedEnv if pd else envs.BatchedJiminyEnv)(scenarios.make(name, n, seed=9), **kw)

    def replay(q_placed):
        bsnap = _np(dev.model_bias_rows).copy()
        shadow._redraw_model_bias = lambda mask: shadow.model_bias.apply_host(shadow.engine, bsnap, mask)
        if dev.model_randomisation is not None:
            msnap = _np(dev.model_rows).copy()
            shadow._redraw_model = lambda mask: shadow.model_randomisation.apply_host(shadow.engine, msnap, mask)
        if dev.sensor_randomisation is not None:
            snap = {k: _np(v).copy() for k, v in dev.sensor_rows.items()}
            snap["seed"] = snap["seed"].astype(np.uint32)
            shadow._redraw_sensors = lambda mask: shadow.sensor_randomisation.apply_host(shadow.engine, snap, mask)
        if dev.disturbance is not None:
            dsnap = {k: _np(v).copy() for k, v in dev.disturbance_rows.items()}
            shadow._redraw_disturbance = lambda mask: shadow.disturbance.apply_host(shadow.engine, dsnap, mask)
        shadow._sample_state = lambda m: (q_placed, np.zeros((n, dev.robot.nv)))

    def same(o_d, o_s):
        np.testing.assert_array_equal(_np(o_d["states"]["agent"]["q"]), o_s["states"]["agent"]["q"])
        np.testing.assert_array_equal(_np(o_d["states"]["agent"]["v"]), o_s["states"]["agent"]["v"])
        for name_, x in o_s["measurements"].items():
            np.testing.assert_array_equal(_np(o_d["measurements"][name_]), x)

    o_d, _ = dev.reset()
    replay(None)
    o_s, _ = shadow.reset()
    same(o_d, o_s)
    restarts = 0
    for k in range(n_steps):
        act = np.zeros((n, shadow.robot.nmotors)) if pd else shadow.sc.sample_targets(k)
        o_d, r_d, te_d, tr_d, info = dev.step(_dev(api, act))
        replay(_np(o_d["states"]["agent"]["q"]).copy())
        o_s, r_s, te_s, tr_s, info_s = shadow.step(act)
        same(o_d, o_s)
        np.testing.assert_array_equal(_np(info["status"]), info_s["status"])
        restarts += int(_np(info["_final_observation"]).sum())
    assert restarts >= n
    rows = dev.engine.get_model_env()
    np.testing.assert_array_equal(rows[:, 1:], _np(dev.model_bias_rows)[:, 1:])
    assert len({rows[e, 2, 0] for e in range(n)}) == n
    for e in (dev, shadow):
        e.close()


SHADOW_CASES = {"alone": (None, False), "randomised": ({"model": 1.0, "sensors": 1.0, "disturbance": 1.0}, False),
                "pd": (None, True)}


@pytest.mark.parametrize("case", list(SHADOW_CASES))
def test_device_env_matches_shadow(api, case):
    env_shadow(api, *SHADOW_CASES[case])


def test_other_rows_unchanged_by_biases(api):
    """The other randomisers' rows are those of a run without biases: their generators are separate."""
    out = []
    for bias in (None, STD):
        env = DeviceBatchedEnv(scenarios.make("anymal_flexible", 3, seed=4), api_=api, reset_states="sample",
                               std_ratio={"model": 1.0, "sensors": 1.0, "disturbance": 1.0}, model_bias_std=bias)
        env.reset()
        env.reset(mask=torch.ones(3, dtype=torch.bool))
        out.append([_np(env.model_rows).copy(), *[_np(v).copy() for v in env.sensor_rows.values()],
                    *[_np(v).copy() for v in env.disturbance_rows.values()]])
        env.close()
    for a, b in zip(*out):
        np.testing.assert_array_equal(a, b)


# ---------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_gpu_sampler_statistics():
    _stats_case("torch", "cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("case", IDENTITY_CASES)
def test_gpu_identity(monkeypatch, case):
    identity(None, monkeypatch, case, n_steps=3)


@pytest.mark.gpu
@pytest.mark.parametrize("case", PARITY_CASES)
def test_gpu_parity_with_oracle(monkeypatch, case):
    parity(None, monkeypatch, case, n_steps=3)


@pytest.mark.gpu
def test_gpu_latch_and_setters(monkeypatch):
    latch_and_setters(None, monkeypatch)


@pytest.mark.gpu
def test_gpu_grounding():
    grounding(None)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(SHADOW_CASES))
def test_gpu_device_env_matches_shadow(case):
    env_shadow(None, *SHADOW_CASES[case])


@pytest.mark.gpu
def test_gpu_step_never_synchronises():
    n = 256
    sc = scenarios.make("anymal", n, seed=0)
    env = DeviceBatchedEnv(sc, simulation_duration_max=0.08, model_bias_std=STD)
    env.reset()
    acts = [torch.as_tensor(sc.sample_targets(k), device="cuda") for k in range(4)]
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
