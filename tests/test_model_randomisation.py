"""Walker model randomisation: per-env stiffness and damping of the flexibility joints, latched at every start
(`jb_enable_per_env_flexibility`, `jb_set_flexibility_env(_device)`), the samplers of `jiminy_b200.model_randomisation` and
the envs' `std_ratio={"model": r}`.

Every kernel scenario is a function of `api`: the CPU suite runs it on the emulated library (device memory is host
memory, torch tensors on the CPU), the `-m gpu` variants on the device with `api=None`.  The oracle has one model per
batch, so each env is compared with a one-env oracle batch built on that env's flexibility parameters."""
import numpy as np
import pytest
import scipy.linalg
import torch

from jiminy_b200 import core, envs, scenarios
from jiminy_b200 import model as M
from jiminy_b200.core import BatchedEngine
from jiminy_b200.model_randomisation import (FLEX_DAMPING_SCALE, FLEX_STIFFNESS_SCALE, WalkerModelRandomisation,
                                             from_std_ratio)
from jiminy_b200.torch_envs import DeviceBatchedEnv, DevicePDControlBatchedEnv

from emul import emul_api
from flexibility_common import _opt, flexible_pendulum
from oracle.oracle import OracleBatch
import parity_common as pc

BAD = core.JB_ENV_NOT_STARTED | core.JB_ENV_BAD_START


@pytest.fixture(scope="module")
def api():
    return emul_api()


def _dev(api, x, dtype=torch.float64):
    """A device copy of x (on the CPU for the emulated library: a copy there too, never a view of x)."""
    return torch.tensor(np.ascontiguousarray(x), dtype=dtype, device="cpu" if api is not None else "cuda")


def _np(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _sync(api):
    if api is None:
        torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- sampler
def _sampler_case(kind, device="cpu", r=1.5):
    robot = scenarios.make("anymal_flexible", 1, seed=0).robot
    s = WalkerModelRandomisation(robot, r)
    n = 2 ** 15
    if kind == "numpy":
        rows = s.draw_numpy(np.random.default_rng(3), n)
    else:
        gen = torch.Generator(device=device)
        gen.manual_seed(4)
        rows = _np(s.draw_torch(gen, n, device))
    nominal = robot.flexibility[robot.flexibility_joint_indices]
    assert rows.shape == (n, 4, 6)
    np.testing.assert_array_equal(s.nominal, nominal)
    dev = rows - nominal
    # the three axes of a flexibility share one shift (up to the rounding of nominal + shift)
    for o in (0, 3):
        np.testing.assert_allclose(dev[:, :, o + 1], dev[:, :, o], rtol=0, atol=1e-12 * np.abs(nominal).max())
        np.testing.assert_allclose(dev[:, :, o + 2], dev[:, :, o], rtol=0, atol=1e-12 * np.abs(nominal).max())
    for o, a in ((0, FLEX_STIFFNESS_SCALE * r), (3, FLEX_DAMPING_SCALE * r)):
        x = dev[:, :, o]
        assert (np.abs(x) <= a).all() and (rows[:, :, o:o + 3] >= 0).all()
        # U(-a, a): mean 0 (var a^2 / 3), variance a^2 / 3 (var of x^2: 4 a^4 / 45)
        assert (np.abs(x.mean(0)) <= 6 * np.sqrt(a ** 2 / 3 / n)).all()
        assert (np.abs((x ** 2).mean(0) - a ** 2 / 3) <= 6 * np.sqrt(4 * a ** 4 / 45 / n)).all()
    # stiffness and damping draws are independent
    assert abs(np.corrcoef(dev[:, 0, 0], dev[:, 0, 3])[0, 1]) <= 6 / np.sqrt(n)


@pytest.mark.parametrize("kind", ["numpy", "torch"])
def test_sampler_statistics(kind):
    _sampler_case(kind)


def test_std_ratio_model(api):
    flex = scenarios.make("anymal_flexible", 1).robot
    rigid = scenarios.make("anymal", 1).robot
    assert from_std_ratio(flex, None) is None and from_std_ratio(flex, {"model": 0.0}) is None
    assert from_std_ratio(flex, {"sensors": 1.0}) is None
    assert from_std_ratio(rigid, {"model": 0.0}) is None
    with pytest.raises(NotImplementedError, match="model"):          # no flexibility joint to randomise
        from_std_ratio(rigid, {"model": 1.0})
    assert from_std_ratio(flex, {"model": 2.0}).n_flex == 4
    # k0 >= 4e3, d0 >= 20: r <= 2
    with pytest.raises(ValueError, match="negative"):
        from_std_ratio(flex, {"model": 2.01})
    with pytest.raises(ValueError):
        from_std_ratio(flex, {"model": -1.0})
    with pytest.raises(ValueError):
        WalkerModelRandomisation(rigid, 1.0)
    for key in ("ground", "flexibility"):
        with pytest.raises(NotImplementedError, match=key):
            envs.BatchedJiminyEnv(scenarios.make("anymal", 2, seed=1), api_=api, std_ratio={"model": 1.0, key: 0.5})


def test_model_key_on_rigid_robot(api):
    """{"model": r} needs flexibility joints: refused on rigid ANYmal by every env (alone or with other keys), while
    r = 0 leaves the run bit-equal to no randomisation and calls no new entry point."""
    for cls in (envs.BatchedJiminyEnv, envs.PDControlBatchedEnv, DeviceBatchedEnv):
        for ratio in ({"model": 1.0}, {"model": 0.5, "sensors": 1.0, "disturbance": 1.0}):
            with pytest.raises(NotImplementedError, match="model"):
                cls(scenarios.make("anymal", 2, seed=1), api_=api, std_ratio=ratio)
    outs = []
    for ratio in (None, {"model": 0.0}):
        env = envs.BatchedJiminyEnv(scenarios.make("anymal", 3, seed=2), api_=api, std_ratio=ratio)
        assert env.model_randomisation is None
        o, _ = env.reset()
        seq = [o["states"]["agent"]["q"].copy()]
        for k in range(2):
            o = env.step(env.sc.sample_targets(k))[0]
            seq.append(o["states"]["agent"]["q"].copy())
        assert "per-env flexibility" not in env.engine.describe()
        outs.append(seq)
        env.close()
    for a, b in zip(*outs):
        np.testing.assert_array_equal(a, b)


# ---------------------------------------------------------------------------------------------- first principles
def sea_per_env(api):
    """The series-elastic actuator of `flexibility_common.series_elastic_actuator` with a different flexibility stiffness
    and damping in every env: each env follows the closed form of its own parameters (1e-4, as the one-parameter test)."""
    J, k_control, nu_control, I = 0.1, 100.0, 1.0, 5.0
    ks, nus = np.array([20.0, 35.0, 12.0]), np.array([0.1, 0.3, 0.05])
    r = flexible_pendulum(J, 20.0, 0.1)
    opt = _opt(odeSolver="runge_kutta_dopri", tolAbs=1e-8, tolRel=1e-8)
    opt["world"]["gravity"] = [0.0] * 6
    v_init = np.array([0.1, -0.05, 0.2])
    n = len(v_init)
    q0 = np.tile([0.0, 0.0, 0.0, 1.0, 0.0], (n, 1))
    v0 = np.zeros((n, 4))
    v0[:, 1] = v_init
    eng = BatchedEngine(r, opt, n, api_=api)
    eng.set_joint_springs([0.0, 0.0, 0.0, k_control], [0.0, 0.0, 0.0, nu_control])
    eng.enable_per_env_flexibility()
    assert "per-env flexibility parameters" in eng.describe()
    np.testing.assert_array_equal(eng.get_flexibility_env(), np.tile([20.0] * 3 + [0.1] * 3, (n, 1, 1)))
    rows = np.concatenate([np.repeat(ks[:, None], 3, 1), np.repeat(nus[:, None], 3, 1)], 1)[:, None, :]
    eng.set_flexibility_env(rows)
    eng.start(q0, v0)
    np.testing.assert_array_equal(eng.get_flexibility_env(), rows)
    log = []
    for _ in range(40):
        eng.step(0.05)
        t1, q1, v1, _ = eng.get_state()
        log.append((t1.copy(), q1.copy(), v1.copy()))
    assert not eng.get_status().any()
    for t1, q1, v1 in log[::4]:
        for e in range(n):
            k, nu = ks[e], nus[e]
            A = np.array([[0.0, 0.0, 1.0, 0.0],
                          [0.0, 0.0, 0.0, 1.0],
                          [-k * (1 / I + 1 / J), k_control / J, -nu * (1 / I + 1 / J), nu_control / J],
                          [k / J, -k_control / J, nu / J, -nu_control / J]])
            x = np.array([2.0 * np.arctan2(q1[e, 1], q1[e, 3]), q1[e, 4], v1[e, 1], v1[e, 3]])
            xa = scipy.linalg.expm(A * t1[e]) @ np.array([0.0, 0.0, v_init[e], 0.0])
            np.testing.assert_allclose(x, xa, atol=1e-4)
    # the parameters matter at that tolerance: env 1's trajectory is not env 0's closed form
    x1 = np.array([2.0 * np.arctan2(log[-1][1][1, 1], log[-1][1][1, 3]), log[-1][1][1, 4]])
    assert np.abs(x1 - np.array([2.0 * np.arctan2(log[-1][1][0, 1], log[-1][1][0, 3]), log[-1][1][0, 4]]) *
                  v_init[1] / v_init[0]).max() > 1e-3


def test_sea_per_env_closed_form(api):
    sea_per_env(api)


# ---------------------------------------------------------------------------------------------- oracle parity
def _flex_robot(rigid, row):
    """The flexible ANYmal with the flexibility parameters of one env's row [n_flex, 6]."""
    cfg = [dict(c, stiffness=list(row[k, :3]), damping=list(row[k, 3:])) for k, c in enumerate(scenarios.FLEXIBLE_ANYMAL_CONFIG)]
    return M.add_flexibility_joints(rigid, cfg)


def _compare(eng, orcs, tol_state, tol_sens):
    t1, q1, v1, a1 = eng.get_state()
    got = [np.concatenate([o.get_state()[i] for o in orcs]) for i in range(4)]
    for x, y, tol in ((t1, got[0], 1e-15), (q1, got[1], tol_state), (v1, got[2], tol_state), (a1, got[3], tol_sens)):
        np.testing.assert_allclose(x, y, rtol=0, atol=tol * max(1.0, np.abs(y).max()))
    s0 = np.concatenate([o.get_sensors() for o in orcs])
    np.testing.assert_allclose(eng.get_sensors(), s0, rtol=0, atol=tol_sens * max(1.0, np.abs(s0).max()))
    u0 = np.concatenate([o.get_efforts()[0] for o in orcs])
    np.testing.assert_allclose(eng.get_efforts()[0], u0, rtol=0, atol=tol_sens * max(1.0, np.abs(u0).max()))
    np.testing.assert_array_equal(eng.get_status(), np.concatenate([o.get_status() for o in orcs]))


def per_env_oracle(api, contact_model=None, n_env=5, n_steps=3, tol_state=1e-9, tol_sens=1e-7):
    """anymal_flexible with a row of its own in every env (r = 2, the largest ratio), each env against a one-env oracle
    built on its parameters; after the first env-step envs 1 and 3 restart with new rows."""
    sc = scenarios.make("anymal_flexible", n_env, seed=3, contact_model=contact_model)
    rigid = scenarios.make("anymal", 1, seed=3, contact_model=contact_model).robot
    s = WalkerModelRandomisation(sc.robot, 2.0)
    rng = np.random.default_rng(12)
    rows = s.draw_numpy(rng, n_env)
    eng = BatchedEngine(sc.robot, sc.options, n_env, api_=api)
    s.register(eng)
    s.apply_host(eng, rows)
    eng.set_pd_controller(sc.kp, sc.kd)
    eng.set_command(sc.target0)

    def oracle(i, row, cmd):
        o = OracleBatch(_flex_robot(rigid, row), sc.options, 1)
        o.set_pd_controller(sc.kp, sc.kd)
        o.set_command(cmd[i:i + 1])
        assert not o.start(sc.q0[i:i + 1], sc.v0[i:i + 1]).any()
        return o

    eng.start(sc.q0, sc.v0)
    orcs = [oracle(i, rows[i], sc.target0) for i in range(n_env)]
    np.testing.assert_array_equal(eng.get_flexibility_env(), rows)
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
            s.apply_host(eng, new, mask)
            eng.start(sc.q0, sc.v0, mask=mask)
            rows = np.where(mask.astype(bool)[:, None, None], new, rows)
            np.testing.assert_array_equal(eng.get_flexibility_env(), rows)
            for i in np.flatnonzero(mask):
                orcs[i] = oracle(i, rows[i], act)
            _compare(eng, orcs, tol_state, tol_sens)
    iq = sc.robot.idx_q[sc.robot.joint_index("LF_HFEFlexibility")]
    assert np.abs(eng.get_state()[1][:, iq:iq + 3]).max() > 1e-6


@pytest.mark.parametrize("contact_model", ["spring_damper", "constraint"])
def test_per_env_rows_match_oracle(api, contact_model):
    per_env_oracle(api, contact_model if contact_model == "constraint" else None, n_steps=3 if contact_model != "constraint" else 2)


# ---------------------------------------------------------------------------------------------- identity, latch
def _pair(api, n, seed=5, enable=(True, False)):
    sc = scenarios.make("anymal_flexible", n, seed=seed)
    out = []
    for on in enable:
        e = BatchedEngine(sc.robot, sc.options, n, api_=api)
        if on:
            e.enable_per_env_flexibility()
        e.set_pd_controller(sc.kp, sc.kd)
        e.set_command(sc.target0)
        out.append(e)
    return sc, out


def _same(a, b):
    for x, y in zip(a.get_state(), b.get_state()):
        np.testing.assert_array_equal(x, y)
    np.testing.assert_array_equal(a.get_sensors(), b.get_sensors())
    np.testing.assert_array_equal(a.get_efforts()[0], b.get_efforts()[0])


def identity(api):
    """Rows equal to the model's values: the bits of the batch without per-env rows (steps and jb_compute_dynamics)."""
    n = 4
    sc, (a, b) = _pair(api, n)
    nominal = sc.robot.flexibility[sc.robot.flexibility_joint_indices]
    np.testing.assert_array_equal(a.get_flexibility_env(), np.broadcast_to(nominal, (n, 4, 6)))
    a.set_flexibility_env(nominal)
    for e in (a, b):
        e.start(sc.q0, sc.v0)
    _same(a, b)
    for k in range(2):
        act = sc.sample_targets(k)
        for e in (a, b):
            e.set_command(act)
            e.step(sc.step_dt)
        _same(a, b)
    q, v = a.get_state()[1:3]
    for x, y in zip(a.compute_dynamics(q, v, sc.target0), b.compute_dynamics(q, v, sc.target0)):
        np.testing.assert_array_equal(x, y)


def test_identity(api):
    identity(api)


def latch(api):
    """A row written to a running env leaves its trajectory bit-unchanged until its next start, which applies it."""
    n = 4
    sc, (a, b) = _pair(api, n, seed=7, enable=(True, True))
    for e in (a, b):
        e.start(sc.q0, sc.v0)
    rows = b.get_flexibility_env()
    new = rows.copy()
    new[2, :, :3] *= 0.5
    new[2, :, 3:] += 7.0
    mask = np.array([0, 0, 1, 0], np.uint8)
    b.set_flexibility_env(new, mask=mask)
    for k in range(2):
        act = sc.sample_targets(k)
        for e in (a, b):
            e.set_command(act)
            e.step(sc.step_dt)
        _same(a, b)
        np.testing.assert_array_equal(b.get_flexibility_env(), rows)
    for e in (a, b):
        e.start(sc.q0, sc.v0, mask=mask)
    np.testing.assert_array_equal(b.get_flexibility_env(), new)
    act = sc.sample_targets(2)
    for e in (a, b):
        e.set_command(act)
        e.step(sc.step_dt)
    keep = ~mask.astype(bool)
    qa, qb = a.get_state()[1], b.get_state()[1]
    np.testing.assert_array_equal(qa[keep], qb[keep])
    assert np.abs(qa[2] - qb[2]).max() > 1e-9


def test_latch(api):
    latch(api)


# ---------------------------------------------------------------------------------------------- setters
def setters(api):
    n = 4
    sc, (a, b) = _pair(api, n, seed=9, enable=(True, True))
    s = WalkerModelRandomisation(sc.robot, 1.0)
    with pytest.raises(ValueError, match="already enabled"):
        a.enable_per_env_flexibility()
    rigid = BatchedEngine(scenarios.make("anymal", 2).robot, sc.options, 2, api_=api)
    with pytest.raises(ValueError, match="no flexibility"):
        rigid.enable_per_env_flexibility()
    with pytest.raises(core.BadControlFlow):
        rigid.set_flexibility_env(np.zeros((2, 0, 6)))
    rows0 = a.get_flexibility_env()
    good = s.draw_numpy(np.random.default_rng(1), n)
    # host form: NaN, inf and negative rows raise with the env index and write nothing
    for bad_value, env in ((np.nan, 1), (-1.0, 3), (np.inf, 2)):
        bad = good.copy()
        bad[env, 1, 4] = bad_value
        with pytest.raises(ValueError, match=f"env {env}"):
            a.set_flexibility_env(bad)
        a.start(sc.q0, sc.v0)
        np.testing.assert_array_equal(a.get_flexibility_env(), rows0)
    # a masked-out bad row is not looked at
    bad = good.copy()
    bad[0] = -1.0
    a.set_flexibility_env(bad, mask=np.array([0, 1, 1, 1], np.uint8))
    # device form: bit-equal to the host form
    g = _dev(api, good)
    b.set_flexibility_env_device(g.data_ptr())
    a.set_flexibility_env(good)
    for e in (a, b):
        e.start(sc.q0, sc.v0)
    _sync(api)
    np.testing.assert_array_equal(a.get_flexibility_env(), b.get_flexibility_env())
    np.testing.assert_array_equal(a.get_flexibility_env(), good)
    # a rejected device row flags its env BAD_START through its starts, until a valid row revives it
    bad = _dev(api, good)
    bad[1, 0, 0] = float("nan")
    bad[3, 2, 5] = -0.5
    mask = _dev(api, np.array([0, 1, 1, 1], np.uint8), torch.uint8)
    b.set_flexibility_env_device(bad.data_ptr(), mask.data_ptr())
    b.start(sc.q0, sc.v0)
    st = b.get_status()
    assert st[1] == BAD and st[3] == BAD and st[0] == 0 and st[2] == 0
    b.step(sc.step_dt)
    assert (b.get_status()[[1, 3]] == BAD).all()
    b.start(sc.q0, sc.v0, mask=np.array([0, 1, 0, 0], np.uint8))
    assert b.get_status()[1] == BAD
    fix, m1 = _dev(api, good), _dev(api, np.array([0, 1, 0, 0], np.uint8), torch.uint8)
    b.set_flexibility_env_device(fix.data_ptr(), m1.data_ptr())
    b.start(sc.q0, sc.v0, mask=np.array([0, 1, 0, 1], np.uint8))
    _sync(api)
    st = b.get_status()
    assert st[1] == 0 and st[3] == BAD
    # the host form's valid row clears the flag too
    b.set_flexibility_env(good, mask=np.array([0, 0, 0, 1], np.uint8))
    b.start(sc.q0, sc.v0)
    assert not b.get_status().any()


def test_setters(api):
    setters(api)


def reject_flags_independent(api):
    """The sensor and flexibility reject flags do not clear each other."""
    from jiminy_b200.sensor_randomisation import WalkerSensorRandomisation
    n = 2
    sc = scenarios.make("anymal_flexible", n, seed=4)
    e = BatchedEngine(sc.robot, sc.options, n, api_=api)
    e.set_pd_controller(sc.kp, sc.kd)
    e.set_command(sc.target0)
    ss = WalkerSensorRandomisation(e, 1.0)
    ss.register(e)
    e.enable_per_env_flexibility()
    srows = ss.draw_numpy(np.random.default_rng(2), n)
    frows = e.get_flexibility_env()
    t = {k: _dev(api, v) for k, v in srows.items() if k != "seed"}
    m0 = _dev(api, np.array([1, 0], np.uint8), torch.uint8)
    # env 0: bad sensor row, good flexibility row -> still refused
    t["delay"][0, 0] = -1.0
    e.set_sensor_options_env_device(t["noise_std"].data_ptr(), t["bias"].data_ptr(), t["delay"].data_ptr(), t["jitter"].data_ptr(), m0.data_ptr())
    f = _dev(api, frows)
    e.set_flexibility_env_device(f.data_ptr(), m0.data_ptr())
    e.start(sc.q0, sc.v0)
    assert e.get_status()[0] == BAD and e.get_status()[1] == 0
    # env 0: good sensor row, bad flexibility row -> still refused
    t["delay"][0, 0] = 0.0
    fb = _dev(api, frows)
    fb[0, 0, 0] = -1.0
    e.set_flexibility_env_device(fb.data_ptr(), m0.data_ptr())
    e.set_sensor_options_env_device(t["noise_std"].data_ptr(), t["bias"].data_ptr(), t["delay"].data_ptr(), t["jitter"].data_ptr(), m0.data_ptr())
    e.start(sc.q0, sc.v0)
    assert e.get_status()[0] == BAD
    e.set_flexibility_env_device(f.data_ptr(), m0.data_ptr())
    e.start(sc.q0, sc.v0)
    _sync(api)
    assert not e.get_status().any()


def test_reject_flags_independent(api):
    reject_flags_independent(api)


# ---------------------------------------------------------------------------------------------- variants, dynamics
def variants(api):
    """Per-env rows over model variants: each env against an oracle built on its group's variant, with the row's stiffness
    and damping; jb_compute_dynamics reads the active rows too."""
    sc0 = scenarios.make("anymal", 1, seed=0)
    rigid = sc0.robot
    rng = np.random.default_rng(17)
    vars_rigid = [M.biased_robot(rigid, rng, mass_std=0.05, com_std=0.01, inertia_std=0.05) for _ in range(2)]
    flex_of = lambda r, row: M.add_flexibility_joints(r, [dict(c, stiffness=list(row[k, :3]), damping=list(row[k, 3:]))
                                                          for k, c in enumerate(scenarios.FLEXIBLE_ANYMAL_CONFIG)])
    sc = scenarios.make("anymal_flexible", 16, seed=6)
    nominal = sc.robot.flexibility[sc.robot.flexibility_joint_indices]
    eng = BatchedEngine(sc.robot, sc.options, sc.n_env, api_=api)
    epg = eng.envs_per_group
    ngroups = -(-sc.n_env // epg)
    vog = np.arange(ngroups) % 2
    eng.set_model_variants([flex_of(r, nominal) for r in vars_rigid], vog)
    eng.enable_per_env_flexibility()
    np.testing.assert_array_equal(eng.get_flexibility_env(), np.broadcast_to(nominal, (sc.n_env, 4, 6)))
    s = WalkerModelRandomisation(sc.robot, 2.0)
    rows = s.draw_numpy(rng, sc.n_env)
    eng.set_flexibility_env(rows)
    eng.set_pd_controller(sc.kp, sc.kd)
    eng.set_command(sc.target0)
    eng.start(sc.q0, sc.v0)
    robots = [flex_of(vars_rigid[vog[i // epg]], rows[i]) for i in range(sc.n_env)]
    orcs = []
    for i in range(sc.n_env):
        o = OracleBatch(robots[i], sc.options, 1)
        o.set_pd_controller(sc.kp, sc.kd)
        o.set_command(sc.target0[i:i + 1])
        assert not o.start(sc.q0[i:i + 1], sc.v0[i:i + 1]).any()
        orcs.append(o)
    _compare(eng, orcs, 1e-13, 1e-11)
    act = sc.sample_targets(0)
    eng.set_command(act)
    eng.step(sc.step_dt)
    for i, o in enumerate(orcs):
        o.set_command(act[i:i + 1])
        assert not o.step(sc.step_dt).any()
    _compare(eng, orcs, 1e-9, 1e-7)
    # jb_compute_dynamics at a deformed, moving state
    q, v = eng.get_state()[1:3]
    v = v + np.random.default_rng(3).normal(size=v.shape) * 0.2
    a1, _, u1 = eng.compute_dynamics(q, v, act)
    for i, o in enumerate(orcs):
        a0, _, u0 = o.compute_dynamics(q[i:i + 1], v[i:i + 1], act[i:i + 1])
        np.testing.assert_allclose(a1[i:i + 1], a0, rtol=0, atol=1e-11 * max(1.0, np.abs(a0).max()))
        np.testing.assert_allclose(u1[i:i + 1], u0, rtol=0, atol=1e-11 * max(1.0, np.abs(u0).max()))


def test_variants_and_compute_dynamics(api):
    variants(api)


# ---------------------------------------------------------------------------------------------- device env vs host shadow
def env_shadow(api, std_ratio, pd=False, n_steps=4):
    """The device env against a host env that replays the device's rows (`model_rows`, `sensor_rows`,
    `disturbance_rows`) and restart rows through the host setters: bit-equal observations through restarts."""
    n = 5
    kw = dict(simulation_duration_max=4.1, api_=api, std_ratio=std_ratio)
    if pd:
        kw["mahony"] = (1.0, 0.1)
    dev = (DevicePDControlBatchedEnv if pd else DeviceBatchedEnv)(scenarios.make("anymal_flexible", n, seed=9), **kw)
    shadow = (envs.PDControlBatchedEnv if pd else envs.BatchedJiminyEnv)(scenarios.make("anymal_flexible", n, seed=9), **kw)
    bank_q, bank_v = (_np(x) for x in dev.reset_states)

    def replay(rows):
        msnap = _np(dev.model_rows).copy()
        shadow._redraw_model = lambda mask: shadow.model_randomisation.apply_host(shadow.engine, msnap, mask)
        if dev.sensor_randomisation is not None:
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
        np.testing.assert_array_equal(dev.engine.get_flexibility_env(), shadow.engine.get_flexibility_env())

    o_d, _ = dev.reset()
    replay(np.zeros(n, np.int64))
    o_s, _ = shadow.reset()
    same(o_d, o_s)
    np.testing.assert_array_equal(dev.engine.get_flexibility_env(), _np(dev.model_rows))
    first = _np(dev.model_rows).copy()
    rng = np.random.default_rng(11)
    for k in range(n_steps):
        act = np.zeros((n, shadow.robot.nmotors)) if pd else shadow.sc.sample_targets(k)
        o_d, _, _, _, info = dev.step(_dev(api, act))
        replay(_np(info["reset_rows"]))
        o_s, _, _, _, info_s = shadow.step(act)
        same(o_d, o_s)
        np.testing.assert_array_equal(_np(info["status"]), info_s["status"])
        if k % 2 == 0:
            mask = (rng.uniform(size=n) < 0.5).astype(np.uint8)
            mask[0] = 1
            o_d, info = dev.reset(mask=_dev(api, mask, torch.uint8))
            replay(_np(info["reset_rows"]))
            o_s, _ = shadow.reset(mask=mask)
            same(o_d, o_s)
    assert np.abs(_np(dev.model_rows)[0] - first[0]).max() > 0        # env 0 restarted with a new draw
    np.testing.assert_array_equal(dev.engine.get_flexibility_env(), _np(dev.model_rows))
    for e in (dev, shadow):
        e.close()


CASES = {"model": {"model": 1.0}, "model+sensors+disturbance": {"model": 1.0, "sensors": 1.0, "disturbance": 1.0}}


@pytest.mark.parametrize("case", ["model", "model+sensors+disturbance", "pd"])
def test_device_env_matches_shadow(api, case):
    env_shadow(api, CASES.get(case, {"model": 2.0}), pd=case == "pd")


# ---------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_gpu_sampler_statistics_torch():
    _sampler_case("torch", "cuda")


@pytest.mark.gpu
def test_gpu_sea_per_env_closed_form():
    sea_per_env(None)


@pytest.mark.gpu
@pytest.mark.parametrize("contact_model", ["spring_damper", "constraint"])
def test_gpu_per_env_rows_match_oracle(contact_model):
    per_env_oracle(None, contact_model if contact_model == "constraint" else None, n_env=8)


@pytest.mark.gpu
def test_gpu_identity():
    identity(None)


@pytest.mark.gpu
def test_gpu_latch():
    latch(None)


@pytest.mark.gpu
def test_gpu_setters():
    setters(None)


@pytest.mark.gpu
def test_gpu_reject_flags_independent():
    reject_flags_independent(None)


@pytest.mark.gpu
def test_gpu_variants_and_compute_dynamics():
    variants(None)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["model", "model+sensors+disturbance", "pd"])
def test_gpu_device_env_matches_shadow(case):
    env_shadow(None, CASES.get(case, {"model": 2.0}), pd=case == "pd")


@pytest.mark.gpu
def test_gpu_model_step_never_synchronises():
    n = 256
    env = DeviceBatchedEnv(scenarios.make("anymal_flexible", n, seed=0), simulation_duration_max=4.1, std_ratio={"model": 1.0})
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
