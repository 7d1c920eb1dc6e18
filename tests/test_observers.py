"""Observer blocks inside the step kernel (`jb_set_mahony_filter_full`, `jb_set_body_observer`, `jiminy_b200.observers`):
gym_jiminy's `MahonyFilter` with its full option set and its `BodyObserver`, refreshed with the filter at the (re)start
and at every sensor breakpoint, on the measured values.

The numpy restatement (tests/observer_reference.py) is pinned to the reference's own functions by
tests/golden/observer_blocks.npz (tools/make_golden_observer_blocks.py); the device is checked against the restatement,
env by env, fed with the measured IMU rows of every refresh, which a `StackObservation` of `measurements.ImuSensor` with
`skip_frames_ratio = 0` and one frame per refresh of an env-step (plus the live one) records.

Every device scenario is a function of `api`: the CPU suite runs it on the emulated library, the `-m gpu` variants on the
H100 with `api=None`."""
import math
import os

import numpy as np
import pytest

from jiminy_b200 import core, envs, observers, scenarios
from jiminy_b200.core import BatchedEngine
from jiminy_b200.observation_stack import StackObservation
from jiminy_b200.observers import BodyObserver, MahonyFilter

import observer_reference as ref
from emul import emul_api

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "observer_blocks.npz"))
RATIO = 8                                   # observer refreshes per ANYmal env-step (40 ms / 5 ms)
GRID = [(e, i, r, tc) for e in (True, False) for i in (False, True) for r in (False, True) for tc in (None, 0.0, 0.3)]
# IMU measurement options: noise and a bias that keeps the accelerometer start off the free-fall fallback
IMU_NOISE, IMU_BIAS = [0.02, 0.02, 0.02, 0.1, 0.1, 0.1], [0.01, -0.02, 0.005, 0.3, -0.2, 2.0]


@pytest.fixture(scope="module")
def api():
    return emul_api()


# ---------------------------------------------------------------------------------------------- restatement vs golden
def test_swing_from_vector_matches_the_reference():
    # (the first 21 vectors are singular: every sub-case of the branch, then v = -e_z)
    for v, q in zip(GOLD["sw_v"], GOLD["sw_q"]):
        np.testing.assert_array_equal(ref.swing_from_vector(v), q)
    assert (GOLD["sw_v"][:21, 2] < -1 + 1e-5).all()


def test_quaternion_functions_match_the_reference():
    for q, q2, v, rt, rpy, mul, app in zip(GOLD["q"], GOLD["q2"], GOLD["vec"], GOLD["rt_q"], GOLD["rpy"], GOLD["mul_rc"],
                                           GOLD["apply"]):
        np.testing.assert_array_equal(ref.remove_twist(q), rt)
        np.testing.assert_array_max_ulp(ref.quat_to_rpy(q), rpy, maxulp=4)
        np.testing.assert_array_equal(ref.quat_multiply_right_conjugate(q, q2), mul)
        np.testing.assert_array_equal(ref.quat_apply(q2, v), app)


def test_update_twist_matches_the_reference():
    for q, tw, om, tc_inv, dt, q_out, tw_out in zip(*(GOLD[k] for k in ("ut_q", "ut_twist", "ut_omega", "ut_tc_inv", "ut_dt",
                                                                          "ut_q_out", "ut_twist_out"))):
        q1, tw1 = ref.update_twist(q, float(tw), om, float(tc_inv), float(dt))
        assert tw1 == tw_out
        np.testing.assert_array_max_ulp(q1, q_out, maxulp=4)


def test_chained_refreshes_match_the_reference():
    """Filter start (either exact_init, free fall, singular swing), iterations with an early return, twist removal, the
    body observer with every twist mode and the rpy, in the reference's refresh order.  Exact operations compare exactly;
    sin / cos / atan2 may round differently in numba and numpy, which the iterations carry on at the 1e-15 level."""
    G_ = GOLD
    for c in range(len(G_["c_kp"])):
        o = ref.Observers(float(G_["c_kp"][c]), float(G_["c_ki"][c]), float(G_["c_dt"][c]), bool(G_["c_exact_init"][c]),
                          bool(G_["c_ignore_twist"][c]), float(G_["c_tc"][c]), G_["c_R_rel"][c])
        o.start()
        for j in range(G_["c_gyro"].shape[1]):
            o.refresh(G_["c_gyro"][c, j], G_["c_acc"][c, j], ref.matrix_to_quat(G_["c_R_true"][c]))
            got = (o.q, o.omega, o.bias, o.rpy, o.body_q, o.body_omega, o.body_rpy, [o.twist])
            for name, x in zip(("mq", "momega", "mbias", "mrpy", "bq", "bomega", "brpy", "twist"), got):
                want = G_["c_" + name][c, j]
                if j == 0 and name in ("mq", "momega", "mbias", "bomega"):
                    np.testing.assert_array_equal(x, want, err_msg=f"chain {c} refresh {j} {name}")
                else:
                    np.testing.assert_allclose(x, want, rtol=0, atol=1e-14, err_msg=f"chain {c} refresh {j} {name}")


# ---------------------------------------------------------------------------------------------- device vs restatement
def _imu_rel(robot):
    return robot.frames[robot.imu_frames[0]].placement.R


def _pd_env(api, sc, mahony, body=None, stack=None, **kw):
    env = envs.PDControlBatchedEnv(sc, api_=api, mahony=mahony, body_observer=body, stack=stack, joint_velocity_limit=4.0,
                                   **kw)
    env.engine.set_sensor_options("ImuSensor", 0, noise_std=IMU_NOISE, bias=IMU_BIAS)
    return env


def _actions(n, k):
    return np.random.default_rng(100 + k).uniform(-0.5, 0.5, (n, 12))


def _check(obs, refs, mahony, body, envs_, where):
    m, b = obs["features"][mahony.name], obs["features"][body.name]
    for e in envs_:
        r = refs[e]
        pairs = [(m["quat"], r.q), (m["omega"], r.omega), (obs["states"][mahony.name]["bias"], r.bias),
                 (b["quat"], r.body_q), (b["omega"], r.body_omega)]
        if mahony.compute_rpy:
            pairs.append((m["rpy"], r.rpy))
        if body.compute_rpy:
            pairs.append((b["rpy"], r.body_rpy))
        for i, (got, want) in enumerate(pairs):
            np.testing.assert_allclose(np.asarray(got)[e, :, 0], want, rtol=0, atol=1e-12, err_msg=f"{where} env {e} leaf {i}")


def device_replay(api, exact_init, ignore_twist, compute_rpy, tc, n=3, n_steps=3):
    """The device observers against the restatement fed with the measured IMU rows of every refresh, with a masked
    restart after the first step and a truncation restart after the third (info["final_observation"] holds the
    pre-restart values); a batch without the observers keeps q, v, sensors and status bit for bit, and its start
    quaternions are the exact ones the restatement starts from (exact_init, or in free fall)."""
    mahony = MahonyFilter(1.0, 0.1, exact_init=exact_init, ignore_twist=ignore_twist, compute_rpy=compute_rpy)
    body = BodyObserver(twist_time_constant=tc, compute_rpy=compute_rpy)
    kw = dict(simulation_duration_max=0.1)
    # (skip_frames_ratio = 0 freezes every refresh and keeps the live value as the latest frame: after an env-step, the
    # frames are the step's RATIO refreshes, then the last one again)
    rec = _pd_env(api, scenarios.make("anymal", n, seed=5), mahony, body,
                  StackObservation(RATIO + 1, [("measurements", "ImuSensor")], 0), **kw)
    plain = _pd_env(api, scenarios.make("anymal", n, seed=5), (1.0, 0.1), **kw)
    dt = rec.sc.options["stepper"]["sensorsUpdatePeriod"]
    refs = [ref.Observers(1.0, 0.1, dt, exact_init, ignore_twist, math.nan if tc is None else tc, _imu_rel(rec.robot))
            for _ in range(n)]

    def start(e, o_rec, o_plain):
        row = o_rec["measurements"]["ImuSensor"][e, -1, :, 0]
        refs[e].start()
        refs[e].refresh(row[:3], row[3:], o_plain["features"]["mahony_filter"][e, :, 0])

    o_rec, o_plain = rec.reset()[0], plain.reset()[0]
    for e in range(n):
        start(e, o_rec, o_plain)
    _check(o_rec, refs, mahony, body, range(n), "reset")
    for k in range(n_steps):
        act = _actions(n, k)
        o_rec, _, _, _, info = rec.step(act)
        o_plain, _, _, _, info_p = plain.step(act)
        np.testing.assert_array_equal(info["status"], info_p["status"])
        for a, b in zip(rec.engine.get_state(), plain.engine.get_state()):
            np.testing.assert_array_equal(a, b)
        np.testing.assert_array_equal(rec.engine.get_sensors(), plain.engine.get_sensors())
        done = info.get("_final_observation", np.zeros(n, dtype=bool))
        np.testing.assert_array_equal(done, info_p.get("_final_observation", np.zeros(n, dtype=bool)))
        fin = info["final_observation"] if done.any() else o_rec
        for e in range(n):
            for j in range(RATIO):
                row = fin["measurements"]["ImuSensor"][e, j, :, 0]
                refs[e].refresh(row[:3], row[3:])
        _check(fin, refs, mahony, body, range(n), f"step {k}")
        for e in np.flatnonzero(done):
            start(e, o_rec, o_plain)
        _check(o_rec, refs, mahony, body, np.flatnonzero(done), f"restart after step {k}")
        if k == 0:
            mask = np.array([0, 1, 0], dtype=np.uint8)
            o_rec, o_plain = rec.reset(mask=mask)[0], plain.reset(mask=mask)[0]
            start(1, o_rec, o_plain)
            _check(o_rec, refs, mahony, body, range(n), "masked restart")
    assert done.any()                                          # the truncation restart happened
    for env in (rec, plain):
        env.close()


@pytest.mark.parametrize("exact_init,ignore_twist,compute_rpy,tc", GRID)
def test_device_matches_the_restatement(api, exact_init, ignore_twist, compute_rpy, tc):
    device_replay(api, exact_init, ignore_twist, compute_rpy, tc)


# ---------------------------------------------------------------------------------------------- start cases
def start_cases(api, n=4):
    """In free fall (no sensor options, the robot starts in the air) exact_init=False keeps the exact start; with the
    IMU frame flipped (rotated by pi about x) and the accelerometer reading a robot upright at rest (-g along the flipped
    frame's z, with horizontal parts that pick every sub-case of the singular branch), the start is the restatement's
    singular swing."""
    sc = scenarios.make("anymal", n, seed=3)
    outs = {}
    for exact in (True, False):
        env = envs.PDControlBatchedEnv(sc, api_=api, mahony=MahonyFilter(exact_init=exact), body_observer=BodyObserver())
        outs[exact] = env.reset()[0]
        env.close()
    for key in ("mahony_filter", "body_observer"):
        np.testing.assert_array_equal(outs[False]["features"][key]["quat"], outs[True]["features"][key]["quat"])

    sc = scenarios.make("anymal", n, seed=3)
    pl = sc.robot.frames[sc.robot.imu_frames[0]].placement
    pl.R = pl.R @ np.diag([1.0, -1.0, -1.0])
    env = envs.PDControlBatchedEnv(sc, api_=api, mahony=MahonyFilter(exact_init=False, compute_rpy=True),
                                   body_observer=BodyObserver(twist_time_constant=0.3))
    eng = env.engine
    lay = eng.width
    eng.enable_per_env_sensor_options(0.0)
    bias = np.zeros((n, lay))
    io = sc.robot.sensor_layout()["ImuSensor"][0]
    g = 9.81
    # (v_x, v_y) of the measured direction: both within 1e-5; x within with a small ratio; y within with a small ratio;
    # x within with a large ratio
    hor = [(3e-6, -4e-6), (2e-9, 1e-3), (-1e-3, 3e-9), (4e-6, 2e-5)]
    for e, (vx, vy) in enumerate(hor):
        bias[e, io + 3:io + 6] = g * np.array([vx, vy, -math.sqrt(1 - vx * vx - vy * vy)])
    eng.set_sensor_options_env(np.zeros((n, lay)), bias, np.zeros((n, eng.n_sensors)), np.zeros((n, eng.n_sensors)))
    obs = env.reset()[0]
    acc = eng.get_sensors()[:, io + 3:io + 6]
    r = ref.Observers(1.0, 0.1, 0.005, False, False, 0.3, pl.R)
    for e in range(n):
        v = acc[e] / np.linalg.norm(acc[e])
        assert v[2] < -1 + 1e-5
        r.start()
        r.refresh(np.zeros(3), acc[e])
        np.testing.assert_allclose(obs["features"]["mahony_filter"]["quat"][e, :, 0], r.q, rtol=0, atol=1e-12)
        np.testing.assert_allclose(obs["features"]["mahony_filter"]["rpy"][e, :, 0], r.rpy, rtol=0, atol=1e-12)
        np.testing.assert_allclose(obs["features"]["body_observer"]["quat"][e, :, 0], r.body_q, rtol=0, atol=1e-12)
    env.close()


def test_start_cases(api):
    start_cases(api)


# ---------------------------------------------------------------------------------------------- nothing existing moves
def tuple_and_object_agree(api, n=3):
    """mahony=(kp, ki) and mahony=MahonyFilter(kp, ki): the same quaternions, bit for bit."""
    out = []
    for m in ((0.75, 0.057), MahonyFilter(0.75, [0.057])):
        env = _pd_env(api, scenarios.make("anymal", n, seed=4), m)
        seq = [env.reset()[0]]
        for k in range(2):
            seq.append(env.step(_actions(n, k))[0])
        out.append([o["features"]["mahony_filter"] for o in seq])
        env.close()
    for a, b in zip(*out):
        np.testing.assert_array_equal(a, b["quat"])


def test_tuple_and_object_agree(api):
    tuple_and_object_agree(api)


# ---------------------------------------------------------------------------------------------- hand-off parity
def _hand_off_engine(api, sc, full, monkeypatch):
    monkeypatch.setenv("JB_NO_FAST_BOUNDS", "1")        # (the quadruped signature would solve the bounds on the hot path)
    monkeypatch.setenv("JB_NO_FAST_KERNEL", "1" if full else "0")
    eng = BatchedEngine(sc.robot, sc.options, sc.n_env, api_=api)
    eng.set_pd_controller(sc.kp, sc.kd)
    eng.set_mahony_filter_full(1.0, 0.1, exact_init=False, ignore_twist=True, compute_rpy=True)
    eng.set_body_observer(True, 0.3, True)
    eng.set_sensor_options("ImuSensor", 0, noise_std=IMU_NOISE, bias=IMU_BIAS)
    eng.set_command(sc.target0)
    eng.start(sc.q0, sc.v0)
    return eng


def hand_off_parity(api, monkeypatch, n=6, n_steps=3):
    """Envs the hot-path body hands to the full body (a hip joint leaves its bounds) refresh their observers exactly once
    per refresh: the same records, twist included, as a batch stepped by the full body only."""
    sc = scenarios.make("anymal", n, seed=8, flagged_fraction=1.0 / 3.0)
    fast, full = _hand_off_engine(api, sc, False, monkeypatch), _hand_off_engine(api, sc, True, monkeypatch)
    for k in range(n_steps):
        act = sc.sample_targets(k)
        for e in (fast, full):
            e.set_command(act)
            e.step(sc.step_dt)
        np.testing.assert_array_equal(fast.get_status(), full.get_status())
        # (the two batches' dynamics agree to ~1e-10, not bit for bit; a refresh done twice would move the estimates and
        # the twist by ~1e-3)
        for get in (fast.get_sensors, fast.get_mahony_filter, fast.get_observers):
            a, b = get(), getattr(full, get.__name__)()
            np.testing.assert_allclose(a, b, rtol=0, atol=1e-7 * max(1.0, float(np.abs(b).max())))
    assert (fast.get_status()[::3] & core.JB_ENV_JOINT_LIMIT).all()      # the flagged envs went through the full body
    for e in (fast, full):
        e.close()


def test_hand_off_refreshes_once(api, monkeypatch):
    hand_off_parity(api, monkeypatch)


# ---------------------------------------------------------------------------------------------- stacking and envs
OBS_PD = dict(mahony=MahonyFilter(1.0, 0.1, exact_init=False, compute_rpy=True),
              body_observer=BodyObserver(twist_time_constant=0.3), joint_velocity_limit=4.0)


def stacked_leaves(api, n=2):
    """Every observer leaf stacks (a whole `features` subtree, and the filter's state): the latest frame is the env's
    own observation."""
    keys = [("features",), ("states", "mahony_filter")]
    env = envs.PDControlBatchedEnv(scenarios.make("anymal", n, seed=5), api_=api, stack=StackObservation(3, keys, 1), **OBS_PD)
    plain = envs.PDControlBatchedEnv(scenarios.make("anymal", n, seed=5), api_=api, **OBS_PD)
    seq = [(env.reset()[0], plain.reset()[0])]
    for k in range(2):
        seq.append((env.step(_actions(n, k))[0], plain.step(_actions(n, k))[0]))
    for o, p in seq:
        for blk in ("mahony_filter", "body_observer"):
            assert set(o["features"][blk]) == {"quat", "rpy", "omega"}
            for leaf, x in o["features"][blk].items():
                assert x.shape == (n, 3) + p["features"][blk][leaf].shape[1:]
                np.testing.assert_array_equal(x[:, -1], p["features"][blk][leaf])
        np.testing.assert_array_equal(o["states"]["mahony_filter"]["bias"][:, -1], p["states"]["mahony_filter"]["bias"])
    for e in (env, plain):
        e.close()


def test_stacked_leaves(api):
    stacked_leaves(api)


def test_device_env_matches_host_env(api):
    from test_device_env import env_equivalence
    env_equivalence(api, dict(OBS_PD, order=1, stack=StackObservation(4, [("features",)], 3)))


# ---------------------------------------------------------------------------------------------- refusals and config
def refusals(api):
    sc = scenarios.make("anymal", 2, seed=0)
    eng = BatchedEngine(sc.robot, sc.options, 2, api_=api)
    with pytest.raises(ValueError):                       # no Mahony filter
        eng.set_body_observer(True, None, True)
    eng.set_mahony_filter_full(1.0, 0.1)
    for tc in (-0.1, math.inf):
        with pytest.raises(ValueError):
            eng.set_body_observer(True, tc, True)
    with pytest.raises(core.BadControlFlow):              # the default path keeps no observer record
        eng.get_observers()
    for leaf in (core.STACK_MAHONY_RPY, core.STACK_BODY_QUAT, core.STACK_BODY_RPY, core.STACK_BODY_OMEGA):
        with pytest.raises(ValueError):
            eng.set_obs_stack(2, 0, [leaf])
    eng.set_body_observer(True, 0.0, False)
    with pytest.raises(ValueError):                       # body rpy off
        eng.set_obs_stack(2, 0, [core.STACK_BODY_RPY])
    eng.set_pd_controller(sc.kp, sc.kd)
    eng.set_command(sc.target0)
    eng.start(sc.q0, sc.v0)
    for args in ((True, 0.3, True), (False,)):
        with pytest.raises(core.BadControlFlow):
            eng.set_body_observer(*args)
    assert eng.get_observers().shape == (2, 1, core.OBSV_N)
    eng.stop()
    eng.set_mahony_filter_full(None)                      # the filter off turns the body observer off
    assert eng.device_observer_views() == 0
    with pytest.raises(core.BadControlFlow):
        eng.get_observers()
    eng.close()


def test_refusals(api):
    refusals(api)


def test_python_refusals(api):
    sc = scenarios.make("anymal", 2, seed=0)
    with pytest.raises(ValueError):                       # body observer without the object form of the filter
        envs.PDControlBatchedEnv(sc, api_=api, mahony=(1.0, 0.1), body_observer=BodyObserver())
    for bad in (dict(update_ratio=2), dict(kp=[1.0, 2.0])):
        with pytest.raises(NotImplementedError):
            MahonyFilter(**bad)
    for bad in (dict(update_ratio=-1), dict(nested_imu_quat_key=("features", "other", "quat"))):
        with pytest.raises(NotImplementedError):
            BodyObserver(**bad)
    with pytest.raises(ValueError):
        BodyObserver(twist_time_constant=-1.0)
    for cls in ("DeformationEstimator", "QuantityObserver"):
        with pytest.raises(NotImplementedError):
            observers.from_config([{"block": {"cls": f"gym_jiminy.common.blocks.{cls}"}}])
    with pytest.raises(NotImplementedError):
        observers.from_config([{"block": {"cls": "gym_jiminy.common.blocks.MahonyFilter", "kwargs": {"update_ratio": 2}}}])


def test_from_config(api):
    from test_observation_stack import ANYMAL_PIPELINE_LAYERS
    found = observers.from_config(ANYMAL_PIPELINE_LAYERS)
    assert found == [MahonyFilter(exact_init=False, kp=1.0, ki=0.1)]
    body = observers.from_config([{"block": {"cls": "gym_jiminy.common.blocks.BodyObserver",
                                             "kwargs": {"twist_time_constant": 0.0, "compute_rpy": False}}}])
    assert body == [BodyObserver(twist_time_constant=0.0, compute_rpy=False)]
    env = _pd_env(api, scenarios.make("anymal", 2, seed=0), found[0])
    obs = env.reset()[0]
    obs = env.step(_actions(2, 0))[0]
    assert obs["features"]["mahony_filter"]["quat"].shape == (2, 4, 1)
    assert obs["states"]["mahony_filter"]["bias"].shape == (2, 3, 1)
    env.close()


# ---------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("exact_init,ignore_twist,compute_rpy,tc", GRID)
def test_gpu_device_matches_the_restatement(exact_init, ignore_twist, compute_rpy, tc):
    device_replay(None, exact_init, ignore_twist, compute_rpy, tc)


@pytest.mark.gpu
def test_gpu_start_cases():
    start_cases(None)


@pytest.mark.gpu
def test_gpu_tuple_and_object_agree():
    tuple_and_object_agree(None)


@pytest.mark.gpu
def test_gpu_hand_off_refreshes_once(monkeypatch):
    hand_off_parity(None, monkeypatch)


@pytest.mark.gpu
def test_gpu_stacked_leaves():
    stacked_leaves(None)


@pytest.mark.gpu
def test_gpu_device_env_matches_host_env():
    from test_device_env import env_equivalence
    env_equivalence(None, dict(OBS_PD, order=1, stack=StackObservation(4, [("features",)], 3)))


@pytest.mark.gpu
def test_gpu_refusals():
    refusals(None)
