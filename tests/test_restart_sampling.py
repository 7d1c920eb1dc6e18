"""Fresh restart states on the device: `jb_start_device_on_ground` (the host rule `robots.ground_base_height` inside the
masked start), the torch draw of the scenario's initial-state distribution (`Scenario.draw_initial_torch`) and the device
envs' `reset_states="sample"`.

Every kernel scenario is a function of `api`: the CPU suite runs it on the emulated library (device memory is host
memory, torch tensors on the CPU), the `-m gpu` variants on the device with `api=None`."""
import numpy as np
import pytest
import torch

from jiminy_b200 import core, envs, robots, scenarios
from jiminy_b200 import model as M
from jiminy_b200.core import BatchedEngine
from jiminy_b200.torch_envs import DeviceBatchedEnv, DevicePDControlBatchedEnv

from emul import emul_api

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


def _draw(sc, n, seed, lift=0.2):
    """Rows of the scenario's distribution (torch draw on the CPU), base raised or lowered by U(-lift, lift)."""
    gen = torch.Generator()
    gen.manual_seed(seed)
    q, v = (_np(x).copy() for x in sc.draw_initial_torch(gen, n, "cpu"))
    q[:, 2] += np.random.default_rng(seed).uniform(-lift, lift, n)
    return q, v


def _contact_z(robot, q):
    pl = robots.frame_placements(robot, q, robot.contact_frame_names)
    return np.array([pl[name].p[2] for name in robot.contact_frame_names])


def _start(eng, api, q, v, mask=None, on_ground=False):
    qd, vd = _dev(api, q), _dev(api, v)
    md = None if mask is None else _dev(api, mask, torch.uint8)
    eng.start_device(qd.data_ptr(), vd.data_ptr(), None if md is None else md.data_ptr(), on_ground=on_ground)
    _sync(api)
    return qd


def _snapshot(eng):
    return [np.array(x, copy=True) for x in (*eng.get_state(), eng.get_sensors(), eng.get_status(), *eng.get_extra_terms())]


# ---------------------------------------------------------------------------------------------- placement
def _with_belly(sc):
    """A contact frame on the floating base next to the feet, 3 mm above the ground in the scenario's posture: for some
    rows a foot stays lowest, for others the belly frame."""
    rob = sc.robot
    base = [name for name, f in rob.frames.items() if f.joint == 1 and f.kind == "body"][0]
    z0 = float(np.median(sc.q0[:, 2]))
    rob.add_frame("belly_contact", base, M.SE3(np.eye(3), np.array([0.05, 0.02, -(z0 - 0.003)])))
    rob.add_contact_points(["belly_contact"])
    return sc


def placement(api, case):
    """`q[2]` after the grounded start against `ground_base_height` of the env's own model (1e-14 m), every other
    coordinate bit-equal to the input row, masked-out envs untouched."""
    name = "anymal" if case in ("variants", "belly") else case
    n = 26
    sc = scenarios.make(name, n, seed=5)
    if case == "belly":
        sc = _with_belly(sc)
    eng = BatchedEngine(sc.robot, sc.options, n, api_=api)
    models = [sc.robot] * n
    if case == "variants":
        rng = np.random.default_rng(12)
        variants = [M.biased_robot(sc.robot, rng, relative_position_std=0.01) for _ in range(2)]
        vog = np.arange(-(-n // eng.envs_per_group), dtype=np.int32) % 2
        eng.set_model_variants(variants, vog)
        models = [variants[vog[e // eng.envs_per_group]] for e in range(n)]
    eng.start(sc.q0, sc.v0)
    before = _snapshot(eng)
    q, v = _draw(sc, n, seed=3)
    mask = (np.random.default_rng(4).uniform(size=n) < 0.7).astype(np.uint8)
    mask[:2] = (1, 0)
    qd = _start(eng, api, q, v, mask, on_ground=True)
    np.testing.assert_array_equal(_np(qd), q)                 # the caller's rows are not written
    after = _snapshot(eng)
    t, q1 = after[0], after[1]
    expect = np.array([robots.ground_base_height(models[e], q[e])[2] for e in range(n)])
    lowest = np.array([np.argmin(_contact_z(models[e], robots.ground_base_height(models[e], q[e]))) for e in range(n)])
    on = mask.astype(bool)
    assert (after[5][on] & BAD == 0).all()
    np.testing.assert_allclose(q1[on, 2], expect[on], rtol=0, atol=1e-14)
    np.testing.assert_array_equal(np.delete(q1[on], 2, axis=1), np.delete(q[on], 2, axis=1))
    np.testing.assert_array_equal(t[on], 0.0)
    for a, b in zip(before, after):
        np.testing.assert_array_equal(a[~on], b[~on])
    if case == "variants":
        # the groups' joint translations differ, and so does the height each puts the same row at
        same = np.array([robots.ground_base_height(sc.robot, q[e])[2] for e in range(n)])
        assert np.abs(expect - same).max() > 1e-4
    # the lowest frame is not the same one for every env (several lanes; the belly is a trunk frame)
    assert len(set(lowest[on].tolist())) >= 2, lowest
    if case == "belly":
        belly = sc.robot.contact_frame_names.index("belly_contact")
        assert (lowest[on] == belly).any() and (lowest[on] != belly).any(), lowest
    eng.close()


PLACEMENT_CASES = ["anymal", "atlas", "anymal_flexible", "variants", "belly"]


@pytest.mark.parametrize("case", PLACEMENT_CASES)
def test_placement_matches_host_rule(api, case):
    placement(api, case)


def only_q2(api, name):
    """A grounded start is bit-equal to a plain `jb_start_device` from the configuration it placed."""
    n = 9
    sc = scenarios.make(name, n, seed=2)
    q, v = _draw(sc, n, seed=8)
    v = v + np.random.default_rng(1).uniform(-0.1, 0.1, v.shape)
    a, b = (BatchedEngine(sc.robot, sc.options, n, api_=api) for _ in range(2))
    for e in (a, b):
        e.set_command(np.zeros((n, max(sc.robot.nmotors, 1))))
    _start(a, api, q, v, on_ground=True)
    placed = a.get_state()[1].copy()
    assert np.abs(placed[:, 2] - q[:, 2]).max() > 1e-3
    _start(b, api, placed, v)
    for x, y in zip(_snapshot(a), _snapshot(b)):
        np.testing.assert_array_equal(x, y)
    for e in (a, b):
        e.close()


@pytest.mark.parametrize("name", ["anymal", "anymal_flexible"])
def test_placement_only_moves_base_height(api, name):
    only_q2(api, name)


def bad_rows(api):
    """A NaN row and an out-of-bounds joint leave their env NOT_STARTED | BAD_START; a later valid start clears them."""
    n = 6
    sc = scenarios.make("anymal", n, seed=1)
    eng = BatchedEngine(sc.robot, sc.options, n, api_=api)
    q, v = _draw(sc, n, seed=2)
    q[1, 9] = np.nan
    q[3, 8] = sc.robot.q_upper[8] + 1e-3
    v[4, 7] = np.nan
    _start(eng, api, q, v, on_ground=True)
    st = eng.get_status()
    np.testing.assert_array_equal(st[[1, 3, 4]], BAD)
    np.testing.assert_array_equal(st[[0, 2, 5]], 0)
    q, v = _draw(sc, n, seed=3)
    _start(eng, api, q, v, np.array([0, 1, 0, 1, 1, 0], np.uint8), on_ground=True)
    np.testing.assert_array_equal(eng.get_status(), 0)
    eng.close()


def test_bad_rows(api):
    bad_rows(api)


def no_free_flyer(api):
    """Cartpole: no free-flyer, so the grounded start is `jb_start_device`."""
    n = 7
    sc = scenarios.make("cartpole", n, seed=3)
    gen = torch.Generator()
    gen.manual_seed(5)
    q, v = (_np(x).copy() for x in sc.draw_initial_torch(gen, n, "cpu"))
    mask = np.array([1, 1, 0, 1, 0, 1, 1], np.uint8)
    a, b = (BatchedEngine(sc.robot, sc.options, n, api_=api) for _ in range(2))
    for e in (a, b):
        e.start(sc.q0, sc.v0)
    _start(a, api, q, v, mask, on_ground=True)
    _start(b, api, q, v, mask)
    for x, y in zip(_snapshot(a), _snapshot(b)):
        np.testing.assert_array_equal(x, y)
    for e in (a, b):
        e.close()


def test_no_free_flyer(api):
    no_free_flyer(api)


# ---------------------------------------------------------------------------------------------- sampler
def sampler_statistics(name, device):
    """The torch draw against the numpy draw of `scenarios.make` (before the ground placement) over 2^15 rows."""
    n = 2 ** 15
    sc = scenarios.make(name, 1, seed=0)
    gen = torch.Generator(device=device)
    gen.manual_seed(6)
    q, v = (_np(x) for x in sc.draw_initial_torch(gen, n, device))
    assert q.shape == (n, sc.robot.nq) and v.shape == (n, sc.robot.nv)
    np.testing.assert_array_equal(v, 0.0)
    rigid = sc.rigid_robot if sc.rigid_robot is not None else sc.robot
    if sc.rigid_robot is not None:
        # the flexibility joints at the identity quaternion, every other coordinate the rigid draw's
        qr = np.empty((n, rigid.nq))
        for j in range(1, rigid.njoints):
            k, t = sc.robot.joint_index(rigid.joint_names[j]), int(rigid.joint_type[j])
            qr[:, rigid.idx_q[j]:rigid.idx_q[j] + M.JOINT_NQ[t]] = q[:, sc.robot.idx_q[k]:sc.robot.idx_q[k] + M.JOINT_NQ[t]]
        np.testing.assert_array_equal(M.extended_state_from_theoretical(sc.robot, rigid, qr), q)
        flex = [j for j in range(1, sc.robot.njoints) if sc.robot.joint_type[j] == M.JB_JOINT_SPHERICAL]
        assert len(flex) == 4
        for j in flex:
            np.testing.assert_array_equal(q[:, sc.robot.idx_q[j]:sc.robot.idx_q[j] + 4], [[0.0, 0.0, 0.0, 1.0]] * n)
        q = qr
    base = "anymal" if name == "anymal_flexible" else name
    qs = scenarios.standing_start(base, rigid)
    np.testing.assert_array_equal(q[:, :7], np.tile(qs[:7], (n, 1)))       # base x, y, z and quaternion of the posture
    # the numpy draw of `make`, same size
    w, lo, hi = scenarios.JOINT_PERTURBATION, rigid.q_lower[7:], rigid.q_upper[7:]
    ref = np.clip(qs[7:] + np.random.default_rng(9).uniform(-w, w, (n, rigid.nq - 7)), lo, hi)
    for x in (q[:, 7:], ref):
        assert (x >= lo).all() and (x <= hi).all() and (np.abs(x - qs[7:]) <= w + 1e-15).all()
    d, dr = q[:, 7:] - qs[7:], ref - qs[7:]
    np.testing.assert_allclose(d.min(0), dr.min(0), rtol=0, atol=2e-3 * w)
    np.testing.assert_allclose(d.max(0), dr.max(0), rtol=0, atol=2e-3 * w)
    sd = np.sqrt(dr.var(0) / n) + 1e-12
    assert (np.abs(d.mean(0) - dr.mean(0)) <= 6 * np.sqrt(2) * sd).all()
    assert (np.abs(d.var(0) - dr.var(0)) <= 6 * np.sqrt(2 * 4 * w ** 4 / 45 / n) + 1e-15).all()
    for edge in (lo, hi):                                                    # mass clipped at the bounds
        p, pr = (x == edge).mean(0), (ref == edge).mean(0)
        assert (np.abs(p - pr) <= 6 * np.sqrt(2 * np.maximum(pr, 1.0 / n) / n)).all()


@pytest.mark.parametrize("name", ["anymal", "atlas", "anymal_flexible"])
def test_sampler_statistics(name):
    sampler_statistics(name, "cpu")


def test_sampler_small_scenarios():
    gen = torch.Generator()
    gen.manual_seed(1)
    n = 2 ** 15
    q, v = (_np(x) for x in scenarios.make("cartpole", 1).draw_initial_torch(gen, n, "cpu"))
    x = np.stack([q[:, 0], np.arctan2(q[:, 2], q[:, 1]), v[:, 0], v[:, 1]], axis=1)
    w = scenarios.CARTPOLE_HALF_WIDTH
    np.testing.assert_allclose(q[:, 1] ** 2 + q[:, 2] ** 2, 1.0, rtol=0, atol=1e-15)
    assert (np.abs(x) <= w + 1e-15).all()
    assert (np.abs(x.mean(0)) <= 6 * np.sqrt(w ** 2 / 3 / n)).all()
    assert (np.abs(x.var(0) - w ** 2 / 3) <= 6 * np.sqrt(4 * w ** 4 / 45 / n)).all()
    q, v = (_np(x) for x in scenarios.make("double_pendulum", 1).draw_initial_torch(gen, 3, "cpu"))
    np.testing.assert_array_equal(q, scenarios.make("double_pendulum", 3).q0)
    np.testing.assert_array_equal(v, 0.0)


# ---------------------------------------------------------------------------------------------- device env vs shadow
def env_shadow(api, std_ratio, pd=False, n_steps=8):
    """The device env with sampled restarts against a host env whose restarts use the states the device env placed
    (read from its post-restart observation, v = 0) and the device's randomisation rows: bit-equal throughout.  Every
    restarted env stands on its lowest contact frame, its joints within the posture +- the perturbation."""
    n = 5
    kw = dict(simulation_duration_max=0.12, api_=api, std_ratio=std_ratio)
    if pd:
        kw["mahony"] = (1.0, 0.1)
    dev = (DevicePDControlBatchedEnv if pd else DeviceBatchedEnv)(scenarios.make("anymal_flexible", n, seed=9),
                                                                  reset_states="sample", **kw)
    shadow = (envs.PDControlBatchedEnv if pd else envs.BatchedJiminyEnv)(scenarios.make("anymal_flexible", n, seed=9), **kw)
    robot, rigid = dev.robot, dev.sc.rigid_robot
    qs = M.extended_state_from_theoretical(robot, rigid, scenarios.standing_start("anymal", rigid))
    joints = np.array([i for j in range(1, robot.njoints) if robot.joint_type[j] not in (M.JB_JOINT_SPHERICAL, M.JB_JOINT_FREEFLYER)
                       for i in range(robot.idx_q[j], robot.idx_q[j] + M.JOINT_NQ[int(robot.joint_type[j])])])
    assert dev.reset_states is None

    def replay(q_placed):
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
        shadow._sample_state = lambda m: (q_placed, np.zeros((n, robot.nv)))

    def same(o_d, o_s):
        np.testing.assert_array_equal(_np(o_d["states"]["agent"]["q"]), o_s["states"]["agent"]["q"])
        np.testing.assert_array_equal(_np(o_d["states"]["agent"]["v"]), o_s["states"]["agent"]["v"])
        for name, x in o_s["measurements"].items():
            np.testing.assert_array_equal(_np(o_d["measurements"][name]), x)
        if pd:
            np.testing.assert_array_equal(_np(o_d["states"]["pd_controller"]), o_s["states"]["pd_controller"])

    def grounded(q, rows):
        for e in np.flatnonzero(rows):
            assert abs(_contact_z(robot, q[e]).min()) <= 1e-12
            assert (np.abs(q[e, joints] - qs[joints]) <= scenarios.JOINT_PERTURBATION + 1e-12).all()
            assert (q[e, joints] >= robot.q_lower[joints]).all() and (q[e, joints] <= robot.q_upper[joints]).all()

    o_d, _ = dev.reset()
    replay(None)
    o_s, _ = shadow.reset()
    same(o_d, o_s)
    restarts = 0
    rng = np.random.default_rng(11)
    for k in range(n_steps):
        act = np.zeros((n, shadow.robot.nmotors)) if pd else shadow.sc.sample_targets(k)
        o_d, r_d, te_d, tr_d, info = dev.step(_dev(api, act))
        assert "reset_rows" not in info
        done = _np(info["_final_observation"])
        q_placed = _np(o_d["states"]["agent"]["q"]).copy()
        replay(q_placed)
        o_s, r_s, te_s, tr_s, info_s = shadow.step(act)
        same(o_d, o_s)
        same(info["final_observation"], info_s.get("final_observation", o_s))
        for a, b in ((r_d, r_s), (te_d, te_s), (tr_d, tr_s), (info["status"], info_s["status"])):
            np.testing.assert_array_equal(_np(a), b)
        grounded(q_placed, done)
        np.testing.assert_array_equal(_np(o_d["states"]["agent"]["v"])[done], 0.0)
        restarts += int(done.sum())
        if k == 3:
            mask = (rng.uniform(size=n) < 0.5).astype(np.uint8)
            mask[0] = 1
            o_d, info = dev.reset(mask=_dev(api, mask, torch.uint8))
            assert "reset_rows" not in info
            q_placed = _np(o_d["states"]["agent"]["q"]).copy()
            replay(q_placed)
            o_s, _ = shadow.reset(mask=mask)
            same(o_d, o_s)
            grounded(q_placed, mask.astype(bool))
    assert restarts >= 2 * n                             # two rounds of restarts
    for e in (dev, shadow):
        e.close()


SHADOW_CASES = {"plain": (None, False), "pd": (None, True),
                "randomised": ({"disturbance": 1.0, "sensors": 1.0, "model": 1.0}, False),
                "pd_randomised": ({"disturbance": 1.0, "sensors": 1.0, "model": 1.0}, True)}


@pytest.mark.parametrize("case", list(SHADOW_CASES))
def test_device_env_matches_shadow(api, case):
    env_shadow(api, *SHADOW_CASES[case])


def test_reset_states_rejects_unknown_mode(api):
    with pytest.raises(ValueError):
        DeviceBatchedEnv(scenarios.make("anymal", 2, seed=0), reset_states="fresh", api_=api)


# ---------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("case", PLACEMENT_CASES)
def test_gpu_placement_matches_host_rule(case):
    placement(None, case)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["anymal", "anymal_flexible"])
def test_gpu_placement_only_moves_base_height(name):
    only_q2(None, name)


@pytest.mark.gpu
def test_gpu_bad_rows():
    bad_rows(None)


@pytest.mark.gpu
def test_gpu_no_free_flyer():
    no_free_flyer(None)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["anymal", "atlas", "anymal_flexible"])
def test_gpu_sampler_statistics(name):
    sampler_statistics(name, "cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(SHADOW_CASES))
def test_gpu_device_env_matches_shadow(case):
    env_shadow(None, *SHADOW_CASES[case])


@pytest.mark.gpu
@pytest.mark.parametrize("pd", [False, True])
def test_gpu_sampled_restart_step_never_synchronises(pd):
    n = 256
    sc = scenarios.make("anymal_flexible", n, seed=0)
    env = (DevicePDControlBatchedEnv if pd else DeviceBatchedEnv)(sc, reset_states="sample", simulation_duration_max=0.08)
    env.reset()
    acts = [torch.as_tensor(np.zeros((n, sc.robot.nmotors)) if pd else sc.sample_targets(k), device="cuda") for k in range(4)]
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
