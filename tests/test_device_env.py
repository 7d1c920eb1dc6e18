"""Device-resident env loop: `jb_start_device` (masked restart from device buffers, input checks in the kernel),
the device `PDAdapter` (`jb_pd_adapter_device`) and the torch envs of `jiminy_b200.torch_envs`.

Every scenario is a function of `api`: the CPU suite runs it on the emulated library (device memory is host memory,
torch tensors on the CPU), the `-m gpu` variants on the H100 with `api=None`."""
import os
import types

import numpy as np
import pytest
import torch

from jiminy_b200 import core, envs, scenarios
from jiminy_b200.blocks import pd_adapter
from jiminy_b200.core import BatchedEngine
from jiminy_b200.torch_envs import DeviceBatchedEnv, DevicePDControlBatchedEnv

from emul import emul_api
import sensor_pipeline_common as spc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pd_adapter.npz")
SAFETY = dict(kp=50.0, kd=0.15, soft_position_margin=0.0, soft_velocity_max=4.0)
BAD = core.JB_ENV_NOT_STARTED | core.JB_ENV_BAD_START


@pytest.fixture(scope="module")
def api():
    return emul_api()


def _dev(api, x, dtype=torch.float64):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype, device="cpu" if api is not None else "cuda").contiguous()


def _sync(api):
    if api is None:
        torch.cuda.synchronize()


def _pd_blocks(eng, sc, mahony=True, safety=True):
    """PDController (+ MotorSafetyLimit, MahonyFilter) on `eng`, with the bounds the PD env derives; returns them."""
    ns = types.SimpleNamespace(robot=sc.robot, step_dt=sc.step_dt, engine=eng)
    envs.configure_pd_blocks(ns, sc.kp, sc.kd, 0.0, 4.0, None, SAFETY if safety else None, 1, 0.0,
                             (1.0, 0.1) if mahony else None, True)
    return ns.command_state_lower, ns.command_state_upper


def _snapshot(eng, pd=True, mahony=True):
    t, q, v, a = eng.get_state()
    sched, held = eng.get_stepper_state()
    out = dict(t=t, q=q, v=v, a=a, sensors=eng.get_sensors(), true=eng.get_sensor_data(), status=eng.get_status(),
               sched=sched, held=held)
    if pd:
        out["pd"] = eng.get_pd_controller_state()
    if mahony:
        out["mahony"] = eng.get_mahony_filter()
    return out


def _assert_same(s1, s0, envs_=slice(None)):
    for k in s0:
        np.testing.assert_array_equal(s1[k][envs_], s0[k][envs_], err_msg=k)


# ---------------------------------------------------------------------------------------------- start parity
def start_parity_anymal(api, mask):
    n = 5
    sc = scenarios.make("anymal", n, seed=3)
    engs = [BatchedEngine(sc.robot, sc.options, n, api_=api) for _ in range(2)]
    seeds = np.arange(n, dtype=np.uint32) * 7919 + 11
    for e in engs:
        _pd_blocks(e, sc)
        spc.configure(e, sc.robot)
        e.set_seeds(seeds)
        e.set_command(np.zeros((n, sc.robot.nmotors)))
    host, dev = engs
    host.start(sc.q0, sc.v0, mask=mask)
    q0, v0 = _dev(api, sc.q0), _dev(api, sc.v0)
    m = None if mask is None else _dev(api, mask, torch.uint8)
    dev.start_device(q0.data_ptr(), v0.data_ptr(), None if m is None else m.data_ptr())
    _sync(api)
    _assert_same(_snapshot(dev), _snapshot(host))
    for k in range(2):
        for e in engs:
            e.set_command(0.1 * sc.sample_targets(k))
            e.step(sc.step_dt)
        _assert_same(_snapshot(dev), _snapshot(host))
    if mask is not None:
        assert (dev.get_status()[mask == 0] == core.JB_ENV_NOT_STARTED).all()


def start_parity_atlas(api):
    n = 3
    sc = scenarios.make("atlas", n, seed=5, contact_model="constraint", solver="euler_explicit", dt_max=0.005)
    fresh = scenarios.make("atlas", n, seed=6)
    engs = [BatchedEngine(sc.robot, sc.options, n, api_=api) for _ in range(2)]
    for e in engs:
        e.set_pd_controller(sc.kp, sc.kd)
        e.set_command(sc.target0)
        e.start(sc.q0, sc.v0)
        e.step(sc.step_dt)
    host, dev = engs
    mask = np.array([1, 0, 1], dtype=np.uint8)
    host.start(fresh.q0, fresh.v0, mask=mask)
    q0, v0, m = _dev(api, fresh.q0), _dev(api, fresh.v0), _dev(api, mask, torch.uint8)
    dev.start_device(q0.data_ptr(), v0.data_ptr(), m.data_ptr())
    _sync(api)
    _assert_same(_snapshot(dev, pd=False, mahony=False), _snapshot(host, pd=False, mahony=False))
    for e in engs:
        e.step(sc.step_dt)
    _assert_same(_snapshot(dev, pd=False, mahony=False), _snapshot(host, pd=False, mahony=False))


@pytest.mark.parametrize("mask", [None, "all", "subset"])
def test_start_device_matches_start_anymal(api, mask):
    m = {None: None, "all": np.ones(5, dtype=np.uint8), "subset": np.array([1, 0, 1, 1, 0], dtype=np.uint8)}[mask]
    start_parity_anymal(api, m)


def test_start_device_matches_start_atlas_constraints(api):
    start_parity_atlas(api)


# ---------------------------------------------------------------------------------------------- validation
def device_validation(api):
    n = 5
    sc = scenarios.make("anymal", n, seed=4)
    q, v = sc.q0.copy(), sc.v0.copy()
    q[1, 9] = np.nan
    q[2, 7] = sc.robot.q_upper[7] + 1e-9
    v[3, 8] = np.nan
    engs = [BatchedEngine(sc.robot, sc.options, n, api_=api) for _ in range(2)]
    for e in engs:
        _pd_blocks(e, sc, mahony=False)
        e.set_command(np.zeros((n, sc.robot.nmotors)))
    host, dev = engs
    good = np.array([1, 0, 0, 0, 1], dtype=np.uint8)
    with pytest.raises(ValueError):
        host.start(q, v)
    with pytest.raises(ValueError):
        host.start(q, v, mask=np.array([0, 0, 1, 0, 0], dtype=np.uint8))
    host.start(q, v, mask=good)
    qd, vd = _dev(api, q), _dev(api, v)
    dev.start_device(qd.data_ptr(), vd.data_ptr())
    _sync(api)
    st = dev.get_status()
    assert st.tolist() == [0, BAD, BAD, BAD, 0]
    ok = good.astype(bool)
    _assert_same(_snapshot(dev, mahony=False), _snapshot(host, mahony=False), ok)
    t_bad = dev.get_state()[0][~ok].copy()
    for e in engs:
        e.step(sc.step_dt)
    assert dev.get_status().tolist() == [0, BAD, BAD, BAD, 0]          # skipped by the step
    np.testing.assert_array_equal(dev.get_state()[0][~ok], t_bad)
    _assert_same(_snapshot(dev, mahony=False), _snapshot(host, mahony=False), ok)
    # a later device start with good rows revives them
    fix = np.array([0, 1, 1, 1, 0], dtype=np.uint8)
    host.start(sc.q0, sc.v0, mask=fix)
    q2, v2, m2 = _dev(api, sc.q0), _dev(api, sc.v0), _dev(api, fix, torch.uint8)
    dev.start_device(q2.data_ptr(), v2.data_ptr(), m2.data_ptr())
    _sync(api)
    assert dev.get_status().tolist() == [0] * n
    _assert_same(_snapshot(dev, mahony=False), _snapshot(host, mahony=False))


def test_start_device_validates_rows_in_the_kernel(api):
    device_validation(api)


# ---------------------------------------------------------------------------------------------- adapter
def adapter_golden(api):
    """Every case of the reference's own `pd_adapter` vectors, the 6-motor vectors tiled over ANYmal's 12 motors."""
    G = np.load(GOLDEN)
    sc = scenarios.make("anymal", 1, seed=0)
    eng = BatchedEngine(sc.robot, sc.options, 1, api_=api)
    nm = sc.robot.nmotors
    tile = lambda x: np.tile(np.asarray(x), (1,) * (np.ndim(x) - 1) + (nm // 6,))
    seen = set()
    for k in range(G["order"].shape[0]):
        eng.set_pd_controller_full(np.full(nm, 100.0), np.full(nm, 0.1), tile(G["lower"][k]), tile(G["upper"][k]))
        eng.set_pd_controller_state(tile(G["state_in"][k])[None])
        eng.set_pd_adapter(int(G["order"][k]), bool(G["instantaneous"][k]), tile(G["deadband"][k]) if G["has_deadband"][k] else None)
        eng.set_command(np.full((1, nm), 7.0))
        act = _dev(api, tile(G["action"][k])[None])
        eng.pd_adapter_device(act.data_ptr(), float(G["step_dt"][k]))
        _sync(api)
        out = eng.get_efforts()[2][0]
        # dt = 0: the reference function returns without touching `out` (the golden vectors keep the caller's fill);
        # the block then holds zero target accelerations (PDAdapter.apply zeroes its buffer first), which is what is written
        want = np.zeros(nm) if float(G["step_dt"][k]) == 0.0 else tile(G["out"][k])
        np.testing.assert_allclose(out, want, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(eng.get_pd_controller_state()[0], tile(G["state_out"][k]), rtol=1e-12, atol=1e-12)
        seen.add((int(G["order"][k]), bool(G["instantaneous"][k]), bool(G["has_deadband"][k]), float(G["step_dt"][k]) == 0.0))
    assert len(seen) == 16


def adapter_random(api, rtol):
    n = 7
    sc = scenarios.make("anymal", n, seed=1)
    eng = BatchedEngine(sc.robot, sc.options, n, api_=api)
    lo, hi = _pd_blocks(eng, sc, mahony=False, safety=False)
    nm = sc.robot.nmotors
    rng = np.random.default_rng(0)
    for order in (0, 1):
        for inst in (False, True):
            for deadband in (None, rng.uniform(0.0, 0.5, nm)):
                for dt in (0.04, 0.0):
                    state = rng.uniform(-1.0, 1.0, (n, 3, nm))
                    action = rng.uniform(-2.0, 2.0, (n, nm))
                    eng.set_pd_controller_state(state)
                    eng.set_pd_adapter(order, inst, deadband)
                    act = _dev(api, action)
                    eng.pd_adapter_device(act.data_ptr(), dt)
                    _sync(api)
                    ref, ref_state = np.zeros((n, nm)), state.copy()
                    pd_adapter(action.copy(), order, ref_state, lo, hi, inst, deadband, dt, ref)
                    for got, want in ((eng.get_efforts()[2], ref), (eng.get_pd_controller_state(), ref_state)):
                        if rtol == 0.0:
                            np.testing.assert_array_equal(got, want)
                        else:
                            np.testing.assert_allclose(got, want, rtol=rtol, atol=rtol)
    with pytest.raises(ValueError):
        eng.set_pd_adapter(2)
    eng.set_pd_controller_full(None, None, None, None)
    with pytest.raises(core.BadControlFlow):
        eng.set_pd_adapter(1)
    with pytest.raises(core.BadControlFlow):
        eng.pd_adapter_device(act.data_ptr(), 0.04)


def test_pd_adapter_device_golden(api):
    adapter_golden(api)


def test_pd_adapter_device_matches_host_block(api):
    adapter_random(api, 0.0)


# ---------------------------------------------------------------------------------------------- envs
def _leaves(obs, prefix=()):
    for k, x in obs.items():
        if isinstance(x, dict):
            yield from _leaves(x, prefix + (k,))
        else:
            yield prefix + (k,), x


def _np(x):
    return x.detach().cpu().numpy()


def _assert_obs(obs_t, obs_n, rows=None):
    lt, ln = dict(_leaves(obs_t)), dict(_leaves(obs_n))
    assert lt.keys() == ln.keys()
    for k in ln:
        a, b = _np(lt[k]), np.asarray(ln[k])
        if rows is not None:
            a, b = a[rows], b[rows]
        np.testing.assert_array_equal(a, b, err_msg=str(k))


KEYS = [("states", "agent", "q"), ("measurements", "EncoderSensor"), ("measurements", "ImuSensor")]


def env_equivalence(api, pd=None, n_steps=7):
    """The torch env against the host env (bit-equal until an env's first restart) and against a shadow host env whose
    restarts use the bank rows the torch env reports (bit-equal throughout)."""
    n = 5
    kw = dict(simulation_duration_max=0.12, api_=api)

    def make(cls):
        sc = scenarios.make("anymal", n, seed=9)
        return cls(sc, **kw, **(pd or {}))
    host_cls, dev_cls = (envs.PDControlBatchedEnv, DevicePDControlBatchedEnv) if pd is not None else \
        (envs.BatchedJiminyEnv, DeviceBatchedEnv)
    host, shadow, dev = make(host_cls), make(host_cls), make(dev_cls)
    bank_q, bank_v = (_np(x) for x in dev.reset_states)
    o_d, _ = dev.reset()
    o_h, _ = host.reset()
    shadow.reset()
    _assert_obs(o_d, o_h)
    fresh = np.ones(n, dtype=bool)                      # envs not yet restarted
    rng = np.random.default_rng(2)
    restarts = 0
    for k in range(n_steps):
        if pd is None:
            act = host.sc.sample_targets(k)
        else:
            act = rng.uniform(-0.5, 0.5, (n, host.robot.nmotors)) + (host.command_state_lower[0] + host.command_state_upper[0]) / 2 * (pd.get("order", 1) == 0)
        act_t = _dev(api, act)
        o_d, r_d, te_d, tr_d, info = dev.step(act_t)
        rows = _np(info["reset_rows"])
        done = _np(info["_final_observation"])
        np.testing.assert_array_equal(rows >= 0, done)
        shadow._sample_state = lambda m, rows=rows: (bank_q[np.maximum(rows, 0)], bank_v[np.maximum(rows, 0)])
        o_s, r_s, te_s, tr_s, info_s = shadow.step(act)
        o_h, r_h, te_h, tr_h, info_h = host.step(act)
        for a, b in ((r_d, r_s), (te_d, te_s), (tr_d, tr_s), (info["status"], info_s["status"])):
            np.testing.assert_array_equal(_np(a), b)
        _assert_obs(o_d, o_s)
        _assert_obs(info["final_observation"], info_s.get("final_observation", o_s))
        for (key, a), (_, b) in zip(_leaves(info["final_observation"]), _leaves(o_d)):
            assert a.untyped_storage().data_ptr() != b.untyped_storage().data_ptr(), key
        _assert_obs(o_d, o_h, fresh & ~done)
        if fresh.any():
            _assert_obs(info["final_observation"], info_h.get("final_observation", o_h), fresh)
        restarts += int(done.sum())
        fresh &= ~done
        flat_t = envs.flatten_observation(o_d, KEYS)
        flat_n = envs.flatten_observation({"states": {"agent": {"q": _np(o_d["states"]["agent"]["q"])}},
                                           "measurements": {k: _np(x) for k, x in o_d["measurements"].items()}}, KEYS)
        np.testing.assert_array_equal(_np(flat_t), flat_n)
    assert restarts >= 2 * n                             # two restart rounds
    if pd is not None:
        keys = [("states", "pd_controller")]
        low, high = {keys[0]: host.command_state_lower[:2]}, {keys[0]: host.command_state_upper[:2]}
        np.testing.assert_array_equal(_np(envs.flatten_observation(o_d, keys, low, high)),
                                      envs.flatten_observation({"states": {"pd_controller": _np(o_d["states"]["pd_controller"])}}, keys, low, high))
    for e in (host, shadow, dev):
        e.close()


PD_VARIANTS = {"order1_mahony_safety": dict(order=1, mahony=(0.75, 0.057), safety=SAFETY, joint_velocity_limit=4.0),
               "order0_instantaneous": dict(order=0, is_instantaneous=True, training=False, joint_velocity_deadband=0.01)}


def test_device_env_matches_host_env(api):
    env_equivalence(api)


@pytest.mark.parametrize("variant", sorted(PD_VARIANTS))
def test_device_pd_env_matches_host_env(api, variant):
    env_equivalence(api, PD_VARIANTS[variant])


def test_reset_bank_is_validated(api):
    sc = scenarios.make("anymal", 2, seed=0)
    q = sc.q0.copy()
    q[0, 7] = sc.robot.q_upper[7] + 1e-6
    with pytest.raises(ValueError):
        DeviceBatchedEnv(sc, reset_states=(q, sc.v0), api_=api)


# ---------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("mask", [None, "all", "subset"])
def test_gpu_start_device_matches_start_anymal(mask):
    m = {None: None, "all": np.ones(5, dtype=np.uint8), "subset": np.array([1, 0, 1, 1, 0], dtype=np.uint8)}[mask]
    start_parity_anymal(None, m)


@pytest.mark.gpu
def test_gpu_start_device_matches_start_atlas_constraints():
    start_parity_atlas(None)


@pytest.mark.gpu
def test_gpu_start_device_validates_rows_in_the_kernel():
    device_validation(None)


@pytest.mark.gpu
def test_gpu_pd_adapter_device_golden():
    adapter_golden(None)


@pytest.mark.gpu
def test_gpu_pd_adapter_device_matches_host_block():
    adapter_random(None, 1e-14)


@pytest.mark.gpu
def test_gpu_device_env_matches_host_env():
    env_equivalence(None)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", sorted(PD_VARIANTS))
def test_gpu_device_pd_env_matches_host_env(variant):
    env_equivalence(None, PD_VARIANTS[variant])


def _rollout(sleep_s: float):
    n = 256
    sc = scenarios.make("anymal", n, seed=0)
    env = DevicePDControlBatchedEnv(sc, order=1, mahony=(0.75, 0.057), safety=SAFETY, joint_velocity_limit=4.0,
                                    simulation_duration_max=0.08)
    env.reset()
    rng = np.random.default_rng(0)
    acts = [torch.as_tensor(rng.uniform(-0.5, 0.5, (n, sc.robot.nmotors)), device="cuda") for _ in range(3)]
    torch.cuda.synchronize()
    outs, pending = [], []
    if sleep_s > 0:
        with torch.cuda.stream(env._stream):
            torch.cuda._sleep(int(sleep_s * 2e9))
    torch.cuda.set_sync_debug_mode("error")
    try:
        for a in acts:
            outs.append(env.step(a))
            pending.append(not env._stream.query())
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    env.close()
    return outs, pending


@pytest.mark.gpu
def test_gpu_step_never_synchronises():
    ref, _ = _rollout(0.0)
    got, pending = _rollout(0.5)
    assert all(pending), pending          # every step returned while the batch stream was still busy
    for (o1, r1, te1, tr1, i1), (o0, r0, te0, tr0, i0) in zip(got, ref):
        _assert_obs(o1, _to_np_tree(o0))
        for a, b in ((r1, r0), (te1, te0), (tr1, tr0), (i1["reset_rows"], i0["reset_rows"]), (i1["status"], i0["status"])):
            np.testing.assert_array_equal(_np(a), _np(b))


def _to_np_tree(obs):
    return {k: _to_np_tree(x) if isinstance(x, dict) else _np(x) for k, x in obs.items()}
