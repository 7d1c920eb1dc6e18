"""Observation stacking inside the step kernel (`jb_set_obs_stack`, `jiminy_b200.observation_stack`): gym_jiminy's
`StackObservation` wrapper (wrappers/observation_stack.py) updated at every observer refresh of every env.

Refresh schedule pinned here.  The reference's observer refreshes once in `reset` (generic.py:702-706; during
`simulator.start` it returns early because no simulation runs yet, bases/interfaces.py:300-302), then at every controller
breakpoint inside a step and once at the end of the step (generic.py:834-838); the next step's first breakpoint is the same
time and is not refreshed again (`__is_observation_refreshed`, interfaces.py:323-329, :361-372).  With
observe_dt = control_dt = 5 ms and 40 ms env-steps that is t = 0 at a (re)start, then 8 refreshes per env-step at
t = 5, 10, ..., 40 ms, the last one at the env's end time.  The kernel refreshes at the start and at every sensor
breakpoint, which is that schedule.

Every scenario is a function of `api`: the CPU suite runs it on the emulated library, the `-m gpu` variants on the H100
with `api=None`."""
from collections import deque

import numpy as np
import pytest

from jiminy_b200 import core, envs, observation_stack, scenarios
from jiminy_b200.core import BatchedEngine
from jiminy_b200.observation_stack import StackObservation

from emul import emul_api

PD = dict(mahony=(1.0, 0.1), augment_observation=True, joint_velocity_limit=4.0)
ALL_KEYS = [("t",), ("measurements",), ("actions",), ("states", "pd_controller"), ("features",)]
CONFIGS = [(3, 2), (4, 3), (2, -1), (1, 0)]
# (env_equivalence normalises the unstacked `states.pd_controller` by its bounds at the end)
DEVICE_KEYS = [("t",), ("measurements",), ("actions",), ("features",)]


@pytest.fixture(scope="module")
def api():
    return emul_api()


def _leaf(obs, path):
    for k in path:
        obs = obs[k]
    return np.asarray(obs)


def _is_breakpoint(t, dt, eps=1e-6):
    """gym_jiminy.common.utils.is_breakpoint (utils/misc.py:37-49)."""
    if dt < eps:
        return True
    r = float(t) % dt
    return r < eps or dt - r <= eps


class RefStack:
    """Deque-based restatement of StackObservation._setup / refresh_observation (observation_stack.py:207-254) for one
    leaf of one env: the deque holds references to the live leaf, frozen copies and the initial zero frames."""

    def __init__(self, num_stack, skip, shape, step_dt):
        self.skip, self.step_dt = skip, step_dt
        self.live = np.zeros(shape)
        self.frames = deque([np.zeros(shape) for _ in range(num_stack)], maxlen=num_stack)
        self.obs = np.zeros((num_stack,) + tuple(shape))
        self.n = skip - 1

    def refresh(self, value, t):
        np.copyto(self.live, value)
        self.n += 1
        update = _is_breakpoint(t, self.step_dt) if self.skip < 0 else self.n == self.skip
        shift = self.n == 0
        if update:
            self.frames[-1] = self.live.copy()
        if shift:
            self.frames.append(self.live)
            np.copyto(self.obs, np.stack(tuple(self.frames)))
        else:
            self.obs[-1, ...] = self.live
        if update:
            self.n = -1


def _pd_env(api, n, stack=None, **kw):
    sc = scenarios.make("anymal", n, seed=5)
    return envs.PDControlBatchedEnv(sc, api_=api, stack=stack, **{**PD, **kw})


def _actions(env, k):
    rng = np.random.default_rng(100 + k)
    return rng.uniform(-0.5, 0.5, (env.n_env, env.robot.nmotors))


# ---------------------------------------------------------------------------------------------- reference replay
def reference_replay(api, n=3, n_steps=3):
    """Every (num_stack, skip) configuration against the deque restatement fed with the refreshes a twin batch records
    (skip_frames_ratio = 0 keeps every refresh: after refresh k the frames end with v[k-1], v[k], v[k]), envs restarted
    mid-rollout included; the stack leaves q, v, sensors and status bit-unchanged; a masked restart re-initialises the
    restarted envs' stacks and leaves the others' bits alone."""
    ratio = 8
    rec_num = ratio * n_steps + 2
    rec = _pd_env(api, n, StackObservation(rec_num, ALL_KEYS, 0))
    plain = _pd_env(api, n)
    cfg = {c: _pd_env(api, n, StackObservation(c[0], ALL_KEYS, c[1])) for c in CONFIGS}
    every = [rec, plain] + list(cfg.values())
    obs = [e.reset()[0] for e in every]
    since = np.zeros(n, dtype=int)                       # env-steps since the env's last (re)start
    paths = [p for p, _ in rec.stack.resolve(rec._obs_shapes())]
    restart = np.array([0, 1, 0], dtype=np.uint8)
    for k in range(n_steps + 1):
        o_rec, o_plain = obs[0], obs[1]
        # the latest recorded frame is the observation the env returns
        for p in paths:
            np.testing.assert_array_equal(_leaf(o_rec, p)[:, -1], _leaf(o_plain, p), err_msg=str(p))
        for o in obs[2:]:
            for p in (("states", "agent", "q"), ("states", "agent", "v")):
                np.testing.assert_array_equal(_leaf(o, p), _leaf(o_plain, p), err_msg=str(p))
        for (num, skip), o in zip(cfg, obs[2:]):
            for e in range(n):
                r = 1 + ratio * since[e]
                t_seq = _leaf(o_rec, ("t",))[e, rec_num - 1 - r:rec_num - 1]
                for p in paths:
                    seq = _leaf(o_rec, p)[e, rec_num - 1 - r:rec_num - 1]
                    ref = RefStack(num, skip, seq.shape[1:], rec.step_dt)
                    for v, t in zip(seq, t_seq):
                        ref.refresh(v, t)
                    np.testing.assert_array_equal(_leaf(o, p)[e], ref.obs, err_msg=f"{(num, skip)} {p} env {e} step {k}")
        if k == n_steps:
            break
        statuses = []
        for i, env in enumerate(every):
            obs[i], _, _, _, info = env.step(_actions(env, k))
            statuses.append(info["status"])
        for env, st in zip(every, statuses):
            np.testing.assert_array_equal(st, statuses[1])
            np.testing.assert_array_equal(env.engine.get_sensors(), plain.engine.get_sensors())
        since += 1
        if k == 0:
            before = {c: env.engine.get_obs_stack() for c, env in cfg.items()}
            for i, env in enumerate(every):
                obs[i], _ = env.reset(mask=restart)
            since[restart.astype(bool)] = 0
            for c, env in cfg.items():
                after = env.engine.get_obs_stack()
                np.testing.assert_array_equal(after[restart == 0], before[c][restart == 0])
                np.testing.assert_array_equal(after[restart == 1][:, :-1], 0.0)
    for env in every:
        env.close()


def test_replay_matches_the_reference_wrapper(api):
    reference_replay(api)


# ---------------------------------------------------------------------------------------------- recording check
def recording_matches_fine_steps(api, n=2, n_steps=2):
    """The recorded frames against a twin batch stepped at step_dt = observe_dt with the same command, observed after
    every one of its steps: the same refreshes, within 1e-12 relative (the two only round their times differently)."""
    ratio = 8
    rec_num = ratio * n_steps + 2
    rec = _pd_env(api, n, StackObservation(rec_num, ALL_KEYS, 0))
    fine = _pd_env(api, n)
    rec.reset()
    seq = [fine.reset()[0]]
    dt = rec.step_dt / ratio
    for k in range(n_steps):
        o_rec = rec.step(_actions(rec, k))[0]
        fine.engine.set_command(rec.engine.get_efforts()[2])
        for _ in range(ratio):
            fine.engine.step(dt)
            seq.append(fine._observation())
    paths = [p for p, _ in rec.stack.resolve(rec._obs_shapes())]
    for p in paths:
        got = _leaf(o_rec, p)[:, :-1]
        want = np.stack([_leaf(o, p) for o in seq], axis=1)
        scale = max(1.0, float(np.abs(want).max()))
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12 * scale, err_msg=str(p))
    for env in (rec, fine):
        env.close()


def test_recording_matches_fine_steps(api):
    recording_matches_fine_steps(api)


# ---------------------------------------------------------------------------------------------- reference unit tests
def reference_unit_tests(api, n=2):
    """test_initial_state and test_stacked_obs (unit_py/test_pipeline_design.py:141-230) on the reference pipeline's
    stacked leaves."""
    keys = [("t",), ("measurements", "ImuSensor"), ("actions",)]
    obs_dt = 0.005
    for num_stack, skip in ((4, 3), (3, 2)):
        env = _pd_env(api, n, StackObservation(num_stack, keys, skip))
        obs, _ = env.reset()
        assert "actions" in obs and "pd_controller" in obs["actions"]
        assert obs["t"].shape == (n, num_stack)
        assert obs["measurements"]["ImuSensor"].shape == (n, num_stack, 6, 1)
        assert obs["actions"]["pd_controller"].shape == (n, num_stack, env.robot.nmotors)
        assert obs["measurements"]["EffortSensor"].ndim == 3           # [n_env, 1, 12]: not stacked
        assert (obs["t"][:, :-1] == 0.0).all()
        assert (obs["measurements"]["ImuSensor"][:, :-1] == 0.0).all()
        assert (obs["actions"]["pd_controller"] == 0.0).all()           # zeroed history, zero action
        np.testing.assert_array_equal(obs["measurements"]["ImuSensor"][:, -1], env._plain_observation()["measurements"]["ImuSensor"])
        np.testing.assert_array_equal(obs["states"]["agent"]["q"], env.engine.get_state()[1])

        action = np.full((n, env.robot.nmotors), 1e-3)
        obs = env.step(action)[0]
        stack_dt = (skip + 1) * obs_dt
        t_last = round(env.step_dt / obs_dt) // (skip + 1) * stack_dt
        shifted = round(env.step_dt / obs_dt) % (skip + 1) > 0
        np.testing.assert_allclose(obs["t"][:, -1], env.engine.get_state()[0], atol=1e-6)
        for i in range(1, num_stack):
            np.testing.assert_allclose(obs["t"][:, ::-1][:, i], max(t_last - (i - shifted) * stack_dt, 0.0), atol=1e-6)
        np.testing.assert_array_equal(obs["actions"]["pd_controller"][:, -1], env.engine.get_efforts()[2])
        np.testing.assert_array_equal(obs["measurements"]["ImuSensor"][:, -1], env._plain_observation()["measurements"]["ImuSensor"])

        # step to the next stacking breakpoint with a full buffer (integer milliseconds: 40 and 5 (skip + 1))
        step_ms, stack_ms = round(env.step_dt * 1000), round(stack_dt * 1000)
        n_bp = stack_ms // np.gcd(step_ms, stack_ms)
        n_full = int(np.ceil(num_stack / (int(np.ceil(step_ms / stack_ms)) + 1)))
        n_steps = n_bp * int(np.ceil(n_full / n_bp))
        for _ in range(1, n_steps):
            obs = env.step(action)[0]
        for i in range(num_stack):
            np.testing.assert_allclose(obs["t"][:, ::-1][:, i], n_steps * env.step_dt - i * stack_dt, atol=1e-6)
        np.testing.assert_array_equal(obs["measurements"]["ImuSensor"][:, -1], env._plain_observation()["measurements"]["ImuSensor"])
        env.close()


def test_reference_unit_tests(api):
    reference_unit_tests(api)


# ---------------------------------------------------------------------------------------------- hand-off parity
def _hand_off_engine(api, sc, full, monkeypatch):
    monkeypatch.setenv("JB_NO_FAST_BOUNDS", "1")        # (the quadruped signature would solve the bounds on the hot path)
    monkeypatch.setenv("JB_NO_FAST_KERNEL", "1" if full else "0")
    eng = BatchedEngine(sc.robot, sc.options, sc.n_env, api_=api)
    eng.set_pd_controller(sc.kp, sc.kd)
    eng.set_mahony_filter(1.0, 0.1)
    eng.set_obs_stack(5, 1, [core.STACK_T, core.STACK_IMU, core.STACK_ENCODER, core.STACK_MAHONY])
    eng.set_command(sc.target0)
    eng.start(sc.q0, sc.v0)
    return eng


def hand_off_parity(api, monkeypatch, n=6, n_steps=3):
    """Envs the hot-path body hands to the full body (a hip joint leaves its bounds) stack exactly once per refresh: the
    same frames as a batch stepped by the full body only."""
    sc = scenarios.make("anymal", n, seed=8, flagged_fraction=1.0 / 3.0)
    fast, full = _hand_off_engine(api, sc, False, monkeypatch), _hand_off_engine(api, sc, True, monkeypatch)
    for k in range(n_steps):
        act = sc.sample_targets(k)
        for e in (fast, full):
            e.set_command(act)
            e.step(sc.step_dt)
        s1, s0 = fast.get_obs_stack(), full.get_obs_stack()
        np.testing.assert_array_equal(s1[:, :, 0], s0[:, :, 0])           # times
        np.testing.assert_allclose(s1, s0, rtol=0, atol=1e-6 * max(1.0, float(np.abs(s0).max())))
    assert (fast.get_status()[::3] & core.JB_ENV_JOINT_LIMIT).all()      # the flagged envs went through the full body
    for e in (fast, full):
        e.close()


def test_hand_off_stacks_once_per_refresh(api, monkeypatch):
    hand_off_parity(api, monkeypatch)


# ---------------------------------------------------------------------------------------------- device env
def test_device_env_matches_host_env(api):
    from test_device_env import env_equivalence
    env_equivalence(api, dict(PD, order=1, stack=StackObservation(4, DEVICE_KEYS, 3)))


# ---------------------------------------------------------------------------------------------- refusals and config
def refusals(api):
    sc = scenarios.make("anymal", 2, seed=0)
    eng = BatchedEngine(sc.robot, sc.options, 2, api_=api)
    T, I = core.STACK_T, core.STACK_IMU
    for bad in (dict(num_stack=-1, leaves=[T]), dict(num_stack=2, skip_frames_ratio=-2, leaves=[T]),
                dict(num_stack=2, leaves=[]), dict(num_stack=2, leaves=[9]), dict(num_stack=2, leaves=[-1]),
                dict(num_stack=2, leaves=[T, I, T]), dict(num_stack=2, leaves=[core.STACK_CONTACT]),
                dict(num_stack=2, leaves=[core.STACK_PD_ACTION]), dict(num_stack=2, leaves=[core.STACK_PD_STATE]),
                dict(num_stack=2, leaves=[core.STACK_MAHONY])):
        with pytest.raises(ValueError):
            eng.set_obs_stack(**bad)
    eng.set_pd_controller(sc.kp, sc.kd)
    eng.set_obs_stack(2, -1, [T, I])
    eng.set_command(sc.target0)
    eng.start(sc.q0, sc.v0)
    with pytest.raises(core.BadControlFlow):
        eng.set_obs_stack(3, 0, [T])
    with pytest.raises(core.BadControlFlow):
        eng.set_obs_stack(0)
    eng.stop()
    eng.set_obs_stack(0)                                  # off between episodes
    with pytest.raises(core.BadControlFlow):
        eng.get_obs_stack()
    eng.close()
    for sp, cp in ((0.0025, 0.005), (0.005, 0.0025)):
        opt = scenarios.make("anymal", 2, seed=0).options
        opt["stepper"]["sensorsUpdatePeriod"], opt["stepper"]["controllerUpdatePeriod"] = sp, cp
        e = BatchedEngine(sc.robot, opt, 2, api_=api)
        with pytest.raises(NotImplementedError):
            e.set_obs_stack(2, 0, [T])
        e.close()


def test_refusals(api):
    refusals(api)


def test_unsupported_leaves_are_refused(api):
    sc = scenarios.make("anymal", 2, seed=0)
    for keys in (None, [("states",)], [("states", "agent", "q")], [("t",), ("states", "agent")]):
        with pytest.raises(NotImplementedError):
            envs.PDControlBatchedEnv(sc, api_=api, stack=StackObservation(2, keys))
    with pytest.raises(ValueError):
        envs.PDControlBatchedEnv(sc, api_=api, stack=StackObservation(2, [("nothing",)]))
    with pytest.raises(ValueError):                       # no `actions` leaf without augment_observation
        envs.PDControlBatchedEnv(sc, api_=api, stack=StackObservation(2, [("actions",)]))
    with pytest.raises(ValueError):
        StackObservation(0)
    with pytest.raises(ValueError):
        StackObservation(2, skip_frames_ratio=-2)


def test_default_observation_is_unchanged(api):
    """stack=None and augment_observation=False: the observation tree the PD env always returned."""
    env = _pd_env(api, 2, augment_observation=False)
    obs, _ = env.reset()
    assert set(obs) == {"t", "states", "measurements", "features"} and obs["t"].shape == (2,)
    env.close()


# the StackObservation entry of python/gym_jiminy/unit_py/data/anymal_pipeline.toml, with the block layers before it
ANYMAL_PIPELINE_LAYERS = [
    {"block": {"cls": "gym_jiminy.common.blocks.PDController",
               "kwargs": {"update_ratio": 2, "kp": [1500.0] * 12, "kd": [0.01] * 12, "joint_position_margin": 0.0,
                          "joint_velocity_limit": 100.0, "joint_acceleration_limit": 10000.0}},
     "wrapper": {"kwargs": {"augment_observation": True}}},
    {"block": {"cls": "gym_jiminy.common.blocks.PDAdapter", "kwargs": {"update_ratio": -1, "order": 1}},
     "wrapper": {"kwargs": {"augment_observation": False}}},
    {"block": {"cls": "gym_jiminy.common.blocks.MahonyFilter",
               "kwargs": {"update_ratio": 1, "exact_init": False, "kp": 1.0, "ki": 0.1}}},
    {"wrapper": {"cls": "gym_jiminy.common.wrappers.StackObservation",
                 "kwargs": {"nested_filter_keys": [["t"], ["measurements", "ImuSensor"], ["actions"]],
                            "num_stack": 4, "skip_frames_ratio": 3}}},
]


def test_from_config(api):
    stack = observation_stack.from_config(ANYMAL_PIPELINE_LAYERS)
    assert (stack.num_stack, stack.skip_frames_ratio) == (4, 3)
    assert stack.nested_filter_keys == [("t",), ("measurements", "ImuSensor"), ("actions",)]
    assert observation_stack.from_config(ANYMAL_PIPELINE_LAYERS[:3]) is None
    with pytest.raises(NotImplementedError):
        observation_stack.from_config([{"wrapper": {"cls": "gym_jiminy.common.wrappers.FlattenObservation"}}])
    env = _pd_env(api, 2, stack)
    obs, _ = env.reset()
    assert obs["t"].shape == (2, 4) and obs["actions"]["pd_controller"].shape == (2, 4, 12)
    assert obs["measurements"]["ImuSensor"].shape == (2, 4, 6, 1) and obs["measurements"]["EncoderSensor"].shape == (2, 2, 12)
    env.close()


# ---------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_gpu_replay_matches_the_reference_wrapper():
    reference_replay(None, n=3, n_steps=4)


@pytest.mark.gpu
def test_gpu_recording_matches_fine_steps():
    recording_matches_fine_steps(None)


@pytest.mark.gpu
def test_gpu_reference_unit_tests():
    reference_unit_tests(None)


@pytest.mark.gpu
def test_gpu_hand_off_stacks_once_per_refresh(monkeypatch):
    hand_off_parity(None, monkeypatch)


@pytest.mark.gpu
def test_gpu_device_env_matches_host_env():
    from test_device_env import env_equivalence
    env_equivalence(None, dict(PD, order=1, stack=StackObservation(4, DEVICE_KEYS, 3)))


@pytest.mark.gpu
def test_gpu_refusals():
    refusals(None)
