"""Reward and termination compositions (`jiminy_b200.compositions`): the numpy terms against closed forms, the device's
contact-frame pass (`jb_contact_positions_device`) against `robots.frame_placements`, the composition kernel
(`jb_compositions_device`) inside the device envs against host envs that replay the same restarts, and the refusal of bad
specs.

Every kernel scenario is a function of `api`: the CPU suite runs it on the emulated library (device memory is host
memory, torch tensors on the CPU), the `-m gpu` variants on the device with `api=None`.

Tolerances: the kernel and the numpy evaluator compute products and sums in the same order without fused multiply-adds,
so power, stack means, safety and mixtures of order 1 are bit-equal.  `pow` (the radial basis function) and
`sin` / `cos` / `atan2` (roll and pitch) come from each side's math library; CUDA documents them within 1-2 ulp of the
exact result, as glibc is, so values built on them are compared within 1e-14 relative.  The contact positions come from
two forward-kinematics codes (the device sweep against the host's SE3 products): 1e-12 m."""
import math

import numpy as np
import pytest
import torch

from jiminy_b200 import compositions as CP
from jiminy_b200 import core, envs, robots, scenarios
from jiminy_b200 import model as M
from jiminy_b200.core import BatchedEngine
from jiminy_b200.torch_envs import DeviceBatchedEnv, DevicePDControlBatchedEnv

from emul import emul_api


@pytest.fixture(scope="module")
def api():
    return emul_api()


def _np(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _dev(api, x, dtype=torch.float64):
    return torch.tensor(np.ascontiguousarray(x), dtype=dtype, device="cpu" if api is not None else "cuda")


def _sync(api):
    if api is None:
        torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- numpy terms
def _rot(axis, angle):
    c, s = math.cos(angle), math.sin(angle)
    return {"x": np.array([[1, 0, 0], [0, c, -s], [0, s, c]]), "y": np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]]),
            "z": np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])}[axis]


def test_matrix_to_rpy_closed_forms():
    for roll, pitch, yaw in [(0.1, -0.2, 0.3), (-0.7, 0.4, -2.5), (0.0, 0.0, 0.0), (1.2, -1.1, 3.0)]:
        R = _rot("z", yaw) @ _rot("y", pitch) @ _rot("x", roll)
        np.testing.assert_allclose(CP.matrix_to_rpy(R[None])[0], [roll, pitch, yaw], atol=1e-14)
    for sign in (1.0, -1.0):      # gimbal lock: pitch exactly +-pi/2, roll and yaw folded into one angle
        R = _rot("z", 0.3) @ _rot("y", sign * math.pi / 2) @ _rot("x", 0.0)
        assert abs(CP.matrix_to_rpy(R[None])[0, 1] - sign * math.pi / 2) < 1e-7
    # the quaternion of a rotation gives that rotation
    axis = np.array([0.3, -0.5, 0.8]) / np.linalg.norm([0.3, -0.5, 0.8])
    th = 0.9
    quat = np.r_[axis * math.sin(th / 2), math.cos(th / 2)]
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    np.testing.assert_allclose(CP.quat_to_matrix(quat[None])[0], np.eye(3) + math.sin(th) * K + (1 - math.cos(th)) * K @ K, atol=1e-15)


def test_compute_power_modes():
    v = np.array([[1.0, -2.0, 3.0]])
    u = np.array([[2.0, 1.0, -1.0]])       # motor powers 2, -2, -3
    E = CP.EnergyGenerationMode
    assert CP.compute_power(E.CHARGE, v, u)[0] == -3.0
    assert CP.compute_power(E.LOST_GLOBAL, v, u)[0] == 0.0
    assert CP.compute_power(E.LOST_EACH, v, u)[0] == 2.0
    assert CP.compute_power(E.PENALIZE, v, u)[0] == 7.0
    assert CP.compute_power(E.LOST_GLOBAL, -v, u)[0] == 3.0


def test_rbf_and_mixtures():
    assert CP.radial_basis_function(np.array([0.0]), 0.5)[0] == 1.0
    assert abs(CP.radial_basis_function(np.array([0.5]), 0.5)[0] - 0.01) < 1e-16
    assert CP.weighted_norm((0.5, 0.5), 1.0, (0.2, None)) == 0.1
    assert CP.weighted_norm((0.5, 0.5), 1.0, (None, None)) is None
    assert CP.weighted_norm((0.5, 2.0), float("inf"), (0.8, 0.3)) == 0.6
    assert abs(CP.weighted_norm((1.0, 1.0), 2.0, (3.0, 4.0)) - 5.0) < 1e-15
    assert CP.geometric_mean((None, None)) is None
    assert CP.geometric_mean((0.25, None, 0.25)) == 0.25
    assert abs(CP.geometric_mean((0.5, 0.125)) - 0.25) < 1e-16
    mix = CP.AdditiveMixtureReward("reward_total", [CP.SurviveReward(), CP.MinimizeMechanicalPowerConsumption(1.0, 0.1)],
                                   weights=[0.0, 1.0])
    assert [type(c) for c in mix.components] == [CP.MinimizeMechanicalPowerConsumption]   # zero weights dropped
    assert CP.AdditiveMixtureReward("r", [CP.SurviveReward()], order="inf").order == float("inf")


def _tiny(n=3, **kw):
    """A Compositions over ANYmal with the given terms and neutral state arrays."""
    sc = scenarios.make("anymal", n, seed=1)
    comp = CP.Compositions(kw.get("reward"), kw.get("terminations", ()), sc.robot, n, 0.01, 20.0, None, kw.get("training", True))
    return sc, comp


def test_power_stack_mean_and_wrap():
    n = 2
    sc, comp = _tiny(n, reward=CP.MinimizeMechanicalPowerConsumption(cutoff=3.0, horizon=0.025))
    i = 0
    assert comp.stack_size[i] == CP.max_stack(0.025, 0.01) == 4
    rob = sc.robot
    nm = rob.nmotors
    cmd = np.ones((n, nm))
    ratio = np.array([m.reduction for m in rob.motors])
    iv = [rob.idx_v[m.joint] for m in rob.motors]
    v = np.zeros((n, rob.nv))
    pushed = [[], []]

    def power_of(x):
        vv = v.copy()
        vv[:, iv] = x / (ratio * nm)
        return vv
    comp.seed(None, power_of(np.array([[1.0], [2.0]])), cmd)
    pushed[0].append(comp.stacks[i][0, 0]); pushed[1].append(comp.stacks[i][1, 0])
    t = np.full(n, 1.0)
    for k in range(7):
        vk = power_of(np.array([[3.0 + k], [10.0 * k]]))
        p = comp.power(comp.nodes[i], vk, cmd)
        pushed[0].append(p[0]); pushed[1].append(p[1])
        reward, *_ , info = comp.evaluate(t, sc.q0, vk, cmd, np.zeros(n, bool), np.zeros(n, bool))
        for e in range(n):
            window = pushed[e][-4:]
            s = 0.0
            for x in window:
                s += x
            assert comp._mean(i)[e] == s / len(window)
            assert reward[e] == info["reward_power_consumption"][e] == np.power(0.01, (s / len(window)) ** 2 / 9.0)
    comp.seed(np.array([0, 1], np.uint8), power_of(np.array([[0.0], [5.0]])), cmd)
    assert comp.count[i, 1] == 1 and comp._mean(i)[1] == comp.stacks[i][1, 0]
    assert comp.count[i, 0] == 8


def test_terminations_gates_and_order():
    n = 4
    sc, comp = _tiny(n, terminations=[
        CP.MechanicalSafetyTermination(position_margin=0.1, velocity_max=1.0, grace_period=0.5),
        CP.BaseRollPitchTermination(low=[-0.1, -0.1], high=[0.1, 0.1], training_only=True),
        CP.FallingTermination(min_base_height=0.3)])
    rob = sc.robot
    q, v = sc.q0.copy(), np.zeros((n, rob.nv))
    m0 = rob.motors[0]
    iq, iv = rob.idx_q[m0.joint], rob.idx_v[m0.joint]
    # env 0: at the lower bound moving down fast; env 1: the same, moving slowly; env 2: near the upper bound moving up;
    # env 3: in the middle, fast
    q[0, iq] = q[1, iq] = rob.q_lower[iq] + 0.05
    q[2, iq] = rob.q_upper[iq] - 0.05
    v[0, iv], v[1, iv], v[2, iv], v[3, iv] = -2.0, -0.5, 2.0, 5.0
    contacts = np.zeros((n, len(rob.contact_frame_names), 3))
    contacts[:, :, 2] = 0.0
    cmd = np.zeros((n, rob.nmotors))
    no = np.zeros(n, bool)
    t = np.full(n, 1.0)
    _, term, trunc, info = comp.evaluate(t, q, v, cmd, no, no, contacts)
    assert term.tolist() == [True, False, True, False] and not trunc.any()
    assert info["terminated"].tolist() == [0, -1, 0, -1]
    assert info["termination_mechanical_safety"].tolist() == [1, 0, 1, 0]
    assert np.isnan(info["termination_base_roll_pitch"][[0, 2]]).all()          # not reached: the first one fired
    # inside the grace period the safety condition continues and the next fires
    q[:, 2] = 0.2                                                                  # base 0.2 m above the lowest contact
    _, term, _, info = comp.evaluate(np.full(n, 0.1), q, v, cmd, no, no, contacts)
    assert info["termination_mechanical_safety"].tolist() == [0, 0, 0, 0]
    assert info["terminated"].tolist() == [2] * 4
    # the env's own rule comes first: nothing is evaluated
    _, term, trunc, info = comp.evaluate(t, q, v, cmd, no, np.ones(n, bool), contacts)
    assert np.isnan(info["termination_mechanical_safety"]).all() and (info["terminated"] == -1).all() and not term.any()
    # training_only: skipped out of training
    _, comp2 = _tiny(n, terminations=[CP.BaseRollPitchTermination(low=[0.5, 0.5], high=None, training_only=True)], training=False)
    _, term, _, info = comp2.evaluate(t, q, v, cmd, no, no, contacts)
    assert not term.any() and (info["termination_base_roll_pitch"] == 0).all()
    _, comp3 = _tiny(n, terminations=[CP.BaseRollPitchTermination(low=[0.5, 0.5], high=None, training_only=True)])
    assert comp3.evaluate(t, q, v, cmd, no, no, contacts)[1].all()


@pytest.mark.parametrize("name", ["anymal", "atlas"])
def test_relative_height_and_lowest_contact(name):
    n = 3
    sc = scenarios.make(name, n, seed=4)
    rob = sc.robot
    q = np.array([robots.ground_base_height(rob, x) for x in sc.q0])
    q[:, 2] += np.array([0.0, 0.05, -0.02])                  # 0, 5 cm above, 2 cm under the ground
    comp = CP.Compositions(None, [CP.FlyingTermination(max_height=0.03), CP.FallingTermination(min_base_height=0.0)],
                           rob, n, sc.step_dt, 20.0, None)
    pos = CP.contact_positions([rob] * n, q)
    np.testing.assert_allclose(pos[:, :, 2].min(axis=1), [0.0, 0.05, -0.02], atol=1e-12)
    no = np.zeros(n, bool)
    _, term, _, info = comp.evaluate(np.ones(n), q, np.zeros((n, rob.nv)), np.zeros((n, rob.nmotors)), no, no, pos)
    assert info["terminated"].tolist() == [-1, 0, -1]
    np.testing.assert_array_equal(info["termination_base_height"][[0, 2]], 0.0)     # base above the lowest frame


def test_from_config_and_bad_specs():
    cfg = {"reward": {"cls": "gym_jiminy.common.compositions.AdditiveMixtureReward",
                      "kwargs": {"name": "reward_total", "weights": [0.6, 0.4], "components": [
                          {"cls": "gym_jiminy.common.compositions.SurviveReward"},
                          {"cls": "gym_jiminy.common.compositions.generic.MinimizeMechanicalPowerConsumption",
                           "kwargs": {"cutoff": 100.0, "horizon": 0.2, "generator_mode": "LOST_EACH"}}]}},
           "terminations": [{"cls": "gym_jiminy.common.compositions.BaseRollPitchTermination",
                             "kwargs": {"low": [-0.2, -0.05], "high": [-0.05, 0.3], "grace_period": 0.1, "training_only": False}}]}
    reward, terms = CP.from_config(cfg)
    assert isinstance(reward, CP.AdditiveMixtureReward) and reward.weights == (0.6, 0.4)
    assert reward.components[1].generator_mode == CP.EnergyGenerationMode.LOST_EACH
    assert terms[0].grace_period == 0.1
    with pytest.raises(NotImplementedError):
        CP.from_config({"reward": {"cls": "gym_jiminy.common.compositions.TrackingBaseOdometryVelocityReward", "kwargs": {}}})
    for bad in (lambda: CP.BaseRollPitchTermination(low=[0.1, 0.2, 0.3], high=None),
                lambda: CP.AdditiveMixtureReward("r", [CP.SurviveReward()], order=0),
                lambda: CP.AdditiveMixtureReward("r", [CP.SurviveReward()], weights=[-1.0]),
                lambda: CP.AdditiveMixtureReward("r", [CP.SurviveReward()], weights=[1.0, 1.0]),
                lambda: CP.MinimizeMechanicalPowerConsumption(cutoff=0.0, horizon=1.0),
                lambda: CP.MinimizeMechanicalPowerConsumption(cutoff=1.0, horizon=-1.0),
                lambda: CP.MechanicalPowerConsumptionTermination(10.0, horizon=0.0)):
        with pytest.raises(ValueError):
            bad()


def spec_refused(api):
    """The C ABI refuses a malformed spec with ValueError and uploads nothing: the good spec set before still runs."""
    n = 2
    sc = scenarios.make("anymal", n, seed=0)
    eng = BatchedEngine(sc.robot, sc.options, n, api_=api)
    comp = CP.Compositions(CP.AdditiveMixtureReward("reward_total", [CP.SurviveReward(), CP.MinimizeMechanicalPowerConsumption(1.0, 0.1)]),
                           [CP.MechanicalPowerConsumptionTermination(1.0, horizon=0.05)], sc.robot, n, sc.step_dt, 20.0, None)
    comp.upload(eng)
    good = (comp.node_int, comp.node_dbl, comp.n_reward, comp.weights, comp.motor_int, comp.motor_dbl, comp.env_dbl, True)

    def variant(i=None, col=None, val=None, dbl=False, **kw):
        args = list(good)
        args[0], args[1], args[3] = good[0].copy(), good[1].copy(), good[3].copy()
        if i is not None:
            (args[1] if dbl else args[0])[i, col] = val
        for k, x in kw.items():
            args[{"n_reward": 2, "weights": 3}[k]] = x
        return args
    bad = [variant(0, 0, 7),                   # unknown kind
           variant(3, 0, 2),                   # a reward kind among the terminations
           variant(1, 2, 9),                   # unknown generator mode
           variant(2, 1, 0.0, dbl=True),       # order 0
           variant(1, 1, -1.0, dbl=True),      # cutoff
           variant(1, 2, 0.0, dbl=True),       # horizon
           variant(3, 2, -1.0, dbl=True),      # termination horizon
           variant(weights=np.array([0.5, -0.5])),
           variant(weights=np.array([1.0])),
           variant(2, 1, 3),                   # more components than the tree holds
           variant(n_reward=2)]                # two roots
    for args in bad:
        with pytest.raises(ValueError):
            eng.set_compositions(*args)
    eng.set_compositions(*good)
    eng.close()


def test_spec_refused(api):
    spec_refused(api)


# ---------------------------------------------------------------------------------------------- contact-frame pass
def contact_pass(api, case):
    """Contact positions of the pass against `robots.frame_placements` on each env's own model (1e-12 m); envs that are
    not started read NaN."""
    name = "anymal" if case in ("variants", "biased") else case
    n = 11
    sc = scenarios.make(name, n, seed=7)
    rob = sc.robot
    eng = BatchedEngine(rob, sc.options, n, api_=api)
    models = [rob] * n
    if case == "variants":
        rng = np.random.default_rng(3)
        variants = [M.biased_robot(rob, rng, relative_position_std=0.005) for _ in range(2)]
        vog = np.arange(-(-n // eng.envs_per_group), dtype=np.int32) % 2
        eng.set_model_variants(variants, vog)
        models = [variants[vog[e // eng.envs_per_group]] for e in range(n)]
    if case == "biased":
        from jiminy_b200 import model_randomisation
        mb = model_randomisation.from_model_bias_std(rob, {"relativePositionBodiesBiasStd": 0.005, "massBodiesBiasStd": 0.02})
        mb.register(eng)
        rows = mb.draw_numpy(np.random.default_rng(5), n)
        mb.apply_host(eng, rows, None)
    eng.set_command(np.zeros((n, max(rob.nmotors, 1))))
    mask = np.ones(n, np.uint8)
    mask[[2, 7]] = 0
    eng.start(sc.q0, sc.v0, mask=mask)
    if case == "biased":
        models = [eng.model(e) for e in range(n)]
    for _ in range(2):
        eng.step(sc.step_dt)
    nc = len(rob.contact_frame_names)
    out = _dev(api, np.full((n, nc, 3), 7.0))
    eng.contact_positions_device(out.data_ptr())
    _sync(api)
    pos = _np(out)
    q = eng.get_state()[1]
    on = (eng.get_status() & (core.JB_ENV_NOT_STARTED | core.JB_ENV_NAN)) == 0
    assert not on[mask == 0].any() and on.sum() >= n - 4, eng.get_status()
    expect = CP.contact_positions([models[e] for e in np.flatnonzero(on)], q[on])
    np.testing.assert_allclose(pos[on], expect, rtol=0, atol=1e-12)
    assert np.isnan(pos[~on]).all()
    if case in ("variants", "biased"):
        nominal = CP.contact_positions([rob] * int(on.sum()), q[on])
        assert np.abs(nominal - expect).max() > 1e-4           # each env is measured on its own body
    eng.close()


CONTACT_CASES = ["anymal", "atlas", "anymal_flexible", "variants", "biased"]


@pytest.mark.parametrize("case", CONTACT_CASES)
def test_contact_positions(api, case):
    contact_pass(api, case)


# ---------------------------------------------------------------------------------------------- device env vs host env
def full_spec(step_dt):
    reward = CP.AdditiveMixtureReward("reward_total", [
        CP.SurviveReward(),
        CP.MultiplicativeMixtureReward("reward_power_mix", [
            CP.MinimizeMechanicalPowerConsumption(cutoff=200.0, horizon=3 * step_dt, generator_mode="LOST_EACH")]),
        CP.MinimizeMechanicalPowerConsumption(cutoff=400.0, horizon=0.5 * step_dt)], order=1, weights=[0.5, 0.3, 0.2])
    # a second power reward needs a name of its own
    reward.components[2].name = "reward_power_consumption_short"
    terms = [CP.BaseRollPitchTermination(low=[-0.08, -0.08], high=[0.08, 0.08], grace_period=2 * step_dt),
             CP.FallingTermination(min_base_height=0.3),
             CP.FlyingTermination(max_height=0.2, training_only=True),
             CP.MechanicalSafetyTermination(position_margin=0.05, velocity_max=4.0),
             CP.MechanicalPowerConsumptionTermination(max_power=400.0, horizon=2 * step_dt, generator_mode="PENALIZE"),
             CP.MechanicalPowerConsumptionTermination(max_power=2000.0, generator_mode="CHARGE")]
    terms[5].name = "termination_power_consumption_instant"
    return reward, terms


EXACT = ("terminated", "truncated", "termination_mechanical_safety", "termination_power_consumption",
         "termination_power_consumption_instant")


def _same_info(info_d, info_s, names):
    for name in names:
        a, b = _np(info_d[name]), np.asarray(info_s[name])
        if name in EXACT:
            np.testing.assert_array_equal(a, b, err_msg=name)
        else:
            np.testing.assert_array_equal(np.isnan(a), np.isnan(b), err_msg=name)
            np.testing.assert_allclose(a, b, rtol=1e-14, atol=0, err_msg=name)


def env_shadow(api, pd, randomised, n_steps=10):
    """A device env with every term against a host env that replays its restart states and randomisation rows: reward,
    terminated, truncated, indices and per-term values (see the module docstring for the tolerances)."""
    n = 6
    sc_d, sc_s = (scenarios.make("anymal", n, seed=21) for _ in range(2))
    reward, terms = full_spec(sc_d.step_dt)
    kw = dict(simulation_duration_max=0.16, api_=api, reward=reward, terminations=terms)
    if randomised:
        kw["std_ratio"] = {"disturbance": 1.0, "sensors": 1.0}
        kw["model_bias_std"] = {"relativePositionBodiesBiasStd": 0.005, "massBodiesBiasStd": 0.02}
    if pd:
        kw["training"] = False
    dev = (DevicePDControlBatchedEnv if pd else DeviceBatchedEnv)(sc_d, reset_states="sample", **kw)
    shadow = (envs.PDControlBatchedEnv if pd else envs.BatchedJiminyEnv)(sc_s, **kw)
    names = ["terminated", "truncated"] + dev.compositions.names

    def replay(q_placed):
        if dev.sensor_randomisation is not None:
            snap = {k: _np(v).copy() for k, v in dev.sensor_rows.items()}
            snap["seed"] = snap["seed"].astype(np.uint32)
            shadow._redraw_sensors = lambda mask: shadow.sensor_randomisation.apply_host(shadow.engine, snap, mask)
        if dev.disturbance is not None:
            dsnap = {k: _np(v).copy() for k, v in dev.disturbance_rows.items()}
            shadow._redraw_disturbance = lambda mask: shadow.disturbance.apply_host(shadow.engine, dsnap, mask)
        if dev.model_bias is not None:
            bsnap = _np(dev.model_bias_rows).copy()
            shadow._redraw_model_bias = lambda mask: shadow.model_bias.apply_host(shadow.engine, bsnap, mask)
        shadow._sample_state = lambda m: (q_placed, np.zeros((n, shadow.robot.nv)))

    dev.reset()
    replay(None)
    shadow.reset()
    rng = np.random.default_rng(2)
    fired, restarts = set(), 0
    for k in range(n_steps):
        act = np.clip(sc_s.sample_targets(k) + rng.normal(0, 0.3, (n, shadow.robot.nmotors)), shadow.action_low, shadow.action_high) \
            if not pd else rng.normal(0, 2.0, (n, shadow.robot.nmotors))
        o_d, r_d, te_d, tr_d, info = dev.step(_dev(api, act))
        q_placed = _np(o_d["states"]["agent"]["q"]).copy()
        replay(q_placed)
        o_s, r_s, te_s, tr_s, info_s = shadow.step(act)
        np.testing.assert_array_equal(_np(o_d["states"]["agent"]["q"]), o_s["states"]["agent"]["q"])
        np.testing.assert_array_equal(_np(te_d), te_s)
        np.testing.assert_array_equal(_np(tr_d), tr_s)
        np.testing.assert_allclose(_np(r_d), r_s, rtol=1e-14, atol=0)
        _same_info(info, info_s, names)
        fired |= set(np.asarray(info_s["terminated"]).tolist())
        restarts += int((te_s | tr_s).sum())
    assert restarts >= 2, restarts
    assert len(fired - {-1}) >= 1, fired
    for e in (dev, shadow):
        e.close()


SHADOW_CASES = {"plain": (False, False), "pd": (True, False), "randomised": (False, True), "pd_randomised": (True, True)}


@pytest.mark.parametrize("case", list(SHADOW_CASES))
def test_device_env_matches_host(api, case):
    env_shadow(api, *SHADOW_CASES[case])


def defaults_unchanged(api):
    """`reward=None, terminations=()` is the plain env; an explicit `SurviveReward` through the kernel gives its bits."""
    n = 5
    out = []
    for kw in ({}, {"reward": None, "terminations": ()}, {"reward": CP.SurviveReward()}):
        env = DeviceBatchedEnv(scenarios.make("anymal", n, seed=3), simulation_duration_max=0.08, api_=api, **kw)
        assert (env.compositions is None) == ("reward" not in kw or kw["reward"] is None)
        env.reset()
        rows = []
        for k in range(6):
            o, r, te, tr, _ = env.step(_dev(api, env.sc.sample_targets(k)))
            rows.append([_np(x).copy() for x in (o["states"]["agent"]["q"], r, te, tr)])
        out.append(rows)
        env.close()
    for other in out[1:]:
        for a, b in zip(out[0], other):
            for x, y in zip(a, b):
                np.testing.assert_array_equal(x, y)


def test_defaults_unchanged(api):
    defaults_unchanged(api)


# ---------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_gpu_spec_refused():
    spec_refused(None)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CONTACT_CASES)
def test_gpu_contact_positions(case):
    contact_pass(None, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(SHADOW_CASES))
def test_gpu_device_env_matches_host(case):
    env_shadow(None, *SHADOW_CASES[case])


@pytest.mark.gpu
def test_gpu_defaults_unchanged():
    defaults_unchanged(None)


@pytest.mark.gpu
@pytest.mark.parametrize("pd", [False, True])
def test_gpu_step_with_compositions_never_synchronises(pd):
    n = 256
    sc = scenarios.make("anymal", n, seed=0)
    reward, terms = full_spec(sc.step_dt)
    env = (DevicePDControlBatchedEnv if pd else DeviceBatchedEnv)(sc, simulation_duration_max=0.08, reward=reward,
                                                                  terminations=terms)
    env.reset()
    acts = [torch.as_tensor(np.zeros((n, sc.robot.nmotors)) if pd else sc.sample_targets(k), device="cuda") for k in range(4)]
    env.step(acts.pop())
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
