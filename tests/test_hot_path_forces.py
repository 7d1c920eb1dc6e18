"""External forces on the quadruped hot path (`env_step_kernel_ext`): impulse, profile and process forces applied in the
composite-rigid-body evaluation, against the full body's force-aware generic sweeps (JB_NO_FAST_KERNEL=1) and the oracle.

Every scenario is a function of `api`: the CPU suite runs it on the warp emulator, the `-m gpu` twins on the device with
`api=None`.  The two paths differ only in rounding (composite-rigid-body form against the articulated-body sweeps)."""
import numpy as np
import pytest

from jiminy_b200 import scenarios
from jiminy_b200.core import BatchedEngine
from jiminy_b200.disturbance import WalkerDisturbance

from emul import emul_api
from oracle.oracle import OracleBatch
from parity_common import compare

HOT = ", external forces applied in the evaluation"
# wrench scale: torques a fifth of the forces (explicit Euler at 1 ms on the 4e6 N/m ground diverges under much more)
W = np.array([1.0, 1.0, 1.0, 0.2, 0.2, 0.2])


@pytest.fixture(scope="module")
def api():
    return emul_api()


def _frames(rob):
    base = rob.frames["base"] if "base" in rob.frames else rob.frames["root_joint"]
    shank = rob.frames[next(n for n in rob.frames if "SHANK" in n.upper())]
    return (base.joint, base.placement.p), (shank.joint, shank.placement.p + [0.0, 0.0, -0.1])


def _engine(api, monkeypatch, sc, full, env=None):
    """A PD-controlled engine of `sc`; `full`: every env-step on the full body (JB_NO_FAST_KERNEL=1)."""
    monkeypatch.setenv("JB_NO_FAST_KERNEL", "1" if full else "0")
    for k, x in (env or {}).items():
        monkeypatch.setenv(k, x)
    eng = BatchedEngine(sc.robot, sc.options, sc.n_env, api_=api)
    eng.set_pd_controller(sc.kp, sc.kd)
    return eng


def _register(eng, sc, case, seed=5):
    """Registers the forces of `case` on `eng` (the same draws for the same seed); returns what to set before env-step k."""
    n, dt = sc.n_env, sc.step_dt
    rng = np.random.default_rng(seed)
    base, shank = _frames(sc.robot)
    if case == "base_impulse":         # crosses inside the first env-step, ends inside it or later
        eng.register_impulse_force(base, rng.uniform(0.005, 0.035, n), rng.uniform(2e-3, 2e-2, n), rng.normal(size=(n, 6)) * W * 100.0)
    elif case == "shank_impulse":      # private joint of one lane, off-origin frame
        eng.register_impulse_force(shank, rng.uniform(0.0, 0.03, n), rng.uniform(1e-3, 3e-2, n), rng.normal(size=(n, 6)) * W * 50.0)
    elif case == "profile":            # held for 10 ms: updates inside the 40 ms env-step
        slots = [eng.register_profile_force(base, 0.01), eng.register_profile_force(shank, 0.01)]
        return lambda k: [eng.set_profile_force(s, rng.normal(size=(n, 6)) * W * w) for s, w in zip(slots, (40.0, 20.0))]
    elif case == "process":            # update period 0: evaluated at every stage time
        tabs = []
        for fr, comp, knots, periods, w in ((base, [0, 1, 5], [10, 12, 8], [1.0, 0.6, 0.8], 60.0), (shank, [2], [9], [0.5], 30.0)):
            slot = eng.register_process_force(fr, comp, knots, periods, 0.0)
            tabs.append((slot, rng.normal(size=(n, sum(knots))) * w, rng.normal(size=(n, sum(knots))) * 10.0 * w))
        for slot, values, grads in tabs:
            eng.set_process_force(slot, values, grads)
    elif case == "walker":             # gym_jiminy's walker disturbance, its first impulse moved into the first env-step
        d = WalkerDisturbance(sc.robot, 1.0)
        d.register(eng)
        draw = d.draw_numpy(rng, n)
        draw["t"][0] = rng.uniform(0.005, dt - 0.005, n)
        d.apply_host(eng, draw)
    else:
        raise ValueError(case)
    return lambda k: None


def _outputs(eng):
    _, q, v, a = eng.get_state()
    return dict(q=q, v=v, a=a, sensors=eng.get_sensors(), fext=eng.get_efforts()[3],
                **dict(zip(("energy", "joint_a", "joint_f"), eng.get_extra_terms()))), eng.get_status()


def hot_vs_full(api, monkeypatch, case, solver, n_steps=1):
    """From identical states, the force-carrying hot path against the full body: q and v within 1e-12 after one env-step;
    accelerations, sensors, external wrenches and extra terms within 1e-9 (through the 4e6 N/m ground a rounding-level
    change of a foot's depth moves them by that much more, as in test_quadruped_stage); status words equal.
    Explicit Euler takes forty 1 ms steps per env-step on that ground, each growing the rounding differences of the two
    evaluations: 1e-9 on q and v, 1e-8 on the rest.  Without any force the two paths already differ by 9e-11 on v and
    4e-10 on a in this scenario."""
    tol_qv, tol_a = (1e-12, 1e-9) if solver == "runge_kutta_4" else (1e-9, 1e-8)
    sc = scenarios.make("anymal", 6, seed=11, solver=solver)
    runs = []
    for full in (True, False):
        eng = _engine(api, monkeypatch, sc, full)
        per_step = _register(eng, sc, case)
        assert (HOT in eng.describe()) == (not full)
        eng.set_command(sc.target0)
        eng.start(sc.q0, sc.v0)
        out = []
        for k in range(n_steps):
            per_step(k)
            eng.set_command(sc.sample_targets(k))
            eng.step(sc.step_dt)
            out.append(_outputs(eng))
        runs.append(out)
    for k, ((ref, st_ref), (hot, st_hot)) in enumerate(zip(*runs)):
        for name, x in ref.items():
            tol = tol_qv if name in ("q", "v") else tol_a
            err = np.abs(hot[name] - x) / np.maximum(np.abs(x), 1.0)
            assert err.max() <= tol, (k, name, err.max())
        np.testing.assert_array_equal(st_hot, st_ref)
        assert not st_ref.any()
    return runs


CASES = ["base_impulse", "shank_impulse", "profile", "process", "walker"]
SOLVERS = ["runge_kutta_4", "euler_explicit"]


@pytest.mark.parametrize("solver", SOLVERS)
@pytest.mark.parametrize("case", CASES)
def test_hot_path_matches_full_body(api, monkeypatch, case, solver):
    hot_vs_full(api, monkeypatch, case, solver)


def handoff(api, monkeypatch, force, in_kernel, n_steps=4):
    """Every third env driven through its hip bounds, solved in the evaluation (default) or by handing the env to the full
    body (JB_NO_FAST_BOUNDS=1), which replays the env-step from its top.  A profile force (against the oracle) or a
    process force (against JB_NO_FAST_KERNEL=1) is sampled every 30 ms: with 40 ms env-steps an update falls inside
    most steps, and a replayed step starts from the value latched before the aborted pass overwrote it."""
    sc = scenarios.make("anymal", 6, seed=8)
    rob = sc.robot
    iq = np.array([rob.idx_q[m.joint] for m in rob.motors])
    haa = [k for k, m in enumerate(rob.motors) if "HAA" in m.name]
    base, _ = _frames(rob)
    env = {} if in_kernel else {"JB_NO_FAST_BOUNDS": "1"}

    def act(k):
        a = sc.sample_targets(k)
        for j in haa:
            a[::3, j] = rob.q_upper[iq[j]] + 0.3
        return a

    if force == "profile":
        eng = _engine(api, monkeypatch, sc, False, env)
        orc = OracleBatch(rob, sc.options, sc.n_env)
        orc.set_pd_controller(sc.kp, sc.kd)
        slot, oslot = eng.register_profile_force(base, 0.03), orc.register_profile_force(base[0], base[1], 0.03)
        assert HOT in eng.describe()
        rng = np.random.default_rng(4)
        for x in (eng, orc):
            x.set_command(sc.target0)
        eng.start(sc.q0, sc.v0)
        assert not orc.start(sc.q0, sc.v0).any()
        for k in range(n_steps):
            w = rng.normal(size=(sc.n_env, 6)) * 80.0
            a = act(k)
            for x, s in ((eng, slot), (orc, oslot)):
                x.set_profile_force(s, w)
                x.set_command(a)
            eng.step(sc.step_dt)
            orc.step(sc.step_dt, parallel=True)
            compare(eng, orc, 1e-9, 1e-7)
        status = eng.get_status()
    else:
        outs = []
        for full in (True, False):
            eng = _engine(api, monkeypatch, sc, full, env)
            rng = np.random.default_rng(6)
            slot = eng.register_process_force(base, [0, 1, 2], [10, 10, 10], [1.0, 1.0, 1.0], 0.03)
            eng.set_process_force(slot, rng.normal(size=(sc.n_env, 30)) * 80.0, rng.normal(size=(sc.n_env, 30)) * 500.0)
            assert (HOT in eng.describe()) == (not full)
            eng.set_command(sc.target0)
            eng.start(sc.q0, sc.v0)
            out = []
            for k in range(n_steps):
                eng.set_command(act(k))
                eng.step(sc.step_dt)
                out.append(_outputs(eng))
            outs.append(out)
        for k, ((ref, st_ref), (hot, st_hot)) in enumerate(zip(*outs)):
            for name, x in ref.items():
                tol = 1e-9 if name in ("q", "v") else 1e-7
                err = np.abs(hot[name] - x) / np.maximum(np.abs(x), 1.0)
                assert err.max() <= tol, (k, name, err.max())
            np.testing.assert_array_equal(st_hot, st_ref)
        status = outs[0][-1][1]
    # the bounds were in play for the driven envs only (JB_ENV_JOINT_LIMIT)
    assert (status[::3] & 8).all() and not (status[1::3] & 8).any()


@pytest.mark.parametrize("in_kernel", [True, False])
@pytest.mark.parametrize("force", ["profile", "process"])
def test_handoff_with_forces(api, monkeypatch, force, in_kernel):
    handoff(api, monkeypatch, force, in_kernel)


def reporting(api, monkeypatch):
    """describe() says that forces ride the hot path for the quadruped signature's composite-rigid-body evaluation with
    spring-damper contacts and Euler / RK4 only; otherwise it reads as if no force were registered."""
    base, _ = _frames(scenarios.make("anymal", 2).robot)

    def describe(force, solver=None, contact_model=None, env=None):
        monkeypatch.delenv("JB_NO_FAST_KERNEL", raising=False)
        monkeypatch.delenv("JB_QUADRUPED_ABA", raising=False)
        for k, x in (env or {}).items():
            monkeypatch.setenv(k, x)
        sc = scenarios.make("anymal", 2, solver=solver, contact_model=contact_model)
        eng = BatchedEngine(sc.robot, sc.options, 2, api_=api)
        before = eng.describe()
        if force:
            eng.register_impulse_force(base, np.zeros(2), np.full(2, 1e-3), np.zeros((2, 6)))
        return before, eng.describe()

    before, after = describe(False)
    assert after == before and HOT not in after
    for solver in ("runge_kutta_4", "euler_explicit"):
        before, after = describe(True, solver=solver)
        assert after == before.replace("; constraints:", HOT + "; constraints:"), (before, after)
    for kw in (dict(solver="runge_kutta_dopri"), dict(contact_model="constraint"), dict(env={"JB_QUADRUPED_ABA": "1"}),
               dict(env={"JB_NO_FAST_KERNEL": "1"})):
        before, after = describe(True, **kw)
        assert after == before and HOT not in after, kw


def test_reporting(api, monkeypatch):
    reporting(api, monkeypatch)


# ---------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("solver", SOLVERS)
@pytest.mark.parametrize("case", CASES)
def test_gpu_hot_path_matches_full_body(monkeypatch, case, solver):
    hot_vs_full(None, monkeypatch, case, solver)


@pytest.mark.gpu
@pytest.mark.parametrize("in_kernel", [True, False])
@pytest.mark.parametrize("force", ["profile", "process"])
def test_gpu_handoff_with_forces(monkeypatch, force, in_kernel):
    handoff(None, monkeypatch, force, in_kernel)


@pytest.mark.gpu
def test_gpu_reporting(monkeypatch):
    reporting(None, monkeypatch)
