"""The linear FSAL repair of the quadruped hot path (`repair_quadruped_crba`: after a controller update the derivative is
the last evaluation's plus M^-1 dtau) against the full re-evaluation at every controller breakpoint.  The full
re-evaluation is what the hot path runs without the one-call RK4 stage (JB_QUADRUPED_STAGE=0), so the two runs also
differ by the stage form's rounding, which test_quadruped_stage.py bounds with the same tolerances.  Iteration counters
and status words must be equal."""
import numpy as np
import pytest

from jiminy_b200 import scenarios
from jiminy_b200.core import BatchedEngine

from emul import emul_api


@pytest.fixture(scope="module")
def api():
    return emul_api()


def _run(api, monkeypatch, repair, sc, q0, v0, n_steps, actions=None):
    monkeypatch.setenv("JB_QUADRUPED_STAGE", "1" if repair else "0")
    eng = BatchedEngine(sc.robot, sc.options, q0.shape[0], api_=api)
    eng.set_pd_controller(sc.kp, sc.kd)
    eng.set_command(sc.target0)
    eng.start(q0, v0)
    out = []
    for k in range(n_steps):
        eng.set_command(actions(k) if actions else sc.sample_targets(k))
        eng.step(sc.step_dt)
        _, q, v, a = eng.get_state()
        out.append((q.copy(), v.copy(), a.copy(), eng.get_sensors().copy(), eng.get_status().copy(),
                    np.array(eng.get_iters()).copy()))
    return out


def _compare(api, monkeypatch, sc, q0, v0, n_steps, tol, tol_a=None, **kw):
    full = _run(api, monkeypatch, False, sc, q0, v0, n_steps, **kw)
    lin = _run(api, monkeypatch, True, sc, q0, v0, n_steps, **kw)
    for k, (o, n) in enumerate(zip(full, lin)):
        for name, x, y, t in zip(("q", "v", "a", "sensors"), o[:4], n[:4], (tol, tol, tol_a or tol, tol_a or tol)):
            err = np.abs(y - x) / np.maximum(np.abs(x), 1.0)
            assert err.max() <= t, (k, name, err.max())
        np.testing.assert_array_equal(o[4], n[4])
        np.testing.assert_array_equal(o[5], n[5])
    return full, lin


def test_contacts_standing_lifted_separating(api, monkeypatch):
    """Standing (feet in contact), lifted (no contact) and thrown upwards (the feet leave the ground during the step)."""
    sc = scenarios.make("anymal", 3, seed=2)
    q0, v0 = sc.q0.copy(), sc.v0.copy()
    q0[1, 2] += 0.1
    v0[2, 2] = 1.5
    _compare(api, monkeypatch, sc, q0, v0, 3, 1e-12, 1e-9)


def test_effort_limit_and_velocity_taper(api, monkeypatch):
    """Targets far from the measured positions saturate the effort limit; fast joints enter the velocity taper."""
    sc = scenarios.make("anymal", 4, seed=5)
    q0, v0 = sc.q0.copy(), sc.v0.copy()
    v0[2:, 7:] = np.where(np.arange(v0.shape[1] - 7) % 2 == 0, 1.0, -1.0) * 12.0   # leg joints spinning

    def act(k):
        a = sc.sample_targets(k)
        a[::2] += np.where(k % 2 == 0, 2.0, -2.0)                                     # far beyond what the effort limit allows
        return a
    _compare(api, monkeypatch, sc, q0, v0, 3, 1e-9, 1e-7, actions=act)


def test_hip_bounds_fall_back(api, monkeypatch):
    """Every third env driven through its hip bounds: the bound solver runs in those envs' evaluations, so their
    breakpoints take the full evaluation; the others are repaired."""
    sc = scenarios.make("anymal", 6, seed=8)
    rob = sc.robot
    iq = np.array([rob.idx_q[m.joint] for m in rob.motors])
    haa = [k for k, m in enumerate(rob.motors) if "HAA" in m.name]

    def act(k):
        a = sc.sample_targets(k)
        for j in haa:
            a[::3, j] = rob.q_upper[iq[j]] + 0.3
        return a
    full, _ = _compare(api, monkeypatch, sc, sc.q0, sc.v0, 4, 1e-9, actions=act)
    assert (full[-1][4][::3] & 8).all() and not (full[-1][4][1::3] & 8).any()


def test_fifty_env_steps(api, monkeypatch):
    sc = scenarios.make("anymal", 2, seed=1)
    _compare(api, monkeypatch, sc, sc.q0, sc.v0, 50, 1e-9)


@pytest.mark.gpu
def test_gpu_fifty_env_steps(monkeypatch):
    """The same on the device, 256 envs over 50 env-steps."""
    from jiminy_b200 import core
    sc = scenarios.make("anymal", 256, seed=4)
    _compare(core.api(), monkeypatch, sc, sc.q0, sc.v0, 50, 1e-9)
