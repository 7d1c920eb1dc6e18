"""The one-call RK4 stage of the quadruped hot path (`stage_quadruped_crba`, default) against the sequence it replaces
(`make_stage` + `rhs_quadruped_crba` + the accumulator loop, JB_QUADRUPED_STAGE=0), on the warp emulator, from
identical states: the two differ only in rounding (quaternion-form base integrate, products with host reciprocals)."""
import numpy as np
import pytest

from jiminy_b200 import scenarios
from jiminy_b200.core import BatchedEngine

from emul import emul_api


@pytest.fixture(scope="module")
def api():
    return emul_api()


def _run(api, monkeypatch, stage, sc, q0, v0, n_steps, actions=None, env=None):
    monkeypatch.setenv("JB_QUADRUPED_STAGE", "1" if stage else "0")
    for k, x in (env or {}).items():
        monkeypatch.setenv(k, x)
    eng = BatchedEngine(sc.robot, sc.options, q0.shape[0], api_=api)
    assert ("one call per RK4 stage" in eng.describe()) == stage
    eng.set_pd_controller(sc.kp, sc.kd)
    eng.set_command(sc.target0)
    eng.start(q0, v0)
    out = []
    for k in range(n_steps):
        eng.set_command(actions(k) if actions else sc.sample_targets(k))
        eng.step(sc.step_dt)
        _, q, v, a = eng.get_state()
        out.append((q.copy(), v.copy(), a.copy(), eng.get_sensors().copy(), eng.get_status().copy()))
    return out


def _compare(api, monkeypatch, sc, q0, v0, n_steps, tol, tol_a=None, **kw):
    """q, v within `tol`; accelerations and sensors within `tol_a`: through the 4e6 N/m ground a rounding-level change of
    a foot's depth moves them by about that much more."""
    old = _run(api, monkeypatch, False, sc, q0, v0, n_steps, **kw)
    new = _run(api, monkeypatch, True, sc, q0, v0, n_steps, **kw)
    for k, (o, n) in enumerate(zip(old, new)):
        for name, x, y, t in zip(("q", "v", "a", "sensors"), o[:4], n[:4], (tol, tol, tol_a or tol, tol_a or tol)):
            err = np.abs(y - x) / np.maximum(np.abs(x), 1.0)
            assert err.max() <= t, (k, name, err.max())
        np.testing.assert_array_equal(o[4], n[4])
    return old, new


def test_one_env_step(api, monkeypatch):
    sc = scenarios.make("anymal", 8, seed=0)
    _compare(api, monkeypatch, sc, sc.q0, sc.v0, 1, 1e-12, 1e-9)


def test_fifty_env_steps(api, monkeypatch):
    sc = scenarios.make("anymal", 2, seed=1)
    _compare(api, monkeypatch, sc, sc.q0, sc.v0, 50, 1e-9)


def test_contacts_on_off_and_separating(api, monkeypatch):
    """Standing (feet in contact), lifted (no contact) and thrown upwards (the feet leave the ground during the step)."""
    sc = scenarios.make("anymal", 3, seed=2)
    q0, v0 = sc.q0.copy(), sc.v0.copy()
    q0[1, 2] += 0.1
    v0[2, 2] = 1.5
    _compare(api, monkeypatch, sc, q0, v0, 3, 1e-12, 1e-9)


@pytest.mark.parametrize("in_kernel", [True, False])
def test_hip_bounds(api, monkeypatch, in_kernel):
    """Every third env driven through its hip bounds: solved in the evaluation from the W / M_ll^-1 rows the stage
    stores (default), or handed to the full body (JB_NO_FAST_BOUNDS=1)."""
    sc = scenarios.make("anymal", 6, seed=8)
    rob = sc.robot
    iq = np.array([rob.idx_q[m.joint] for m in rob.motors])
    haa = [k for k, m in enumerate(rob.motors) if "HAA" in m.name]

    def act(k):
        a = sc.sample_targets(k)
        for j in haa:
            a[::3, j] = rob.q_upper[iq[j]] + 0.3
        return a
    old, _ = _compare(api, monkeypatch, sc, sc.q0, sc.v0, 4, 1e-9, actions=act,
                      env={} if in_kernel else {"JB_NO_FAST_BOUNDS": "1"})
    assert (old[-1][4][::3] & 8).all() and not (old[-1][4][1::3] & 8).any()


@pytest.mark.parametrize("omega", [40.0, 1e-9, 0.0, 1.220703125e-4 / 5e-4, 1.220703125e-4 / 1e-3])
@pytest.mark.parametrize("flip", [False, True])
def test_base_integrate(api, monkeypatch, omega, flip):
    """Quaternion-form base integrate against integrate_free through one env-step: a fast spin, tiny and zero rates,
    rates whose half-step / full-step rotation is at the Taylor threshold of exp6, and the quaternion with its sign
    flipped."""
    sc = scenarios.make("anymal", 2, seed=3)
    q0, v0 = sc.q0.copy(), sc.v0.copy()
    q0[:, 2] += 0.2                                        # in the air: only the rotation matters
    ax = np.array([0.3, -0.5, 0.8]) / np.linalg.norm([0.3, -0.5, 0.8])
    v0[:, 3:6] = omega * ax
    v0[:, 0:3] = [0.2, -0.1, 0.05]
    if flip:
        q0[:, 3:7] *= -1.0
    _compare(api, monkeypatch, sc, q0, v0, 1, 1e-12, 1e-10)
