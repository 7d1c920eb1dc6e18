"""Parity gate on the GPU (`pytest -m gpu`): the CUDA path, called through the C ABI, against the
oracle on the same seeded inputs (sizes the oracle finishes in seconds), then size-independent
properties at the BASELINE batch size (4096 envs)."""
import numpy as np
import pytest

from jiminy_b200 import robots as R
from jiminy_b200 import scenarios
from jiminy_b200.core import BatchedEngine
from oracle.oracle import OracleBatch

from conftest import DATA
import parity_common as pc

pytestmark = pytest.mark.gpu

# fp64 tolerances: a single RHS agrees to ~1e-15 relative; over an env-step the stiff contact
# (k = 4e6 N/m) amplifies rounding differences, hence the looser trajectory bounds (north-star: 1e-10
# relative on state trajectories).
RHS_TOL = 1e-12
TRAJ_TOL = 1e-9
# one env-step from identical inputs, relative (measured: <= 1e-12 on ANYmal and Atlas, emulator with GPU rounding)
RESYNC_TOL = 1e-11


@pytest.mark.parametrize("name", R.ROBOT_NAMES)
def test_rhs_matches_oracle(name):
    robot, opt = R.load_robot(name)
    opt = R.baseline_options(name, opt)
    rng = np.random.default_rng(11)
    n = 100
    q, v = pc.random_states(robot, n, rng)
    cmd = rng.uniform(-20, 20, size=(n, max(robot.nmotors, 1)))
    a0, f0, u0 = OracleBatch(robot, opt, n).compute_dynamics(q, v, cmd)
    a1, f1, u1 = BatchedEngine(robot, opt, n).compute_dynamics(q, v, cmd)
    np.testing.assert_allclose(a1, a0, rtol=0, atol=RHS_TOL * max(1.0, np.abs(a0).max()))
    np.testing.assert_allclose(f1, f0, rtol=0, atol=RHS_TOL * max(1.0, np.abs(f0).max()))
    np.testing.assert_allclose(u1, u0, rtol=0, atol=RHS_TOL)


@pytest.mark.parametrize("name,n_env,n_steps", [("anymal", 96, 5), ("atlas", 40, 3), ("cartpole", 512, 50),
                                               ("double_pendulum", 1, 300)])
def test_env_steps_match_oracle(name, n_env, n_steps):
    tol = 1e-13 if name in ("cartpole", "double_pendulum") else TRAJ_TOL
    pc.run_scenario(name, n_env, n_steps, tol_state=tol, tol_sens=max(tol, 1e-7) if tol > 1e-12 else 1e-11)


def test_masked_restart():
    sc = scenarios.make("anymal", 70)
    eng, orc = pc.make_pair(sc)
    for k in range(2):
        eng.step(sc.step_dt)
        orc.step(sc.step_dt, parallel=True)
    mask = (np.arange(70) % 3 == 0).astype(np.uint8)
    eng.start(sc.q0, sc.v0, mask=mask)
    orc.start(sc.q0, sc.v0, mask=mask)
    eng.step(sc.step_dt)
    orc.step(sc.step_dt, parallel=True)
    pc.compare(eng, orc, TRAJ_TOL, 1e-6)


def test_full_size_properties():
    """4096 ANYmal envs: (i) bit-determinism across runs, (ii) env permutation invariance -- an env's
    trajectory does not depend on its position in the batch or on its warp neighbours, (iii) no env
    leaves the well-posed regime, (iv) a sampled subset agrees with the oracle."""
    n = 4096
    sc = scenarios.make("anymal", n)
    perm = np.random.default_rng(0).permutation(n)

    def run(order):
        eng = BatchedEngine(sc.robot, sc.options, n)
        eng.set_pd_controller(sc.kp, sc.kd)
        eng.set_command(sc.target0[order])
        eng.start(sc.q0[order], sc.v0[order])
        for k in range(3):
            eng.set_command(sc.sample_targets(k)[order])
            eng.step(sc.step_dt)
        return eng.get_state(), eng.get_sensors().copy(), eng.get_status()
    (t1, q1, v1, a1), s1, st1 = run(np.arange(n))
    (t2, q2, v2, a2), s2, st2 = run(np.arange(n))
    assert np.array_equal(q1, q2) and np.array_equal(v1, v2) and np.array_equal(s1, s2)       # (i)
    (t3, q3, v3, a3), s3, st3 = run(perm)
    assert np.array_equal(q3, q1[perm]) and np.array_equal(v3, v1[perm]) and np.array_equal(s3, s1[perm])   # (ii)
    assert (st1 == 0).all() and np.isfinite(q1).all()                                         # (iii)
    np.testing.assert_allclose(t1, 0.12, atol=1e-15)
    idx = np.arange(0, n, 64)                                                                 # (iv)
    orc = OracleBatch(sc.robot, sc.options, len(idx))
    orc.set_pd_controller(sc.kp, sc.kd)
    orc.set_command(sc.target0[idx])
    assert not orc.start(sc.q0[idx], sc.v0[idx]).any()
    for k in range(3):
        orc.set_command(sc.sample_targets(k)[idx])
        orc.step(sc.step_dt, parallel=True)
    _, q0, v0, _ = orc.get_state()
    np.testing.assert_allclose(q1[idx], q0, rtol=0, atol=TRAJ_TOL)
    np.testing.assert_allclose(v1[idx], v0, rtol=0, atol=TRAJ_TOL * max(1.0, np.abs(v0).max()))


def test_graft_smoke():
    import __graft_entry__ as g
    g.smoke()


def test_dopri_adaptive_matches_oracle():
    """Per-env adaptive Dormand-Prince on the device (config 1's solver): accepted and rejected step
    counts equal the oracle's for every env, states agree to 1e-9."""
    robot, opt = R.load_robot("double_pendulum")
    opt = R.baseline_options("double_pendulum", opt)
    opt["stepper"].update(odeSolver="runge_kutta_dopri", tolAbs=1e-9, tolRel=1e-9, dtMax=0.02,
                          sensorsUpdatePeriod=1e-3, controllerUpdatePeriod=1e-3)
    n = 64
    rng = np.random.default_rng(4)
    q0, v0 = rng.uniform(-1.0, 1.0, size=(n, 2)), rng.uniform(-2.0, 2.0, size=(n, 2))
    eng, orc = BatchedEngine(robot, opt, n), OracleBatch(robot, opt, n)
    eng.start(q0, v0)
    assert not orc.start(q0, v0).any()
    for _ in range(25):
        eng.step(0.02)
        assert not orc.step(0.02, parallel=True).any()
    pc.compare(eng, orc, 1e-9, 1e-8)
    np.testing.assert_array_equal(eng.get_iters()[1], orc.get_iters()[1])
    # ANYmal with the engine's default adaptive solver
    sc = scenarios.make("anymal", 16, solver="runge_kutta_dopri", dt_max=0.02)
    eng, orc = pc.make_pair(sc)
    for k in range(2):
        eng.set_command(sc.sample_targets(k)); orc.set_command(sc.sample_targets(k))
        eng.step(sc.step_dt)
        assert not orc.step(sc.step_dt, parallel=True).any()
    pc.compare(eng, orc, 1e-7, 1e-5)


def test_cuda_path_vs_closed_forms():
    """The reference's analytical tests run on the CUDA path directly: rotor inertia + spring vs expm,
    prismatic chain vs expm, contact equilibrium / sensors / friction steady state, energy conservation."""
    import analytic_device as ad
    ad.armature_spring()
    ad.joint_position_limits()
    ad.foot_pendulum(t_end=0.02)                 # (2000 RK4 steps of a single env: the full second is run on the oracle)
    ad.velocity_bounds()
    ad.two_masses()
    ad.contact_equilibrium_and_friction()
    ad.energy_conservation()
    ad.force_impulse()
    ad.constraint_closed_forms()


def test_external_forces_match_oracle():
    """Impulse + profile forces (Engine::computeExternalForces, impulse breakpoints) on 70 ANYmal envs."""
    pc.external_forces_scenario(None, n_env=70, n_steps=4)


@pytest.mark.parametrize("model", ["spring_damper", "constraint"])
def test_joint_bounds_constraint_path(model):
    pc.bounds_scenario(None, DATA, model)


def test_start_on_joint_bounds():
    pc.start_on_bounds_scenario(None, DATA)


def test_constraint_contact_matches_oracle():
    """contacts.model = "constraint" (boxed PGS): point mass (rest / slide / spin, torsion), 40 ANYmal envs,
    Atlas (78 constraint rows at most)."""
    pc.point_mass_constraint_scenario(None, DATA)
    pc.point_mass_constraint_scenario(None, DATA, n_steps=15, torsion=0.05)
    eng, orc, sc = pc.robot_constraint_scenario("anymal", 40, 3, seed=2)
    assert (eng.get_state()[1][:, 2] > 0.4).all()
    pc.robot_constraint_scenario("atlas", 6, 1, seed=1, tol_state=1e-7, tol_sens=1e-5)


@pytest.mark.parametrize("robot,toggle", [("atlas", None), ("atlas", "JB_NO_BODY_CONS"), ("atlas", "JB_NO_BLOCK_CONS"),
                                          ("anymal", "JB_NO_STRUCTURED_CONS"), ("atlas", "torsion")])
def test_constraint_solver_variants(monkeypatch, robot, toggle):
    """Every device formulation of the constraint solve against the oracle (see tests/test_kernel_emul.py), 24 envs."""
    torsion = 0.05 if toggle == "torsion" else None      # torsional friction block of the sweep
    if toggle and torsion is None:
        monkeypatch.setenv(toggle, "1")
    eng, orc, sc = pc.robot_constraint_scenario(robot, 24, 2, seed=3, torsion=torsion, solver="euler_explicit", dt_max=0.005, tol_state=1e-7, tol_sens=1e-5)
    want = {None: "body-space", "JB_NO_BODY_CONS": "lane-block", "JB_NO_BLOCK_CONS": "generic", "JB_NO_STRUCTURED_CONS": "body-space", "torsion": "body-space"}[toggle]
    assert want in eng.describe()


@pytest.mark.parametrize("robot", ["atlas", "anymal"])
def test_masked_restart_with_constraint_contacts(robot):
    pc.masked_restart_constraint_scenario(None, robot, n_env=21, tol_state=1e-7, tol_sens=1e-5)


def test_atlas_pd_standing_like_the_reference_test():
    """gym_jiminy/unit_py/test_pipeline_control.py:46-113 on the device: 9 s of zero target velocities, then every
    generalised velocity of the last second below 1e-3 (and the final state equal to the oracle's)."""
    v_dev, v_orc, sc = pc.atlas_pd_standing_on_device(None, 9.0, tol_state=1e-6)
    last = int(round(1.0 / sc.step_dt))
    assert np.all(v_dev[-last:] < 1.0e-3), v_dev[-last:].max()


def test_restart_is_exactly_repeatable():
    pc.atlas_repeatability_scenario(None, n_env=9)


def test_atlas_bounds_and_contacts_together():
    pc.atlas_bounds_and_contacts_scenario(None, n_env=16, n_steps=8, tol_state=1e-7, tol_sens=1e-5)


def test_constraint_solvers_agree_at_scale():
    """1024 ANYmal envs with the constraint contact model: the structured quadruped solver and the generic dense
    solver (two independent formulations of the same boxed LCP) give the same trajectories; bit-identical when
    repeated; nobody falls or fails."""
    import os
    sc = scenarios.make("anymal", 1024, seed=4, contact_model="constraint")
    runs = []
    for mode in ("0", "0", "1"):
        os.environ["JB_NO_STRUCTURED_CONS"] = mode
        try:
            eng = BatchedEngine(sc.robot, sc.options, sc.n_env)
        finally:
            os.environ.pop("JB_NO_STRUCTURED_CONS", None)
        assert ("structured" in eng.describe()) == (mode == "0")
        eng.set_pd_controller(sc.kp, sc.kd)
        eng.set_command(sc.target0)
        eng.start(sc.q0, sc.v0)
        for k in range(3):
            eng.set_command(sc.sample_targets(k))
            eng.step(sc.step_dt)
        t, q, v, a = eng.get_state()
        assert not eng.get_status().any()
        runs.append((q.copy(), v.copy(), eng.get_sensors().copy()))
    np.testing.assert_array_equal(runs[0][0], runs[1][0])
    np.testing.assert_array_equal(runs[0][2], runs[1][2])
    np.testing.assert_allclose(runs[0][0], runs[2][0], rtol=0, atol=1e-8)
    np.testing.assert_allclose(runs[0][1], runs[2][1], rtol=0, atol=1e-6)
    assert (runs[0][0][:, 2] > 0.4).all()


@pytest.mark.parametrize("name,n_env,n_steps,free_tol", [("anymal", 64, 250, 1e-10), ("atlas", 16, 50, None)])
def test_long_horizon_resynchronised(name, n_env, n_steps, free_tol):
    """The full BASELINE horizon (ANYmal: 250 env-steps = 10 s), compared step by step from identical inputs (the device
    is handed the oracle's state after every env-step): the error the CUDA path adds per env-step stays at rounding
    level all along the trajectory.  For ANYmal the FREE-RUNNING device trajectory (never re-synchronised) must also
    stay within north-star's 1e-10 relative of the oracle over the whole horizon; for Atlas on the stiff spring-damper
    ground the free-running deviation is recorded only (it is amplified by the dynamics, not produced by the path)."""
    resync, free = pc.resync_long_horizon_scenario(name, n_env, n_steps, tol_rel=RESYNC_TOL)
    print(f"{name}: one-step (re-synchronised) max {resync.max():.2e}; free-running after {n_steps} env-steps {free[-1].max():.2e}, "
          f"max over the horizon {free.max():.2e}")
    if free_tol is not None:
        assert free.max() <= free_tol, free.max()


@pytest.mark.parametrize("safety", [False, True])
def test_pd_controller_block(safety):
    """Device-side PDController (+ MotorSafetyLimit) block vs the oracle restatement (pinned by golden vectors of the
    reference's own functions), 64 ANYmal envs."""
    pc.pd_block_scenario(None, n_env=64, n_steps=4, safety=safety)


@pytest.mark.parametrize("order,instantaneous", [(0, False), (1, True)])
def test_pd_adapter_pipeline(order, instantaneous):
    pc.pd_adapter_scenario(None, n_env=40, n_steps=4, order=order, instantaneous=instantaneous)


@pytest.mark.parametrize("in_kernel", [True, False])
def test_joint_bounds_at_scale(monkeypatch, in_kernel):
    """600 ANYmal envs, every third pushed into its joint bounds: solved inside the hot-path evaluation, or (the path of
    every robot without a static signature) aborted and replayed by the full body inside the same launch."""
    if not in_kernel:
        monkeypatch.setenv("JB_NO_FAST_BOUNDS", "1")
    pc.bounds_handoff_scenario(None, n_env=600, n_steps=5)


@pytest.mark.parametrize("in_kernel", [True, False])
def test_handoff_with_stateful_blocks_at_scale(monkeypatch, in_kernel):
    if not in_kernel:
        monkeypatch.setenv("JB_NO_FAST_BOUNDS", "1")
    pc.stateful_handoff_scenario(None, n_env=300, n_steps=7)


def test_mahony_filter_observer():
    pc.mahony_scenario(None, "anymal", n_env=70, n_steps=4)
    pc.mahony_scenario(None, "atlas", n_env=5, n_steps=1)


# ---- the single-env `Engine` facade on the CUDA library (the same test bodies the CPU suite runs on the emulator)
def test_engine_facade_python_controller_on_device():
    import test_kernel_emul as tke
    tke.test_engine_facade_python_controller(None)


def test_engine_facade_forces_on_device():
    import test_kernel_emul as tke
    tke.test_engine_facade_impulse_forces(None)
    tke.test_engine_facade_profile_force_function(None)


def test_engine_facade_telemetry_log_on_device(tmp_path):
    import test_kernel_emul as tke
    tke.test_engine_facade_telemetry_log(None, tmp_path)


def test_batched_env_reset_step_autoreset_on_device():
    import test_kernel_emul as tke
    tke.test_batched_env_reset_step_autoreset(None)
    tke.test_pd_control_pipeline_env(None)


def test_sensor_measurement_pipeline_matches_oracle():
    """Delay ring / jitter / white noise / bias of every sensor type on the device against the oracle's restatement
    (abstract_sensor.hxx:305-522): identical noise draws, delayed values within the physics tolerance; restart of one env
    with the same seed reproduces its noise."""
    import sensor_pipeline_common as spc
    spc.pipeline_scenario(None, n_env=48, n_steps=3)


@pytest.mark.gpu
def test_state_views_on_device():
    import test_kernel_emul as tke
    tke.test_state_views_are_stable_and_current(None)


@pytest.mark.gpu
def test_model_variants_on_device():
    import test_kernel_emul as tke
    tke.test_model_variants_match_per_variant_oracles(None)



def test_flexibility_joints_on_device():
    """Flexibility joints (spherical records, Engine::computeInternalDynamics engine.cc:3367-3391): the reference's
    series-elastic-actuator test on the CUDA path (closed form + oracle, adaptive steps), the flexible branched arm with
    RK4 and Dormand-Prince, and ANYmal with a flexibility in every leg."""
    import flexibility_common as fc
    assert fc.series_elastic_actuator() < 1e-10
    fc.branched_arm_parity()
    fc.branched_arm_parity(solver="runge_kutta_dopri")
    fc.flexible_anymal_parity(n_env=70, n_steps=2)
    # ... and through the constraint path (generic solver): joint bounds behind a flexibility, constraint contacts
    for model in ("spring_damper", "constraint"):
        fc.flexible_pendulum_on_its_bounds(model=model)
    fc.flexible_anymal_parity(n_env=40, n_steps=2, contact_model="constraint", tol_state=1e-8, tol_sens=1e-6)


def test_backlash_joints_on_device():
    """Transmission backlash (robot.cc:582-629): free play, impact and locked motion of the reference's `test_backlash`
    system on the CUDA path against the oracle."""
    import flexibility_common as fc
    fc.backlash_pendulum_parity()
