"""Whole-robot dynamics, contact wrenches, efforts, sensors and `computeExtraTerms` outputs against the extended-precision
first-principles reference of tests/first_principles.py (FK composition + finite differences + Newton-Euler per body).

Every check runs on three implementations: the kernel source under the warp emulator (CPU suite), the CUDA library
(`-m gpu`, same function bodies) and the oracle -- so that an error the kernel and the oracle share shows which side
is wrong.  Sensor noise, delay and bias stay off.

Limits, from the measured values printed by the tests (worst over all robots and paths):
* equation-of-motion residual ||M a + h - u - sum J^T f||_inf / scale <= 1e-12: double-precision evaluations give
  < 2e-16, a wrong term of the dynamics gives >= 1e-6;
* forward error ||a - a_ref||_inf / max(1, ||a_ref||_inf) <= 64 cond(M) eps, a_ref = M^-1 (u + sum J^T f - h) from the
  reference laws: the measured values stay below 1.5 cond(M) eps (cond(M) up to 2.2e3 on Atlas);
* contact wrenches, efforts and sensors: 1e-12 relative to the largest value of the quantity (1e-10 for sensors, each
  type against its own largest value); contact wrenches also allow the stiffness times the double rounding of the
  contact position (`check_wrenches`).  The measured errors are at rounding level.
"""
import os

import numpy as np
import pytest

import first_principles as fp
from jiminy_b200 import model as M
from jiminy_b200 import robots as R
from jiminy_b200 import scenarios
from jiminy_b200.core import BatchedEngine
from oracle.oracle import OracleBatch

from conftest import DATA, has_cuda
import parity_common as pc

RESIDUAL_TOL = 1e-12
WRENCH_TOL = 1e-12
EPS64 = float(np.finfo(np.float64).eps)
FORWARD_FACTOR = 64.0       # measured: <= 1.5 (emulator, oracle and H100)
IMPLS = ["emul", "oracle", pytest.param("gpu", marks=pytest.mark.gpu)]


def _engine(impl, robot, opt, n):
    if impl == "oracle":
        return OracleBatch(robot, opt, n)
    if impl == "gpu":
        if not has_cuda():
            pytest.skip("no CUDA device")
        return BatchedEngine(robot, opt, n)
    from emul import emul_api
    return BatchedEngine(robot, opt, n, api_=emul_api())


def _start(eng, q, v):
    st = eng.start(q, v)
    assert st is None or not np.asarray(st).any()


def _step(eng, dt):
    st = eng.step(dt) if isinstance(eng, BatchedEngine) else eng.step(dt, parallel=True)
    assert st is None or not np.asarray(st).any()


# --------------------------------------------------------------------------- robots
def _branched_arm():
    robot = M.build_robot_table(os.path.join(DATA, "branched_arm.urdf"), True)
    robot.add_contact_points(["b_sole", "a_tool"])
    for jn in ("a_shoulder", "a_elbow", "a_spin", "b_hip", "b_slide", "b_skew_slide", "b_ankle_z", "c_spin_skew"):
        M.attach_motor(robot, jn, jn, enableVelocityLimit=(jn == "b_hip"), velocityEffortInvSlope=0.05,
                       enableArmature=True, armature=0.01 * (1 + len(jn) % 3), enableFriction=(jn == "a_elbow"),
                       frictionViscousPositive=-0.1, frictionViscousNegative=-0.2, frictionDryPositive=-0.05,
                       frictionDryNegative=-0.07, frictionDrySlope=3.0)
        M.attach_sensor(robot, "EncoderSensor", jn, motor_name=jn)
        M.attach_sensor(robot, "EffortSensor", jn, motor_name=jn)
    # an IMU and a force sensor away from their joint origin, rotated, on moving bodies
    robot.add_frame("imu_off", "a_hand", M.SE3(M.rpy_to_matrix([0.3, -0.4, 0.7]), np.array([0.05, -0.03, 0.08])))
    robot.add_frame("force_off", "b_toe", M.SE3(M.rpy_to_matrix([-0.5, 0.2, 1.1]), np.array([-0.04, 0.06, 0.03])))
    M.attach_sensor(robot, "ImuSensor", "imu", frame_name="imu_off")
    M.attach_sensor(robot, "ForceSensor", "sole", frame_name="force_off")
    M.attach_sensor(robot, "ContactSensor", "sole_c", frame_name="b_sole")
    opt = M.default_engine_options()
    opt["contacts"].update(model="spring_damper", stiffness=1e5, damping=5e2, transitionEps=2e-3, transitionVelocity=1e-2)
    opt["stepper"].update(odeSolver="runge_kutta_4", dtMax=5e-4, sensorsUpdatePeriod=2e-3, controllerUpdatePeriod=2e-3)
    return robot, opt


def _with_offset_sensors(robot):
    """ANYmal with its IMU moved on the base and its LF force sensor moved on the shank, both off their joint origin and rotated."""
    base = "base" if "base" in robot.frames else "root_joint"
    robot.add_frame("imu_off", base, M.SE3(M.rpy_to_matrix([0.4, 0.3, -0.6]), np.array([0.12, -0.07, 0.05])))
    robot.imu_frames[0] = "imu_off"
    shank = next(n for n in robot.frames if "SHANK" in n.upper() and n.upper().startswith("LF"))
    robot.add_frame("force_off", shank, M.SE3(M.rpy_to_matrix([-0.3, 0.6, 0.2]), np.array([0.03, 0.05, -0.1])))
    k = next(i for i, f in enumerate(robot.force_frames) if f.upper().startswith("LF"))
    assert robot.frames[robot.force_frames[k]].joint == robot.frames["force_off"].joint
    robot.force_frames[k] = "force_off"
    return robot


def _robot(name):
    """(robot, options) of every robot of the RHS checks."""
    if name in R.ROBOT_NAMES:
        robot, opt = R.load_robot(name)
        return robot, R.baseline_options(name, opt)
    if name == "branched_arm":
        return _branched_arm()
    if name == "anymal_flexible":
        sc = scenarios.make("anymal_flexible", 1)
        return sc.robot, sc.options
    if name == "atlas_flexible_trunk":
        sc = scenarios.make("atlas", 1, seed=1)
        cfg = [dict(frameName=jn, stiffness=[8e3, 9e3, 7e3], damping=[40.0, 30.0, 35.0], inertia=[0.2, 0.3, 0.25])
               for jn in ("back_bky", "l_leg_kny", "r_arm_shx")]
        return M.add_flexibility_joints(sc.robot, cfg), sc.options
    if name == "anymal_variant":
        sc = scenarios.make("anymal", 1, seed=6)
        rng = np.random.default_rng(11)
        return M.biased_robot(sc.robot, rng, mass_std=0.05, com_std=0.05, inertia_std=0.05, relative_position_std=0.002), sc.options
    raise KeyError(name)


def _model(robot, opt):
    frames = list(robot.contact_frame_names) + list(robot.imu_frames) + list(robot.force_frames)
    return fp.Model(robot, opt["world"]["gravity"], frames=frames)


# --------------------------------------------------------------------------- states
def _base_quat(axis, angle):
    axis = np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis)
    return np.concatenate([np.sin(angle / 2) * axis, [np.cos(angle / 2)]])


def _states(robot, opt, m, rng):
    """Random states, then the edges: quaternion sign flipped, base upside down (w ~ 0), spinning, unbounded revolute
    angles on either side of +-pi, contacts above / at / below the ground, sliding slower / faster than
    transitionVelocity at depths below / above transitionEps, a separating contact whose damping cancels the spring."""
    q, v = pc.random_states(robot, 2, rng, base_height=0.6)
    out = [(q[0], v[0]), (q[1], v[1] * 4.0)]
    ff = robot.has_freeflyer and int(robot.joint_type[1]) == M.JB_JOINT_FREEFLYER
    unb = [j for j in range(1, robot.njoints) if int(robot.joint_type[j]) in fp.UNBOUNDED]
    if ff:
        x = q[0].copy()
        x[3:7] = -x[3:7]
        out.append((x, v[0]))                                            # same rotation, other sign
        x = q[1].copy()
        x[2] += 1.0
        x[3:7] = _base_quat([1.0, 0.3, 0.0], np.pi - 2e-3)              # upside down, w ~ 1e-3
        out.append((x, v[1]))
    vs = v[0].copy()
    vs[:] = rng.uniform(-25.0, 25.0, size=robot.nv)                     # fast joints; gyroscopic terms dominate
    if ff:
        vs[3:6] = rng.normal(size=3)
        vs[3:6] *= 45.0 / np.linalg.norm(vs[3:6])
    out.append((q[1].copy(), vs))
    if unb:
        x = q[0].copy()
        for s, j in enumerate(unb):
            ang = np.pi - 1e-3 if s % 2 == 0 else -np.pi + 1e-3
            x[robot.idx_q[j]:robot.idx_q[j] + 2] = np.cos(ang), np.sin(ang)
        out.append((x, v[1]))
    nc = len(robot.contact_frame_names)
    if ff and nc:
        c = opt["contacts"]
        eps, tv = c["transitionEps"], c["transitionVelocity"]
        k, d = c["stiffness"], c["damping"]
        base = q[0].copy()
        base[3:7] = _base_quat([0.2, -0.3, 1.0], 0.4) * (1 if rng.uniform() > 0.5 else -1)
        z = min(float(p[1][2]) for p in m.fk(m.config(base))[m.nj:m.nj + nc])
        Rb = np.array([[float(e) for e in r] for r in fp.quat_to_rot(*[fp.mpf(t) for t in base[3:7]])])
        # depth 0.0: the lowest contact point on the surface to double rounding (|depth| ~ 1e-17, either sign), where
        # the force must vanish continuously
        for depth, slide, vz in ((0.01, 0.0, 0.0), (0.0, 0.5 * tv, 0.0), (-0.3 * eps, 0.3 * tv, -0.01),
                                 (-3.0 * eps, 3.0 * tv, 0.02), (-0.3 * eps, 2.0 * tv, 2.0 * 0.3 * eps * k / d)):
            x = base.copy()
            x[2] += depth - z
            vw = np.array([slide * 0.6, slide * 0.8, vz])
            y = np.zeros(robot.nv)
            y[0:3] = Rb.T @ vw                                               # free-flyer velocity: base frame
            out.append((x, y))
    return out


_CACHE = {}


def _reference_states(name):
    """Per robot: (robot, options, model, [(q, v, cmd, fp.State)]), computed once for the three implementations."""
    if name not in _CACHE:
        robot, opt = _robot(name)
        m = _model(robot, opt)
        rng = np.random.default_rng(sum(name.encode()))
        sts = []
        for q, v in _states(robot, opt, m, rng):
            cmd = rng.uniform(-30, 30, size=max(robot.nmotors, 1))
            sts.append((q, v, cmd, fp.State(m, q, v)))
        _CACHE[name] = (robot, opt, m, sts)
    return _CACHE[name]


# --------------------------------------------------------------------------- checks
def check_residual(st, a, u, fext):
    r, scale = st.residual(a, u, fext)
    res = float(max(abs(x) for x in r) / scale)
    assert res <= RESIDUAL_TOL, f"equation-of-motion residual {res:.3e}"
    return res


def check_forward(st, a, u_ref, fext_ref):
    gf = st.generalized_force(fext_ref)
    rhs = [fp.mpf(float(x)) + g - h for x, g, h in zip(u_ref, gf, st.h)]
    a_ref = fp.to_np(st.solve(rhs))
    err = float(np.abs(a - a_ref).max() / max(1.0, np.abs(a_ref).max()))
    cond = float(np.linalg.cond(st.M_np()))
    assert err <= FORWARD_FACTOR * cond * EPS64, f"forward error {err:.3e} (cond(M) = {cond:.2e})"
    return err, cond


def expected_contacts(st, robot, opt):
    fe, forces = fp.contact_wrenches(st, opt, range(len(robot.contact_frame_names)))
    return np.array([[float(x) for x in row] for row in fe]), forces


def check_wrenches(fext, fe, opt):
    """Contact wrenches to WRENCH_TOL relative, plus what the stiff law makes of the rounding of its inputs: a double
    FK knows a contact point to ~32 eps of its distance from the origin (a few metres at most), i.e. the stiffness times
    ~1e-14 m on the normal force (4e-8 N at 4e6 N/m; measured up to 4e-10 N)."""
    scale = max(1.0, np.abs(fe).max())
    err = float(np.abs(fext - fe).max() / scale)
    assert err <= WRENCH_TOL + opt["contacts"]["stiffness"] * 32 * EPS64 * 3.0 / scale, \
        f"contact wrenches off by {err:.3e} (largest {scale:.3e})"
    return err


def expected_efforts(robot, q, v, cmd):
    u, um = fp.motor_efforts(robot, v, cmd)
    return u + fp.to_np(fp.flexibility_efforts(robot, q, v)), um


def check_efforts(robot, u, u_ref):
    np.testing.assert_allclose(u, u_ref, rtol=0, atol=1e-12 * max(1.0, np.abs(u_ref).max()))
    if robot.has_freeflyer and int(robot.joint_type[1]) == M.JB_JOINT_FREEFLYER:
        assert np.all(u[0:6] == 0.0), "free-flyer efforts must be exactly zero"


RHS_ROBOTS = list(R.ROBOT_NAMES) + ["branched_arm", "anymal_flexible", "atlas_flexible_trunk", "anymal_variant"]


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("name", RHS_ROBOTS)
def test_one_rhs_against_first_principles(impl, name):
    """One full-body right-hand side (`compute_dynamics`) on random and edge states: equation-of-motion residual with
    the implementation's own (a, u, fext), forward error against M^-1 (u + J^T f - h), contact wrenches from the
    spring-damper law at the reference's depth and contact-point velocity, efforts from the motor / flexibility laws."""
    robot, opt, m, sts = _reference_states(name)
    n = len(sts)
    q = np.stack([s[0] for s in sts])
    v = np.stack([s[1] for s in sts])
    cmd = np.stack([s[2] for s in sts])
    if name == "anymal_variant" and impl != "oracle":
        base = scenarios.make("anymal", 1, seed=6).robot
        eng = _engine(impl, base, opt, n)
        eng.set_model_variants([base, robot], np.ones(-(-n // eng.envs_per_group), dtype=np.int32))
    else:
        eng = _engine(impl, robot, opt, n)
    a, fext, u = eng.compute_dynamics(q, v, cmd)
    worst = [0.0, 0.0, 0.0, 0.0]
    pen = 0
    for e, (qe, ve, ce, st) in enumerate(sts):
        fe, forces = expected_contacts(st, robot, opt)
        pen += sum(1 for F in forces if F[2] > 0)
        u_ref, _ = expected_efforts(robot, qe, ve, ce)
        res = check_residual(st, a[e], u[e], fext[e])
        err, cond = check_forward(st, a[e], u_ref, fe)
        werr = check_wrenches(fext[e], fe, opt)
        check_efforts(robot, u[e], u_ref)
        worst = [max(worst[0], res), max(worst[1], err / (cond * EPS64)), max(worst[2], cond), max(worst[3], werr)]
    if robot.contact_frame_names and robot.has_freeflyer:
        assert pen > 0                                       # some states really load the contacts
    print(f"{impl} {name}: residual {worst[0]:.2e}, forward error / (cond(M) eps) {worst[1]:.2f} (cond(M) <= {worst[2]:.1e}), wrenches {worst[3]:.2e}")


# --------------------------------------------------------------------------- the state a step ends on
def expected_sensors(st, robot, opt, a, um, forces):
    """Sensor row of the accepted state: IMU (gyroscope = angular velocity in the IMU frame, accelerometer =
    R_imu^T (pddot_imu - g) on the path of (v, a)), force sensors (wrench of the contacts of the sensor's joint about
    the sensor origin, in the sensor frame), encoders, effort sensors, contact sensors (contact force, contact frame)."""
    m, nj = st.m, st.m.nj
    nc, ni = len(robot.contact_frame_names), len(robot.imu_frames)
    lay = robot.sensor_layout()
    row = np.zeros(lay["width"][0])
    acc = st.accelerations(a)
    g = m.gravity[0:3]
    for k in range(ni):
        f = nj + nc + k
        w = st.V[f][3:6]
        lin_acc = fp.sub(acc[f][2], fp.tvec(st.T[f][0], g))
        for e, x in enumerate(w + lin_acc):
            row[lay["ImuSensor"][0] + e * ni + k] = float(x)
    nfs = len(robot.force_frames)
    for k in range(nfs):
        f = nj + nc + ni + k
        js = m.frames[nc + ni + k][0]
        lin, ang = [fp.ZERO] * 3, [fp.ZERO] * 3
        for c in range(nc):
            if m.frames[c][0] == js:
                lin = fp.add(lin, forces[c])
                ang = fp.add(ang, fp.cross(fp.sub(st.world_point(nj + c), st.world_point(f)), forces[c]))
        for e, x in enumerate(fp.tvec(st.T[f][0], lin) + fp.tvec(st.T[f][0], ang)):
            row[lay["ForceSensor"][0] + e * nfs + k] = float(x)
    ne = len(robot.encoder_names)
    for k, (j, red) in enumerate(zip(robot.encoder_joints, robot.encoder_reduction)):
        iq, iv = int(robot.idx_q[j]), int(robot.idx_v[j])
        pos = np.arctan2(st.q[iq + 1], st.q[iq]) if int(robot.joint_type[j]) in fp.UNBOUNDED else st.q[iq]
        row[lay["EncoderSensor"][0] + k] = pos * red
        row[lay["EncoderSensor"][0] + ne + k] = st.v[iv] * red
    for k, mi in enumerate(robot.effort_motors):
        row[lay["EffortSensor"][0] + k] = um[mi]
    ncs = len(robot.contact_sensor_names)
    for k, c in enumerate(robot.contact_sensor_index):
        for e, x in enumerate(fp.tvec(st.T[nj + c][0], forces[c])):
            row[lay["ContactSensor"][0] + e * ncs + k] = float(x)
    return row, acc


def expected_extra_terms(st, robot, a, fext):
    """computeExtraTerms (engine.cc:800-905) from the first-principles quantities: kinetic energy 1/2 v^T M v, potential
    energy -sum m g.c (Pinocchio's sign), joint spatial accelerations (local frame, gravity-free), joint internal
    wrenches sum over the subtree of I (a - g) + v x* I v - fext (gravity included, external forces removed), subtree
    mass / centre of mass / its velocity, centroidal momentum and its derivative about com[0], which is the centre of mass
    of the subtree of joint 1 (engine.cc:898)."""
    m, nj, nv = st.m, st.m.nj, st.m.nv
    vm = st.vm
    kin = sum(vm[k] * st.M[k][l] * vm[l] for k in range(nv) for l in range(nv)) / 2
    g = m.gravity[0:3]
    pot = fp.ZERO
    for b in range(1, nj):
        c = fp.add(st.T[b][1], fp.mvec(st.T[b][0], m.lever[b]))
        pot -= m.mass[b] * fp.dot(g, c)
    acc = st.accelerations(a)
    ja, body_f, body_dh, body_h = [[0.0] * 6], [None], [None], [None]
    for b in range(1, nj):
        lin, w, cl, wd = acc[b]
        alpha = fp.sub(cl, fp.cross(w, lin)) + wd
        ja.append([float(x) for x in alpha])
        Vb = st.V[b]
        Iv = fp.inertia_apply(m.mass[b], m.lever[b], m.Ic[b], Vb)
        gyro = fp.force_cross(Vb, Iv)
        gb = fp.tvec(st.T[b][0], m.gravity[0:3]) + fp.tvec(st.T[b][0], m.gravity[3:6])
        fa = fp.inertia_apply(m.mass[b], m.lever[b], m.Ic[b], alpha)
        fg = fp.inertia_apply(m.mass[b], m.lever[b], m.Ic[b], [x - y for x, y in zip(alpha, gb)])
        body_f.append([x + y - fp.mpf(float(z)) for x, y, z in zip(fg, gyro, fext[b])])
        body_dh.append([x + y for x, y in zip(fa, gyro)])
        body_h.append(Iv)
    world = (fp.eye3(), [fp.ZERO] * 3)
    jf = [[0.0] * 6]
    for i in range(1, nj):
        tot = [fp.ZERO] * 6
        for b in range(1, nj):
            if i in m.ancestors[b]:
                tot = [x + y for x, y in zip(tot, fp.transport_wrench(st.T[i], st.T[b], body_f[b]))]
        jf.append([float(x) for x in tot])
    # subtree of joint 1: mass, centre of mass (world), momentum and its rate about the world origin
    sub1 = [b for b in range(1, nj) if 1 in m.ancestors[b]]
    mass = sum(m.mass[b] for b in sub1)
    com0 = [fp.ZERO] * 3
    for b in sub1:
        com0 = fp.add(com0, fp.scl(m.mass[b], fp.add(st.T[b][1], fp.mvec(st.T[b][0], m.lever[b]))))
    com0 = fp.scl(1 / mass, com0)
    h0, dh0 = [fp.ZERO] * 6, [fp.ZERO] * 6
    for b in range(1, nj):
        h0 = [x + y for x, y in zip(h0, fp.transport_wrench(world, st.T[b], body_h[b]))]
        dh0 = [x + y for x, y in zip(dh0, fp.transport_wrench(world, st.T[b], body_dh[b]))]
    hg = h0[0:3] + fp.add(h0[3:6], fp.cross(h0[0:3], com0))
    dhg = dh0[0:3] + fp.add(dh0[3:6], fp.cross(dh0[0:3], com0))
    mtot = sum(m.mass[b] for b in range(1, nj))
    return dict(energy=np.array([float(kin), float(pot)]), ja=np.array(ja), jf=np.array(jf), com0=fp.to_np(com0),
                vcom0=fp.to_np(fp.scl(1 / mtot, h0[0:3])), hg=fp.to_np(hg), dhg=fp.to_np(dhg))


def _close(x, ref, tol, what):
    scale = max(1.0, float(np.abs(ref).max()))
    err = float(np.abs(np.asarray(x) - ref).max()) / scale
    assert err <= tol, f"{what}: off by {err:.3e} relative to {scale:.3e}"
    return err


def _close_sensors(row, ref, robot, tol):
    """Sensor rows compared type by type, each relative to the largest value of its own type."""
    for key, (off, nf, ns) in robot.sensor_layout().items():
        if key != "width" and ns:
            _close(row[off:off + nf * ns], ref[off:off + nf * ns], tol, key)


def check_end_state(eng, robot, opt, envs, bounds=False, sensors=True, torque=False):
    """(i)-(iv), sensors and computeExtraTerms at the accepted state of the sampled envs.  `torque`: the command is the
    effort itself (no controller block), so the motor law is checked from it; with a PD block the held effort command
    comes from the controller at its last update and only the part of the law after the command is checked."""
    t, q, v, a = eng.get_state()
    u, um, cmd, fext = eng.get_efforts()
    s_all = eng.get_sensors()
    (e_all, ja_all, jf_all), cen = eng.get_extra_terms(), eng.get_centroidal()
    m = _model(robot, opt)
    constraint = opt["contacts"]["model"] == "constraint"
    worst, n_enabled = 0.0, 0
    je, jl, ce, cl = eng.get_constraints()
    for e in envs:
        st = fp.State(m, q[e], v[e])
        u_ref, um_ref = expected_efforts(robot, q[e], v[e], cmd[e] if torque else um[e])
        _close(um[e], um_ref, 1e-12, "motor efforts")
        u_applied = u[e].copy()
        if bounds:
            # the only other thing u may hold: the multiplier of an enabled bound constraint.  The reference adds the
            # multiplier itself to u whatever the side of the bound (engine.cc:3770-3788), while the generalised force
            # it applies is J^T lambda, J = -1 on an upper bound: the residual uses the applied force.
            d = u[e] - u_ref
            n_enabled += int(je[e].sum())
            for j in range(1, robot.njoints):
                iq, iv = int(robot.idx_q[j]), int(robot.idx_v[j])
                if je[e, j]:
                    assert abs(d[iv] - jl[e, j]) <= 1e-12 * max(1.0, abs(jl[e, j])) and jl[e, j] >= 0.0
                    upper = robot.q_upper[iq] - q[e, iq] < q[e, iq] - robot.q_lower[iq]
                    u_applied[iv] = u_ref[iv] + (-d[iv] if upper else d[iv])
                elif fp.Mo.JOINT_NV[int(robot.joint_type[j])] == 1:
                    assert abs(d[iv]) <= 1e-12 * max(1.0, np.abs(u_ref).max())
        else:
            check_efforts(robot, u[e], u_ref)
        worst = max(worst, check_residual(st, a[e], u_applied, fext[e]))
        if constraint:
            mu = opt["contacts"]["friction"]
            for c in np.flatnonzero(ce[e]):
                lam = cl[e, c]
                assert lam[2] >= -1e-8, lam
                assert np.hypot(lam[0], lam[1]) <= mu * lam[2] * (1 + 1e-6) + 1e-8, lam
            continue
        fe, forces = expected_contacts(st, robot, opt)
        check_wrenches(fext[e], fe, opt)
        if sensors:
            row, _ = expected_sensors(st, robot, opt, a[e], um[e], forces)
            _close_sensors(s_all[e], row, robot, 1e-10)
        x = expected_extra_terms(st, robot, a[e], fext[e])
        _close(e_all[e], x["energy"], 1e-12, "energies")
        _close(ja_all[e], x["ja"], 1e-11, "joint accelerations data.a")
        _close(jf_all[e], x["jf"], 1e-11, "joint wrenches data.f")
        ycrb, com, vcom, hg, dhg = [np.asarray(y)[e] for y in cen]
        _close(com[0], x["com0"], 1e-12, "com[0]")
        _close(vcom[0], x["vcom0"], 1e-12, "vcom[0]")
        _close(hg, x["hg"], 1e-12, "hg")
        _close(dhg, x["dhg"], 1e-11, "dhg")
    if bounds:
        assert n_enabled > 0, "no sampled env ends on an enabled bound constraint"
    return worst


def _warps(robot, opt):
    """(n_env, sampled envs): three warps, the last one partial, and an env of the first, the middle and the last warp
    (the last env included)."""
    from emul import emul_api
    epg = BatchedEngine(robot, opt, 1, api_=emul_api()).envs_per_group
    assert epg >= 2
    n = 2 * epg + epg // 2
    return n, (0, epg + epg // 2, n - 1)


def _run(impl, sc, n_steps, targets=None):
    eng = _engine(impl, sc.robot, sc.options, sc.n_env)
    if impl != "oracle":
        epg = eng.envs_per_group
        assert sc.n_env % epg and sc.n_env // epg == 2
    if sc.kp is not None:
        eng.set_pd_controller(sc.kp, sc.kd)
    eng.set_command(sc.target0)
    _start(eng, sc.q0, sc.v0)
    for k in range(n_steps):
        act = sc.sample_targets(k) if targets is None else targets(k)
        eng.set_command(act)
        _step(eng, sc.step_dt)
    return eng


STEP_CASES = {
    "anymal_rk4": dict(name="anymal"),
    "anymal_rk4_full_body": dict(name="anymal", env={"JB_NO_FAST_KERNEL": "1"}),
    "anymal_bounds_in_kernel": dict(name="anymal", bounds=True),
    "anymal_bounds_handoff": dict(name="anymal", bounds=True, env={"JB_NO_FAST_BOUNDS": "1"}),
    "anymal_constraint": dict(name="anymal", contact_model="constraint", solver="euler_explicit", dt_max=0.005),
    "atlas_constraint": dict(name="atlas", contact_model="constraint", solver="euler_explicit", dt_max=0.005),
    "atlas_spring_damper": dict(name="atlas"),
    "anymal_dopri": dict(name="anymal", solver="runge_kutta_dopri"),
    "anymal_torque_sensors_period_0": dict(name="anymal", action="torque", sensors_period=0.0),
}


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("case", list(STEP_CASES))
def test_step_end_state_against_first_principles(impl, case, monkeypatch):
    """The accepted (q, v, a), efforts, sensors and computeExtraTerms outputs after a few env-steps, on every kernel path:
    the quadruped hot path and the full body, joint bounds solved in the evaluation and by hand-off, PGS contacts,
    spring-damper Atlas, Dormand-Prince."""
    cfg = dict(STEP_CASES[case])
    for k, val in cfg.pop("env", {}).items():
        monkeypatch.setenv(k, val)
    bounds = cfg.pop("bounds", False)
    name = cfg.pop("name")
    period = cfg.pop("sensors_period", None)
    sc = scenarios.make(name, 1, seed=4, **cfg)
    n_env, envs = _warps(sc.robot, sc.options)
    sc = scenarios.make(name, n_env, seed=4, **cfg)
    if period is not None:
        sc.options["stepper"]["sensorsUpdatePeriod"] = period
    if sc.kp is None:
        sc.torque_amplitude = 120.0           # beyond the effort limits of some motors: the clipping is exercised
    if name == "anymal" and sc.options["contacts"]["model"] == "spring_damper":
        sc.robot = _with_offset_sensors(sc.robot)
    targets = None
    if bounds:
        rob = sc.robot
        iq = np.array([rob.idx_q[mo.joint] for mo in rob.motors])
        haa = [k for k, mo in enumerate(rob.motors) if "HAA" in mo.name]

        def targets(k):
            act = sc.sample_targets(k)
            for j in haa:
                act[::2, j] = rob.q_upper[iq[j]] + 0.3
            return act
    eng = _run(impl, sc, 2, targets)
    if impl != "oracle" and case == "anymal_rk4":
        assert "hot path: quadruped signature" in eng.describe()
    if bounds:
        assert (eng.get_status()[::2] & 8).any()
    worst = check_end_state(eng, sc.robot, sc.options, envs, bounds=bounds, torque=sc.kp is None)
    print(f"{impl} {case}: residual {worst:.2e}")


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("period", [0.0, 2e-3])
def test_branched_arm_sensors_against_first_principles(impl, period):
    """Every joint model of the path (revolute, unbounded, prismatic, skewed prismatic, free-flyer) under a spinning,
    accelerating base, its foot pressed into the ground: IMU and force sensor away from their joint origin and rotated,
    encoders, effort and contact sensors, efforts, contact wrenches and computeExtraTerms at the end of an env-step,
    with sensors refreshed at every internal step (period 0) and on a period."""
    robot, opt = _branched_arm()
    opt["stepper"].update(sensorsUpdatePeriod=period, controllerUpdatePeriod=period)
    n, envs = _warps(robot, opt)
    m = _model(robot, opt)
    rng = np.random.default_rng(8)
    q, v = pc.random_states(robot, n, rng, base_height=0.55)
    sole, tool = (m.nj + robot.contact_frame_names.index(f) for f in ("b_sole", "a_tool"))
    for e in range(n):
        while True:                                                # the sole 1 mm into the ground, the tool above it
            x = pc.random_states(robot, 1, rng, base_height=0.55)[0][0]
            T = m.fk(m.config(x))
            x[2] += -1e-3 - float(T[sole][1][2])
            if float(T[tool][1][2] - T[sole][1][2]) > 0.05:
                q[e] = x
                break
        v[e, 3:6] = rng.normal(size=3) * 4.0                       # spinning base
        v[e, 6:] = rng.uniform(-2.0, 2.0, size=robot.nv - 6)
    cmd = rng.uniform(-40.0, 40.0, size=(n, robot.nmotors))
    eng = _engine(impl, robot, opt, n)
    eng.set_command(cmd)
    _start(eng, q, v)
    _step(eng, 2e-3)
    check_end_state(eng, robot, opt, envs, torque=True)
    lay, s_all = robot.sensor_layout(), eng.get_sensors()
    off, nf, ns = lay["ForceSensor"]
    assert np.abs(s_all[list(envs), off:off + nf * ns]).max() > 1.0          # the foot is loaded
    off = lay["ImuSensor"][0]
    assert np.abs(s_all[list(envs), off:off + 3]).max() > 2.0                 # the IMU spins


# --------------------------------------------------------------------------- self-tests of the reference
def test_reference_point_mass_and_pendulum_closed_forms():
    """A free-flying body: M = [m I, -m [c]x; m [c]x, Ic - m [c]x^2] (local frame), h = gyroscopic - m R^T g; a pendulum:
    M = a^T (Ic - m [c]x^2) a, h = -a.(c x m R^T g), both to 1e-20."""
    robot = M.build_robot_table(os.path.join(DATA, "point_mass.urdf"), True)
    robot.inertia[1, 1:4] = [0.03, -0.02, 0.05]                     # centre of mass off the joint origin
    robot.inertia[1, 4:10] = [0.2, 0.01, 0.3, -0.02, 0.015, 0.25]
    m = fp.Model(robot)
    q = np.array([0.1, -0.2, 0.3, 0.5, -0.5, 0.5, 0.5])                # an exactly unit quaternion
    v = np.array([0.3, -0.5, 0.2, 4.0, -7.0, 5.5])
    st = fp.State(m, q, v)
    mass, c, Ic = m.mass[1], m.lever[1], m.Ic[1]
    cx = fp.hat(c)
    ref = [[fp.ZERO] * 6 for _ in range(6)]
    for i in range(3):
        ref[i][i] = mass
        for j in range(3):
            ref[i][3 + j] = -mass * cx[i][j]
            ref[3 + i][j] = mass * cx[i][j]
            ref[3 + i][3 + j] = Ic[i][j] - mass * fp.mm(cx, cx)[i][j]
    assert max(abs(st.M[i][j] - ref[i][j]) for i in range(6) for j in range(6)) < 1e-20
    V = fp.mv(v)
    gl = fp.tvec(st.T[1][0], m.gravity[0:3])
    h_ref = fp.force_cross(V, fp.inertia_apply(mass, c, Ic, V))
    h_ref = [x - y for x, y in zip(h_ref, fp.inertia_apply(mass, c, Ic, gl + [fp.ZERO] * 3))]
    assert max(abs(x - y) for x, y in zip(st.h, h_ref)) < 1e-20
    # pendulum
    robot = M.build_robot_table(os.path.join(DATA, "simple_pendulum.urdf"), False)
    m = fp.Model(robot)
    th, w = 0.7, 1.3
    st = fp.State(m, [th], [w])
    j = 1
    a, c, mass = m.axis[j], m.lever[j], m.mass[j]
    Ip = fp.madd(m.Ic[j], fp.mm(fp.hat(c), fp.hat(c)), -mass)
    assert abs(st.M[0][0] - fp.dot(a, fp.mvec(Ip, a))) < 1e-20
    gl = fp.tvec(st.T[j][0], m.gravity[0:3])
    assert abs(st.h[0] + fp.dot(a, fp.cross(c, fp.scl(mass, gl)))) < 1e-20


@pytest.mark.parametrize("name", ["anymal", "branched_arm"])
def test_reference_properties(name):
    """M symmetric positive definite, q and -q (same rotation) give the same M and h, and a finite difference of the
    body positions along integrate(q, t v) matches the twists J v."""
    robot, opt, m, sts = _reference_states(name)
    q, v, _, st = sts[0]
    Mn = st.M_np()
    np.testing.assert_allclose(Mn, Mn.T, rtol=0, atol=1e-25)
    assert np.linalg.eigvalsh(Mn).min() > 0
    if robot.has_freeflyer:
        x = q.copy()
        x[3:7] = -x[3:7]
        st2 = fp.State(m, x, v)
        assert max(abs(a - b) for r1, r2 in zip(st.M, st2.M) for a, b in zip(r1, r2)) < 1e-25
        assert max(abs(a - b) for a, b in zip(st.h, st2.h)) < 1e-25
    for f in range(1, len(st.T)):
        lin, w = st.bias[f][0], st.bias[f][1]           # five-point difference of the poses along the path
        assert max(abs(x - y) for x, y in zip(lin + w, st.V[f])) < 1e-22 * max(1, max(abs(x) for x in st.V[f]))


def test_reference_double_pendulum_closed_form():
    """Double pendulum from its kinetic and potential energy: with r2 the centre of mass of link 2 in frame 1, b the
    axis of joint 2 in frame 1 and I2 its inertia about its centre of mass in frame 1,
    M11 = a.I1o.a + m2 |a x r2|^2 + a.I2.a,  M12 = m2 (a x r2).(b x (r2 - p)) + a.I2.b,  M22 = m2 |b x (r2 - p)|^2 + b.I2.b
    (+ rotor inertias), h = C(q, qd) qd + dV/dq with the Christoffel symbols of that M; both to 1e-20."""
    robot, _ = R.load_robot("double_pendulum")
    m = fp.Model(robot)
    assert m.nj == 3 and m.parent[2] == 1
    P1, P2 = m.place[1], m.place[2]

    def rot(j, th):
        return m.joint_motion(j, th)[0]

    def energy_terms(q1, q2):
        a = m.axis[1]
        R2 = fp.mm(P2[0], rot(2, q2))
        b = fp.mvec(P2[0], m.axis[2])
        p = P2[1]
        r2 = fp.add(p, fp.mvec(R2, m.lever[2]))
        c1 = fp.hat(m.lever[1])
        I1o = fp.madd(m.Ic[1], fp.mm(c1, c1), -m.mass[1])
        I2 = fp.mm(fp.mm(R2, m.Ic[2]), fp.tr(R2))
        ar, br = fp.cross(a, r2), fp.cross(b, fp.sub(r2, p))
        M = [[fp.dot(a, fp.mvec(I1o, a)) + m.mass[2] * fp.dot(ar, ar) + fp.dot(a, fp.mvec(I2, a)) + m.rotor[0],
              m.mass[2] * fp.dot(ar, br) + fp.dot(a, fp.mvec(I2, b))],
             [None, m.mass[2] * fp.dot(br, br) + fp.dot(b, fp.mvec(I2, b)) + m.rotor[1]]]
        M[1][0] = M[0][1]
        W1 = fp.mm(P1[0], rot(1, q1))                              # frame 1 in the world
        g = m.gravity[0:3]
        V = -m.mass[1] * fp.dot(g, fp.add(P1[1], fp.mvec(W1, m.lever[1]))) - m.mass[2] * fp.dot(g, fp.add(P1[1], fp.mvec(W1, r2)))
        return M, V

    q, qd = [fp.mpf(0.7), fp.mpf(-1.3)], [fp.mpf(2.1), fp.mpf(-3.4)]        # exact doubles
    st = fp.State(m, [float(x) for x in q], [float(x) for x in qd])
    M, _ = energy_terms(*q)
    assert max(abs(st.M[i][j] - M[i][j]) for i in range(2) for j in range(2)) < 1e-20
    dM = [[[fp.mp.diff(lambda t, i=i, j=j, k=k: energy_terms(*[t if l == k else q[l] for l in range(2)])[0][i][j], q[k])
            for k in range(2)] for j in range(2)] for i in range(2)]
    dV = [fp.mp.diff(lambda t, k=k: energy_terms(*[t if l == k else q[l] for l in range(2)])[1], q[k]) for k in range(2)]
    h = [sum((dM[i][j][k] - dM[j][k][i] / 2) * qd[j] * qd[k] for j in range(2) for k in range(2)) + dV[i] for i in range(2)]
    assert max(abs(x - y) for x, y in zip(st.h, h)) < 1e-20

