"""Extended-precision first-principles reference for whole-robot dynamics, written without any recursion of the
repository (no ABA, CRBA or RNEA) and without the oracle, so that a convention error shared by the kernel and the oracle
shows up as a disagreement with this module.

It reads only the tables of `jiminy_b200.model.RobotTable` (parents, joint types, axes, placements, inertias, rotor
inertias, frames, motors, flexibility stiffness / damping) and the engine options, and works in mpmath at `DPS` digits:

* forward kinematics composes one homogeneous transform per joint (`fk`);
* `integrate(q, d)` follows Pinocchio's conventions joint by joint: vector spaces add, SO(2) rotates (cos, sin), the
  free-flyer and the spherical joint right-multiply the exponential of the local twist;
* body twists and Jacobians in the local frame of every joint / frame come from central differences of the FK along
  `integrate(q, eps e_i)`;
* bias terms and accelerations come from second differences of the FK along the path `q(t) = integrate(q, t v + t^2 a / 2)`:
  with `a = 0` the generalised velocity is constant, so the body acceleration is the bias `Jdot v`;
* dynamics by Newton-Euler per body projected with the Jacobians: `M = sum J_b^T I_b J_b + diag(armature)`,
  `h = sum J_b^T (I_b (Jdot v)_b + v_b x* I_b v_b - I_b g_b)`.

Step sizes (DPS = 50 significant digits, rounding unit u = 1e-50):
* Jacobian columns, central first difference with EPS_J = 1e-15: truncation eps^2 |T'''| / 6 ~ 1e-31 for O(1) link
  lengths, rounding u / eps ~ 1e-35.
* Path derivatives, five-point stencils with H_PATH = 1e-7 / max(1, |v|, |a|^(1/2)) (the path parameter is scaled so that
  one step moves every joint by at most ~1e-7): truncation of the second derivative h^4 |T^(6)| / 90 ~ 1e-30 relative to
  the acceleration, rounding 64 u / (12 h^2) ~ 1e-35 relative.
Both stay below 1e-25 relative, far below the double-precision quantities they are compared with.
"""
from __future__ import annotations

import math

import mpmath as mp
import numpy as np

from jiminy_b200 import model as Mo

DPS = 50
mp.mp.dps = DPS
mpf = mp.mpf
EPS_J = mpf("1e-15")
H_PATH = mpf("1e-7")
ZERO, ONE, HALF = mpf(0), mpf(1), mpf("0.5")

REVOLUTE = (Mo.JB_JOINT_RX, Mo.JB_JOINT_RY, Mo.JB_JOINT_RZ, Mo.JB_JOINT_RU)
UNBOUNDED = (Mo.JB_JOINT_RUBX, Mo.JB_JOINT_RUBY, Mo.JB_JOINT_RUBZ, Mo.JB_JOINT_RUBU)
PRISMATIC = (Mo.JB_JOINT_PX, Mo.JB_JOINT_PY, Mo.JB_JOINT_PZ, Mo.JB_JOINT_PU)


# --------------------------------------------------------------------------- 3-vectors and 3x3 matrices as lists of mpf
def mv(x):
    return [mpf(float(t)) for t in x]       # exact: every double is an mpf


def add(a, b):
    return [a[0] + b[0], a[1] + b[1], a[2] + b[2]]


def sub(a, b):
    return [a[0] - b[0], a[1] - b[1], a[2] - b[2]]


def scl(s, a):
    return [s * a[0], s * a[1], s * a[2]]


def dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def eye3():
    return [[ONE, ZERO, ZERO], [ZERO, ONE, ZERO], [ZERO, ZERO, ONE]]


def mm(A, B):
    return [[A[i][0] * B[0][j] + A[i][1] * B[1][j] + A[i][2] * B[2][j] for j in range(3)] for i in range(3)]


def mvec(A, x):
    return [A[i][0] * x[0] + A[i][1] * x[1] + A[i][2] * x[2] for i in range(3)]


def tr(A):
    return [[A[j][i] for j in range(3)] for i in range(3)]


def tvec(A, x):
    return mvec(tr(A), x)


def hat(w):
    return [[ZERO, -w[2], w[1]], [w[2], ZERO, -w[0]], [-w[1], w[0], ZERO]]


def vee_skew(A):
    """Axial vector of the skew-symmetric part of A."""
    return [(A[2][1] - A[1][2]) / 2, (A[0][2] - A[2][0]) / 2, (A[1][0] - A[0][1]) / 2]


def madd(A, B, s=ONE):
    return [[A[i][j] + s * B[i][j] for j in range(3)] for i in range(3)]


def rot_axis(axis, c, s):
    """Rotation about the unit `axis` by the angle whose cosine / sine are (c, s): c I + s [a]x + (1 - c) a a^T."""
    K = hat(axis)
    return madd(madd([[c if i == j else ZERO for j in range(3)] for i in range(3)], K, s),
                [[axis[i] * axis[j] for j in range(3)] for i in range(3)], 1 - c)


def quat_to_rot(x, y, z, w):
    return [[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
            [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
            [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]


def exp3(w):
    th = mp.sqrt(dot(w, w))
    if th == 0:
        return eye3()
    K = hat(w)
    return madd(madd(eye3(), K, mp.sin(th) / th), mm(K, K), (1 - mp.cos(th)) / th ** 2)


def exp6(v, w):
    """SE(3) exponential of the twist (v, w): (exp3(w), V(w) v)."""
    th = mp.sqrt(dot(w, w))
    if th == 0:
        return eye3(), list(v)
    K = hat(w)
    V = madd(madd(eye3(), K, (1 - mp.cos(th)) / th ** 2), mm(K, K), (th - mp.sin(th)) / th ** 3)
    return exp3(w), mvec(V, v)


def se3(flat):
    f = mv(flat)
    return [f[0:3], f[3:6], f[6:9]], f[9:12]


def compose(A, B):
    return mm(A[0], B[0]), add(mvec(A[0], B[1]), A[1])


# --------------------------------------------------------------------------- model
class Model:
    """Extended-precision copy of the tables of one robot."""

    def __init__(self, robot: Mo.RobotTable, gravity=(0.0, 0.0, -9.81, 0.0, 0.0, 0.0), frames=()):
        self.robot = robot
        self.nj, self.nq, self.nv = robot.njoints, robot.nq, robot.nv
        self.jt = [int(t) for t in robot.joint_type]
        self.parent = [int(p) for p in robot.parent]
        self.iq = [int(i) for i in robot.idx_q]
        self.iv = [int(i) for i in robot.idx_v]
        self.place = [se3(robot.placement[j]) for j in range(self.nj)]
        self.axis = [mv(robot.axis[j]) for j in range(self.nj)]
        self.mass, self.lever, self.Ic = [], [], []
        for j in range(self.nj):
            y = mv(robot.inertia[j])
            self.mass.append(y[0])
            self.lever.append(y[1:4])
            self.Ic.append([[y[4], y[5], y[7]], [y[5], y[6], y[8]], [y[7], y[8], y[9]]])
        self.rotor = mv(robot.rotor_inertia)
        self.gravity = mv(gravity)
        # extra frames: (joint, placement) of every frame whose motion is wanted besides the joint frames
        self.frames = [(robot.frames[f].joint, se3(robot.frames[f].placement.flat())) if isinstance(f, str)
                       else (int(f[0]), se3(f[1])) for f in frames]
        # joints whose motion moves joint j: j and its ancestors
        self.ancestors = []
        for j in range(self.nj):
            s, k = set(), j
            while k > 0:
                s.add(k)
                k = self.parent[k]
            self.ancestors.append(s)
        self.dofs = []          # velocity indices that move joint j
        for j in range(self.nj):
            self.dofs.append(sorted(self.iv[k] + d for k in self.ancestors[j] for d in range(Mo.JOINT_NV[self.jt[k]])))

    # ---- configuration: one entry per joint, in the form its FK needs
    def config(self, q):
        q = mv(q)
        cfg = [None]
        for j in range(1, self.nj):
            t, i = self.jt[j], self.iq[j]
            if t == Mo.JB_JOINT_FREEFLYER:
                cfg.append((quat_to_rot(*q[i + 3:i + 7]), q[i:i + 3]))
            elif t == Mo.JB_JOINT_SPHERICAL:
                cfg.append(quat_to_rot(*q[i:i + 4]))
            elif t in UNBOUNDED:
                cfg.append((q[i], q[i + 1]))
            else:
                cfg.append(q[i])
        return cfg

    def integrate(self, cfg, d):
        """Pinocchio's `integrate(q, d)` joint by joint (d: list of mpf, length nv)."""
        out = [None]
        for j in range(1, self.nj):
            t, i, c = self.jt[j], self.iv[j], cfg[j]
            if t == Mo.JB_JOINT_FREEFLYER:
                R, p = c
                if any(d[i:i + 6]):
                    dR, dp = exp6(d[i:i + 3], d[i + 3:i + 6])
                    c = (mm(R, dR), add(p, mvec(R, dp)))
            elif t == Mo.JB_JOINT_SPHERICAL:
                if any(d[i:i + 3]):
                    c = mm(c, exp3(d[i:i + 3]))
            elif t in UNBOUNDED:
                if d[i]:
                    cw, sw = mp.cos(d[i]), mp.sin(d[i])
                    c = (cw * c[0] - sw * c[1], sw * c[0] + cw * c[1])
            else:
                c = c + d[i]
            out.append(c)
        return out

    def joint_motion(self, j, c):
        t = self.jt[j]
        if t == Mo.JB_JOINT_FREEFLYER:
            return c
        if t == Mo.JB_JOINT_SPHERICAL:
            return c, [ZERO] * 3
        if t in REVOLUTE:
            return rot_axis(self.axis[j], mp.cos(c), mp.sin(c)), [ZERO] * 3
        if t in UNBOUNDED:
            return rot_axis(self.axis[j], c[0], c[1]), [ZERO] * 3
        return eye3(), scl(c, self.axis[j])

    def fk(self, cfg):
        """World transform of every joint frame, then of every extra frame."""
        T = [(eye3(), [ZERO] * 3)]
        for j in range(1, self.nj):
            T.append(compose(compose(T[self.parent[j]], self.place[j]), self.joint_motion(j, cfg[j])))
        return T + [compose(T[j], P) for j, P in self.frames]


# --------------------------------------------------------------------------- differentiation of the FK
def _local(T, dT):
    """(R^T dp, R^T dR) of a derivative (dR, dp) of T = (R, p)."""
    return tvec(T[0], dT[1]), mm(tr(T[0]), dT[0])


def _diff(Ta, Tb, s):
    return [[(Ta[0][i][k] - Tb[0][i][k]) * s for k in range(3)] for i in range(3)], [(Ta[1][i] - Tb[1][i]) * s for i in range(3)]


def jacobians(m: Model, cfg, T0):
    """Body Jacobians (6 x nv, rows lin | ang, local frame) of every joint and extra frame, by central differences."""
    nf = len(T0)
    J = [[[ZERO] * m.nv for _ in range(6)] for _ in range(nf)]
    for k in range(m.nv):
        e = [ZERO] * m.nv
        e[k] = EPS_J
        Tp = m.fk(m.integrate(cfg, e))
        e[k] = -EPS_J
        Tm = m.fk(m.integrate(cfg, e))
        for f in range(nf):
            if Tp[f] == Tm[f]:
                continue
            lin, A = _local(T0[f], _diff(Tp[f], Tm[f], 1 / (2 * EPS_J)))
            col = lin + vee_skew(A)
            for r in range(6):
                J[f][r][k] = col[r]
    return J


def path_derivatives(m: Model, cfg, T0, v, a=None):
    """Along q(t) = integrate(q, t v + t^2 a / 2): per frame the body twist (lin, ang) by a five-point first difference,
    the classical linear acceleration R^T pddot and the angular acceleration (local frame) by a five-point second one."""
    v = mv(v)
    a = [ZERO] * m.nv if a is None else mv(a)
    scale = max(ONE, max(abs(x) for x in v), mp.sqrt(max(abs(x) for x in a)) if m.nv else ONE)
    h = H_PATH / scale
    Ts = {}
    for s in (-2, -1, 1, 2):
        t = s * h
        Ts[s] = m.fk(m.integrate(cfg, [t * vi + t * t / 2 * ai for vi, ai in zip(v, a)]))
    out = []
    for f in range(len(T0)):
        d1 = [[(-Ts[2][f][0][i][k] + 8 * Ts[1][f][0][i][k] - 8 * Ts[-1][f][0][i][k] + Ts[-2][f][0][i][k]) / (12 * h)
               for k in range(3)] for i in range(3)], \
             [(-Ts[2][f][1][i] + 8 * Ts[1][f][1][i] - 8 * Ts[-1][f][1][i] + Ts[-2][f][1][i]) / (12 * h) for i in range(3)]
        d2 = [[(-Ts[2][f][0][i][k] + 16 * Ts[1][f][0][i][k] - 30 * T0[f][0][i][k] + 16 * Ts[-1][f][0][i][k] - Ts[-2][f][0][i][k])
               / (12 * h * h) for k in range(3)] for i in range(3)], \
             [(-Ts[2][f][1][i] + 16 * Ts[1][f][1][i] - 30 * T0[f][1][i] + 16 * Ts[-1][f][1][i] - Ts[-2][f][1][i]) / (12 * h * h)
              for i in range(3)]
        lin, A = _local(T0[f], d1)
        acc, B = _local(T0[f], d2)
        out.append((lin, vee_skew(A), acc, vee_skew(B)))     # v, w, R^T pddot, wdot   (R^T Rddot = [wdot]x + [w]x^2)
    return out


# --------------------------------------------------------------------------- spatial algebra of one body
def inertia_apply(m, c, Ic, V):
    """Momentum (lin, ang about the frame origin) of a body of mass m, centre of mass c, inertia Ic about c, twist V."""
    lin = scl(m, add(V[0:3], cross(V[3:6], c)))
    return lin + add(mvec(Ic, V[3:6]), cross(c, lin))


def force_cross(V, f):
    """V x* f, twist (v, w), wrench (f, n)."""
    v, w = V[0:3], V[3:6]
    return cross(w, f[0:3]) + add(cross(w, f[3:6]), cross(v, f[0:3]))


def jt_times(J, f, dofs, out):
    for k in dofs:
        out[k] += sum(J[r][k] * f[r] for r in range(6))


def matvec(Jm, x, dofs):
    return [sum(Jm[r][k] * x[k] for k in dofs) for r in range(6)]


def transport_wrench(Ti, Tb, f):
    """Wrench f expressed at frame b -> the same wrench expressed at frame i."""
    R = mm(tr(Ti[0]), Tb[0])
    p = tvec(Ti[0], sub(Tb[1], Ti[1]))
    lin = mvec(R, f[0:3])
    return lin + add(mvec(R, f[3:6]), cross(p, lin))


# --------------------------------------------------------------------------- one state
class State:
    """Everything the checks need at one (q, v): FK, Jacobians, twists, bias, M, h."""

    def __init__(self, m: Model, q, v):
        self.m = m
        self.q, self.v = np.asarray(q, dtype=np.float64), np.asarray(v, dtype=np.float64)
        self.cfg = m.config(q)
        self.T = m.fk(self.cfg)
        self.J = jacobians(m, self.cfg, self.T)
        vm = mv(v)
        self.vm = vm
        self.bias = path_derivatives(m, self.cfg, self.T, v)
        nv = m.nv
        self.V = []       # body twist (lin, ang) of every joint / frame, J v
        for f in range(len(self.T)):
            self.V.append(matvec(self.J[f], vm, range(nv)))
        # mass matrix and bias forces
        M = [[ZERO] * nv for _ in range(nv)]
        h = [ZERO] * nv
        g6 = m.gravity
        for b in range(1, m.nj):
            if m.mass[b] == 0 and not any(any(r) for r in m.Ic[b]):
                continue
            Jb, dofs, R = self.J[b], m.dofs[b], self.T[b][0]
            IJ = {k: inertia_apply(m.mass[b], m.lever[b], m.Ic[b], [Jb[r][k] for r in range(6)]) for k in dofs}
            for k in dofs:
                for l in dofs:
                    M[k][l] += sum(Jb[r][k] * IJ[l][r] for r in range(6))
            Vb = self.V[b]
            lin, w, acc, wd = self.bias[b]
            alpha = sub(acc, cross(w, lin)) + wd                       # spatial acceleration Jdot v (local frame)
            gb = tvec(R, g6[0:3]) + tvec(R, g6[3:6])
            ag = [alpha[r] - gb[r] for r in range(6)]
            fb = inertia_apply(m.mass[b], m.lever[b], m.Ic[b], ag)
            fb = [x + y for x, y in zip(fb, force_cross(Vb, inertia_apply(m.mass[b], m.lever[b], m.Ic[b], Vb)))]
            jt_times(Jb, fb, dofs, h)
        for k in range(nv):
            M[k][k] += m.rotor[k]
        self.M, self.h = M, h

    # ---- numpy views
    def M_np(self):
        return np.array([[float(x) for x in r] for r in self.M])

    def h_np(self):
        return np.array([float(x) for x in self.h])

    def world_point(self, f):
        return self.T[f][1]

    def world_velocity(self, f):
        """Velocity of the origin of frame f in the world frame (R of the frame times the linear part of its twist)."""
        return mvec(self.T[f][0], self.V[f][0:3])

    def generalized_force(self, fext):
        """sum_j J_j^T f_j, f_j the wrench on joint j expressed in its frame (fext [njoints, 6] as the C ABI returns it)."""
        out = [ZERO] * self.m.nv
        for j in range(1, self.m.nj):
            fj = mv(fext[j])
            if any(fj):
                jt_times(self.J[j], fj, self.m.dofs[j], out)
        return out

    def residual(self, a, u, fext):
        """M a + h - u - sum J^T f (mpf list) and the scale ||M|| ||a|| + ||h|| + ||u|| + ||sum J^T f|| (inf-norms)."""
        am, um = mv(a), mv(u)
        gf = self.generalized_force(fext)
        nv = self.m.nv
        Ma = [sum(self.M[k][l] * am[l] for l in range(nv)) for k in range(nv)]
        r = [Ma[k] + self.h[k] - um[k] - gf[k] for k in range(nv)]
        nM = max(sum(abs(x) for x in row) for row in self.M)
        scale = nM * max(abs(x) for x in am) + max(abs(x) for x in self.h) + max(abs(x) for x in um) + max(abs(x) for x in gf)
        return r, scale

    def solve(self, rhs):
        """M^{-1} rhs in extended precision."""
        x = mp.lu_solve(mp.matrix(self.M), mp.matrix(rhs))
        return [x[k] for k in range(self.m.nv)]

    def accelerations(self, a):
        """Per joint / frame (twist lin, twist ang, classical linear acceleration R^T pddot, angular acceleration) along
        q(t) = integrate(q, t v + t^2 a / 2)."""
        return path_derivatives(self.m, self.cfg, self.T, self.v, a)


# --------------------------------------------------------------------------- laws restated from the reference engine
def spring_damper_contact(opt, depth, vel):
    """Ground reaction in the world frame at a point of the flat ground z = 0, normal +z (Engine::computeContactDynamics,
    engine.cc:3197-3238): below the ground the normal force is the spring-damper force, never pulling; friction opposes
    the tangential velocity with a coefficient that ramps up to `friction` until `transitionVelocity` and is applied to
    the tangential velocity vector itself; the whole force fades in with tanh(2 * penetration / transitionEps)."""
    c = opt["contacts"]
    if depth >= 0:
        return [ZERO] * 3
    k, d, mu = mpf(c["stiffness"]), mpf(c["damping"]), mpf(c["friction"])
    fn = -min(k * depth + d * vel[2], ZERO)
    vt = [vel[0], vel[1], ZERO]
    ratio = min(mp.sqrt(dot(vt, vt)) / mpf(c["transitionVelocity"]), ONE)
    F = [-mu * ratio * fn * vt[0], -mu * ratio * fn * vt[1], fn]
    eps = mpf(c["transitionEps"])
    if eps > mpf(float(np.finfo(np.float64).eps)):
        F = scl(mp.tanh(2 * (-depth) / eps), F)
    return F


def contact_wrenches(st: State, opt, contact_frames):
    """Expected fext [njoints, 6] (joint frames) and world forces of the contacts.  `contact_frames[c]` is the index of
    contact c among the extra frames of the model."""
    m = st.m
    fext = [[ZERO] * 6 for _ in range(m.nj)]
    forces = []
    for fi in contact_frames:
        f = m.nj + fi
        j, P = m.frames[fi]
        p = st.world_point(f)
        F = spring_damper_contact(opt, p[2], st.world_velocity(f))
        forces.append(F)
        lin = tvec(st.T[j][0], F)                 # force applied at the contact point, moved to the joint origin
        w = lin + cross(P[1], lin)
        fext[j] = [x + y for x, y in zip(fext[j], w)]
    return fext, forces


def motor_efforts(robot: Mo.RobotTable, v, command):
    """SimpleMotor (basic_motors.cc, abstract_motor.cc): motor effort = command clipped to the effort limit, the limit
    tapered linearly to zero over `effortLimit * velocityEffortInvSlope` below the velocity limit; joint effort = reduction
    * motor effort + viscous / dry friction on the joint velocity.  Returns (u [nv] from the motors, motor efforts)."""
    u, um = np.zeros(robot.nv), np.zeros(robot.nmotors)
    for k, mo in enumerate(robot.motors):
        iv = int(robot.idx_v[mo.joint])
        vj = float(v[iv])
        lo, hi = -math.inf, math.inf
        if mo.enable_effort_limit:
            lo, hi = -mo.effort_limit, mo.effort_limit
            dv = mo.effort_limit * mo.velocity_effort_inv_slope
            if mo.enable_velocity_limit and dv > 0:
                vm, vl = mo.reduction * vj, mo.velocity_limit
                band = vl - max(vl - dv, 0.0)
                lo *= min(max((vl + vm) / band, 0.0), 1.0)
                hi *= min(max((vl - vm) / band, 0.0), 1.0)
        um[k] = min(max(float(command[k]), lo), hi)
        ut = mo.reduction * um[k]
        if mo.enable_friction:
            if vj > 0:
                ut += mo.friction_viscous_positive * vj + mo.friction_dry_positive * math.tanh(mo.friction_dry_slope * vj)
            else:
                ut += mo.friction_viscous_negative * vj + mo.friction_dry_negative * math.tanh(mo.friction_dry_slope * vj)
        u[iv] += ut
    return u, um


def flexibility_efforts(robot: Mo.RobotTable, q, v):
    """Spring-damper of the spherical flexibility joints (engine.cc:3367-3391): with r = log3(quaternion) (angle-axis),
    u -= Jlog3(r) (k * r) + d * v, Jlog3 the inverse right Jacobian of SO(3)."""
    u = [ZERO] * robot.nv
    if robot.flexibility is None:
        return u
    for j in range(1, robot.njoints):
        if int(robot.joint_type[j]) != Mo.JB_JOINT_SPHERICAL:
            continue
        iq, iv = int(robot.idx_q[j]), int(robot.idx_v[j])
        x, y, z, w = mv(q[iq:iq + 4])
        if w < 0:
            x, y, z, w = -x, -y, -z, -w
        s = mp.sqrt(x * x + y * y + z * z)
        th = 2 * mp.atan2(s, w)
        r = [ZERO] * 3 if s == 0 else scl(th / s, [x, y, z])
        K = hat(r)
        Jl = eye3() if th == 0 else madd(madd(eye3(), K, HALF), mm(K, K), 1 / th ** 2 - (1 + mp.cos(th)) / (2 * th * mp.sin(th)))
        kd = mv(robot.flexibility[j])
        t = mvec(Jl, [kd[0] * r[0], kd[1] * r[1], kd[2] * r[2]])
        vj = mv(v[iv:iv + 3])
        for e in range(3):
            u[iv + e] -= t[e] + kd[3 + e] * vj[e]
    return u


def to_np(x):
    return np.array([float(t) for t in x])
