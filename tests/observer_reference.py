"""numpy restatement of gym_jiminy's observer blocks, one IMU at a time: `MahonyFilter.refresh_observation` with its
full option set (blocks/mahony_filter.py:28-101, :337-393) and `BodyObserver.refresh_observation`
(blocks/body_orientation_observer.py:26-72, :237-266), with the utils/math.py functions they call.  Pinned to the
reference's own code by tests/golden/observer_blocks.npz (tools/make_golden_observer_blocks.py); the device observers are
checked against it.  Quaternions are (x, y, z, w) arrays of 4 floats."""
import math

import numpy as np

G = 9.81                 # EARTH_SURFACE_GRAVITY
THR = 1e-5               # TWIST_SWING_SINGULAR_THR


def tilt(q):
    """compute_tilt_from_quat: R(q)^T e_z."""
    q_x, q_y, q_z, q_w = q
    return 2 * (q_x * q_z - q_y * q_w), 2 * (q_y * q_z + q_w * q_x), 1 - 2 * (q_x * q_x + q_y * q_y)


def _renormalise(q):
    s = (3.0 - (((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3])) / 2
    return [x * s for x in q]


def swing_from_vector(v):
    """swing_from_vector on one column of a batch: the singular branch is the per-column recursion of the batched call,
    so it is renormalised twice."""
    v_x, v_y, v_z = (float(x) for x in v)
    if v_z < -1.0 + THR:
        eps_thr = math.sqrt(THR)
        eps_x, eps_y = -THR < v_x < THR, -THR < v_y < THR
        ratio, eps_ratio = 0.0, False
        if eps_x and not eps_y:
            ratio = v_x / v_y
            eps_ratio = -eps_thr < ratio < eps_thr
        elif eps_y and not eps_x:
            ratio = v_y / v_x
            eps_ratio = -eps_thr < ratio < eps_thr
        w_2 = (1.0 + max(v_z, -1.0)) / 2.0
        if eps_x and eps_y:
            q = [0.0, math.sqrt(1.0 - w_2)]
        elif eps_ratio and eps_x:
            q = [-math.sqrt(1.0 - w_2) * (1 - 0.5 * (ratio * ratio)), math.sqrt(1.0 - w_2) * (ratio - 0.5 * (ratio * ratio * ratio))]
        elif eps_ratio and eps_y:
            q = [-math.sqrt(1.0 - w_2) * (ratio - 0.5 * (ratio * ratio * ratio)), math.sqrt(1.0 - w_2) * (1 - 0.5 * (ratio * ratio))]
        else:
            q = [-math.sqrt((1.0 - w_2) / (1 + (v_x / v_y) * (v_x / v_y))), math.sqrt((1.0 - w_2) / (1 + (v_y / v_x) * (v_y / v_x)))]
        q = _renormalise(q + [0.0, math.sqrt(w_2)])
    else:
        s = math.sqrt(2.0 * (1.0 + v_z))
        q = [v_y / s, -v_x / s, 0.0, s / 2]
    return np.array(_renormalise(q))


def remove_twist(q):
    return swing_from_vector(tilt(q))


def quat_to_rpy(q):
    x, y, z, w = (float(c) for c in q)
    q_xx, q_xy, q_xz, q_xw, q_yy, q_yz, q_yw = x * x, x * y, x * z, x * w, y * y, y * z, y * w
    q_zz, q_zw, q_ww = z * z, z * w, w * w
    n = (3.0 - (((q_xx + q_yy) + q_zz) + q_ww)) / 2
    q_yw, q_xz = q_yw * n, q_xz * n
    return np.array([math.atan2(2 * (q_xw + q_yz), 1.0 - 2 * (q_xx + q_yy)),
                     -math.pi / 2 + 2 * math.atan2(math.sqrt(1.0 + 2 * (q_yw - q_xz)), math.sqrt(1.0 - 2 * (q_yw - q_xz))),
                     math.atan2(2 * (q_zw + q_xy), 1.0 - 2 * (q_yy + q_zz))])


def quat_multiply_right_conjugate(l, r):
    """quat_multiply(l, r, is_right_conjugate=True): its sign convention negates the real part of r."""
    lx, ly, lz, lw = (float(c) for c in l)
    rx, ry, rz, rw = (float(c) for c in r)
    return np.array([((lw * rx + (-lx) * rw) + ly * rz) - lz * ry,
                     ((lw * ry - lx * rz) + (-ly) * rw) + lz * rx,
                     ((lw * rz + lx * ry) - ly * rx) + (-lz) * rw,
                     (((-lw) * rw - lx * rx) - ly * ry) - lz * rz])


def quat_apply(q, v):
    x_, y_, z_, w_ = (float(c) for c in q)
    q_xx, q_xy, q_xz, q_xw = x_ * x_, x_ * y_, x_ * z_, x_ * w_
    q_yy, q_yz, q_yw, q_zz, q_zw, q_ww = y_ * y_, y_ * z_, y_ * w_, z_ * z_, z_ * w_, w_ * w_
    x, y, z = (float(c) for c in v)
    return np.array([(x * (((q_xx + q_ww) - q_yy) - q_zz) + y * (2 * q_xy - 2 * q_zw)) + z * (2 * q_xz + 2 * q_yw),
                     (x * (2 * q_zw + 2 * q_xy) + y * (((q_ww - q_xx) + q_yy) - q_zz)) + z * (-2 * q_xw + 2 * q_yz),
                     (x * (-2 * q_yw + 2 * q_xz) + y * (2 * q_xw + 2 * q_yz)) + z * (((q_ww - q_xx) - q_yy) + q_zz)])


def matrix_to_quat(R):
    """matrices_to_quat for one matrix."""
    R = np.asarray(R, dtype=np.float64)
    if R[2, 2] < 0:
        if R[0, 0] > R[1, 1]:
            t = 1 + R[0, 0] - R[1, 1] - R[2, 2]
            o = [t, R[1, 0] + R[0, 1], R[0, 2] + R[2, 0], R[2, 1] - R[1, 2]]
        else:
            t = 1 - R[0, 0] + R[1, 1] - R[2, 2]
            o = [R[1, 0] + R[0, 1], t, R[2, 1] + R[1, 2], R[0, 2] - R[2, 0]]
    else:
        if R[0, 0] < -R[1, 1]:
            t = 1 - R[0, 0] - R[1, 1] + R[2, 2]
            o = [R[0, 2] + R[2, 0], R[2, 1] + R[1, 2], t, R[1, 0] - R[0, 1]]
        else:
            t = 1 + R[0, 0] + R[1, 1] + R[2, 2]
            o = [R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1], t]
    d = 2 * math.sqrt(t)
    return np.array([x / d for x in o])


def update_twist(q, twist, omega, tc_inv, dt):
    """update_twist: returns (quaternion, twist)."""
    q_x, q_y, _, q_w = (float(c) for c in q)
    dtwist = ((-q_y) * omega[0] + q_x * omega[1]) / q_w + omega[2]
    twist = twist * max(0.0, 1.0 - tc_inv * dt)
    twist = twist + dtwist * dt
    p_z, p_w = math.sin(0.5 * twist), math.cos(0.5 * twist)
    return np.array([p_w * q_x - p_z * q_y, p_z * q_x + p_w * q_y, p_z * q_w, p_w * q_w]), twist


def mahony_filter(q, bias, gyro, acc, kp, ki, dt):
    """mahony_filter: returns (quaternion, omega, bias)."""
    v_x, v_y, v_z = tilt(q)
    omega = np.array([gyro[0] - bias[0], gyro[1] - bias[1], gyro[2] - bias[2]])
    ax, ay, az = acc[0] / G, acc[1] / G, acc[2] / G
    om = np.array([ay * v_z - az * v_y, az * v_x - ax * v_z, ax * v_y - ay * v_x])
    cf = omega + kp * om
    if (np.abs(cf) < 1e-6).all():
        return np.array(q, dtype=np.float64), omega, np.array(bias, dtype=np.float64)
    theta = math.sqrt((cf[0] * cf[0] + cf[1] * cf[1]) + cf[2] * cf[2])
    axis = cf / theta
    theta *= dt / 2
    p_x, p_y, p_z = axis * math.sin(theta)
    p_w = math.cos(theta)
    q_x, q_y, q_z, q_w = (float(c) for c in q)
    n = [q_x * p_w + q_w * p_x - q_z * p_y + q_y * p_z, q_y * p_w + q_z * p_x + q_w * p_y - q_x * p_z,
         q_z * p_w - q_y * p_x + q_x * p_y + q_w * p_z, q_w * p_w - q_x * p_x - q_y * p_y - q_z * p_z]
    return np.array(_renormalise(n)), omega, np.asarray(bias, dtype=np.float64) - ki * dt * om


class Observers:
    """MahonyFilter (kp, ki, exact_init, ignore_twist) then BodyObserver(twist_time_constant=tc; NaN = None) for one IMU
    whose frame has the rotation `R_rel` in its parent body; `refresh` is one observer refresh, the first after `start`
    the (re)start one (the true IMU orientation `q_exact` is used by exact_init and in free fall)."""

    def __init__(self, kp, ki, dt, exact_init=True, ignore_twist=False, tc=float("nan"), R_rel=np.eye(3)):
        self.kp, self.ki, self.dt, self.exact_init, self.ignore_twist = kp, ki, dt, exact_init, ignore_twist
        self.tc_inv = None if math.isnan(tc) else (1.0 / tc if tc > 0.0 else math.inf)
        self.q_rel = matrix_to_quat(R_rel)

    def start(self):
        self.q, self.omega, self.bias, self.twist, self.started = None, np.zeros(3), np.zeros(3), 0.0, False

    def refresh(self, gyro, acc, q_exact=None):
        if not self.started:
            self.started = True
            acc = np.asarray(acc, dtype=np.float64)
            if not self.exact_init and not (np.abs(acc) < 0.1 * G).all():
                nrm = math.sqrt((acc[0] * acc[0] + acc[1] * acc[1]) + acc[2] * acc[2])
                self.q = swing_from_vector(acc / nrm)
            else:
                self.q = np.array(q_exact, dtype=np.float64)
        else:
            self.q, self.omega, self.bias = mahony_filter(self.q, self.bias, gyro, acc, self.kp, self.ki, self.dt)
            if self.ignore_twist:
                self.q = remove_twist(self.q)
        self.rpy = quat_to_rpy(self.q)
        self.body_q = quat_multiply_right_conjugate(self.q, self.q_rel)
        self.body_omega = quat_apply(self.q_rel, self.omega)
        if self.tc_inv is not None:
            self.body_q = remove_twist(self.body_q)
            if math.isfinite(self.tc_inv):
                self.body_q, self.twist = update_twist(self.body_q, self.twist, self.body_omega, self.tc_inv, self.dt)
        self.body_rpy = quat_to_rpy(self.body_q)
