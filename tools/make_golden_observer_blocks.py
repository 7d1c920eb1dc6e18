"""Generates tests/golden/observer_blocks.npz by RUNNING THE REFERENCE'S OWN CODE in this container.

The device observers (jb_set_mahony_filter_full, jb_set_body_observer) restate gym_jiminy's `MahonyFilter` options and
`BodyObserver`: `mahony_filter` (blocks/mahony_filter.py:28-101), `update_twist` (blocks/body_orientation_observer.py:
26-72) and, from utils/math.py, `compute_tilt_from_quat`, `swing_from_vector`, `remove_twist_from_quat`, `quat_to_rpy`,
`quat_multiply`, `quat_apply` and `matrices_to_quat`.  As in tools/make_golden_controller_blocks.py, their source text is
extracted from the reference tree with `ast` and compiled unchanged (numpy and numba only); only the numeric vectors are
committed.  The chained sequences apply the functions in the order the blocks' `refresh_observation` methods do
(mahony_filter.py:337-393, body_orientation_observer.py:237-266): the first refresh is the (re)start one.

Run once (reference at /root/reference, numba installed):  python tools/make_golden_observer_blocks.py
"""
import importlib.util
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden_controller_blocks import REF, extract  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "observer_blocks.npz")
G = 9.81
K = 12          # refreshes per chained sequence, the first one the (re)start


def load():
    tmp = tempfile.mkdtemp(prefix="jb_golden_")
    path = os.path.join(tmp, "ref_observer_blocks.py")
    with open(path, "w") as fh:
        fh.write("from typing import Optional, Tuple, Union\nimport numpy as np\nimport numba as nb\n\n")
        fh.write("ArrayOrScalar = Union[np.ndarray, float]\nTWIST_SWING_SINGULAR_THR = 1e-5   # utils/math.py:15\n")
        fh.write("EARTH_SURFACE_GRAVITY = 9.81   # blocks/mahony_filter.py:23\n\n")
        fh.write(extract(os.path.join(REF, "..", "utils", "math.py"),
                         {"compute_tilt_from_quat", "swing_from_vector", "remove_twist_from_quat", "quat_to_rpy",
                          "quat_multiply", "quat_apply", "matrices_to_quat"}))
        fh.write("\n\n")
        fh.write(extract(os.path.join(REF, "mahony_filter.py"), {"mahony_filter"}))
        fh.write("\n\n")
        fh.write(extract(os.path.join(REF, "body_orientation_observer.py"), {"update_twist"}))
        fh.write("\n")
    spec = importlib.util.spec_from_file_location("ref_observer_blocks", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def rot(quat):
    x, y, z, w = quat / np.linalg.norm(quat)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def singular_vectors(rng):
    """Unit vectors with v_z < -1 + 1e-5, one per sub-case of the singular branch: both horizontal components within
    the threshold, only x (resp. y) within it with a small ratio, only one within it with a large ratio, neither."""
    out = []
    for _ in range(4):
        for vx, vy in ((rng.uniform(-9e-6, 9e-6), rng.uniform(-9e-6, 9e-6)),
                       (rng.uniform(-9e-6, 9e-6) * 1e-3, rng.choice([-1, 1]) * rng.uniform(2e-5, 3e-3)),
                       (rng.choice([-1, 1]) * rng.uniform(2e-5, 3e-3), rng.uniform(-9e-6, 9e-6) * 1e-3),
                       (rng.uniform(-9e-6, 9e-6), rng.choice([-1, 1]) * rng.uniform(1e-3, 3e-3)),
                       (rng.choice([-1, 1]) * rng.uniform(1e-3, 3e-3), rng.choice([-1, 1]) * rng.uniform(1e-3, 3e-3))):
            out.append(np.array([vx, vy, -np.sqrt(1.0 - vx * vx - vy * vy)]))
    out.append(np.array([0.0, 0.0, -1.0]))
    return out


def chain(mod, rng, exact_init, ignore_twist, tc, start, rel):
    """One observer sequence: MahonyFilter (kp, ki) then BodyObserver(twist_time_constant=tc) over K refreshes."""
    kp, ki, dt = float(rng.uniform(0.5, 2.0)), float(rng.uniform(0.0, 0.3)), 0.005
    R_true = rot(rng.normal(size=4))
    R_rel = {"identity": np.eye(3), "flip": rot(np.array([1.0, 0.0, 0.0, 0.0])), "random": rot(rng.normal(size=4))}[rel]
    gyro = rng.normal(size=(K, 3)) * 0.8
    acc = rng.normal(size=(K, 3)) * 1.5 + np.array([0.0, 0.0, G])
    if start == "free_fall":
        acc[0] = rng.uniform(-0.9, 0.9, 3)
    elif start == "upside_down":
        acc[0] = G * singular_vectors(rng)[int(rng.integers(21))] * rng.uniform(0.9, 1.1)
    quat, omega, cf, bias = np.zeros((4, 1)), np.zeros((3, 1)), np.zeros((3, 1)), np.zeros((3, 1))
    quat[-1] = 1.0
    rpy, q_rel = np.zeros((3, 1)), mod.matrices_to_quat((R_rel,))
    b_quat, b_omega, b_rpy, twist = np.zeros((4, 1)), np.zeros((3, 1)), np.zeros((3, 1)), np.zeros((1, 1))
    tc_inv = None if tc is None else (1.0 / tc if tc > 0.0 else float("inf"))
    rec = {k: [] for k in ("mq", "momega", "mbias", "mrpy", "bq", "bomega", "brpy", "twist")}
    still = int(rng.integers(3, K))          # a refresh with no IMU motion: the filter's early return
    for j in range(K):
        if j == still:
            gyro[j] = bias[:, 0]
            acc[j] = G * np.stack(mod.compute_tilt_from_quat(quat))[:, 0]
        g, a = gyro[j][:, None].copy(), acc[j][:, None].copy()
        if j == 0:
            done = False
            if not exact_init and not (np.abs(a) < 0.1 * mod.EARTH_SURFACE_GRAVITY).all():
                mod.swing_from_vector(a / np.linalg.norm(a, axis=0), quat)
                done = True
            if not done:
                mod.matrices_to_quat((R_true,), quat)
        else:
            mod.mahony_filter(quat, omega, cf, g, a, bias, kp, ki, dt)
            if ignore_twist:
                mod.remove_twist_from_quat(quat)
        mod.quat_to_rpy(quat, rpy)
        mod.quat_multiply(quat, q_rel, out=b_quat, is_right_conjugate=True)
        mod.quat_apply(q_rel, omega, out=b_omega)
        if tc_inv is not None:
            mod.remove_twist_from_quat(b_quat)
            if np.isfinite(tc_inv):
                mod.update_twist(b_quat, twist, b_omega, tc_inv, dt)
        mod.quat_to_rpy(b_quat, b_rpy)
        for k, x in zip(rec, (quat, omega, bias, rpy, b_quat, b_omega, b_rpy, twist)):
            rec[k].append(x[:, 0].copy())
    inputs = dict(kp=kp, ki=ki, dt=dt, exact_init=exact_init, ignore_twist=ignore_twist,
                  tc=np.nan if tc is None else tc, R_true=R_true, R_rel=R_rel, gyro=gyro, acc=acc)
    return inputs, {k: np.array(v) for k, v in rec.items()}


def main():
    mod = load()
    rng = np.random.default_rng(20261019)
    out = {}
    # swing_from_vector on [3][1] columns: every singular sub-case, then regular unit vectors
    vs = singular_vectors(rng) + [v / np.linalg.norm(v) for v in rng.normal(size=(40, 3))]
    sw = []
    for v in vs:
        q = np.zeros((4, 1))
        mod.swing_from_vector(tuple(v[:, None]), q)
        sw.append(q[:, 0].copy())
    out["sw_v"], out["sw_q"] = np.array(vs), np.array(sw)
    # remove_twist_from_quat, quat_to_rpy (pitch near +-pi/2 included), quat_multiply / quat_apply, matrices_to_quat,
    # update_twist
    qs = rng.normal(size=(60, 4))
    qs /= np.linalg.norm(qs, axis=1)[:, None]
    qs[:4] = [[0.0, 0.7071067811865476, 0.0, 0.7071067811865476], [0.0, -0.7071067811865476, 0.0, 0.7071067811865476],
              [0.5, 0.5, -0.5, 0.5], [1.0, 0.0, 0.0, 1e-9]]
    out["q"] = qs
    rt, rpy = [], []
    for q in qs:
        a = q[:, None].copy()
        mod.remove_twist_from_quat(a)
        rt.append(a[:, 0].copy())
        r = np.zeros((3, 1))
        mod.quat_to_rpy(q[:, None].copy(), r)
        rpy.append(r[:, 0].copy())
    out["rt_q"], out["rpy"] = np.array(rt), np.array(rpy)
    q2 = rng.normal(size=(60, 4))
    q2 /= np.linalg.norm(q2, axis=1)[:, None]
    vec = rng.normal(size=(60, 3))
    mul, app = [], []
    for a, b, v in zip(qs, q2, vec):
        o = np.zeros((4, 1))
        mod.quat_multiply(a[:, None].copy(), b[:, None].copy(), out=o, is_right_conjugate=True)
        mul.append(o[:, 0].copy())
        p = np.zeros((3, 1))
        mod.quat_apply(b[:, None].copy(), v[:, None].copy(), out=p)
        app.append(p[:, 0].copy())
    out["q2"], out["vec"], out["mul_rc"], out["apply"] = q2, vec, np.array(mul), np.array(app)
    ut_in = {k: [] for k in ("ut_q", "ut_twist", "ut_omega", "ut_tc_inv", "ut_dt", "ut_q_out", "ut_twist_out")}
    for j in range(40):
        q = np.zeros((4, 1))
        v = rng.normal(size=3)
        mod.swing_from_vector(tuple((v / np.linalg.norm(v))[:, None]), q)
        tw, om = np.array([[rng.uniform(-3, 3)]]), rng.normal(size=(3, 1))
        tc_inv, dt = float(rng.choice([0.1, 1.0 / 0.3, 50.0, 400.0])), float(rng.choice([0.005, 0.01]))
        qo, two = q.copy(), tw.copy()
        mod.update_twist(qo, two, om, tc_inv, dt)
        for k, x in zip(ut_in, (q[:, 0], tw[0, 0], om[:, 0], tc_inv, dt, qo[:, 0], two[0, 0])):
            ut_in[k].append(np.array(x))
    out.update({k: np.array(v) for k, v in ut_in.items()})
    # chained sequences
    ch_in, ch_out = {}, {}
    for exact_init in (True, False):
        for ignore_twist in (False, True):
            for tc in (None, 0.0, 0.3):
                for start, rel in (("standing", "random"), ("free_fall", "identity"), ("upside_down", "flip")):
                    i, o = chain(mod, rng, exact_init, ignore_twist, tc, start, rel)
                    for k, v in i.items():
                        ch_in.setdefault("c_" + k, []).append(v)
                    for k, v in o.items():
                        ch_out.setdefault("c_" + k, []).append(v)
    out.update({k: np.array(v) for k, v in {**ch_in, **ch_out}.items()})
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    sys.exit(main())
