"""States on and next to the thresholds of the kernels' discrete decisions (test infrastructure), and the reference's float64
predicates on them.  The authority for an angle is the Bullet stand-in's getEulerFromQuaternion, evaluated drone by drone with
the host libm (the reference's own); the oracle's NumPy trigonometry is not used for decisions."""
import math
from fractions import Fraction

import numpy as np

from oracle.standins import pybullet as pb

TILT = 0.4
TERM_DIST = 1e-4
XY_BOUND = {"hover": 1.5, "multihover": 2.0}
Z_BOUND = 2.0
HALF_PI = math.pi / 2
GUARD = 0.99999


def ulps(x, k):
    """x moved by k ulps (k may be negative)."""
    x = np.float64(x)
    for _ in range(abs(int(k))):
        x = np.nextafter(x, np.inf if k > 0 else -np.inf)
    return float(x)


def quat(rpy):
    return np.array([pb.getQuaternionFromEuler(r) for r in np.asarray(rpy, np.float64).reshape(-1, 3)])


def euler(q):
    return np.array([pb.getEulerFromQuaternion(v) for v in np.asarray(q, np.float64).reshape(-1, 4)])


def tilt_poses(yaws=(0.0, 1.0, -2.5, 3.0), k=6):
    """S1: roll or pitch at +-0.4 + j*delta, delta from 1e-9 down to one ulp of 0.4, over several yaws -> rpy [n, 3]."""
    angles = set()
    for s in (1.0, -1.0):
        for delta in (1e-9, 1e-11, 1e-13, 1e-15):
            angles.update(s * (TILT + j * delta) for j in range(-k, k + 1))
        angles.update(s * ulps(TILT, j) for j in range(-4 * k, 4 * k + 1))
    rows = []
    for a in sorted(angles):
        for y in yaws:
            rows.append((a, 0.0, y))
            rows.append((0.0, a, y))
    return np.array(rows)


def tilted(q, bound=TILT):
    """HoverAviary._computeTruncated's tilt term on the stand-in's float64 rpy -> bool [n]."""
    r = euler(q)
    return (np.abs(r[:, 0]) > bound) | (np.abs(r[:, 1]) > bound)


def tilt_margin(q, bound=TILT):
    """Distance of the nearer of |roll|, |pitch| to the bound, in ulps of the bound."""
    r = np.abs(euler(q)[:, :2])
    return np.min(np.abs(r - bound), axis=1) / np.spacing(bound)


def bound_positions(task, k=4):
    """S2: x or y at +-xy_bound + j ulps, z at 2.0 + j ulps (the others well inside) -> pos [n, 3]."""
    b = XY_BOUND[task]
    rows = []
    for j in range(-k, k + 1):
        for s in (1.0, -1.0):
            rows.append((s * ulps(b, j), 0.0, 1.0))
            rows.append((0.0, s * ulps(b, j), 1.0))
        rows.append((0.0, 0.0, ulps(Z_BOUND, j)))
    return np.array(rows)


def out_of_bounds(pos, task):
    b = XY_BOUND[task]
    return (np.abs(pos[:, 0]) > b) | (np.abs(pos[:, 1]) > b) | (pos[:, 2] > Z_BOUND)


def guard_quats(k=40, step=2.5e-14, rng_seed=0):
    """S4: quaternions whose sarg = -2(xz - wy) lies within a few ulps of +-0.99999 on both sides, plus pitch within 1e-3 of +-pi/2."""
    rng = np.random.default_rng(rng_seed)
    p0 = math.asin(GUARD)
    rows = []
    for s in (1.0, -1.0):
        for j in range(-k, k + 1):
            rows.append((rng.uniform(-3, 3), s * (p0 + j * step), rng.uniform(-3, 3)))
        for p in np.linspace(HALF_PI - 1e-3, HALF_PI, 41):
            rows.append((rng.uniform(-3, 3), s * p, rng.uniform(-3, 3)))
    return quat(rows)


def sarg(q):
    q = np.asarray(q, np.float64).reshape(-1, 4)
    x, y, z, w = q.T
    return -2.0 * (x * z - w * y)


def upright_quats(n=4000, rng_seed=0):
    """S5: roll at +-pi/2 + ~1e-16 (rb tiny positive, zero or negative), random pitch and yaw."""
    rng = np.random.default_rng(rng_seed)
    rows = []
    for _ in range(n):
        r = HALF_PI + int(rng.integers(-50, 50)) * 1e-17 * (1 + rng.random())
        rows.append((r * rng.choice([-1.0, 1.0]), rng.uniform(-1, 1), rng.uniform(-3, 3)))
    q = quat(rows)
    # roll exactly +-pi/2 of a hand-made quaternion: rb = 0 exactly
    c = math.sqrt(0.5)
    extra = [(c, 0.0, 0.0, c), (-c, 0.0, 0.0, c), (c, 0.0, 0.0, -c)]
    return np.concatenate([q, np.array(extra)])


def upright(q):
    """BaseAviary._groundEffect's switch (BaseAviary.py:742) on the stand-in's float64 rpy -> bool [n]."""
    r = euler(q)
    return (np.abs(r[:, 0]) < np.pi / 2) & (np.abs(r[:, 1]) < np.pi / 2)


def pid_states(rng_seed=0):
    """S4 + S6 inputs of DSLPIDControl.computeControl, all float32-representable (the device controller takes float32):
    pitch at the gimbal guard with last_rpy next to it, and yaw at +-pi + j ulps with last_rpy's yaw on the other side of the
    wrap -> dict(pos, quat, vel, last_rpy, target_pos, target_rpy), float64 [n, k]."""
    rng = np.random.default_rng(rng_seed)
    qg = guard_quats()
    rows, last = [], []
    for s in (1.0, -1.0):
        for j in range(-8, 9):
            yaw = ulps(s * math.pi, j * 4000)                                  # float32 rounding keeps both sides of +-pi
            rows.append((rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2), yaw))
            last.append((0.0, 0.0, -yaw))
    q = np.concatenate([qg, quat(rows)])
    f32 = lambda a: np.asarray(a, np.float32).astype(np.float64)      # noqa: E731
    q = f32(q)
    eg = euler(qg)
    last_rpy = np.concatenate([eg + rng.uniform(-1e-3, 1e-3, eg.shape), np.array(last)])
    n = q.shape[0]
    return dict(pos=f32(rng.uniform(-0.5, 0.5, (n, 3)) + [0, 0, 1]), quat=q, vel=f32(rng.uniform(-0.3, 0.3, (n, 3))),
                last_rpy=last_rpy, target_pos=f32(np.tile([0.1, -0.1, 1.2], (n, 1))),
                target_rpy=f32(np.stack([np.zeros(n), np.zeros(n), np.where(np.arange(n) % 2 == 0, math.pi, -math.pi)], axis=1)))


def oracle_pid(st, dt):
    """One teacher-forced call of the oracle's DSLPIDControl -> (rpm [n, 4], last_rpy [n, 3])."""
    from oracle import dyn_oracle as O
    o = O.OraclePID(st["pos"].shape[0])
    o.last_rpy = st["last_rpy"].copy()
    rpm, _, _ = o.compute(dt, st["pos"], st["quat"], st["vel"], st["target_pos"], target_rpy=st["target_rpy"])
    return rpm, o.last_rpy


def _norm2_is_one(q):
    """quad_core.cuh's quat_norm2 (fma(w,w, fma(z,z, fma(y,y, x*x))), each step rounded once) == 1.0 exactly."""
    x, y, z, w = (Fraction(float(v)) for v in q)
    r = float(x * x)
    for v in (y, z, w):
        r = float(v * v + Fraction(r))
    return r == 1.0


def ground_effect_states(n=800):
    """S5 states for a one-substep tick: the S5 and S4 attitudes whose |q|^2 is exactly 1 in the kernels' arithmetic (so the
    renormalisation on entry, rsqrt on the device and 1/sqrt on the host, leaves q untouched and the switch sees the bits the
    reference sees), each at heights below, near and above GND_EFF_H_CLIP -> (pos [m, 3], quat [m, 4])."""
    q = np.concatenate([upright_quats(n=n), guard_quats()])
    q = q[[_norm2_is_one(v) for v in q]]
    heights = np.array([0.0, 0.05, 0.5])
    pos = np.zeros((q.shape[0] * heights.size, 3))
    pos[:, 2] = np.tile(heights, q.shape[0])
    return pos, np.repeat(q, heights.size, axis=0)


def oracle_ground_effect_tick(pos, q, action, pyb_freq=240, flip=False):
    """One PYB_GND substep of the float64 oracle from rest, RPM action `action` (float32), with the upright decision taken from
    the stand-in (flip=True: the other decision, the negative control) -> (pos, quat, vel, rpy_rates)."""
    from oracle import dyn_oracle as O
    P = O.OracleParams("cf2x", pyb_freq, pyb_freq)
    n = pos.shape[0]
    rpm = np.full((n, 4), P.HOVER_RPM * float(np.float32(1.0) + np.float32(0.05) * np.float32(action)))
    up = upright(q)
    if flip:
        up = ~up
    rpy = np.where(up[:, None], [[0.0, 0.0, 0.0]], [[np.pi, 0.0, 0.0]])       # stands for the decision only
    z = np.zeros((n, 3))
    p1, q1, v1, w1, _ = O.dynamics_substep(P, rpm, pos, q, z, z, effects=O.EFFECT_GND, rpm_prev=np.zeros((n, 4)), rpy=rpy)
    return p1, q1, v1, w1
