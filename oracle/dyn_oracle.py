"""Tier-2 oracle: batched float64 NumPy restatement of the reference hot path.

ORACLE / TEST INFRASTRUCTURE -- not product code.  Only tests/, smoke() and
bench.py's CPU-baseline legs import this module; the product package never does.

Parity status: PINNED against the unmodified reference (tier 1, run through the
stand-ins of oracle/standins/) by the golden vectors in tests/golden/*.npz, which
tests/golden/make_golden.py regenerates in the build container.  The three
Bullet quaternion helpers are restated from Bullet's published algorithm
(pybullet ^3.2.7, absent here) and cross-checked against scipy only.

All file:line citations are into /root/reference/gym_pybullet_drones/.

Everything is vectorised over a leading drone axis N (or [E, D]); `dtype`
defaults to float64 like the reference (numpy default + Bullet doubles) and can
be set to float32 to study rounding.
"""
import math

import numpy as np

# --------------------------------------------------------------------------
# Constants (assets/cf2x.urdf:5,11-12,34,42-78; cf2p.urdf; racer.urdf) and the
# derived constants of envs/BaseAviary.py:116-128.
# --------------------------------------------------------------------------
_URDF = {
    "cf2x": dict(m=0.027, arm=0.0397, kf=3.16e-10, km=7.94e-12, t2w=2.25, max_speed_kmh=30.0,
                 gnd_eff_coeff=11.36859, prop_radius=2.31348e-2, drag_xy=9.1785e-7, drag_z=10.311e-7,
                 dw1=2267.18, dw2=0.16, dw3=-0.11, ixx=1.4e-5, iyy=1.4e-5, izz=2.17e-5,
                 coll_h=0.025, coll_r=0.06, coll_z=0.0,
                 props=[[0.028, -0.028, 0.0], [-0.028, -0.028, 0.0], [-0.028, 0.028, 0.0], [0.028, 0.028, 0.0]]),
    "cf2p": dict(m=0.027, arm=0.0397, kf=3.16e-10, km=7.94e-12, t2w=2.25, max_speed_kmh=30.0,
                 gnd_eff_coeff=11.36859, prop_radius=2.31348e-2, drag_xy=9.1785e-7, drag_z=10.311e-7,
                 dw1=2267.18, dw2=0.16, dw3=-0.11, ixx=2.3951e-5, iyy=2.3951e-5, izz=3.2347e-5,
                 coll_h=0.025, coll_r=0.06, coll_z=0.0,
                 props=[[0.0397, 0.0, 0.0], [0.0, 0.0397, 0.0], [-0.0397, 0.0, 0.0], [0.0, -0.0397, 0.0]]),
    "racer": dict(m=0.830, arm=0.109, kf=8.47e-9, km=2.13e-11, t2w=4.17, max_speed_kmh=200.0,
                  gnd_eff_coeff=11.36859, prop_radius=12.7e-2, drag_xy=9.1785e-7, drag_z=10.311e-7,
                  dw1=2267.18, dw2=0.16, dw3=-0.11, ixx=0.003113, iyy=0.003113, izz=0.003113,
                  coll_h=0.025, coll_r=0.06, coll_z=0.0,
                  props=[[0.0850, 0.0675, 0.0], [-0.0850, 0.0675, 0.0], [-0.085, -0.0675, 0.0], [0.085, -0.0675, 0.0]]),
}

EFFECT_GND = 1
EFFECT_DRAG = 2
EFFECT_DW = 4


class OracleParams:
    """BaseAviary.__init__ constants (envs/BaseAviary.py:74-128)."""

    def __init__(self, drone_model="cf2x", pyb_freq=240, ctrl_freq=240, g=9.8):
        u = _URDF[drone_model]
        self.model = drone_model
        self.G = g
        self.M, self.L, self.KF, self.KM = u["m"], u["arm"], u["kf"], u["km"]
        self.T2W = u["t2w"]
        self.J = np.array([u["ixx"], u["iyy"], u["izz"]])
        self.J_INV = 1.0 / self.J                      # np.linalg.inv of a diagonal matrix
        self.MAX_SPEED_KMH = u["max_speed_kmh"]
        self.GND_EFF_COEFF, self.PROP_RADIUS = u["gnd_eff_coeff"], u["prop_radius"]
        self.DRAG_COEFF = np.array([u["drag_xy"], u["drag_xy"], u["drag_z"]])
        self.DW = (u["dw1"], u["dw2"], u["dw3"])
        self.COLLISION_H, self.COLLISION_Z_OFFSET = u["coll_h"], u["coll_z"]
        self.PROPS = np.array(u["props"])
        self.PYB_FREQ, self.CTRL_FREQ = pyb_freq, ctrl_freq
        if pyb_freq % ctrl_freq != 0:
            raise ValueError("pyb_freq is not divisible by ctrl_freq")    # BaseAviary.py:79-80
        self.S = pyb_freq // ctrl_freq
        self.CTRL_TIMESTEP = 1.0 / ctrl_freq
        self.PYB_TIMESTEP = 1.0 / pyb_freq
        self.GRAVITY = self.G * self.M                                        # :117
        self.HOVER_RPM = math.sqrt(self.GRAVITY / (4 * self.KF))              # :118
        self.MAX_RPM = math.sqrt((self.T2W * self.GRAVITY) / (4 * self.KF))   # :119
        self.MAX_THRUST = 4 * self.KF * self.MAX_RPM ** 2                     # :120
        if drone_model == "cf2p":
            self.MAX_XY_TORQUE = self.L * self.KF * self.MAX_RPM ** 2         # :123-124
        else:
            self.MAX_XY_TORQUE = (2 * self.L * self.KF * self.MAX_RPM ** 2) / math.sqrt(2)
        self.MAX_Z_TORQUE = 2 * self.KM * self.MAX_RPM ** 2                   # :127
        self.GND_EFF_H_CLIP = 0.25 * self.PROP_RADIUS * math.sqrt(
            (15 * self.MAX_RPM ** 2 * self.KF * self.GND_EFF_COEFF) / self.MAX_THRUST)   # :128

    def default_init_xyzs(self, num_drones):
        """envs/BaseAviary.py:194-197."""
        i = np.arange(num_drones, dtype=np.float64)
        z = np.ones(num_drones) * (self.COLLISION_H / 2 - self.COLLISION_Z_OFFSET + 0.1)
        return np.stack([i * 4 * self.L, i * 4 * self.L, z], axis=1)


# --------------------------------------------------------------------------
# Bullet quaternion helpers (quaternion order x,y,z,w), batched on axis 0.
# --------------------------------------------------------------------------
def quat_to_matrix(q):
    """p.getMatrixFromQuaternion (call sites BaseAviary.py:836, DSLPIDControl.py:187,240).
    Returns R[..., 3, 3]; normalises implicitly through s = 2/|q|^2."""
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    s = 2.0 / (x * x + y * y + z * z + w * w)
    xs, ys, zs = x * s, y * s, z * s
    wx, wy, wz = w * xs, w * ys, w * zs
    xx, xy, xz = x * xs, x * ys, x * zs
    yy, yz, zz = y * ys, y * zs, z * zs
    R = np.empty(q.shape[:-1] + (3, 3), dtype=q.dtype)
    R[..., 0, 0] = 1.0 - (yy + zz); R[..., 0, 1] = xy - wz;         R[..., 0, 2] = xz + wy
    R[..., 1, 0] = xy + wz;         R[..., 1, 1] = 1.0 - (xx + zz); R[..., 1, 2] = yz - wx
    R[..., 2, 0] = xz - wy;         R[..., 2, 1] = yz + wx;         R[..., 2, 2] = 1.0 - (xx + yy)
    return R


def quat_to_euler(q):
    """p.getEulerFromQuaternion (BaseAviary.py:518, DSLPIDControl.py:144,241):
    ZYX (roll,pitch,yaw) with Bullet's +-0.99999 gimbal guard, no normalisation."""
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    sarg = -2.0 * (x * z - w * y)
    roll = np.arctan2(2.0 * (y * z + w * x), w * w - x * x - y * y + z * z)
    pitch = np.arcsin(np.clip(sarg, -1.0, 1.0))
    yaw = np.arctan2(2.0 * (x * y + w * z), w * w + x * x - y * y - z * z)
    lo, hi = sarg <= -0.99999, sarg >= 0.99999
    half_pi = q.dtype.type(0.5 * math.pi)
    roll = np.where(lo | hi, 0.0, roll)
    pitch = np.where(lo, -half_pi, np.where(hi, half_pi, pitch))
    yaw = np.where(lo, 2.0 * np.arctan2(x, -y), np.where(hi, 2.0 * np.arctan2(-x, y), yaw))
    return np.stack([roll, pitch, yaw], axis=-1).astype(q.dtype)


def euler_to_quat(rpy):
    """p.getQuaternionFromEuler (BaseAviary.py:488)."""
    h = rpy * 0.5
    cr, sr = np.cos(h[..., 0]), np.sin(h[..., 0])
    cp, sp = np.cos(h[..., 1]), np.sin(h[..., 1])
    cy, sy = np.cos(h[..., 2]), np.sin(h[..., 2])
    q = np.stack([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy,
                  cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy], axis=-1)
    return q / np.linalg.norm(q, axis=-1, keepdims=True)


# --------------------------------------------------------------------------
# Physics.DYN: _dynamics + _integrateQ, with the DYN+ aerodynamic terms.
# --------------------------------------------------------------------------
def integrate_q(q, omega, dt):
    """BaseAviary._integrateQ (envs/BaseAviary.py:879-892): exact exponential map
    for constant body rate omega over dt; identity when np.isclose(|omega|, 0)."""
    n = np.sqrt(np.sum(omega * omega, axis=-1))
    p_, q_, r_ = omega[..., 0], omega[..., 1], omega[..., 2]
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    still = np.abs(n) <= 1e-8                      # np.isclose(n, 0): atol 1e-8 + rtol*0
    nn = np.where(still, 1.0, n)
    th = nn * dt / 2
    c, s = np.cos(th), np.sin(th) / nn             # (2/|w|)*lambda*sin = (sin/|w|)*Omega
    out = np.stack([c * x + s * (r_ * y - q_ * z + p_ * w),
                    c * y + s * (-r_ * x + p_ * z + q_ * w),
                    c * z + s * (q_ * x - p_ * y + r_ * w),
                    c * w + s * (-p_ * x - q_ * y - r_ * z)], axis=-1)
    return np.where(still[..., None], q, out).astype(q.dtype)


def ground_effect_thrust(P, rpm, pos, R, rpy):
    """BaseAviary._groundEffect (envs/BaseAviary.py:715-750): per-propeller extra
    thrust along the link z axis; zero unless |roll|,|pitch| < pi/2."""
    prop_z = pos[..., None, 2] + np.einsum("...j,kj->...k", R[..., 2, :], P.PROPS.astype(pos.dtype))
    h = np.clip(prop_z, P.GND_EFF_H_CLIP, np.inf)                                        # :739-740
    g = rpm ** 2 * P.KF * P.GND_EFF_COEFF * (P.PROP_RADIUS / (4 * h)) ** 2               # :741
    ok = (np.abs(rpy[..., 0]) < np.pi / 2) & (np.abs(rpy[..., 1]) < np.pi / 2)           # :742
    return np.where(ok[..., None], g, 0.0).astype(pos.dtype)


def drag_force_world(P, rpm_prev, vel):
    """BaseAviary._drag (envs/BaseAviary.py:754-781).  The reference rotates
    drag_factors*vel into the body frame and applies it in LINK_FRAME, i.e. the
    world-frame force is drag_factors (.) vel_world."""
    factors = -1 * P.DRAG_COEFF.astype(vel.dtype) * np.sum(2 * np.pi * rpm_prev / 60, axis=-1, keepdims=True)
    return factors * vel


def downwash_body_z(P, pos, group_size=None):
    """BaseAviary._downwash (envs/BaseAviary.py:785-811): for every drone n, the sum
    over drones i above it (dz>0) and within 10 m in xy of -alpha*exp(-.5 (dxy/beta)^2),
    a force along n's BODY z axis.  `pos` is [E, D, 3]; pairs are taken within an aviary."""
    dz = pos[:, None, :, 2] - pos[:, :, None, 2]            # [E, n, i] = z_i - z_n
    dxy = np.sqrt((pos[:, None, :, 0] - pos[:, :, None, 0]) ** 2 + (pos[:, None, :, 1] - pos[:, :, None, 1]) ** 2)
    act = (dz > 0) & (dxy < 10)
    dzs = np.where(act, dz, 1.0)
    alpha = P.DW[0] * (P.PROP_RADIUS / (4 * dzs)) ** 2
    beta = P.DW[1] * dzs + P.DW[2]
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        f = -alpha * np.exp(-0.5 * (dxy / beta) ** 2)
    return np.sum(np.where(act, f, 0.0), axis=2).astype(pos.dtype)


def adjacency_matrix(pos, radius):
    """BaseAviary._getAdjacencyMatrix (envs/BaseAviary.py:658-675): identity plus 1 where
    |pos_i - pos_j| < NEIGHBOURHOOD_RADIUS.  `pos` is [E, D, 3]; returns float64 [E, D, D]."""
    d = pos[:, :, None, :] - pos[:, None, :, :]
    dist = np.sqrt(np.sum(d * d, axis=-1))
    adj = (dist < radius).astype(np.float64)
    idx = np.arange(pos.shape[1])
    adj[:, idx, idx] = 1.0
    return adj


def dynamics_substep(P, rpm, pos, quat, vel, rpy_rates, effects=0, rpm_prev=None, dw_fz=None, rpy=None):
    """BaseAviary._dynamics (envs/BaseAviary.py:815-877) for a batch [..., ] of drones.

    DYN+ (SURVEY.md 8a rows 6-8): with `effects` flags the reference's PYB-only
    force models are added as explicit terms evaluated on the substep-start state:
      GND  : f_i <- f_i + g_i in the collective thrust and the x/y torques
      DRAG : + drag_force_world(rpm_prev, vel)
      DW   : + R [0,0,dw_fz]
    Returns (pos, quat, vel, rpy_rates, ang_v)."""
    dt = P.PYB_TIMESTEP
    R = quat_to_matrix(quat)                                                     # :836
    forces = rpm ** 2 * P.KF                                                     # :838
    if effects & EFFECT_GND:
        if rpy is None:
            rpy = quat_to_euler(quat)
        forces = forces + ground_effect_thrust(P, rpm, pos, R, rpy)
    thrust = np.sum(forces, axis=-1)
    force_world = R[..., :, 2] * thrust[..., None]                               # :839-840
    force_world[..., 2] -= P.GRAVITY                                             # :841
    if effects & EFFECT_DRAG:
        force_world = force_world + drag_force_world(P, rpm_prev, vel)
    if effects & EFFECT_DW:
        force_world = force_world + R[..., :, 2] * dw_fz[..., None]
    zt = rpm ** 2 * P.KM                                                         # :842
    if P.model == "racer":
        zt = -zt                                                                 # :843-844
    z_torque = -zt[..., 0] + zt[..., 1] - zt[..., 2] + zt[..., 3]                # :845
    f0, f1, f2, f3 = forces[..., 0], forces[..., 1], forces[..., 2], forces[..., 3]
    if P.model == "racer":                                                       # :846-848
        x_torque = (f0 + f1 - f2 - f3) * (P.L / np.sqrt(2))
        y_torque = (-f0 + f1 + f2 - f3) * (P.L / np.sqrt(2))
    elif P.model == "cf2x":                                                      # :849-851
        x_torque = -(f0 + f1 - f2 - f3) * (P.L / np.sqrt(2))
        y_torque = (-f0 + f1 + f2 - f3) * (P.L / np.sqrt(2))
    else:                                                                        # cf2p :852-854
        x_torque = (f1 - f3) * P.L
        y_torque = (-f0 + f2) * P.L
    J = P.J.astype(pos.dtype)
    torques = np.stack([x_torque, y_torque, z_torque], axis=-1)
    torques = torques - np.cross(rpy_rates, J * rpy_rates)                       # :856
    rates_deriv = torques * P.J_INV.astype(pos.dtype)                            # :857
    acc = force_world / P.M                                                      # :858
    vel = vel + dt * acc                                                         # :860
    rpy_rates = rpy_rates + dt * rates_deriv                                     # :861
    pos = pos + dt * vel                                                         # :862
    quat_new = integrate_q(quat, rpy_rates, dt)                                  # :863
    ang_v = np.einsum("...ij,...j->...i", R, rpy_rates)                          # :873
    dtp = quat.dtype
    return pos.astype(dtp), quat_new.astype(dtp), vel.astype(dtp), rpy_rates.astype(dtp), ang_v.astype(dtp)


# --------------------------------------------------------------------------
# DSLPIDControl (control/DSLPIDControl.py), batched with per-drone state.
# --------------------------------------------------------------------------
_MIXER = {
    "cf2x": np.array([[-.5, -.5, -1], [-.5, .5, 1], [.5, .5, -1], [.5, -.5, 1]]),       # :49-54
    "cf2p": np.array([[0, -1, -1], [1, 0, 1], [0, 1, -1], [-1, 0, 1]], dtype=float),   # :55-61
}


class OraclePID:
    """DSLPIDControl for N drones (control/DSLPIDControl.py:37-259)."""

    def __init__(self, n, drone_model="cf2x", g=9.8, dtype=np.float64):
        if drone_model not in ("cf2x", "cf2p"):
            raise ValueError("DSLPIDControl requires CF2X or CF2P")             # :33-35
        u = _URDF[drone_model]
        self.n, self.dtype = n, dtype
        self.GRAVITY, self.KF, self.KM = g * u["m"], u["kf"], u["km"]           # BaseControl.py:35-40
        self.P_FOR = np.array([.4, .4, 1.25]); self.I_FOR = np.array([.05, .05, .05]); self.D_FOR = np.array([.2, .2, .5])
        self.P_TOR = np.array([70000., 70000., 60000.]); self.I_TOR = np.array([.0, .0, 500.])
        self.D_TOR = np.array([20000., 20000., 12000.])
        self.PWM2RPM_SCALE, self.PWM2RPM_CONST, self.MIN_PWM, self.MAX_PWM = 0.2685, 4070.3, 20000, 65535
        self.MIXER = _MIXER[drone_model]
        self.reset()

    def reset(self, mask=None):
        """DSLPIDControl.reset (:65-78)."""
        if mask is None:
            self.control_counter = 0
            self.last_rpy = np.zeros((self.n, 3), self.dtype)
            self.integral_pos_e = np.zeros((self.n, 3), self.dtype)
            self.integral_rpy_e = np.zeros((self.n, 3), self.dtype)
        else:
            for a in (self.last_rpy, self.integral_pos_e, self.integral_rpy_e):
                a[mask] = 0

    def compute(self, dt, pos, quat, vel, target_pos, target_rpy=None, target_vel=None, target_rpy_rates=None):
        """computeControl (:82-145) -> (rpm[N,4], pos_e[N,3], yaw_e[N])."""
        z3 = np.zeros((self.n, 3), self.dtype)
        target_rpy = z3 if target_rpy is None else target_rpy
        target_vel = z3 if target_vel is None else target_vel
        target_rpy_rates = z3 if target_rpy_rates is None else target_rpy_rates
        self.control_counter += 1
        R = quat_to_matrix(quat)                                                              # :187
        pos_e = target_pos - pos
        vel_e = target_vel - vel
        ipe = np.clip(self.integral_pos_e + pos_e * dt, -2., 2.)                              # :190-191
        ipe[:, 2] = np.clip(ipe[:, 2], -0.15, 0.15)                                           # :192
        self.integral_pos_e = ipe
        tt = self.P_FOR * pos_e + self.I_FOR * ipe + self.D_FOR * vel_e                       # :194-196
        tt[:, 2] += self.GRAVITY
        scalar = np.maximum(0., np.sum(tt * R[:, :, 2], axis=1))                              # :197
        thrust = (np.sqrt(scalar / (4 * self.KF)) - self.PWM2RPM_CONST) / self.PWM2RPM_SCALE  # :198
        z_ax = tt / np.linalg.norm(tt, axis=1, keepdims=True)                                 # :199
        x_c = np.stack([np.cos(target_rpy[:, 2]), np.sin(target_rpy[:, 2]), np.zeros(self.n)], axis=1)
        yc = np.cross(z_ax, x_c)
        y_ax = yc / np.linalg.norm(yc, axis=1, keepdims=True)                                 # :201
        x_ax = np.cross(y_ax, z_ax)                                                           # :202
        Rd = np.stack([x_ax, y_ax, z_ax], axis=2)                                             # columns :203
        # scipy Rotation.from_matrix(Rd).as_euler('XYZ') (:205), closed form for R=Rx(a)Ry(b)Rz(c)
        a = np.arctan2(-Rd[:, 1, 2], Rd[:, 2, 2])
        b = np.arcsin(np.clip(Rd[:, 0, 2], -1., 1.))
        c = np.arctan2(-Rd[:, 0, 1], Rd[:, 0, 0])
        target_euler = np.stack([a, b, c], axis=1)
        # attitude loop (:240-259); from_euler('XYZ').as_quat()->from_quat->as_matrix is an identity round trip
        ca, sa, cb, sb, cc, sc = np.cos(a), np.sin(a), np.cos(b), np.sin(b), np.cos(c), np.sin(c)
        Rt = np.empty((self.n, 3, 3), self.dtype)
        Rt[:, 0, 0] = cb * cc;                Rt[:, 0, 1] = -cb * sc;               Rt[:, 0, 2] = sb
        Rt[:, 1, 0] = ca * sc + sa * sb * cc; Rt[:, 1, 1] = ca * cc - sa * sb * sc; Rt[:, 1, 2] = -sa * cb
        Rt[:, 2, 0] = sa * sc - ca * sb * cc; Rt[:, 2, 1] = sa * cc + ca * sb * sc; Rt[:, 2, 2] = ca * cb
        cur_rpy = quat_to_euler(quat)                                                         # :241
        Em = np.einsum("nji,njk->nik", Rt, R) - np.einsum("nji,njk->nik", R, Rt)              # :245
        rot_e = np.stack([Em[:, 2, 1], Em[:, 0, 2], Em[:, 1, 0]], axis=1)                     # :246
        rates_e = target_rpy_rates - (cur_rpy - self.last_rpy) / dt                           # :247
        self.last_rpy = cur_rpy                                                               # :248
        ire = np.clip(self.integral_rpy_e - rot_e * dt, -1500., 1500.)                        # :249-250
        ire[:, 0:2] = np.clip(ire[:, 0:2], -1., 1.)                                           # :251
        self.integral_rpy_e = ire
        tq = -self.P_TOR * rot_e + self.D_TOR * rates_e + self.I_TOR * ire                    # :253-255
        tq = np.clip(tq, -3200, 3200)                                                         # :256
        pwm = np.clip(thrust[:, None] + tq @ self.MIXER.T, self.MIN_PWM, self.MAX_PWM)        # :257-258
        rpm = self.PWM2RPM_SCALE * pwm + self.PWM2RPM_CONST                                   # :259
        return rpm.astype(self.dtype), pos_e, target_euler[:, 2] - cur_rpy[:, 2]              # :145


# --------------------------------------------------------------------------
# Env-level restatement: BaseAviary.step / BaseRLAviary / Hover / MultiHover / Ctrl
# --------------------------------------------------------------------------
_ACT_WIDTH = {"rpm": 4, "vel": 4, "pid": 3, "one_d_rpm": 1, "one_d_pid": 1}       # BaseRLAviary.py:141-146


def next_waypoint(cur, dest, step_size=1.0):
    """BaseAviary._calculateNextStep (envs/BaseAviary.py:1108-1150)."""
    d = dest - cur
    dist = np.linalg.norm(d, axis=-1, keepdims=True)
    safe = np.where(dist > 0, dist, 1.0)
    return np.where(dist <= step_size, dest, cur + d / safe * step_size)


class OracleAviary:
    """E independent aviaries of D drones, stepped in lockstep.

    kind = "hover" (HoverAviary.py), "multihover" (MultiHoverAviary.py) or "ctrl"
    (CtrlAviary.py).  Follows BaseAviary.step (envs/BaseAviary.py:259-383) in order:
    preprocess action -> S x dynamics -> refresh cache -> obs/reward/term/trunc ->
    step_counter += S.  The reference quirks are kept: the action buffer and the
    embedded PID controllers are NOT cleared by reset() (SURVEY.md 3.3)."""

    def __init__(self, kind="hover", num_envs=1, num_drones=1, drone_model="cf2x", pyb_freq=240, ctrl_freq=None,
                 act="rpm", initial_xyzs=None, initial_rpys=None, effects=0, dtype=np.float64):
        if ctrl_freq is None:
            ctrl_freq = 240 if kind in ("ctrl", "velocity") else 30    # CtrlAviary.py:19-20, VelocityAviary.py:22-23, HoverAviary.py:16-17
        if kind == "hover":
            num_drones = 1                                             # HoverAviary.py:54
        self.kind, self.E, self.D, self.dtype = kind, num_envs, num_drones, dtype
        self.P = OracleParams(drone_model, pyb_freq, ctrl_freq)
        self.effects = effects
        self.act = act
        P = self.P
        base_xyz = P.default_init_xyzs(num_drones) if initial_xyzs is None else np.asarray(initial_xyzs, dtype=np.float64)
        base_rpy = np.zeros((num_drones, 3)) if initial_rpys is None else np.asarray(initial_rpys, dtype=np.float64)
        self.INIT_XYZS = np.broadcast_to(base_xyz, (self.E, self.D, 3)).astype(dtype).copy()
        self.INIT_RPYS = np.broadcast_to(base_rpy, (self.E, self.D, 3)).astype(dtype).copy()
        self.EPISODE_LEN_SEC = 8                                       # HoverAviary.py:52
        if kind == "hover":
            self.TARGET_POS = np.broadcast_to(np.array([0., 0., 1.]), (self.E, 1, 3)).astype(dtype)   # HoverAviary.py:51
            self.xy_bound = 1.5
        elif kind == "multihover":
            off = np.array([[0, 0, 1 / (i + 1)] for i in range(num_drones)])
            self.TARGET_POS = (self.INIT_XYZS + off).astype(dtype)     # MultiHoverAviary.py:71
            self.xy_bound = 2.0
        if kind == "velocity":                                         # VelocityAviary.py:59-78
            self.act, self.A, self.B = "vel", 4, 0
            self.action_buffer = []
            self.ctrl = OraclePID(self.E * self.D, "cf2x", dtype=dtype)
            self.SPEED_LIMIT = 0.03 * P.MAX_SPEED_KMH * (1000 / 3600)
        elif kind != "ctrl":
            self.A = _ACT_WIDTH[act]
            self.B = int(ctrl_freq // 2)                               # BaseRLAviary.py:66
            self.action_buffer = [np.zeros((self.E, self.D, self.A), dtype) for _ in range(self.B)]   # :153-154
            if act in ("pid", "vel", "one_d_pid"):
                self.ctrl = OraclePID(self.E * self.D, "cf2x", dtype=dtype)   # BaseRLAviary.py:76 (always CF2X)
            if act == "vel":
                self.SPEED_LIMIT = 0.03 * P.MAX_SPEED_KMH * (1000 / 3600)     # BaseRLAviary.py:95
        self._housekeeping()

    # -- BaseAviary._housekeeping (:451-505) + _updateAndStoreKinematicInformation (:509-519)
    def _housekeeping(self, mask=None):
        if mask is None:
            self.step_counter = np.zeros(self.E, dtype=np.int64)
            self.pos = self.INIT_XYZS.copy()
            self.quat = euler_to_quat(self.INIT_RPYS).astype(self.dtype)
            self.vel = np.zeros((self.E, self.D, 3), self.dtype)
            self.ang_v = np.zeros((self.E, self.D, 3), self.dtype)
            self.rpy_rates = np.zeros((self.E, self.D, 3), self.dtype)
            self.last_clipped_action = np.zeros((self.E, self.D, 4), self.dtype)
        else:
            self.step_counter[mask] = 0
            self.pos[mask] = self.INIT_XYZS[mask]
            self.quat[mask] = euler_to_quat(self.INIT_RPYS[mask])
            for a in (self.vel, self.ang_v, self.rpy_rates, self.last_clipped_action):
                a[mask] = 0
        self.rpy = quat_to_euler(self.quat)

    def reset(self, mask=None):
        """BaseAviary.reset (:220-255); `mask` [E] bool resets a subset (vector-env autoreset)."""
        self._housekeeping(mask)
        return self._obs()

    # -- action -> rpm : CtrlAviary.py:121-140, BaseRLAviary.py:160-239
    def _preprocess(self, action):
        P = self.P
        action = np.asarray(action)
        if self.kind == "ctrl":
            return np.clip(action.astype(self.dtype), 0, P.MAX_RPM)
        if self.kind != "velocity" and self.B > 0:                                # deque(maxlen=0) at ctrl_freq 1: no buffer
            self.action_buffer.pop(0)
            self.action_buffer.append(action.copy())                             # :187 (deque maxlen)
        # NumPy-2 promotion (reference pins numpy ^2.2, pyproject.toml:15): python scalars are weak,
        # so with float32 actions `1+0.05*target` is evaluated in float32 and only the product with
        # the np.float64 HOVER_RPM is float64; the VEL target velocity is float32 end to end.
        if self.act == "rpm":
            return np.float64(P.HOVER_RPM) * (1 + 0.05 * action)                # :192
        if self.act == "one_d_rpm":
            return np.repeat(np.float64(P.HOVER_RPM) * (1 + 0.05 * action), 4, axis=-1)   # :225
        n = self.E * self.D
        pos, quat, vel = self.pos.reshape(n, 3), self.quat.reshape(n, 4), self.vel.reshape(n, 3)
        a = action.reshape(n, self.A)
        if self.act == "pid":
            tgt = next_waypoint(pos, a.astype(self.dtype), 1.0)                  # :195-199
            rpm, _, _ = self.ctrl.compute(P.CTRL_TIMESTEP, pos, quat, vel, tgt)  # :200-206
        elif self.act == "vel":
            # np.linalg.norm of a 1-D float32 slice (sqrt(dot(x,x)) in the action dtype): call it row by
            # row like the reference so float32 rounding is identical
            nv = np.array([[np.linalg.norm(r)] for r in a[:, 0:3]], dtype=a.dtype)
            unit = np.where(nv != 0, a[:, 0:3] / np.where(nv != 0, nv, 1), 0).astype(a.dtype)   # :210-213
            trpy = np.zeros((n, 3), self.dtype); trpy[:, 2] = self.rpy.reshape(n, 3)[:, 2]       # :219
            tvel = (a.dtype.type(self.SPEED_LIMIT) * np.abs(a[:, 3:4])) * unit                   # :220
            rpm, _, _ = self.ctrl.compute(P.CTRL_TIMESTEP, pos, quat, vel, pos, target_rpy=trpy,
                                          target_vel=tvel.astype(self.dtype))                    # :214-221
        elif self.act == "one_d_pid":
            tgt = pos + 0.1 * np.concatenate([np.zeros((n, 2), self.dtype), a[:, 0:1].astype(self.dtype)], axis=1)   # :233
            rpm, _, _ = self.ctrl.compute(P.CTRL_TIMESTEP, pos, quat, vel, tgt)
        else:
            raise ValueError(self.act)
        return rpm.reshape(self.E, self.D, 4)

    def _obs(self):
        if self.kind in ("ctrl", "velocity"):                                    # CtrlAviary.py:106-117, VelocityAviary.py:111-125
            return self.state_vector()
        kin = np.concatenate([self.pos, self.rpy, self.vel, self.ang_v], axis=-1).astype(np.float32)   # BaseRLAviary.py:310-315
        return np.concatenate([kin] + [b.astype(np.float32) for b in self.action_buffer], axis=-1)    # :317-318

    def state_vector(self):
        """BaseAviary._getDroneStateVector (:541-561): [pos3 quat4 rpy3 vel3 ang_v3 last_clipped_action4]."""
        return np.concatenate([self.pos, self.quat, self.rpy, self.vel, self.ang_v, self.last_clipped_action], axis=-1)

    def step(self, action):
        P = self.P
        rpm = self._preprocess(action).astype(self.dtype)                        # :341
        for _ in range(P.S):                                                     # :343
            if P.S > 1:
                self.rpy = quat_to_euler(self.quat)                              # :346-347 cache refresh
            dw = None
            if self.effects & EFFECT_DW:
                dw = downwash_body_z(P, self.pos)
            self.pos, self.quat, self.vel, self.rpy_rates, self.ang_v = dynamics_substep(
                P, rpm, self.pos, self.quat, self.vel, self.rpy_rates, self.effects,
                rpm_prev=self.last_clipped_action, dw_fz=dw, rpy=self.rpy)       # :349-353
            self.last_clipped_action = rpm                                       # :372
        self.rpy = quat_to_euler(self.quat)                                      # :374
        obs = self._obs()                                                        # :376
        if self.kind in ("ctrl", "velocity"):
            reward = -np.ones(self.E); term = np.zeros(self.E, bool); trunc = np.zeros(self.E, bool)
        else:
            e = np.linalg.norm(self.TARGET_POS - self.pos, axis=-1)              # [E, D]
            reward = np.sum(np.maximum(0, 2 - e ** 4), axis=1)                   # HoverAviary.py:77-78, MultiHover :84-88
            term = np.sum(e, axis=1) < .0001                                     # HoverAviary.py:91, MultiHover :104-106
            oob = ((np.abs(self.pos[..., 0]) > self.xy_bound) | (np.abs(self.pos[..., 1]) > self.xy_bound)
                   | (self.pos[..., 2] > 2.0) | (np.abs(self.rpy[..., 0]) > .4) | (np.abs(self.rpy[..., 1]) > .4))
            trunc = np.any(oob, axis=1) | (self.step_counter / P.PYB_FREQ > self.EPISODE_LEN_SEC)   # HoverAviary.py:109-115
        self.step_counter = self.step_counter + P.S                              # :382
        return obs, reward, term, trunc
