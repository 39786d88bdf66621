"""Drone model constants and the derived constants of the reference's BaseAviary.

The reference parses these from URDF `<properties>` at construction
(gym_pybullet_drones/envs/BaseAviary.py:985-1017, assets/cf2x.urdf:5,11-12,34,42-78,
assets/cf2p.urdf, assets/racer.urdf) and derives the rest in
BaseAviary.__init__ (envs/BaseAviary.py:116-128).  Here the three models are a
table; `AviaryConstants` reproduces the derivations in float64 in the same
operation order, and `fill_params` packs everything the kernels need into the
C-ABI `QsParams` (include/quadsim.h).
"""
import math
from dataclasses import dataclass

import numpy as np

from . import _native as N
from .utils.enums import DroneModel

# arm, kf, km, thrust2weight, max_speed_kmh, gnd_eff_coeff, prop_radius, drag_xy, drag_z, dw1, dw2, dw3,
# mass, ixx, iyy, izz, collision cylinder (h, r, z offset), propeller link COM offsets
DRONE_PROPERTIES = {
    DroneModel.CF2X: dict(arm=0.0397, kf=3.16e-10, km=7.94e-12, thrust2weight=2.25, max_speed_kmh=30.0,
                          gnd_eff_coeff=11.36859, prop_radius=2.31348e-2, drag_coeff_xy=9.1785e-7, drag_coeff_z=10.311e-7,
                          dw_coeff_1=2267.18, dw_coeff_2=0.16, dw_coeff_3=-0.11,
                          m=0.027, ixx=1.4e-5, iyy=1.4e-5, izz=2.17e-5, length=0.025, radius=0.06, collision_z_offset=0.0,
                          props=((0.028, -0.028, 0.0), (-0.028, -0.028, 0.0), (-0.028, 0.028, 0.0), (0.028, 0.028, 0.0))),
    DroneModel.CF2P: dict(arm=0.0397, kf=3.16e-10, km=7.94e-12, thrust2weight=2.25, max_speed_kmh=30.0,
                          gnd_eff_coeff=11.36859, prop_radius=2.31348e-2, drag_coeff_xy=9.1785e-7, drag_coeff_z=10.311e-7,
                          dw_coeff_1=2267.18, dw_coeff_2=0.16, dw_coeff_3=-0.11,
                          m=0.027, ixx=2.3951e-5, iyy=2.3951e-5, izz=3.2347e-5, length=0.025, radius=0.06, collision_z_offset=0.0,
                          props=((0.0397, 0.0, 0.0), (0.0, 0.0397, 0.0), (-0.0397, 0.0, 0.0), (0.0, -0.0397, 0.0))),
    DroneModel.RACE: dict(arm=0.109, kf=8.47e-9, km=2.13e-11, thrust2weight=4.17, max_speed_kmh=200.0,
                          gnd_eff_coeff=11.36859, prop_radius=12.7e-2, drag_coeff_xy=9.1785e-7, drag_coeff_z=10.311e-7,
                          dw_coeff_1=2267.18, dw_coeff_2=0.16, dw_coeff_3=-0.11,
                          m=0.830, ixx=0.003113, iyy=0.003113, izz=0.003113, length=0.025, radius=0.06, collision_z_offset=0.0,
                          props=((0.0850, 0.0675, 0.0), (-0.0850, 0.0675, 0.0), (-0.085, -0.0675, 0.0), (0.085, -0.0675, 0.0))),
}

# _dynamics torque mixing (envs/BaseAviary.py:842-854): tau_x = kx * sum_i sx_i f_i, tau_y = ky * sum_i sy_i f_i,
# tau_z = sum_i sz_i KM rpm_i^2 (all z torques negated for RACE, :843-844)
_MIXING = {
    DroneModel.CF2X: dict(sx=(1, 1, -1, -1), sy=(-1, 1, 1, -1), sz=(-1, 1, -1, 1), kx_sign=-1.0, diag=True),
    DroneModel.RACE: dict(sx=(1, 1, -1, -1), sy=(-1, 1, 1, -1), sz=(1, -1, 1, -1), kx_sign=1.0, diag=True),
    DroneModel.CF2P: dict(sx=(0, 1, 0, -1), sy=(-1, 0, 1, 0), sz=(-1, 1, -1, 1), kx_sign=1.0, diag=False),
}

# DSLPIDControl mixer matrices (control/DSLPIDControl.py:48-61)
_PID_MIXER = {
    DroneModel.CF2X: ((-.5, -.5, -1), (-.5, .5, 1), (.5, .5, -1), (.5, -.5, 1)),
    DroneModel.CF2P: ((0, -1, -1), (1, 0, 1), (0, 1, -1), (-1, 0, 1)),
}


@dataclass
class PIDCoefficients:
    """DSLPIDControl gains (control/DSLPIDControl.py:37-42)."""
    P_COEFF_FOR: np.ndarray
    I_COEFF_FOR: np.ndarray
    D_COEFF_FOR: np.ndarray
    P_COEFF_TOR: np.ndarray
    I_COEFF_TOR: np.ndarray
    D_COEFF_TOR: np.ndarray

    @staticmethod
    def default():
        return PIDCoefficients(np.array([.4, .4, 1.25]), np.array([.05, .05, .05]), np.array([.2, .2, .5]),
                               np.array([70000., 70000., 60000.]), np.array([.0, .0, 500.]), np.array([20000., 20000., 12000.]))


class AviaryConstants:
    """The attribute names and values of BaseAviary.__init__ (envs/BaseAviary.py:74-128)."""

    def __init__(self, drone_model=DroneModel.CF2X, pyb_freq=240, ctrl_freq=240, g=9.8):
        u = DRONE_PROPERTIES[drone_model]
        self.DRONE_MODEL = drone_model
        self.G = g
        self.RAD2DEG = 180 / np.pi
        self.DEG2RAD = np.pi / 180
        self.CTRL_FREQ = ctrl_freq
        self.PYB_FREQ = pyb_freq
        if self.PYB_FREQ % self.CTRL_FREQ != 0:
            raise ValueError('[ERROR] in BaseAviary.__init__(), pyb_freq is not divisible by env_freq.')   # BaseAviary.py:79-80
        self.PYB_STEPS_PER_CTRL = int(self.PYB_FREQ / self.CTRL_FREQ)
        self.CTRL_TIMESTEP = 1. / self.CTRL_FREQ
        self.PYB_TIMESTEP = 1. / self.PYB_FREQ
        self.URDF = drone_model.value + ".urdf"
        self.M, self.L, self.THRUST2WEIGHT_RATIO = u["m"], u["arm"], u["thrust2weight"]
        self.J = np.diag([u["ixx"], u["iyy"], u["izz"]])
        self.J_INV = np.linalg.inv(self.J)
        self.KF, self.KM = u["kf"], u["km"]
        self.COLLISION_H, self.COLLISION_R, self.COLLISION_Z_OFFSET = u["length"], u["radius"], u["collision_z_offset"]
        self.MAX_SPEED_KMH = u["max_speed_kmh"]
        self.GND_EFF_COEFF, self.PROP_RADIUS = u["gnd_eff_coeff"], u["prop_radius"]
        self.DRAG_COEFF = np.array([u["drag_coeff_xy"], u["drag_coeff_xy"], u["drag_coeff_z"]])
        self.DW_COEFF_1, self.DW_COEFF_2, self.DW_COEFF_3 = u["dw_coeff_1"], u["dw_coeff_2"], u["dw_coeff_3"]
        self.PROP_OFFSETS = np.array(u["props"])
        self.GRAVITY = self.G * self.M                                                      # :117
        self.HOVER_RPM = np.sqrt(self.GRAVITY / (4 * self.KF))                              # :118
        self.MAX_RPM = np.sqrt((self.THRUST2WEIGHT_RATIO * self.GRAVITY) / (4 * self.KF))   # :119
        self.MAX_THRUST = (4 * self.KF * self.MAX_RPM ** 2)                                 # :120
        if drone_model == DroneModel.CF2P:
            self.MAX_XY_TORQUE = (self.L * self.KF * self.MAX_RPM ** 2)                     # :123-124
        else:
            self.MAX_XY_TORQUE = (2 * self.L * self.KF * self.MAX_RPM ** 2) / np.sqrt(2)    # :121-126
        self.MAX_Z_TORQUE = (2 * self.KM * self.MAX_RPM ** 2)                               # :127
        self.GND_EFF_H_CLIP = 0.25 * self.PROP_RADIUS * np.sqrt(
            (15 * self.MAX_RPM ** 2 * self.KF * self.GND_EFF_COEFF) / self.MAX_THRUST)      # :128

    def default_init_xyzs(self, num_drones):
        """envs/BaseAviary.py:194-197."""
        return np.vstack([np.array([x * 4 * self.L for x in range(num_drones)]),
                          np.array([y * 4 * self.L for y in range(num_drones)]),
                          np.ones(num_drones) * (self.COLLISION_H / 2 - self.COLLISION_Z_OFFSET + .1)]).transpose().reshape(num_drones, 3)


# ---- per-aviary physical constants (QsState.phys, include/quadsim.h) ------------------------------------------------------
# The properties a user may vary per aviary (names of DRONE_PROPERTIES) and the columns of one table row derived from them.
PHYS_KEYS = ("m", "ixx", "iyy", "izz", "kf", "km", "arm", "thrust2weight")
PHYS_COLUMNS = ("inv_m", "gravity", "kf", "km", "kx", "ky", "jx", "jy", "jz", "jx_inv", "jy_inv", "jz_inv", "hover_rpm", "max_rpm")


def _sqrt(t):
    # correctly rounded like np.sqrt: CUDA's float64 sqrt is; torch's vectorised CPU sqrt is not (1 ulp apart now and then)
    if t.device.type == "cpu":
        import torch
        r = torch.from_numpy(np.sqrt(t.detach().numpy()))
        if t.requires_grad:                  # np.sqrt's value with sqrt's derivative (s - s.detach() is exactly 0)
            s = t.sqrt()
            r = r + (s - s.detach())
        return r
    return t.sqrt()


def physical_rows(drone_model, props, g=9.8):
    """[E, 16] float64 rows of QsState.phys from the properties `props` (dict PHYS_KEYS -> [E] float64 torch tensors, any device),
    derived in float64 with BaseAviary.__init__'s formulas and operation order (envs/BaseAviary.py:117-119, :1000 J^-1, the
    _dynamics arm L/sqrt(2) of :846-851).  fill_params packs its QsParams fields from the same function, so a row of nominal
    properties has exactly their bits."""
    import torch
    m, kf, km, arm, t2w = props["m"], props["kf"], props["km"], props["arm"], props["thrust2weight"]
    j = torch.stack([props["ixx"], props["iyy"], props["izz"]], dim=1)
    gravity = g * m                                                                         # :117
    mix = _MIXING[drone_model]
    a = arm / math.sqrt(2) if mix["diag"] else arm                                          # np.sqrt(2) == math.sqrt(2)
    out = torch.zeros((m.shape[0], N.PHYS_WIDTH), dtype=torch.float64, device=m.device)
    out[:, 0] = 1.0 / m
    out[:, 1] = gravity
    out[:, 2], out[:, 3] = kf, km
    out[:, 4], out[:, 5] = mix["kx_sign"] * a, a
    out[:, 6:9] = j
    out[:, 9:12] = 1.0 / j                                                                  # np.linalg.inv of the diagonal J
    out[:, 12] = _sqrt(gravity / (4 * kf))                                                  # :118
    out[:, 13] = _sqrt((t2w * gravity) / (4 * kf))                                          # :119
    return out


def nominal_properties(drone_model):
    """The model's PHYS_KEYS values (DRONE_PROPERTIES)."""
    u = DRONE_PROPERTIES[drone_model]
    return {k: float(u[k]) for k in PHYS_KEYS}


def coerce_physical_args(n_envs, device, values, single=False):
    """Validates the arguments of BaseAviary.set_physical_params: `values` maps PHYS_KEYS to a scalar, an [E] NumPy array or an
    [E] torch tensor (None = keep).  Returns {key: [E] float64 tensor on `device`}.  Wrong keys, types or shapes raise
    ValueError, and so do non-finite or non-positive scalars and NumPy values (checked on the host).  Tensors are not read
    back (no synchronisation): set_physical_params screens them on the device.  single = the single-env API: scalars only."""
    import torch
    out = {}
    for k, v in values.items():
        if k not in PHYS_KEYS:
            raise ValueError("unknown physical parameter %r (expected one of %s)" % (k, ", ".join(PHYS_KEYS)))
        if v is None:
            continue
        if isinstance(v, torch.Tensor):
            if single and v.numel() != 1:
                raise ValueError("%s: the single-env API takes scalars" % k)
            if v.dim() > 1 or (v.dim() == 1 and v.shape[0] != n_envs) or not (v.dtype.is_floating_point or v.dtype in (torch.int32, torch.int64)):
                raise ValueError("%s must be a scalar or a [%d] float tensor, got %s %s" % (k, n_envs, v.dtype, tuple(v.shape)))
            out[k] = v.to(device=device, dtype=torch.float64).reshape(-1).expand(n_envs)
            continue
        a = np.asarray(v)
        if a.dtype.kind not in "fiu" or (a.ndim == 1 and single) or a.ndim > 1 or (a.ndim == 1 and a.shape[0] != n_envs):
            raise ValueError("%s must be a scalar or a [%d] array of floats, got %s %s" % (k, n_envs, a.dtype, a.shape))
        a = a.astype(np.float64)
        if not np.all(np.isfinite(a)) or not np.all(a > 0):
            raise ValueError("%s must be finite and positive" % k)
        out[k] = torch.as_tensor(np.broadcast_to(a, (n_envs,)).copy(), device=device)
    return out


def fill_params(c, *, episode_len_sec=8.0, xy_bound=1.5, z_bound=2.0, tilt_bound=0.4, term_dist=1e-4,
                pid_model=DroneModel.CF2X, pid_coeffs=None, pid_g=9.8):
    """Packs an AviaryConstants (+ task and controller constants) into the C-ABI QsParams."""
    import torch
    P = N.QsParams()
    P.dt, P.ctrl_dt, P.pyb_freq = c.PYB_TIMESTEP, c.CTRL_TIMESTEP, float(c.PYB_FREQ)
    props = dict(m=c.M, ixx=c.J[0, 0], iyy=c.J[1, 1], izz=c.J[2, 2], kf=c.KF, km=c.KM, arm=c.L, thrust2weight=c.THRUST2WEIGHT_RATIO)
    row = physical_rows(c.DRONE_MODEL, {k: torch.tensor([float(v)], dtype=torch.float64) for k, v in props.items()}, c.G)[0].tolist()
    P.m = c.M
    P.inv_m, P.gravity, P.kf, P.km, P.kx, P.ky = row[0:6]
    for k in range(3):
        P.j[k], P.j_inv[k] = row[6 + k], row[9 + k]
        P.drag_coeff[k] = c.DRAG_COEFF[k]
    P.hover_rpm, P.max_rpm = row[12], row[13]
    mix = _MIXING[c.DRONE_MODEL]
    for k in range(4):
        P.sx[k], P.sy[k], P.sz[k] = mix["sx"][k], mix["sy"][k], mix["sz"][k]
        for a in range(3):
            P.prop_xyz[k][a] = c.PROP_OFFSETS[k, a]
    P.gnd_eff_coeff, P.prop_radius, P.gnd_eff_h_clip = c.GND_EFF_COEFF, c.PROP_RADIUS, float(c.GND_EFF_H_CLIP)
    P.dw_coeff[0], P.dw_coeff[1], P.dw_coeff[2] = c.DW_COEFF_1, c.DW_COEFF_2, c.DW_COEFF_3
    P.episode_len_sec, P.xy_bound, P.z_bound, P.tilt_bound, P.term_dist = episode_len_sec, xy_bound, z_bound, tilt_bound, term_dist
    P.speed_limit = 0.03 * c.MAX_SPEED_KMH * (1000 / 3600)                                  # BaseRLAviary.py:95
    co = pid_coeffs or PIDCoefficients.default()
    for k in range(3):
        P.pid_p_for[k], P.pid_i_for[k], P.pid_d_for[k] = co.P_COEFF_FOR[k], co.I_COEFF_FOR[k], co.D_COEFF_FOR[k]
        P.pid_p_tor[k], P.pid_i_tor[k], P.pid_d_tor[k] = co.P_COEFF_TOR[k], co.I_COEFF_TOR[k], co.D_COEFF_TOR[k]
    if pid_model in _PID_MIXER:
        for r in range(4):
            for k in range(3):
                P.pid_mixer[r][k] = _PID_MIXER[pid_model][r][k]
        pu = DRONE_PROPERTIES[pid_model]
        P.pid_gravity, P.pid_kf = pid_g * pu["m"], pu["kf"]                                 # BaseControl.py:35-38
    P.pid_pwm2rpm_scale, P.pid_pwm2rpm_const, P.pid_min_pwm, P.pid_max_pwm = 0.2685, 4070.3, 20000.0, 65535.0   # DSLPIDControl.py:43-46
    P.drone_model = {DroneModel.CF2X: N.MODEL_CF2X, DroneModel.CF2P: N.MODEL_CF2P, DroneModel.RACE: N.MODEL_RACE}[c.DRONE_MODEL]
    return P


def quaternion_from_euler(rpy):
    """pybullet.getQuaternionFromEuler (call site envs/BaseAviary.py:488), float64, [..., 3] -> [..., 4] (x,y,z,w)."""
    h = np.asarray(rpy, dtype=np.float64) * 0.5
    cr, sr = np.cos(h[..., 0]), np.sin(h[..., 0])
    cp, sp = np.cos(h[..., 1]), np.sin(h[..., 1])
    cy, sy = np.cos(h[..., 2]), np.sin(h[..., 2])
    q = np.stack([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy,
                  cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy], axis=-1)
    return q / np.linalg.norm(q, axis=-1, keepdims=True)


def euler_from_quaternion(quat):
    """pybullet.getEulerFromQuaternion (call site envs/BaseAviary.py:518) on a float64 tensor [..., 4] (x,y,z,w) -> [..., 3],
    with Bullet's gimbal guard: where sarg = -2(xz - wy) reaches +-0.99999, roll = 0, pitch = +-pi/2 and yaw = 2 atan2(-+x, +-y)."""
    import torch
    x, y, z, w = quat.unbind(-1)
    sarg = -2.0 * (x * z - w * y)
    lo, hi = sarg <= -0.99999, sarg >= 0.99999
    roll = torch.where(lo | hi, 0.0, torch.atan2(2.0 * (y * z + w * x), w * w - x * x - y * y + z * z))
    pitch = torch.where(lo, -0.5 * math.pi, torch.where(hi, 0.5 * math.pi, torch.asin(sarg.clamp(-1, 1))))
    yaw = torch.where(lo, 2.0 * torch.atan2(x, -y),
                      torch.where(hi, 2.0 * torch.atan2(-x, y), torch.atan2(2.0 * (x * y + w * z), w * w + x * x - y * y - z * z)))
    return torch.stack([roll, pitch, yaw], dim=-1)
