"""Float64 torch restatement of DSLPIDControl.computeControl (oracle.dyn_oracle.OraclePID, control/DSLPIDControl.py:82-259) for
batches, made to follow the derivative decisions of the closed-loop differentiable_rollout (DESIGN.md 4.5), and its composition
with diff_ref.tick into a closed-loop rollout.  Its autograd is the reference gradient of the closed-loop kernels (test
infrastructure, CPU or CUDA tensors).

The decisions: every clip is torch.clamp (the gradient passes for lo <= x <= hi); `max(scalar, 0)` then sqrt has a zero gradient
where scalar <= 0 (torch.where, no nan at 0); the Euler angles are differentiated on the branch of the gimbal guard the forward
takes; the rate term (rpy - last_rpy) / dt has no angle unwrap.  `flip` names decisions to turn the other way -- negative
controls only: "integral" and "torque" and "pwm" pass the gradient straight through their clips, "scalar" passes it through
max(scalar, 0) (with sqrt's derivative at 1e-6 where scalar <= 0), "gimbal" differentiates the atan2 / asin branch everywhere.

A controller state is 9 numbers: integral_pos_e, last_rpy, integral_rpy_e.  Gains are [B, 18]: P_FOR, I_FOR, D_FOR, P_TOR,
I_TOR, D_TOR."""
import math

import torch

import diff_ref as R


def controller_constants(CP, device=None):
    """The constants a DSLPIDControl reads from its QsParams `CP` (ctypes), as floats and float64 tensors."""
    t = lambda v: torch.tensor(v, dtype=torch.float64, device=device)
    return dict(gravity=float(CP.pid_gravity), kf=float(CP.pid_kf), scale=float(CP.pid_pwm2rpm_scale),
                const=float(CP.pid_pwm2rpm_const), min_pwm=float(CP.pid_min_pwm), max_pwm=float(CP.pid_max_pwm),
                mixer=t([[CP.pid_mixer[j][a] for a in range(3)] for j in range(4)]), max_rpm=float(CP.max_rpm))


def gains_of(CP, device=None):
    """[18] float64: the gains of QsParams `CP` in QsDynCtrlTrajIO.gains' order."""
    return torch.tensor([float(getattr(CP, f)[a]) for f in ("pid_p_for", "pid_i_for", "pid_d_for", "pid_p_tor", "pid_i_tor", "pid_d_tor")
                         for a in range(3)], dtype=torch.float64, device=device)


def _clip(x, lo, hi, straight):
    y = torch.clamp(x, lo, hi)
    return x + (y - x).detach() if straight else y


def quat_to_matrix(q):
    """Bullet's getMatrixFromQuaternion with s = 2 / |q|^2: [B, 3, 3]."""
    x, y, z, w = q.unbind(1)
    s = 2.0 / (x * x + y * y + z * z + w * w)
    return torch.stack([1 - s * (y * y + z * z), s * (x * y - w * z), s * (x * z + w * y),
                        s * (x * y + w * z), 1 - s * (x * x + z * z), s * (y * z - w * x),
                        s * (x * z - w * y), s * (y * z + w * x), 1 - s * (x * x + y * y)], dim=1).reshape(-1, 3, 3)


def quat_to_euler(q, branch_free=False):
    """getEulerFromQuaternion (no normalisation) with the +-0.99999 gimbal guard, differentiated on the taken branch."""
    x, y, z, w = q.unbind(1)
    sarg = -2.0 * (x * z - w * y)
    lo, hi = sarg <= -0.99999, sarg >= 0.99999
    guard = (lo | hi) & (not branch_free)
    roll = torch.atan2(2.0 * (y * z + w * x), w * w - x * x - y * y + z * z)
    pitch = torch.asin(torch.where(guard, torch.zeros_like(sarg), sarg))
    yaw = torch.atan2(2.0 * (x * y + w * z), w * w + x * x - y * y - z * z)
    yaw_g = torch.where(lo, 2.0 * torch.atan2(x, -y), 2.0 * torch.atan2(-x, y))
    half = math.pi / 2
    roll = torch.where(guard, torch.zeros_like(roll), roll)
    pitch = torch.where(guard, torch.where(lo, torch.full_like(pitch, -half), torch.full_like(pitch, half)), pitch)
    yaw = torch.where(guard, yaw_g, yaw)
    return torch.stack([roll, pitch, yaw], dim=1)


def pid(Cc, gains, st, dt, x, tp, tyaw, tv, trr, flip=(), probe=None):
    """One computeControl for B drones: x [B, 13] (pos, quat, vel, rates), st [B, 9], targets tp / tv / trr [B, 3] and tyaw [B],
    gains [B, 18] -> (raw rpm [B, 4], the updated state [B, 9], pos_e [B, 3], yaw_e [B]).  probe: a dict that receives the inputs
    of the decisions (scalar [B], sarg [B], the torques and PWMs before their clips [B, 3] / [B, 4]), for tests that show a
    decision is taken."""
    pos, q, vel = x[:, 0:3], x[:, 3:7], x[:, 7:10]
    Kp, Ki, Kd, Tp, Ti, Td = (gains[:, 3 * j:3 * j + 3] for j in range(6))
    Rm = quat_to_matrix(q)
    e, ev = tp - pos, tv - vel
    si = "integral" in flip
    ip0 = st[:, 0:3] + e * dt
    ip = torch.cat([_clip(ip0[:, 0:2], -2.0, 2.0, si), _clip(_clip(ip0[:, 2:3], -2.0, 2.0, si), -0.15, 0.15, si)], dim=1)
    tt = Kp * e + Ki * ip + Kd * ev
    tt = tt + torch.tensor([0.0, 0.0, Cc["gravity"]], dtype=tt.dtype, device=tt.device)
    scalar = (tt * Rm[:, :, 2]).sum(1)
    live = scalar > 0
    if "scalar" in flip:                     # value max(scalar, 1e-6), gradient straight through
        root = torch.sqrt((scalar + (scalar.clamp(min=1e-6) - scalar).detach()) / (4 * Cc["kf"]))
    else:
        root = torch.where(live, torch.sqrt(torch.where(live, scalar, torch.ones_like(scalar)) / (4 * Cc["kf"])), torch.zeros_like(scalar))
    thrust = (root - Cc["const"]) / Cc["scale"]
    z = tt / torch.linalg.vector_norm(tt, dim=1, keepdim=True)
    xc = torch.stack([torch.cos(tyaw), torch.sin(tyaw), torch.zeros_like(tyaw)], dim=1)
    yc = torch.cross(z, xc, dim=1)
    yax = yc / torch.linalg.vector_norm(yc, dim=1, keepdim=True)
    xax = torch.cross(yax, z, dim=1)
    Rd = torch.stack([xax, yax, z], dim=2)
    rpy = quat_to_euler(q, branch_free="gimbal" in flip)
    Em = Rd.transpose(1, 2) @ Rm - Rm.transpose(1, 2) @ Rd
    re = torch.stack([Em[:, 2, 1], Em[:, 0, 2], Em[:, 1, 0]], dim=1)
    rr = trr - (rpy - st[:, 3:6]) / dt
    ir0 = st[:, 6:9] - re * dt
    ir1 = _clip(ir0, -1500.0, 1500.0, si)
    ir = torch.cat([_clip(ir1[:, 0:2], -1.0, 1.0, si), ir1[:, 2:3]], dim=1)
    tq = _clip(-Tp * re + Td * rr + Ti * ir, -3200.0, 3200.0, "torque" in flip)
    pwm = _clip(thrust[:, None] + tq @ Cc["mixer"].T, Cc["min_pwm"], Cc["max_pwm"], "pwm" in flip)
    rpm = Cc["scale"] * pwm + Cc["const"]
    if probe is not None:
        probe.update(scalar=scalar, sarg=-2.0 * (q[:, 0] * q[:, 2] - q[:, 3] * q[:, 1]), torque=-Tp * re + Td * rr + Ti * ir,
                     pwm=thrust[:, None] + tq @ Cc["mixer"].T)
    ec = torch.atan2(-Rd[:, 0, 1], Rd[:, 0, 0])
    return rpm, torch.cat([ip, rpy, ir], dim=1), e, ec - rpy[:, 2]


def closed_loop(K, Cc, rows, gains, x0, pid0, tpos, tyaw, tv, trr, last_rpm, dt, S, effects, flip=()):
    """T ticks of the TRACK loop from x0 [B, 13] and pid0 [B, 9] with target_pos [T, B, 3]: the controller, its max_rpm clip, the
    env's clip and S substeps (diff_ref.tick).  Returns (states [T, B, 13], applied rpm [T, B, 4])."""
    xs, us, x, st, up = [], [], x0, pid0, last_rpm
    for k in range(tpos.shape[0]):
        raw, st, _, _ = pid(Cc, gains, st, dt, x, tpos[k], tyaw, tv, trr, flip)
        u1 = torch.clamp(raw, 0.0, Cc["max_rpm"])
        x, up = R.tick(K, rows, x, u1, up, S, effects)
        xs.append(x)
        us.append(up)
    return torch.stack(xs), torch.stack(us)
