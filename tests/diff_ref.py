"""Float64 torch restatement of oracle.dyn_oracle.dynamics_substep for batches, made to follow the derivative decisions of
BaseAviary.differentiable_rollout (DESIGN.md 4.5).  Its autograd is the reference gradient of the differentiable-trajectory
kernels (test infrastructure, CPU or CUDA tensors).

Where it departs from the NumPy oracle, it does so as the kernels do, so that both define the same function and derivative:
  * the quaternion is renormalised on tick entry (and Bullet's s = 2/|q|^2 is then 2);
  * _integrateQ is the exponential map everywhere (no np.isclose(|w|, 0) identity), with cos(theta) and sin(theta)/|w| as series
    in theta^2 below theta^2 = 1/4, so nothing takes sqrt(|w|^2) at w = 0;
  * the RPM clip is torch.clamp(rpm, 0, MAX_RPM) with a tensor MAX_RPM, the ground-effect height clip is `hz < clip ? clip : hz`,
    and the upright switch is the kernels' trig-free predicate (quad_core.cuh, upright), with no derivative.

A drone is 13 numbers: pos (3), quat (x, y, z, w), vel (3), rpy_rates (3).  `rows` are QsState.phys rows ([B, 16], per drone),
e.g. params.physical_rows of per-aviary properties indexed by each drone's aviary; `P` is the env's QsParams (ctypes), from which
only the model-wide constants are read (time step, mixing signs, propeller offsets, ground-effect and drag coefficients)."""
import math

import torch

EFFECT_GND, EFFECT_DRAG = 1, 2
_UPRIGHT_T = 1.722546424198833e-16


def model_constants(P, device=None):
    """The model-wide constants of QsParams `P` as float64 tensors on `device`."""
    t = lambda v: torch.tensor(v, dtype=torch.float64, device=device)
    return dict(dt=float(P.dt), sx=t(list(P.sx)), sy=t(list(P.sy)), sz=t(list(P.sz)),
                props=t([[P.prop_xyz[i][a] for a in range(3)] for i in range(4)]), gnd_coeff=float(P.gnd_eff_coeff),
                prop_radius=float(P.prop_radius), h_clip=float(P.gnd_eff_h_clip), drag=t(list(P.drag_coeff)))


def half_angle(n2, dt, exact_branch=False):
    """cos(theta) and sin(theta)/|w| for theta = |w| dt / 2, from n2 = |w|^2.  exact_branch=True: the reference's
    np.isclose(|w|, 0) identity (c = 1, s = 0 where |w| <= 1e-8), whose derivative is zero there -- a negative control only."""
    h = 0.5 * dt
    t = n2 * h * h                                   # half_angle_terms' order: both take the same side of t = 1/4
    small = t < 0.25
    ts = torch.where(small, t, torch.zeros_like(t))
    c_ser = torch.zeros_like(t)
    s_ser = torch.zeros_like(t)
    for k in range(9, -1, -1):
        c_ser = c_ser * ts + (-1) ** k / math.factorial(2 * k)
        s_ser = s_ser * ts + (-1) ** k / math.factorial(2 * k + 1)
    nl = torch.sqrt(torch.where(small, torch.ones_like(n2), n2))
    c = torch.where(small, c_ser, torch.cos(nl * h))
    s = torch.where(small, s_ser * h, torch.sin(nl * h) / nl)
    if exact_branch:
        still = n2 <= 1e-16
        c = torch.where(still, torch.ones_like(c), c)
        s = torch.where(still, torch.zeros_like(s), s)
    return c, s


def upright(sarg, ra, rb):
    """quad_core.cuh upright(): |roll| < pi/2 and |pitch| < pi/2 of the reference's float64 rpy, without trig."""
    return (sarg > -0.99999) & (sarg < 0.99999) & ((rb > _UPRIGHT_T * ra.abs()) | ((rb == 0) & (ra == 0)))


def substep(K, rows, x, u, ds, effects, exact_branch=False, gnd_clip_le=False):
    """One _dynamics substep (BaseAviary.py:815-877) from x [B, 13] with clipped rpm u [B, 4] and drag sum ds [B].
    gnd_clip_le=True: the height clip as `hz <= clip`, which clips at equality -- a negative control only."""
    dt = K["dt"]
    p, q, v, w = x[:, 0:3], x[:, 3:7], x[:, 7:10], x[:, 10:13]
    X, Y, Z, W = q.unbind(1)
    inv_m, gravity, kf, km, kx, ky = (rows[:, j] for j in range(6))
    J, J_inv = rows[:, 6:9], rows[:, 9:12]
    r02, r12, r22 = 2 * (X * Z + W * Y), 2 * (Y * Z - W * X), 1 - 2 * (X * X + Y * Y)
    f = u * u * kf[:, None]
    if effects & EFFECT_GND:                                                    # :715-750
        r20, r21 = 2 * (X * Z - W * Y), 2 * (Y * Z + W * X)
        up = upright(-2.0 * (X * Z - W * Y), 2.0 * (Y * Z + W * X), W * W - X * X - Y * Y + Z * Z).detach()
        Pp = K["props"]
        hz = p[:, 2:3] + r20[:, None] * Pp[:, 0] + r21[:, None] * Pp[:, 1] + r22[:, None] * Pp[:, 2]
        h = torch.where(hz <= K["h_clip"] if gnd_clip_le else hz < K["h_clip"], torch.full_like(hz, K["h_clip"]), hz)
        rr = K["prop_radius"] / (4 * h)
        g = u * u * kf[:, None] * K["gnd_coeff"] * (rr * rr)
        f = f + torch.where(up[:, None], g, torch.zeros_like(g))
    thrust = f.sum(1)
    tx = (f * K["sx"]).sum(1) * kx
    ty = (f * K["sy"]).sum(1) * ky
    tz = (u * u * km[:, None] * K["sz"]).sum(1)
    F = torch.stack([r02 * thrust, r12 * thrust, r22 * thrust - gravity], dim=1)
    if effects & EFFECT_DRAG:
        F = F - K["drag"] * ds[:, None] * v
    vn = v + (dt * inv_m)[:, None] * F
    tt = torch.stack([tx, ty, tz], dim=1) - torch.cross(w, J * w, dim=1)
    wn = w + dt * J_inv * tt
    pn = p + dt * vn
    a, b, c3 = wn.unbind(1)
    C, S = half_angle((wn * wn).sum(1), dt, exact_branch)
    om = torch.stack([c3 * Y - b * Z + a * W, -c3 * X + a * Z + b * W, b * X - a * Y + c3 * W, -a * X - b * Y - c3 * Z], dim=1)
    qn = C[:, None] * q + S[:, None] * om
    return torch.cat([pn, qn, vn, wn], dim=1)


def tick(K, rows, x, rpm, up, S, effects, renormalise=True, strict_clamp=False, **sub):
    """One control tick: clip(rpm, 0, MAX_RPM) for S substeps from x [B, 13]; up = the previous tick's clipped rpm (drag).
    strict_clamp=True: a clip whose gradient reaches rpm only strictly below MAX_RPM (at equality it goes to MAX_RPM) -- a
    negative control only.  `sub`: substep's exact_branch and gnd_clip_le."""
    mx = rows[:, 13:14].expand_as(rpm)
    u = torch.clamp(rpm, min=torch.zeros_like(rpm), max=mx)
    if strict_clamp:
        u = torch.where(rpm < mx, u, mx)
    if renormalise:
        q = x[:, 3:7]
        x = torch.cat([x[:, 0:3], q / torch.sqrt((q * q).sum(1, keepdim=True)), x[:, 7:13]], dim=1)
    k = 2 * math.pi
    ds_prev, ds_cur = (k * up / 60).sum(1), (k * u / 60).sum(1)
    for s in range(S):
        x = substep(K, rows, x, u, ds_prev if s == 0 else ds_cur, effects, **sub)
    return x, u


def rollout(K, rows, x0, rpm, last_rpm, S, effects, **kw):
    """T ticks from x0 [B, 13] with rpm [T, B, 4]: the states after every tick, [T, B, 13]."""
    out, x, up = [], x0, last_rpm
    for k in range(rpm.shape[0]):
        x, up = tick(K, rows, x, rpm[k], up, S, effects, **kw)
        out.append(x)
    return torch.stack(out)


def relerr(got, want):
    """Normwise relative error ||got - want|| / ||want|| (0 when both are 0)."""
    got, want = torch.as_tensor(got, dtype=torch.float64), torch.as_tensor(want, dtype=torch.float64)
    n = float(torch.linalg.vector_norm(want))
    d = float(torch.linalg.vector_norm(got - want))
    return d / n if n > 0 else d
