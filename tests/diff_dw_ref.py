"""Float64 torch reference of differentiable_rollout(downwash=True) (DESIGN.md 4.5, downwash adjoint): mppi_ref.rollout_dw's
aviary tick -- every substep renormalises the quaternion, takes its pair force from the aviary's start positions and runs one
diff_ref substep -- with the pair term written so that autograd gives the kernels' derivative (test infrastructure, CPU or CUDA
tensors).

The pair term of a receiver i and a source q is p = -alpha exp(-dxy2 / (2 beta^2)) with dz = z_q - z_i, dxy2 = dx^2 + dy^2,
alpha = c0 (R / (4 dz))^2 and beta = c1 dz + c2.  The predicate (dz > 0 and sqrt(dxy2) < 10, the oracle's) is taken without
gradient, and every branch reads masked safe inputs, so no NaN reaches the gradient: the sqrt is never differentiated (stacked
drones have finite derivatives), and where beta = 0 the term is the constant 0 the forward gives there.

Negative controls only: source=False / receiver=False detach the source's / receiver's position in the pair term (dropping its
side of the adjoint), sqrt_form=True writes the exponent as (sqrt(dxy2) / beta)^2 (whose autograd is NaN at dxy2 = 0),
lt100=True tests dxy2 < 100 and renorm_per_tick=True renormalises on tick entry only."""
import math

import torch

import diff_ref as DR

EFFECT_GND, EFFECT_DRAG, EFFECT_DW = 1, 2, 4


def dw_fz(P, pos, source=True, receiver=True, sqrt_form=False, lt100=False):
    """fz [G, D]: each drone's downwash force along body z from the drones of its group, pos [G, D, 3], summed over the
    group in drone order from 0.0."""
    G, D, _ = pos.shape
    c0, c1, c2 = (float(c) for c in P.dw_coeff)
    r = float(P.prop_radius)
    fz = torch.zeros((G, D), dtype=pos.dtype, device=pos.device)
    rcv = pos if receiver else pos.detach()
    for q in range(D):
        src = pos[:, q:q + 1] if source else pos[:, q:q + 1].detach()
        dz = src[..., 2] - rcv[..., 2]
        dx, dy = src[..., 0] - rcv[..., 0], src[..., 1] - rcv[..., 1]
        dxy2 = dx * dx + dy * dy
        with torch.no_grad():
            act = (dz > 0) & (dxy2 < 100.0 if lt100 else torch.sqrt(dxy2) < 10.0)
        dzs = torch.where(act, dz, torch.ones_like(dz))
        beta = c1 * dzs + c2
        live = act & (beta != 0)                          # beta = 0 (dxy2 > 0): the forward's term is exp(-inf) = 0
        betas = torch.where(live, beta, torch.ones_like(beta))
        d2 = torch.where(live, dxy2, torch.zeros_like(dxy2))
        rr = r / (4.0 * dzs)
        if sqrt_form:
            u = torch.sqrt(d2) / betas
            e = torch.exp(-0.5 * (u * u))
        else:
            e = torch.exp(-d2 / (2.0 * betas * betas))
        fz = torch.where(live, fz + (-(c0 * (rr * rr)) * e), fz)
    return fz


def tick(K, P, rows, x, rpm, up, S, effects, D, renorm_per_tick=False, **pair):
    """One aviary tick from x [B, 13] (B / D groups of D consecutive drones) with the raw rpm [B, 4] clipped to [0, MAX_RPM]
    (torch.clamp); up = drag's previous clipped rpm.  Returns (x', u)."""
    mx = rows[:, 13:14].expand_as(rpm)
    u = torch.clamp(rpm, min=torch.zeros_like(rpm), max=mx)
    k2 = 2 * math.pi
    ds_prev, ds_cur = (k2 * up / 60).sum(1), (k2 * u / 60).sum(1)
    B = x.shape[0]
    for s in range(S):
        if s == 0 or not renorm_per_tick:
            q = x[:, 3:7]
            x = torch.cat([x[:, 0:3], q / torch.sqrt((q * q).sum(1, keepdim=True)), x[:, 7:13]], dim=1)
        fz = dw_fz(P, x[:, 0:3].reshape(B // D, D, 3), **pair).reshape(B)
        x = DR.substep(K, rows, x, u, ds_prev if s == 0 else ds_cur, effects, fz=fz)
    return x, u


def rollout(K, P, rows, x0, rpm, last_rpm, S, effects, D, **kw):
    """T aviary ticks from x0 [B, 13] with rpm [T, B, 4]: the states after every tick, [T, B, 13]."""
    out, x, up = [], x0, last_rpm
    for k in range(rpm.shape[0]):
        x, up = tick(K, P, rows, x, rpm[k], up, S, effects, D, **kw)
        out.append(x)
    return torch.stack(out)


# ---- pair geometry at the decisions of the downwash adjoint (exact in float64: x_i = y_i = 0, z_i = 0 or 1) -----------------

def _ulp_step(v, k):
    import numpy as np
    for _ in range(abs(k)):
        v = float(np.nextafter(v, math.inf if k > 0 else -math.inf))
    return v


def pair_offset_for(dxy2):
    """(dx, dy) with dx * dx + dy * dy == dxy2 exactly in float64 (the kernels' operation order, no fma), dx near sqrt(dxy2)."""
    r = math.sqrt(dxy2)
    for k in range(0, 16):
        dx = _ulp_step(r, -k)
        a = dx * dx
        if a == dxy2:
            return dx, 0.0
        if a < dxy2:
            y0 = math.sqrt(dxy2 - a)
            for j in range(-64, 65):
                dy = _ulp_step(y0, j)
                if a + dy * dy == dxy2:
                    return dx, dy
    raise AssertionError("no exact offset for dxy2 = %r" % dxy2)


def beta_zero_dz(P):
    """A dz with c1 dz + c2 == 0 exactly (z_i = 0, z_q = dz), or None when no double within 4096 ulps of -c2 / c1 gives it."""
    c1, c2 = float(P.dw_coeff[1]), float(P.dw_coeff[2])
    z0 = -c2 / c1
    for k in range(0, 4097):
        for dz in (_ulp_step(z0, k), _ulp_step(z0, -k)):
            if c1 * dz + c2 == 0.0:
                return dz
    return None


def closed_loop(K, P, Cc, rows, gains, x0, pid0, tpos, tyaw, tv, trr, last_rpm, dt, S, effects, D):
    """diff_pid_ref.closed_loop with the aviary tick above: T ticks of the TRACK loop from x0 [B, 13] and pid0 [B, 9].  Returns
    (states [T, B, 13], applied rpm [T, B, 4])."""
    import diff_pid_ref as PR
    xs, us, x, st, up = [], [], x0, pid0, last_rpm
    for k in range(tpos.shape[0]):
        raw, st, _, _ = PR.pid(Cc, gains, st, dt, x, tpos[k], tyaw, tv, trr)
        u1 = torch.clamp(raw, 0.0, Cc["max_rpm"])
        x, up = tick(K, P, rows, x, u1, up, S, effects, D)
        xs.append(x)
        us.append(up)
    return torch.stack(xs), torch.stack(us)
