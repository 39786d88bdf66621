"""Float64 restatement of mppi() (DESIGN.md 4.5.2) for the tests: Philox4x32-10 in Python integers, Box-Muller in NumPy, the
sample rollouts' cost through ilqr_ref / diff_ref, and the weights, candidate and commit rules of qs_mppi_update and
qs_mppi_commit."""
import math

import numpy as np
import torch

import diff_ref as DR
import ilqr_ref as IR

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF


def philox(ctr, key):
    """Philox4x32-10 of the 4-word counter and the 2-word key (Python ints) -> 4 words"""
    c0, c1, c2, c3 = ctr
    k0, k1 = key
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
        p0, p1 = M0 * c0, M1 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & MASK, p1 & MASK, ((p0 >> 32) ^ c3 ^ k1) & MASK, p0 & MASK
    return c0, c1, c2, c3


def uniform(hi, lo):
    """(x + 0.5) 2^-53 from the top 53 bits x of (hi << 32) | lo"""
    return (float(((hi << 32) | lo) >> 11) + 0.5) * 2.0 ** -53


def box_muller(w):
    ua, ub = uniform(w[0], w[1]), uniform(w[2], w[3])
    r = np.sqrt(-2.0 * np.log(ua))
    a = (2.0 * np.pi) * ub
    return r * np.cos(a), r * np.sin(a)


def eps(seed, k, s, i, it):
    """the four normals of drone i at tick k of sample s in iteration it (zeros for s = 0)"""
    if s == 0:
        return np.zeros(4)
    key = (seed & MASK, seed >> 32)
    out = []
    for h in range(2):
        out += box_muller(philox((k, s, i, 2 * it + h), key))
    return np.array(out)


def eps_vec(seed, k, s, i, it):
    """eps of Philox4x32-10 vectorised in NumPy: k, s, i, it integer arrays (broadcast, s >= 1 where not masked) -> [..., 4]; the
    same normals as eps() where s >= 1, zeros where s == 0"""
    u = lambda a: np.asarray(a, dtype=np.uint64)
    k, s, i, it = np.broadcast_arrays(u(k), u(s), u(i), u(it))
    m = np.uint64(MASK)
    out = []
    for h in range(2):
        c0, c1, c2, c3 = k & m, s & m, i & m, (np.uint64(2) * it + np.uint64(h)) & m
        k0, k1 = np.full_like(c0, seed & MASK), np.full_like(c0, seed >> 32)
        for r in range(10):
            if r:
                k0, k1 = (k0 + np.uint64(W0)) & m, (k1 + np.uint64(W1)) & m
            p0, p1 = np.uint64(M0) * c0, np.uint64(M1) * c2
            c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ k0) & m, p1 & m, ((p0 >> np.uint64(32)) ^ c3 ^ k1) & m, p0 & m
        ua = (((c0 << np.uint64(32)) | c1) >> np.uint64(11)).astype(np.float64) + 0.5
        ub = (((c2 << np.uint64(32)) | c3) >> np.uint64(11)).astype(np.float64) + 0.5
        r_ = np.sqrt(-2.0 * np.log(ua * 2.0 ** -53))
        a = (2.0 * np.pi) * (ub * 2.0 ** -53)
        out += [r_ * np.cos(a), r_ * np.sin(a)]
    e = np.stack(out, axis=-1)
    return np.where((s == 0)[..., None], 0.0, e)


def noise(seed, it, K, T, N):
    """eps [K, T, N, 4]"""
    return np.array([[[eps(seed, k, s, i, it) for i in range(N)] for k in range(T)] for s in range(K)])


def samples(u, sig, e, lo=None, hi=None):
    """(commands v, perturbations delta) [K, T, N, 4] of the nominal u [T, N, 4] with sig [N] and eps e [K, T, N, 4]: with a box
    v is clamped and delta = v - u where it binds, sig eps elsewhere"""
    v = u[None] + sig[None, None, :, None] * e
    if lo is None:
        return v, sig[None, None, :, None] * e
    c = np.minimum(np.maximum(v, lo), hi)                   # clampd: the bounds are ordered
    return c, np.where(c == v, sig[None, None, :, None] * e, c - u[None])


def weights(J, temperature, order="s"):
    """w [K] and the best sample of a unit's costs J [K] (the rule of qs_mppi_update): J_min, its lowest s and the sum of the
    finite J in one scan in s order, lambda = temperature (sum / count - J_min).  order="numpy": the mean by np.mean, whose
    pairwise partial sums round otherwise from K = 8 -- a negative control only."""
    J = np.asarray(J, dtype=np.float64)
    fin = np.isfinite(J)
    jmin, best, tot, count = math.inf, 0, 0.0, 0
    for s, j in enumerate(J.tolist()):
        if not math.isfinite(j):
            continue
        if j < jmin:
            jmin, best = j, s
        tot += j
        count += 1
    if count == 0:
        return np.zeros_like(J), 0
    mean = float(J[fin].mean()) if order == "numpy" else tot / count
    lam = temperature * (mean - jmin)
    w = [0.0 if not math.isfinite(j) else 1.0 if lam == 0 else math.exp(-(j - jmin) / lam) for j in J.tolist()]   # libm exp
    return np.array(w), best


def unit_sum(J, D, reverse=False):
    """[K, n] per-drone J -> [K, n / D] per-aviary J summed in drone order from 0.0 (the unit cost of qs_mppi_update and
    qs_mppi_commit with downwash).  reverse=True sums from the last drone -- a negative control only."""
    J = np.asarray(J, dtype=np.float64)
    out = np.zeros((J.shape[0], J.shape[1] // D))
    for q in (range(D - 1, -1, -1) if reverse else range(D)):
        out += J[:, q::D]
    return out


def candidate(u, delta, w):
    """u + sum_s w_s delta_s / sum_s w_s (u when no weight is positive); delta [K, ...]"""
    ws = w.sum()
    if not ws > 0:
        return u.copy()
    return u + np.tensordot(w, delta, axes=1) / ws


def pick(jc, J, tie="first", strict=False):
    """-1 keeps the candidate (jc <= the best sample's J), else the best sample (the lowest s of J_min).  Negative controls
    only: tie="last" takes the highest s of a tie, strict=True keeps the candidate only when jc < J[best]."""
    J = np.asarray(J, dtype=np.float64)
    _, best = weights(J, 1.0)
    if tie == "last" and np.isfinite(J).any():
        best = int(np.flatnonzero(J == J[best])[-1])
    return -1 if (jc < J[best] if strict else jc <= J[best]) else best


def rollout_cost(K_dyn, rows, x0, last_rpm, v, targets, W, Rt, uref, S, effects):
    """J [B] of the commands v [T, B, 4] (after the box) on diff_ref's tick, the cost of ilqr_ref (torch float64 tensors)"""
    return IR.rollout_cost(K_dyn, rows, x0, last_rpm, v, v, None, None, 0.0, targets, W, Rt, uref, S, effects)["J"]   # no gains: no dz


def dw_fz(P, pos, order=1, lt100=False):
    """fz [G, D]: each drone's downwash force along body z from the drones of its group, pos [G, D, 3] (torch float64), summed
    over the group in drone order from 0.0 (qs::downwash_pair of the kernels).  A pair acts when dz > 0 and
    sqrt(dx*dx + dy*dy) < 10, the oracle's predicate (oracle/dyn_oracle.py, downwash_body_z); alpha and beta as BaseAviary._downwash.
    Negative controls only: order=-1 sums from the last drone, lt100=True tests dx*dx + dy*dy < 100."""
    G, D, _ = pos.shape
    c0, c1, c2 = (float(c) for c in P.dw_coeff)
    r = float(P.prop_radius)
    fz = torch.zeros((G, D), dtype=pos.dtype, device=pos.device)
    for q in (range(D) if order > 0 else range(D - 1, -1, -1)):
        dz = pos[:, q:q + 1, 2] - pos[:, :, 2]
        dx, dy = pos[:, q:q + 1, 0] - pos[:, :, 0], pos[:, q:q + 1, 1] - pos[:, :, 1]
        dxy2 = dx * dx + dy * dy
        act = (dz > 0) & (dxy2 < 100.0 if lt100 else torch.sqrt(dxy2) < 10.0)
        dzs = torch.where(act, dz, torch.ones_like(dz))
        rr = r / (4.0 * dzs)
        u = torch.sqrt(dxy2) / (c1 * dzs + c2)
        fz = torch.where(act, fz + (-(c0 * (rr * rr)) * torch.exp(-0.5 * (u * u))), fz)
    return fz


def rollout_dw(K_dyn, P, rows, x0, last_rpm, v, S, effects, D, order=1, drag_up0=True, lt100=False):
    """The states [T, B, 13] of commands v [T, B, 4] (after the box) with downwash, for B / D groups of D consecutive drones
    (an (aviary, sample) group each): every substep takes fz from that substep's start positions (dw_fz) and renormalises the
    quaternion, as ctrl_rollout_kernel and mppi_rollout run one dyn_tick_k substep at a time; drag reads the previous tick's
    clipped rpm in substep 0 (last_rpm at tick 0).  Negative controls only: drag_up0=False reads the current rpm there;
    order and lt100 as dw_fz."""
    B = x0.shape[0]
    x, up, xs = x0, last_rpm, []
    mx = rows[:, 13:14]
    k2 = 2 * math.pi
    for k in range(v.shape[0]):
        u = torch.clamp(v[k], min=torch.zeros_like(v[k]), max=mx.expand_as(v[k]))
        ds_prev, ds_cur = (k2 * up / 60).sum(1), (k2 * u / 60).sum(1)
        for s in range(S):
            q = x[:, 3:7]
            x = torch.cat([x[:, 0:3], q / torch.sqrt((q * q).sum(1, keepdim=True)), x[:, 7:13]], dim=1)
            fz = dw_fz(P, x[:, 0:3].reshape(B // D, D, 3), order, lt100).reshape(B)
            x = DR.substep(K_dyn, rows, x, u, ds_prev if s == 0 and drag_up0 else ds_cur, effects, fz=fz)
        up = u
        xs.append(x)
    return torch.stack(xs)


def rollout_cost_dw(K_dyn, P, rows, x0, last_rpm, v, targets, W, Rt, uref, S, effects, D, **kw):
    """J [B] per drone of rollout_dw's states (the stage cost of ilqr_ref on the commands v), and the states [T, B, 13]"""
    x = rollout_dw(K_dyn, P, rows, x0, last_rpm, v, S, effects, D, **kw)
    return IR.cost(x, targets, W, v, uref, Rt), x
