"""Float64 restatement of mppi() (DESIGN.md 4.5.2) for the tests: Philox4x32-10 in Python integers, Box-Muller in NumPy, the
sample rollouts' cost through ilqr_ref / diff_ref, and the weights, candidate and commit rules of qs_mppi_update and
qs_mppi_commit."""
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


def weights(J, temperature):
    """w [K] and the best sample of a unit's costs J [K] (the rule of qs_mppi_update)"""
    J = np.asarray(J, dtype=np.float64)
    fin = np.isfinite(J)
    if not fin.any():
        return np.zeros_like(J), 0
    jmin = J[fin].min()
    best = int(np.flatnonzero(fin & (J == jmin))[0])
    lam = temperature * (J[fin].mean() - jmin)
    w = np.where(fin, 1.0 if lam == 0 else np.exp(-(np.where(fin, J, jmin) - jmin) / (lam if lam else 1.0)), 0.0)
    return w, best


def candidate(u, delta, w):
    """u + sum_s w_s delta_s / sum_s w_s (u when no weight is positive); delta [K, ...]"""
    ws = w.sum()
    if not ws > 0:
        return u.copy()
    return u + np.tensordot(w, delta, axes=1) / ws


def pick(jc, J):
    """-1 keeps the candidate (jc <= the best sample's J), else the best sample"""
    _, best = weights(J, 1.0)
    return -1 if jc <= J[best] else best


def rollout_cost(K_dyn, rows, x0, last_rpm, v, targets, W, Rt, uref, S, effects):
    """J [B] of the commands v [T, B, 4] (after the box) on diff_ref's tick, the cost of ilqr_ref (torch float64 tensors)"""
    return IR.rollout_cost(K_dyn, rows, x0, last_rpm, v, v, None, None, 0.0, targets, W, Rt, uref, S, effects)["J"]   # no gains: no dz
