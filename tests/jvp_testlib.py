"""Shared helpers of the forward-mode tests (test infrastructure): the g++ build of dyn_tangent.cuh (the tick tangent of the JVP and
Jacobian kernels, dyn_jvp.cu) and one tick's Jacobian per drone and input block, from that build, from the transpose of the
host-built adjoint (diff_host.cpp) and from torch.func.jacfwd of the reference tests/diff_ref.py."""
import ctypes as C

import numpy as np

from diff_testlib import host_tick_vjp, per_drone_relerr
from qs_testlib import harness

# input blocks of one tick and their widths: the tick-start state, the raw RPMs, drag's previous clipped RPMs, the 16-column row
BLOCKS = (("state", 13), ("rpm", 4), ("up", 4), ("row", 16))


def jvp_harness():
    """tests/host_harness/jvp_host.cpp: the kernels' tick tangent compiled for the host."""
    L = harness("jvp_host")
    L.jh_tick_jvp.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_int, C.c_int] + [C.c_void_p] * 9
    return L


def host_tick_jvp(P, effects, S, state, raw, up, rows, t_state, t_raw, t_up, t_rows):
    """The host-built tick tangent for n drones: (out [n, 13], t_out [n, 13])."""
    L = jvp_harness()
    a = lambda x: np.ascontiguousarray(x, dtype=np.float64)
    ins = [a(x) for x in (state, raw, up, t_state, t_raw, t_up, t_rows)]
    rows = None if rows is None else a(rows)
    n = ins[0].shape[0]
    out, t_out = np.zeros((n, 13)), np.zeros((n, 13))
    p = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)
    L.jh_tick_jvp(C.addressof(P), p(rows), effects, S, n, *[p(x) for x in ins[:6]], p(ins[6]), p(out), p(t_out))
    return out, t_out


def _units(n, block, j):
    """Tangents of the four blocks for n drones: a unit in column j of `block`, zero elsewhere."""
    t = {k: np.zeros((n, w)) for k, w in BLOCKS}
    t[block][:, j] = 1.0
    return t


def host_tick_jac(P, effects, S, state, raw, up, rows):
    """{block: [n, 13, width]} of the host-built tick tangent, one unit tangent per column."""
    n = len(state)
    jac = {}
    for blk, w in BLOCKS:
        cols = []
        for j in range(w):
            t = _units(n, blk, j)
            cols.append(host_tick_jvp(P, effects, S, state, raw, up, rows, t["state"], t["rpm"], t["up"], t["row"])[1])
        jac[blk] = np.stack(cols, axis=2)
    return jac


def vjp_tick_jac(P, effects, S, state, raw, up, rows):
    """{block: [n, 13, width]} of the host-built adjoint, transposed: one unit cotangent per row of the end state."""
    n = len(state)
    rows_out = []
    for r in range(13):
        g = np.zeros((n, 13))
        g[:, r] = 1.0
        _, g_state, g_raw, g_up, g_row = host_tick_vjp(P, effects, S, state, raw, up, g, rows)
        rows_out.append({"state": g_state, "rpm": g_raw, "up": g_up, "row": g_row})
    return {blk: np.stack([x[blk] for x in rows_out], axis=1) for blk, _ in BLOCKS}


def ref_tick_jac(P, effects, S, state, raw, up, rows, device=None, **kw):
    """{block: [n, 13, width]}: torch.func.jacfwd of diff_ref.tick, the diagonal (per-drone) blocks.  `kw`: diff_ref.tick's
    switches (the negative controls)."""
    import torch
    import diff_ref as R
    t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64), device=device)
    K = R.model_constants(P, device)
    args = tuple(t(a) for a in (state, raw, up, rows))
    f = lambda x, r, u, rw: R.tick(K, rw, x, r, u, S, effects, **kw)[0]
    J = torch.func.jacfwd(f, argnums=(0, 1, 2, 3))(*args)
    return {blk: torch.diagonal(j, dim1=0, dim2=2).permute(2, 0, 1).cpu().numpy() for (blk, _), j in zip(BLOCKS, J)}


def worst_per_block(got, want):
    """{block: worst per-drone normwise relative error} of two {block: [n, 13, width]} Jacobians."""
    return {k: float(np.max(per_drone_relerr(got[k], want[k]))) for k in got}
