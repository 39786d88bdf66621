"""Shared helpers of the closed-loop forward-mode tests (test infrastructure): the g++ build of pid_tangent.cuh with the closed-loop
tick of dyn_ctrl_jvp.cu, and one closed-loop tick's Jacobian per drone and input block from that build, from the transpose of the
host-built closed-loop adjoint (diff_ctrl_host.cpp) and from torch.func.jacfwd of the reference (tests/diff_pid_ref.py +
tests/diff_ref.py)."""
import ctypes as C

import numpy as np
import torch

import diff_pid_ref as PR
import diff_ref as R
from diff_ctrl_testlib import host_ctrl_tick_vjp
from qs_testlib import harness

# input blocks of one closed-loop tick and their widths (diff_ctrl_testlib.BLOCKS' order), and the 26 output rows: the end
# state (13), the updated controller state (9), the applied RPMs (4)
BLOCKS = (("state", 13), ("pid", 9), ("targets", 10), ("last_rpm", 4), ("phys", 16), ("gains", 18))
OUTS = (("out", 13), ("pid_out", 9), ("rpm", 4))


def ctrl_jvp_harness():
    """tests/host_harness/ctrl_jvp_host.cpp: the kernels' closed-loop tick tangent compiled for the host."""
    L = harness("ctrl_jvp_host")
    L.cj_ctrl_tick_jvp.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_int, C.c_double, C.c_int] + [C.c_void_p] * 18
    return L


def host_ctrl_tick_jvp(P, CP, effects, S, dt, rows, gains, state, pid, tg, up, tan):
    """The host-built closed-loop tick and its tangent for n drones along tan = {block: [n, width]}.  Returns {out, rpm, pid_out}
    and their tangents {t_out, t_rpm, t_pid_out}."""
    L = ctrl_jvp_harness()
    n = state.shape[0]
    a = lambda x: np.ascontiguousarray(x, dtype=np.float64)
    ins = [a(x) for x in (rows, gains, state, pid, tg, up)]
    tans = [a(tan[k]) for k in ("phys", "gains", "state", "pid", "targets", "last_rpm")]
    outs = [np.zeros((n, w)) for w in (13, 4, 9, 13, 4, 9)]
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    L.cj_ctrl_tick_jvp(C.addressof(P), C.addressof(CP), effects, S, dt, n, *[p(x) for x in ins + tans], *[p(o) for o in outs])
    return dict(zip(("out", "rpm", "pid_out", "t_out", "t_rpm", "t_pid_out"), outs))


def _stack_rows(t):
    """[n, 26] rows of the outputs' tangents in OUTS order"""
    return np.concatenate([t["t_out"], t["t_pid_out"], t["t_rpm"]], axis=1)


def host_ctrl_tick_jac(P, CP, effects, S, dt, rows, gains, state, pid, tg, up):
    """{block: [n, 26, width]} of the host-built tangent, one unit tangent per column."""
    n = len(state)
    jac = {}
    for blk, w in BLOCKS:
        cols = []
        for j in range(w):
            tan = {k: np.zeros((n, wk)) for k, wk in BLOCKS}
            tan[blk][:, j] = 1.0
            cols.append(_stack_rows(host_ctrl_tick_jvp(P, CP, effects, S, dt, rows, gains, state, pid, tg, up, tan)))
        jac[blk] = np.stack(cols, axis=2)
    return jac


def vjp_ctrl_tick_jac(P, CP, effects, S, dt, rows, gains, state, pid, tg, up):
    """{block: [n, 26, width]} of the host-built closed-loop adjoint, transposed: one unit cotangent per output row."""
    n = len(state)
    per_row = []
    for r in range(26):
        g = np.zeros((n, 26))
        g[:, r] = 1.0
        res = host_ctrl_tick_vjp(P, CP, effects, S, dt, rows, gains, state, pid, tg, up, g[:, 0:13], g[:, 22:26], g[:, 13:22])
        per_row.append(res)
    return {blk: np.stack([x[blk] for x in per_row], axis=1) for blk, _ in BLOCKS}


def ref_ctrl_tick_jac(P, CP, effects, S, dt, rows, gains, state, pid, tg, up, flip=()):
    """{block: [n, 26, width]}: torch.func.jacfwd of diff_pid_ref.pid + diff_ref.tick, the diagonal (per-drone) blocks.  flip:
    diff_pid_ref's decisions to turn the other way (the negative controls)."""
    K, Cc = R.model_constants(P), PR.controller_constants(CP)
    t = lambda v: torch.tensor(np.asarray(v, dtype=np.float64))
    args = tuple(t(v) for v in (state, pid, tg, up, rows, gains))

    def f(x, st, tgt, u_prev, rw, gn):
        raw, st1, _, _ = PR.pid(Cc, gn, st, dt, x, tgt[:, 0:3], tgt[:, 3], tgt[:, 4:7], tgt[:, 7:10], flip)
        out, u = R.tick(K, rw, x, torch.clamp(raw, 0.0, Cc["max_rpm"]), u_prev, S, effects)
        return torch.cat([out, st1, u], dim=1)

    J = torch.func.jacfwd(f, argnums=tuple(range(6)))(*args)
    return {blk: torch.diagonal(j, dim1=0, dim2=2).permute(2, 0, 1).numpy() for (blk, _), j in zip(BLOCKS, J)}
