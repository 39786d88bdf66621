"""Shared helpers of the policy loop's forward-mode tests (test infrastructure): the g++ build of mlp_tangent.cuh
(tests/host_harness/policy_jvp_host.cpp), and one aviary tick's Jacobian per input block from that build, from the transpose of
the host-built adjoint (diff_policy_host.cpp) and from torch.func.jacfwd of a restatement of tests/diff_policy_ref.one_tick that
takes the observation's ang_v as part of the loop state.

One aviary tick maps the loop state (per drone: the stored state [13], the observation's ang_v [3], the history [B, A], drag's
previous applied rpm [4]), the aviary's constants [16] and an additive perturbation raw_in [D A] of the raw action to the next
state, ang_v, history, applied rpm and the raw action (OUTS)."""
import ctypes as C

import numpy as np
import torch

import diff_policy_ref as PR
import diff_ref as R
from qs_testlib import harness

BLOCKS = ("state", "ang", "hist", "up", "row", "raw_in")
OUTS = ("state", "ang", "hist", "u", "raw")


def _arr(x):
    return np.ascontiguousarray(torch.as_tensor(x).detach().numpy(), dtype=np.float64)


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _actor_ptrs(theta):
    depth = len(theta) // 2 - 1
    th = [_arr(t) for t in theta]
    Ws = (C.c_void_p * (depth + 1))(*[_ptr(th[2 * l]).value for l in range(depth + 1)])
    bs = (C.c_void_p * (depth + 1))(*[_ptr(th[2 * l + 1]).value for l in range(depth + 1)])
    width = (C.c_int * 4)(*([th[2 * l].shape[1] for l in range(depth)] + [0] * (4 - depth)))
    return th, depth, width, Ws, bs


def widths(D, A, B):
    """{block: flattened width} of the inputs and {output: width} of one aviary tick"""
    ins = dict(state=13 * D, ang=3 * D, hist=B * A * D, up=4 * D, row=16, raw_in=D * A)
    outs = dict(state=13 * D, ang=3 * D, hist=B * A * D, u=4 * D, raw=D * A)
    return ins, outs


def host_tick_jvp(P, effects, S, activation, theta, noise, x, tan):
    """The host-built aviary tick and its tangent: x = {state [D, 13], ang [D, 3], hist [D, B, A], up [D, 4], row [16]},
    tan = {block: array of the block's shape}.  Returns ({output: value}, {output: tangent}), flattened."""
    lib = harness("policy_jvp_host")
    D, B, A = x["hist"].shape
    th, depth, width, Ws, bs = _actor_ptrs(theta)
    ins = [_arr(x[k]) for k in ("row", "state", "ang", "hist", "up")]
    tans = [_arr(tan[k]) for k in ("row", "state", "ang", "hist", "up", "raw_in")]
    _, ow = widths(D, A, B)
    outs = [np.zeros(ow[k]) for k in OUTS] + [np.zeros(ow[k]) for k in OUTS]
    nz = None if noise is None else _arr(noise)
    lib.pj_tick_jvp(C.c_void_p(C.addressof(P)), C.c_uint(effects), S, D, A, B, 0 if activation == "tanh" else 1, depth, width, Ws, bs, _ptr(th[-1]),
                    None if nz is None else _ptr(nz), *[_ptr(a) for a in ins], *[_ptr(a) for a in tans], *[_ptr(o) for o in outs])
    return dict(zip(OUTS, outs[:5])), dict(zip(OUTS, outs[5:]))


def host_tick_jac(P, effects, S, activation, theta, noise, x):
    """{block: [rows, width]} of the host-built tangent, one unit tangent per column; rows are OUTS' entries in order"""
    D, B, A = x["hist"].shape
    iw, _ = widths(D, A, B)
    shapes = dict(state=(D, 13), ang=(D, 3), hist=(D, B, A), up=(D, 4), row=(16,), raw_in=(D * A,))
    jac = {}
    for blk in BLOCKS:
        cols = []
        for j in range(iw[blk]):
            tan = {k: np.zeros(shapes[k]) for k in BLOCKS}
            tan[blk].reshape(-1)[j] = 1.0
            _, t = host_tick_jvp(P, effects, S, activation, theta, noise, x, tan)
            cols.append(np.concatenate([t[k] for k in OUTS]))
        jac[blk] = np.stack(cols, axis=1)
    return jac


def ref_tick(P, effects, S, activation, theta, noise, flip=(), device=None):
    """f(state, ang, hist, up, row, raw_in) -> OUTS' entries concatenated: diff_policy_ref.one_tick with ang_v as state.  flip:
    diff_policy_ref's decisions to turn the other way, and "ang_start": the next ang_v through the tick's start attitude instead
    of the last substep's (negative controls only).  The end-of-tick attitude would give the same function: the last substep
    turns the attitude about w_end itself, which R(q_end) w_end = R(q_last) w_end leaves fixed."""
    K = R.model_constants(P, device)
    th = [torch.as_tensor(t, dtype=torch.float64, device=device) for t in theta]
    eps = None if noise is None else torch.as_tensor(noise, dtype=torch.float64, device=device)

    def f(x, ang, hist, up, row, raw_in):
        n, B, A = hist.shape
        rows = row[None].expand(n, 16)
        obs = torch.cat([x[:, 0:3], PR.PR.quat_to_euler(x[:, 3:7]), x[:, 7:10], ang, hist.reshape(n, B * A)], dim=1).reshape(1, -1)
        raw = PR.actor(th, activation, obs, flip)[0]
        if eps is not None:
            raw = raw + torch.exp(th[-1]) * eps
        raw = (raw + raw_in).reshape(n, A)
        a = torch.clamp(raw, -1.0, 1.0)
        if "clip" in flip:
            a = raw + (a - raw).detach()
        hist1 = torch.cat([hist[:, 1:], a[:, None, :]], dim=1)
        rpm = (rows[:, 12:13] * (1.0 + 0.05 * a)).expand(n, 4)
        x1, u, ql1 = PR.tick(K, rows, x, rpm, up, S, effects)
        q0 = x[:, 3:7] / torch.sqrt((x[:, 3:7] ** 2).sum(1, keepdim=True))
        ang1 = (PR.matrix_unit(q0 if "ang_start" in flip else ql1) @ x1[:, 10:13, None])[:, :, 0]
        return torch.cat([x1.reshape(-1), ang1.reshape(-1), hist1.reshape(-1), u.reshape(-1), raw.reshape(-1)])
    return f


def ref_tick_jac(P, effects, S, activation, theta, noise, x, flip=(), device=None):
    """{block: [rows, width]}: torch.func.jacfwd of ref_tick on `device` (x's entries may be arrays or tensors), as NumPy arrays"""
    D = x["state"].shape[0]
    t = lambda v: torch.as_tensor(v, dtype=torch.float64, device=device)
    args = tuple(t(x[k]) for k in ("state", "ang", "hist", "up", "row")) + (torch.zeros(D * x["hist"].shape[2], dtype=torch.float64,
                                                                                        device=device),)
    J = torch.func.jacfwd(ref_tick(P, effects, S, activation, theta, noise, flip, device), argnums=tuple(range(6)))(*args)
    return {blk: j.reshape(j.shape[0], -1).cpu().numpy() for blk, j in zip(BLOCKS, J)}


def kernel_layout(D, A, B, drag):
    """Where linearise(policy=)'s [R, R] tick Jacobian of one aviary sits in ref_tick_jac's blocks: (rows, cols, groups) with
    rows [R] the reference row of each kernel row, cols [R] the column of each kernel column in the reference blocks laid side by
    side in BLOCKS order, and groups {block: kernel columns} (state, ang, hist, up with drag, delta = raw_in).  The loop state is
    drone-major in the kernel (quadsim.h: pos, quat, vel, rpy_rates, ang_v, history, drag's previous rpm per drone) and
    block-major in the reference."""
    iw, ow = widths(D, A, B)
    BA, nzd = B * A, 16 + B * A + (4 if drag else 0)
    z = []
    for d in range(D):
        z += [13 * d + j for j in range(13)] + [13 * D + 3 * d + j for j in range(3)]
        z += [16 * D + d * BA + j for j in range(BA)] + ([16 * D + D * BA + 4 * d + j for j in range(4)] if drag else [])
    raw_row = ow["state"] + ow["ang"] + ow["hist"] + ow["u"]
    raw_col = iw["state"] + iw["ang"] + iw["hist"] + iw["up"] + iw["row"]
    rows = np.array(z + [raw_row + i for i in range(D * A)])
    cols = np.array(z + [raw_col + i for i in range(D * A)])
    entry = np.array([j for d in range(D) for j in range(nzd)])
    groups = dict(state=np.flatnonzero(entry < 13), ang=np.flatnonzero((entry >= 13) & (entry < 16)),
                  hist=np.flatnonzero((entry >= 16) & (entry < 16 + BA)))
    if drag:
        groups["up"] = np.flatnonzero(entry >= 16 + BA)
    groups["delta"] = np.arange(D * nzd, D * nzd + D * A)
    return rows, cols, groups


def vjp_tick_jac(P, effects, S, activation, theta, noise, x, ql):
    """{block: [rows, width]} of the host-built adjoint (diff_policy_host.cpp), transposed, for the rows of the outputs it has
    (state, ang, hist, raw: not u), in the tangent's coordinates: the adjoint takes the attitude ql that ang_v = R(ql) w is formed
    from.  Returns (J, dw, dq) with dw [D, 3, 3] = d ang / d w and dq [D, 3, 4] = d ang / d ql per drone, which map the
    tangent's blocks into the adjoint's coordinates (compose_for_vjp).  x["ang"] must be R(ql) w."""
    lib = harness("diff_policy_host")
    D, B, A = x["hist"].shape
    th, depth, width, Ws, bs = _actor_ptrs(theta)
    ins = [_arr(v) for v in (x["row"], x["state"], ql, x["hist"], x["up"])]
    nz = np.zeros(D * A) if noise is None else _arr(noise)
    _, ow = widths(D, A, B)
    rows = [k for k in OUTS if k != "u"]
    nrow = sum(ow[k] for k in rows)
    got = {k: [] for k in ("state", "ql", "hist", "up", "row", "raw_in")}
    for r in range(nrow):
        g = np.zeros(nrow)
        g[r] = 1.0
        parts, o = {}, 0
        for k in rows:
            parts[k] = np.ascontiguousarray(g[o:o + ow[k]])
            o += ow[k]
        shapes = [(D, 13), (D, A), (D, B, A), (D, 4), (D, 13), (D, 4), (D, B, A), (D, 4), (16,), (D, A)]
        outs = [np.zeros(s) for s in shapes]
        lib.dph_tick_vjp(C.c_void_p(C.addressof(P)), C.c_uint(effects), S, D, A, B, 0 if activation == "tanh" else 1, depth, width, Ws, bs,
                         _ptr(th[-1]), _ptr(nz), *[_ptr(a) for a in ins], _ptr(parts["state"]), _ptr(parts["raw"]), _ptr(parts["ang"]),
                         _ptr(parts["hist"]), *[_ptr(o) for o in outs])
        for k, v in zip(("state", "ql", "hist", "up", "row", "raw_in"), outs[4:]):
            got[k].append(v.reshape(-1))
    J = {k: np.stack(v, axis=0) for k, v in got.items()}              # [rows, width]: row r of J
    qt, wt = torch.as_tensor(_arr(ql)), torch.as_tensor(_arr(x["state"]))[:, 10:13]
    dw = torch.func.vmap(lambda q, w: torch.func.jacfwd(lambda w_: (PR.matrix_unit(q[None]) @ w_[:, None])[0, :, 0])(w))(qt, wt).numpy()
    dq = torch.func.vmap(lambda q, w: torch.func.jacfwd(lambda q_: (PR.matrix_unit(q_[None]) @ w[:, None])[0, :, 0])(q))(qt, wt).numpy()
    return J, dw, dq


def compose_for_vjp(jac, D, dw, dq):
    """The tangent's {block: [rows, width]} in the adjoint's coordinates (vjp_tick_jac): w's columns gain ang's through
    d ang / d w, and ql's columns are ang's through d ang / d ql"""
    state = jac["state"].copy()
    for d in range(D):
        state[:, 13 * d + 10:13 * d + 13] += jac["ang"][:, 3 * d:3 * d + 3] @ dw[d]
    ql = np.concatenate([jac["ang"][:, 3 * d:3 * d + 3] @ dq[d] for d in range(D)], axis=1)
    return dict(state=state, ql=ql, hist=jac["hist"], up=jac["up"], row=jac["row"], raw_in=jac["raw_in"])


def drop_u_rows(jac, D, A, B):
    """rows of `jac` without the applied rpm's"""
    _, ow = widths(D, A, B)
    o = ow["state"] + ow["ang"] + ow["hist"]
    keep = np.r_[0:o, o + ow["u"]:o + ow["u"] + ow["raw"]]
    return {k: v[keep] for k, v in jac.items()}
