"""Float64 references of the control-limited iLQR backward pass of qs_ilqr_box_backward (csrc/riccati.cuh, DESIGN.md 4.5.1)
and of the clamped rollout its line search and commit evaluate (test infrastructure).

The box QP of one tick, min 1/2 x'H x + g'x subject to lo <= x <= hi with H symmetric positive definite, has one solution.  Two
independent references find it:
  * kkt_enum: every one of the 3^4 assignments of each dimension to free, at lo or at hi; the free block is solved with the
    others fixed and the assignment kept whose x lies in the box and whose gradient has the multipliers' signs (>= 0 at lo,
    <= 0 at hi);
  * bvls: scipy.optimize.lsq_linear(method="bvls") on the Cholesky form || L'x + L^-1 g ||^2 / 2 (H = L L').
The backward pass (backward_pass_box) restates the kernel's recursion in torch with the QP's k from kkt_enum, K's free rows
-(Quu_mu,ff)^-1 Qux,f and its held rows 0; full_factor_K=True takes K = -Quu_mu^-1 Qux on every row, a negative control."""
import itertools

import numpy as np
import scipy.optimize
import torch

import ilqr_ref as IR


def kkt_enum(H, g, lo, hi, tol=1e-9):
    """(x [4], act [4]: -1 at lo, +1 at hi, 0 free) of the assignment that satisfies the KKT conditions; among several (only
    in degenerate cases) the one with the smallest value.  tol: the relative slack of the feasibility and sign checks."""
    H, g, lo, hi = (np.asarray(a, dtype=np.float64) for a in (H, g, lo, hi))
    n = len(g)
    best = None
    scale = np.abs(g) + np.abs(H).sum(1) * np.maximum(np.abs(lo), np.abs(hi)) + 1e-300
    for asg in itertools.product((0, -1, 1), repeat=n):
        a = np.array(asg)
        x = np.where(a == -1, lo, np.where(a == 1, hi, 0.0))
        f = a == 0
        if f.any():
            x[f] = np.linalg.solve(H[np.ix_(f, f)], -(g[f] + H[np.ix_(f, ~f)] @ x[~f]))
        span = np.maximum(hi - lo, 1e-300)
        if np.any(x < lo - tol * span) or np.any(x > hi + tol * span):
            continue
        gr = g + H @ x
        if np.any(gr[a == -1] < -tol * scale[a == -1]) or np.any(gr[a == 1] > tol * scale[a == 1]):
            continue
        val = 0.5 * x @ H @ x + g @ x
        if best is None or val < best[0]:
            best = (val, x, a)
    assert best is not None, "no KKT point: H is not positive definite?"
    return best[1], best[2]


def bvls(H, g, lo, hi):
    """x of the QP by bounded-variable least squares on the Cholesky form"""
    H, g, lo, hi = (np.asarray(a, dtype=np.float64) for a in (H, g, lo, hi))
    L = np.linalg.cholesky(H)
    b = -np.linalg.solve(L, g)
    # lsq_linear needs lo < hi: a dimension with lo == hi is fixed and moved to the right-hand side
    fixed = lo == hi
    x = np.where(fixed, lo, 0.0)
    free = ~fixed
    if free.any():
        A = L.T
        r = scipy.optimize.lsq_linear(A[:, free], b - A[:, fixed] @ x[fixed], bounds=(lo[free], hi[free]), method="bvls", tol=1e-15,
                                      max_iter=200)
        assert r.status > 0                                  # 0: the iteration limit
        x[free] = r.x
    return x


def qp_value(H, g, x):
    return float(0.5 * x @ H @ x + g @ x)


def backward_tick_box(F, V, vx, Rt, du, lo, hi, mu, full_factor_K=False):
    """One tick for one drone: F [nz, nz + 4], V [nz, nz], vx [nz], Rt, du, lo, hi [4] (the box of k), mu a float.  As
    ilqr_ref.backward_tick with k the box QP's and K's held rows 0.  Returns {K, k, V, vx, dV1, dV2, act}."""
    nz = F.shape[-2]
    A, B = F[:, :nz], F[:, nz:]
    Qx = A.T @ vx
    Qu = Rt * du + B.T @ vx
    Qxx = A.T @ V @ A
    Quu = torch.diag(Rt) + B.T @ V @ B
    Quu = 0.5 * (Quu + Quu.T)
    Qux = B.T @ V @ A
    Qr = Quu + mu * torch.diag(torch.diagonal(Quu))
    x, act = kkt_enum(Qr.numpy(), Qu.numpy(), lo.numpy(), hi.numpy())
    k = torch.as_tensor(x, dtype=F.dtype)
    act = torch.as_tensor(act)
    free = act == 0
    K = torch.zeros((4, nz), dtype=F.dtype)
    if full_factor_K:
        K = -torch.linalg.solve(Qr, Qux)
    elif free.any():
        K[free] = -torch.linalg.solve(Qr[free][:, free], Qux[free])
    vx_new = Qx + K.T @ (Quu @ k) + K.T @ Qu + Qux.T @ k
    Vn = Qxx + K.T @ Quu @ K + K.T @ Qux + Qux.T @ K
    Vn = 0.5 * (Vn + Vn.T)
    return dict(K=K, k=k, V=Vn, vx=vx_new, dV1=float(k @ Qu), dV2=float(0.5 * k @ (Quu @ k)), act=act)


def backward_pass_box(F, dx, W, Rt, du, lo, hi, mu, V=None, vx=None, **kw):
    """T ticks, t = T-1 .. 0, for one drone: F [T, nz, nz + 4], dx and W [T, 13], du, lo, hi [T, 4]; V, vx the value after
    the last tick (None: zero).  Returns {K [T, 4, nz], k [T, 4], act [T, 4], V, vx, dV1, dV2}."""
    T, nz = F.shape[0], F.shape[-2]
    V = torch.zeros((nz, nz), dtype=F.dtype) if V is None else V
    vx = torch.zeros(nz, dtype=F.dtype) if vx is None else vx
    Ks, ks, acts = [None] * T, [None] * T, [None] * T
    dV1 = dV2 = 0.0
    for t in range(T - 1, -1, -1):
        V, vx = IR.stage(V, vx, dx[t], W[t])
        r = backward_tick_box(F[t], V, vx, Rt, du[t], lo[t], hi[t], mu, **kw)
        Ks[t], ks[t], acts[t], V, vx = r["K"], r["k"], r["act"], r["V"], r["vx"]
        dV1, dV2 = dV1 + r["dV1"], dV2 + r["dV2"]
    return dict(K=torch.stack(Ks), k=torch.stack(ks), act=torch.stack(acts), V=V, vx=vx, dV1=dV1, dV2=dV2)


def rollout_cost_box(K_dyn, rows, x0, last_rpm, rpm_nom, states_nom, Kfb, kff, alpha, targets, W, Rt, uref, S, effects, lo, hi,
                     clamp=True):
    """J(alpha) of qs_ilqr_box_line_search: ilqr_ref.rollout_cost with u_k clamped to [lo_k, hi_k] (lo, hi [T, B, 4]) before the
    tick and the stage cost, as torch.clamp does, i.e. min(max(u, lo), hi).  clamp=False is ilqr_ref.rollout_cost -- a negative
    control.  Returns {J [B], u [T, B, 4], x [T, B, 13]}."""
    import diff_ref as DR
    drag = bool(effects & DR.EFFECT_DRAG)
    alpha = torch.as_tensor(alpha, dtype=torch.float64, device=x0.device)
    x, xn, up, upn = x0, x0, last_rpm, last_rpm
    us, xs = [], []
    for k in range(rpm_nom.shape[0]):
        raw = rpm_nom[k]
        u = raw
        if kff is not None:
            u = u + alpha[..., None] * kff[k]
        if Kfb is not None:
            dz = x - xn
            if drag:
                dz = torch.cat([dz, up - upn], dim=-1)
            u = u + (Kfb[k] @ dz[..., None])[..., 0]
        if clamp:
            u = torch.minimum(torch.maximum(u, lo[k]), hi[k])
        x, up = DR.tick(K_dyn, rows, x, u, up, S, effects)
        xn = states_nom[k]
        upn = torch.clamp(raw, min=torch.zeros_like(raw), max=rows[:, 13:14].expand_as(raw))
        us.append(u)
        xs.append(x)
    u, x = torch.stack(us), torch.stack(xs)
    return dict(J=IR.cost(x, targets, W, u, uref, Rt), u=u, x=x)
