"""Float64 torch restatement of the iLQR backward pass of qs_ilqr_backward (csrc/riccati.cuh, DESIGN.md 4.5.1) and of the cost
the line search and the commit evaluate (test infrastructure, CPU or CUDA tensors, batched over leading dimensions).

A tick maps z_k to z_{k+1} with F = [A | B] (n_z rows, n_z + 4 columns).  The backward tick is the textbook Gauss-Newton DDP step
with Tassa's value update: Qx = A'V_x, Qu = Rt du + B'V_x, Qxx = A'V_xx A, Quu = Rt + B'V_xx B (symmetrised), Qux = B'V_xx A;
Quu_mu = Quu + mu diag(Quu); k = -Quu_mu^-1 Qu, K = -Quu_mu^-1 Qux; V_x = Qx + K'Quu k + K'Qu + Qux'k,
V_xx = Qxx + K'Quu K + K'Qux + Qux'K, symmetrised.

The line search's J(alpha) (rollout_cost, on diff_ref.tick), the commit rule (commit) and the backward's restart ladder (mu_ladder)
are restated operation for operation in the kernels' order: the kernels are built with -fmad=false, so Python floats give the
same bits."""
import torch

import diff_ref as DR


def backward_tick(F, V, vx, Rt, du, mu, symmetrise=True, regularised_value=False):
    """One tick for batches: F [..., nz, nz + 4], V [..., nz, nz], vx [..., nz], Rt [..., 4], du [..., 4], mu [...].  Returns
    {K [..., 4, nz], k [..., 4], V, vx, dV1, dV2, ok}.  symmetrise=False and regularised_value=True (Quu_mu in the value
    update) are negative controls."""
    nz = F.shape[-2]
    A, B = F[..., :nz], F[..., nz:]
    At, Bt = A.mT, B.mT
    Qx = (At @ vx[..., None])[..., 0]
    Qu = Rt * du + (Bt @ vx[..., None])[..., 0]
    Qxx = At @ V @ A
    Quu = torch.diag_embed(Rt) + Bt @ V @ B
    Quu = 0.5 * (Quu + Quu.mT)
    Qux = Bt @ V @ A
    mu = torch.as_tensor(mu, dtype=F.dtype, device=F.device)
    Qr = Quu + mu[..., None, None] * torch.diag_embed(torch.diagonal(Quu, dim1=-2, dim2=-1))
    L, info = torch.linalg.cholesky_ex(Qr)
    ok = (info == 0) & torch.isfinite(torch.diagonal(L, dim1=-2, dim2=-1)).all(-1)   # chol4: a pivot must be > 0 and finite
    k = -torch.cholesky_solve(Qu[..., None], L)[..., 0]
    K = -torch.cholesky_solve(Qux, L)
    Qv = Qr if regularised_value else Quu
    Kt = K.mT
    vx_new = Qx + (Kt @ (Qv @ k[..., None]))[..., 0] + (Kt @ Qu[..., None])[..., 0] + (Qux.mT @ k[..., None])[..., 0]
    Vn = Qxx + Kt @ Qv @ K + Kt @ Qux + Qux.mT @ K
    if symmetrise:
        Vn = 0.5 * (Vn + Vn.mT)
    dV1 = (k * Qu).sum(-1)
    dV2 = 0.5 * (k * (Quu @ k[..., None])[..., 0]).sum(-1)
    return dict(K=K, k=k, V=Vn, vx=vx_new, dV1=dV1, dV2=dV2, ok=ok)


def stage(V, vx, dx, W):
    """V, vx plus the cost 1/2 sum_r W_r dx_r^2 of the 13 state components (the first 13 of z)."""
    nz = V.shape[-1]
    pad = lambda x: torch.nn.functional.pad(x, (0, nz - 13))
    return V + torch.diag_embed(pad(W)), vx + pad(W * dx)


def backward_pass(F, dx, W, Rt, du, mu, V=None, vx=None, **kw):
    """T ticks, t = T-1 .. 0: F [T, ..., nz, nz + 4], dx and W [T, ..., 13] of the state after tick t, du [T, ..., 4]; V, vx: the
    value after the last tick (None: zero).  Returns {K [T, ..., 4, nz], k [T, ..., 4], V, vx (at z_0), dV1, dV2, ok}."""
    T, nz = F.shape[0], F.shape[-2]
    V = torch.zeros(F.shape[1:-1] + (nz,), dtype=F.dtype, device=F.device) if V is None else V
    vx = torch.zeros(F.shape[1:-1], dtype=F.dtype, device=F.device) if vx is None else vx
    Ks, ks = [None] * T, [None] * T
    dV1 = dV2 = 0.0
    ok = torch.ones(F.shape[1:-2], dtype=torch.bool, device=F.device)
    for t in range(T - 1, -1, -1):
        V, vx = stage(V, vx, dx[t], W[t])
        r = backward_tick(F[t], V, vx, Rt, du[t], mu, **kw)
        Ks[t], ks[t], V, vx = r["K"], r["k"], r["V"], r["vx"]
        dV1, dV2, ok = dV1 + r["dV1"], dV2 + r["dV2"], ok & r["ok"]
    return dict(K=torch.stack(Ks), k=torch.stack(ks), V=V, vx=vx, dV1=dV1, dV2=dV2, ok=ok)


def f_from_jac(jac, raw, max_rpm):
    """F [..., nz, nz + 4] from qs_dyn_tick_jac's tick block jac [..., 13, C] (C = 17, or 21 with drag) and the raw rpm [..., 4]
    of the tick: with drag z = (x, clipped previous RPMs), whose rows are the clip's derivative of u."""
    C = jac.shape[-1]
    if C == 17:
        return jac.clone()
    cd = ((raw >= 0) & (raw <= max_rpm[..., None])).to(jac.dtype)
    top = torch.cat([jac[..., :13], jac[..., 17:21], jac[..., 13:17]], dim=-1)
    bottom = torch.cat([torch.zeros(jac.shape[:-2] + (4, 17), dtype=jac.dtype, device=jac.device), torch.diag_embed(cd)], dim=-1)
    return torch.cat([top, bottom], dim=-2)


def cost(x, ref, W, u, uref, Rt):
    """J = 1/2 sum_t (sum_r W_t,r (x - ref)^2 + sum_j Rt_j (u - uref)^2): x, ref, W [T, ..., 13], u [T, ..., 4], uref and Rt
    [..., 4]."""
    return 0.5 * ((W * (x - ref) ** 2).sum(-1) + (Rt * (u - uref) ** 2).sum(-1)).sum(0)


def rollout_cost(K_dyn, rows, x0, last_rpm, rpm_nom, states_nom, Kfb, kff, alpha, targets, W, Rt, uref, S, effects,
                 drag_prev_raw=False):
    """J(alpha) of the line search: the rollout u_k = rpm_nom[k] + alpha kff[k] + Kfb[k] (z_k - z_nom,k) from x0 on diff_ref.tick,
    with dz taken against the nominal that is passed in (teacher-forced on states_nom [T, B, 13], the states after each tick).
    z = x, and with drag also the previous clipped RPMs (last_rpm at k = 0, then the rollout's clip(u) and the nominal's
    clip(rpm_nom)).  rows [B, 16], x0 [B, 13], last_rpm [B, 4], rpm_nom [T, B, 4], Kfb [T, B, 4, nz] and kff [T, B, 4] (None:
    zero), alpha a float or [B], targets and W [T, B, 13], Rt and uref [B, 4].  The control cost is on the raw u.
    drag_prev_raw=True takes the nominal's previous RPMs unclipped -- a negative control only.
    Returns {J [B], u [T, B, 4], x [T, B, 13]}."""
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
        x, up = DR.tick(K_dyn, rows, x, u, up, S, effects)
        xn = states_nom[k]
        upn = raw if drag_prev_raw else torch.clamp(raw, min=torch.zeros_like(raw), max=rows[:, 13:14].expand_as(raw))
        us.append(u)
        xs.append(x)
    u, x = torch.stack(us), torch.stack(xs)
    return dict(J=cost(x, targets, W, u, uref, Rt), u=u, x=x)


def commit(alpha, J, Jn, dV1, dV2, mu, status, converged, Jc=None, first_accepted=False):
    """ilqr_commit_kernel for one drone, in its operations and order: alpha [n_alpha] and J [n_alpha] of the line search, the
    nominal's cost Jn, dV1, dV2, mu, status and converged (Python scalars).  Jc: the committed rollout's J (default J[best], which
    the kernel reproduces bit for bit).  first_accepted=True takes the first accepted alpha instead of the largest -- a negative
control only.  Returns (best: index of the chosen alpha or -1, new mu, converged)."""
    alpha, J = [float(a) for a in alpha], [float(j) for j in J]
    Jn, dV1, dV2, mu = float(Jn), float(dV1), float(dV2), float(mu)
    if converged:
        return -1, mu, True
    best = -1
    if status == 0:
        for s, (al, Ja) in enumerate(zip(alpha, J)):
            expected = -(al * dV1 + al * al * dV2)
            if Ja < Jn and Jn - Ja >= 1e-4 * expected and (best < 0 or (al > alpha[best] and not first_accepted)):
                best = s
    if best >= 0:
        Jc = J[best] if Jc is None else float(Jc)
        mu = mu / 10.0
        if mu < 1e-6:
            mu = 0.0
        return best, mu, Jn - Jc < 1e-9 * Jn
    return best, max(1e-6, 10.0 * mu), False


def converged_boundary(Jn):
    """The largest committed J that does not set `converged` (Jn - Jc >= 1e-9 Jn): one ulp above it does."""
    import numpy as np
    t = 1e-9 * Jn
    Jc = Jn - t
    while not Jn - Jc >= t:
        Jc = np.nextafter(Jc, -np.inf)
    while Jn - np.nextafter(Jc, np.inf) >= t:
        Jc = np.nextafter(Jc, np.inf)
    return float(Jc)


def armijo_boundary(Jn, al, dV1, dV2):
    """The largest J(al) that passes Jn - J >= 1e-4 (-(al dV1 + al^2 dV2)): one ulp above it fails."""
    import numpy as np
    t = 1e-4 * -(al * dV1 + al * al * dV2)
    Ja = Jn - t
    while not Jn - Ja >= t:
        Ja = np.nextafter(Ja, -np.inf)
    while Jn - np.nextafter(Ja, np.inf) >= t:
        Ja = np.nextafter(Ja, np.inf)
    return float(Ja)


def mu_ladder(mu0, ok_at):
    """The backward's restart ladder from the incoming mu0: while the pass fails at mu, mu = fmax(1e-6, 10 mu), at most 8
    restarts.  ok_at(mu) -> bool says whether the pass succeeds at mu (a float t stands for mu >= t).  Returns (mu, status)."""
    ok = ok_at if callable(ok_at) else (lambda m: m >= ok_at)
    mu = float(mu0)
    for restarts in range(9):
        if ok(mu):
            return mu, 0
        mu = max(1e-6, 10.0 * mu)
    return mu, 1


def tick_jac(K_dyn, rows, x, raw, up, S, effects):
    """qs_dyn_tick_jac's tick blocks [B, 13, C] (columns: state, raw rpm, and with drag the previous clipped rpm) of diff_ref.tick
    by forward mode: the B drones are independent, so one tangent per column, the same for every drone, gives each drone's
    own column (linear in B, where jacfwd of the batch is quadratic).  rows [B, 16], x [B, 13], raw and up [B, 4]."""
    drag = bool(effects & DR.EFFECT_DRAG)
    C = 21 if drag else 17
    eye = torch.eye(C, dtype=x.dtype, device=x.device)
    tx = eye[:, None, :13].expand(C, x.shape[0], 13)
    tr = eye[:, None, 13:17].expand(C, x.shape[0], 4)
    tu = eye[:, None, 17:21].expand(C, x.shape[0], 4) if drag else torch.zeros((C, x.shape[0], 4), dtype=x.dtype, device=x.device)
    f = lambda a, r, u: DR.tick(K_dyn, rows, a, r, u, S, effects)[0]
    J = torch.func.vmap(lambda a, b, c: torch.func.jvp(f, (x, raw, up), (a, b, c))[1])(tx, tr, tu)
    return J.permute(1, 2, 0).contiguous()
