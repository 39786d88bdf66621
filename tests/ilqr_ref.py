"""Float64 torch restatement of the iLQR backward pass of qs_ilqr_backward (csrc/riccati.cuh, DESIGN.md 4.5.1) and of the cost
the line search and the commit evaluate (test infrastructure, CPU or CUDA tensors, batched over leading dimensions).

A tick maps z_k to z_{k+1} with F = [A | B] (n_z rows, n_z + 4 columns).  The backward tick is the textbook Gauss-Newton DDP step
with Tassa's value update: Qx = A'V_x, Qu = Rt du + B'V_x, Qxx = A'V_xx A, Quu = Rt + B'V_xx B (symmetrised), Qux = B'V_xx A;
Quu_mu = Quu + mu diag(Quu); k = -Quu_mu^-1 Qu, K = -Quu_mu^-1 Qux; V_x = Qx + K'Quu k + K'Qu + Qux'k,
V_xx = Qxx + K'Quu K + K'Qux + Qux'K, symmetrised."""
import torch


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
    return dict(K=K, k=k, V=Vn, vx=vx_new, dV1=dV1, dV2=dV2, ok=info == 0)


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
