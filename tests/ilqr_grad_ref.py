"""Float64 restatements of the derivative of an iLQR solution (DESIGN.md 4.5.1 "Gradients of the solution") for the tests:
the dense Gauss-Newton system of one drone (H_SS w_S = G_S from the tick blocks F = [A | B]) and the host harness of the adjoint
kernels (tests/host_harness/ilqr_adjoint_host.cpp).  Test infrastructure."""
import ctypes as C

import numpy as np

from qs_testlib import harness


def dense_jacobian(F):
    """J [T, 13, T, 4]: d x_t / d w_s of dz_{t+1} = F_t [dz_t; w_t] from dz_0 = 0 (x_t the first 13 entries of dz_{t+1})."""
    T, nz = F.shape[0], F.shape[1]
    Z = np.zeros((T, nz, T, 4))                       # dz_{t+1} / dw_s
    prev = np.zeros((nz, T, 4))
    for t in range(T):
        A, B = F[t, :, :nz], F[t, :, nz:]
        cur = np.einsum("ab,bsj->asj", A, prev)
        cur[:, t, :] += B
        Z[t] = cur
        prev = cur
    return Z[:, :13]


def dense_solve(F, W, Rt, gx, gu, held=None, mu=0.0):
    """(w [T, 4], dx [T, 13]) of H_SS w_S = G_S, H = J'diag(W)J + Rt (+ mu diag(H) as a negative control), G = gu + J'gx, w = 0
    on held rotor-ticks (held [T, 4] bool)."""
    T = F.shape[0]
    J = dense_jacobian(F).reshape(T * 13, T * 4)
    H = J.T @ (W.reshape(-1)[:, None] * J) + np.diag(np.tile(Rt, T))
    H = H + mu * np.diag(np.diag(H))
    G = gu.reshape(-1) + J.T @ gx.reshape(-1)
    free = np.ones(T * 4, bool) if held is None else ~np.asarray(held, bool).reshape(-1)
    w = np.zeros(T * 4)
    w[free] = np.linalg.solve(H[np.ix_(free, free)], G[free])
    return w.reshape(T, 4), (J @ w).reshape(T, 13)


def _lib():
    L = harness("ilqr_adjoint_host")
    L.ih_adjoint_pass.restype = C.c_int
    L.ih_adjoint_pass.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 8
    L.ih_adjoint_rollout.restype = None
    L.ih_adjoint_rollout.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 6
    return L


def host_adjoint(F, W, Rt, gx, gu, held=None):
    """The host build of qs_ilqr_adjoint + qs_ilqr_adjoint_rollout for one drone: (rc, K [T, 4, nz], k [T, 4], w [T, 4],
    dz [T, nz])."""
    T, nz = F.shape[0], F.shape[1]
    a = lambda x: np.ascontiguousarray(x, dtype=np.float64)
    F, W, Rt, gx, gu = (a(x) for x in (F, W, Rt, gx, gu))
    act = None if held is None else np.ascontiguousarray(np.asarray(held) != 0, dtype=np.int32)
    K, k, w, dz = np.zeros((T, 4, nz)), np.zeros((T, 4)), np.zeros((T, 4)), np.zeros((T, nz))
    p = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)
    L = _lib()
    rc = L.ih_adjoint_pass(nz, T, p(F), p(W), p(Rt), p(gx), p(gu), p(act), p(K), p(k))
    if rc == 0:
        L.ih_adjoint_rollout(nz, T, p(F), p(K), p(k), p(act), p(w), p(dz))
    return rc, K, k, w, dz

