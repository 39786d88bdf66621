"""CPU tests of the iLQR backward pass (csrc/riccati.cuh, built for the host by tests/host_harness/ilqr_host.cpp; DESIGN.md 4.5.1):
one tick against the float64 restatement tests/ilqr_ref.py for n_z = 13 and 17, a long pass with constant (A, B) from the hover
Jacobian of the reference dynamics against the discrete algebraic Riccati equation, the stage cost, a Cholesky failure, and the
C ABI's refusals of qs_ilqr_backward / qs_ilqr_line_search / qs_ilqr_commit without a GPU."""
import ctypes as C

import numpy as np
import pytest
import scipy.linalg
import torch

import ilqr_ref as IR
from diff_testlib import params_of
from jvp_testlib import ref_tick_jac
from qs_testlib import harness

def _lib():
    L = harness("ilqr_host")
    L.ih_backward_pass.restype = C.c_int
    L.ih_backward_pass.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 5 + [C.c_double] + [C.c_void_p] * 5
    L.ih_stage_cost.restype = C.c_double
    L.ih_stage_cost.argtypes = [C.c_void_p] * 6
    return L


def host_pass(F, dx, W, Rt, du, mu, V, vx):
    """ih_backward_pass over F [T, nz, nz + 4]: (rc, K [T, 4, nz], k [T, 4], V, vx, dV [2])."""
    T, nz = F.shape[0], F.shape[1]
    a = lambda x: np.ascontiguousarray(x, dtype=np.float64)
    F, dx, W, Rt, du, V, vx = (a(x) for x in (F, dx, W, Rt, du, V, vx))
    V, vx = V.copy(), vx.copy()
    K, k, dV = np.zeros((T, 4, nz)), np.zeros((T, 4)), np.zeros(2)
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    rc = _lib().ih_backward_pass(nz, T, p(F), p(dx), p(W), p(Rt), p(du), mu, p(V), p(vx), p(K), p(k), p(dV))
    return rc, K, k, V, vx, dV


def rel(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(np.asarray(b)), 1e-300))


def _random_tick(nz, rng, clipped=1):
    """F [1, nz, nz + 4] with random A and B; with n_z = 17 the augmented rows [0 | diag(cd)], rotor `clipped` with cd = 0."""
    F = np.zeros((1, nz, nz + 4))
    F[0, :13] = rng.normal(size=(13, nz + 4))
    if nz == 17:
        cd = np.ones(4)
        cd[clipped] = 0.0
        F[0, 13:, 17:] = np.diag(cd)
    else:
        F[0, :, 13 + clipped] = 0.0                      # a clipped rotor: its B column is zero
    return F


# ---- H1: one tick against the restatement -----------------------------------------------------------------------------------

@pytest.mark.parametrize("nz", [13, 17])
@pytest.mark.parametrize("mu", [0.0, 0.3])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_backward_tick_matches_restatement(nz, mu, seed):
    rng = np.random.default_rng(seed * 10 + nz)
    F = _random_tick(nz, rng)
    G = rng.normal(size=(nz, nz))
    V = G @ G.T + np.eye(nz)
    vx = rng.normal(size=nz)
    dx, W = rng.normal(size=(1, 13)), rng.uniform(0.0, 2.0, (1, 13))
    Rt, du = rng.uniform(0.5, 2.0, 4), rng.normal(size=(1, 4))
    rc, K, k, Vh, vxh, dV = host_pass(F, dx, W, Rt, du, mu, V, vx)
    assert rc == 0
    t = lambda x: torch.as_tensor(x, dtype=torch.float64)
    r = IR.backward_pass(t(F), t(dx), t(W), t(Rt), t(du), mu, V=t(V), vx=t(vx))
    errs = {"K": rel(K, r["K"]), "k": rel(k, r["k"]), "V": rel(Vh, r["V"]), "vx": rel(vxh, r["vx"]),
            "dV1": rel(dV[0], r["dV1"]), "dV2": rel(dV[1], r["dV2"])}
    print("backward tick nz=%d mu=%g: %s" % (nz, mu, {k: "%.1e" % v for k, v in errs.items()}))
    for name, e in errs.items():
        assert e <= 1e-12, (name, e)
    assert np.array_equal(Vh, Vh.T)                          # symmetrised
    assert np.all(K[0, 1] == 0.0) if nz == 13 else True      # no gain on a clipped rotor without drag
    # the negative control: the regularised Quu in the value update is a different recursion when mu > 0
    bad = IR.backward_pass(t(F), t(dx), t(W), t(Rt), t(du), mu, V=t(V), vx=t(vx), regularised_value=True)
    assert (rel(Vh, bad["V"]) > 1e-6) == (mu > 0)


# ---- H2: the discrete algebraic Riccati equation ----------------------------------------------------------------------------

def _hover_AB(model="cf2x", S=5):
    """A [13, 13], B [13, 4] of one tick at hover (pyb 240 Hz, S substeps per tick) by jacfwd of the reference dynamics."""
    P, c = params_of(model, 240, 240 // S)
    from diff_testlib import aviary_rows
    _, rows = aviary_rows(model, 1, np.random.default_rng(0))
    rows = rows.numpy()
    state = np.zeros((1, 13))
    state[0, 2], state[0, 6] = 1.0, 1.0
    raw = np.full((1, 4), rows[0, 12])
    jac = ref_tick_jac(P, 0, S, state, raw, np.zeros((1, 4)), rows)
    return jac["state"][0], jac["rpm"][0], rows[0, 12]


def test_long_pass_solves_the_dare():
    A, B, hover = _hover_AB()
    q = np.array([1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.1, 0.1, 0.1, 0.01, 0.01, 0.01])
    Rt = np.full(4, 1e-2) / hover ** 2
    T = 3000
    F = np.broadcast_to(np.concatenate([A, B], 1), (T, 13, 17))
    rc, K, k, V, vx, dV = host_pass(F, np.zeros((T, 13)), np.broadcast_to(q, (T, 13)), Rt, np.zeros((T, 4)), 0.0, np.zeros((13, 13)),
                                    np.zeros(13))
    assert rc == 0
    X = scipy.linalg.solve_discrete_are(A, B, np.diag(q), np.diag(Rt))
    K_dare = -np.linalg.solve(np.diag(Rt) + B.T @ X @ B, B.T @ X @ A)
    eV, eK = rel(V + np.diag(q), X), rel(K[0], K_dare)
    print("DARE: V_0 + Q %.1e, K_0 %.1e; rho(A + B K_0) = %.4f" % (eV, eK, max(abs(np.linalg.eigvals(A + B @ K[0])))))
    assert eV <= 1e-8 and eK <= 1e-8
    assert max(abs(np.linalg.eigvals(A + B @ K[0]))) < 1.0
    assert np.all(k == 0.0) and np.all(vx == 0.0)             # at the target with du = 0 there is nothing to feed forward
    # the negative control: a short pass has not reached the fixed point
    rc, K5, _, V5, _, _ = host_pass(F[:5], np.zeros((5, 13)), np.broadcast_to(q, (5, 13)), Rt, np.zeros((5, 4)), 0.0,
                                    np.zeros((13, 13)), np.zeros(13))
    assert rel(V5 + np.diag(q), X) > 1e-3 and rel(K5[0], K_dare) > 1e-3


# ---- H3: the stage cost, a failed factorisation, the ABI's refusals ---------------------------------------------------------

def test_stage_cost():
    rng = np.random.default_rng(3)
    x, ref, W, u, uref, Rt = (rng.normal(size=s) for s in (13, 13, 13, 4, 4, 4))
    W, Rt = np.abs(W), np.abs(Rt)
    p = lambda a: np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)
    got = _lib().ih_stage_cost(p(x), p(ref), p(W), p(u), p(uref), p(Rt))
    assert got == pytest.approx(0.5 * (W @ (x - ref) ** 2 + Rt @ (u - uref) ** 2), rel=1e-15)


@pytest.mark.parametrize("nz", [13, 17])
def test_indefinite_quu_fails_the_factorisation(nz):
    rng = np.random.default_rng(4)
    F = np.repeat(_random_tick(nz, rng), 3, axis=0)
    Rt = np.array([1.0, 1.0, -1e6, 1.0])                       # Quu indefinite at every tick
    args = (F, np.zeros((3, 13)), np.ones((3, 13)), Rt, np.zeros((3, 4)))
    rc = host_pass(*args, 0.0, np.zeros((nz, nz)), np.zeros(nz))[0]
    assert rc == 3                                            # the first tick of the pass, t = T - 1
    assert host_pass(F, args[1], args[2], np.ones(4), args[4], 0.0, np.zeros((nz, nz)), np.zeros(nz))[0] == 0


def test_abi_exports_struct_and_refusals():
    from gym_pybullet_drones_b200 import _native as N
    L = N.lib()
    for name in ("qs_ilqr_backward", "qs_ilqr_line_search", "qs_ilqr_commit", "qs_sizeof_ilqr_io"):
        assert name in N.EXPORTS
        getattr(L, name)
    assert L.qs_sizeof_ilqr_io() == C.sizeof(N.QsIlqrIO) == 8 + 19 * 8
    P, _ = params_of("cf2x")
    buf = (C.c_double * 64)()
    a = C.addressof(buf)
    needs = [(L.qs_ilqr_backward, ("jac", "mu", "K", "k", "dV", "status")),
             (L.qs_ilqr_line_search, ("alpha", "J")),
             (L.qs_ilqr_commit, ("alpha", "J", "mu", "dV", "status", "converged", "cost_in", "cost_out"))]
    for f, outs in needs:
        io = N.QsIlqrIO()
        io.T, io.n_alpha = 2, 1
        call = lambda io_, *args: f(C.byref(P), C.byref(io_), *args, None)
        assert f(None, C.byref(io), 1, 1, 1, 0, None) == -1
        assert f(C.byref(P), None, 1, 1, 1, 0, None) == -1
        assert call(io, 1, 1, 1, 0) == -1
        for k in ("state0", "rpm", "states", "targets", "weights", "rpm_ref"):
            setattr(io, k, a)
        for k in outs:
            assert call(io, 1, 1, 1, 0) == -1, k                  # each missing pointer is refused
            assert L.qs_last_error().startswith(f.__name__.encode() + b": ")
            setattr(io, k, a)
        assert call(io, 1, 1, 1, N.EFFECT_DW) == -5
        assert b"downwash" in L.qs_last_error() and L.qs_last_error().startswith(f.__name__.encode() + b": ")
        assert call(io, 1, 1, 1, 8) == -4
        assert call(io, 0, 1, 1, 0) == -3
        assert call(io, 1, 0, 1, 0) == -3
        assert call(io, 1, 1, 0, 0) == -3
        assert call(io, 65536, 65536, 1, 0) == -3
        io.T = 0
        assert call(io, 1, 1, 1, 0) == -3
        io.T = 1
        if f is not L.qs_ilqr_backward:
            for na in (0, 17):
                io.n_alpha = na
                assert call(io, 1, 1, 1, 0) == -3
                assert b"n_alpha" in L.qs_last_error()
            io.n_alpha = 1
        io.phys = a + 8
        assert call(io, 1, 1, 1, 0) == -2
