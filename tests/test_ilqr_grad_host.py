"""CPU tests of the adjoint LQR behind differentiable_ilqr() (csrc/riccati.cuh's adjoint phases, built for the host by
tests/host_harness/ilqr_adjoint_host.cpp; DESIGN.md 4.5.1 "Gradients of the solution"): the Riccati pass plus the linear
rollout against a dense solve of H_SS w_S = G_S on random tick blocks, with n_z 13 and 17 (drag's rows of the clipped RPMs),
with no held set, several held sets, every rotor of a tick held and T = 1; negative controls that must miss (mu > 0, the held
set ignored, the g_X term dropped); the adjoint's K against the solve's backward pass at mu = 0 bit for bit; and the C ABI's
refusals of qs_ilqr_adjoint / qs_ilqr_adjoint_rollout without a GPU."""
import ctypes as C

import numpy as np
import pytest

from diff_testlib import params_of
from ilqr_grad_ref import dense_solve, host_adjoint
from test_ilqr_host import host_pass

TOL = 1e-10


def rel(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(np.asarray(b)), 1e-300))


def problem(nz, T, seed, clipped=None):
    """Random tick blocks F [T, nz, nz + 4] (with n_z 17 the augmented rows [0 | diag(cd)], rotor `clipped` with cd = 0), stage
    weights, Rt and cotangents of one drone.  A is scaled so that the horizon stays well conditioned."""
    rng = np.random.default_rng(seed)
    F = np.zeros((T, nz, nz + 4))
    F[:, :13, :nz] = 0.3 * rng.normal(size=(T, 13, nz))
    F[:, :13, nz:] = rng.normal(size=(T, 13, 4))
    if nz == 17:
        cd = np.ones(4)
        if clipped is not None:
            cd[clipped] = 0.0
        F[:, 13:, nz:] = np.diag(cd)
    W = rng.uniform(0.1, 2.0, size=(T, 13))
    Rt = rng.uniform(0.05, 0.5, size=4)
    gx, gu = rng.normal(size=(T, 13)), rng.normal(size=(T, 4))
    return F, W, Rt, gx, gu


def held_sets(T, rng):
    """None, a random held set, every rotor of tick 0 held, every rotor of the last tick held"""
    out = [None, rng.random((T, 4)) < 0.3]
    for t in (0, T - 1):
        h = np.zeros((T, 4), bool)
        h[t] = True
        out.append(h)
    return out


@pytest.mark.parametrize("nz", [13, 17])
@pytest.mark.parametrize("T", [1, 2, 12])
@pytest.mark.parametrize("seed", [0, 1])
def test_adjoint_equals_dense_solve(nz, T, seed):
    F, W, Rt, gx, gu = problem(nz, T, seed, clipped=1 if seed else None)
    for held in held_sets(T, np.random.default_rng(seed + 100)):
        rc, K, k, w, dz = host_adjoint(F, W, Rt, gx, gu, held)
        assert rc == 0
        w_ref, dx_ref = dense_solve(F, W, Rt, gx, gu, held)
        assert rel(w, w_ref) < TOL, (held, rel(w, w_ref))
        assert rel(dz[:, :13], dx_ref) < TOL
        if held is not None:
            assert np.all(w[held] == 0.0)                                 # held rotors: exactly zero
            assert np.all(K[held] == 0.0) and np.all(k[held] == 0.0)
        if nz == 17:                                                      # the augmented rows carry the clipped w
            assert np.array_equal(dz[:, 13:], w * F[:, 13:, 17:].diagonal(axis1=1, axis2=2))


@pytest.mark.parametrize("nz", [13, 17])
def test_negative_controls_miss(nz):
    T = 8
    F, W, Rt, gx, gu = problem(nz, T, 7)
    held = np.zeros((T, 4), bool)
    held[2, 1] = held[5] = True
    _, _, _, w, dz = host_adjoint(F, W, Rt, gx, gu, held)
    w_ref, _ = dense_solve(F, W, Rt, gx, gu, held)
    assert rel(w, w_ref) < TOL
    assert rel(w, dense_solve(F, W, Rt, gx, gu, held, mu=1e-3)[0]) > 1e3 * TOL        # mu > 0 is another derivative
    assert rel(w, dense_solve(F, W, Rt, gx, gu, None)[0]) > 1e3 * TOL                  # the held set matters
    _, _, _, w0, _ = host_adjoint(F, W, Rt, np.zeros_like(gx), gu, held)               # dropping g_X misses
    assert rel(w0, w_ref) > 1e3 * TOL


@pytest.mark.parametrize("nz", [13, 17])
def test_gains_are_the_backward_pass_at_mu_zero(nz):
    """Without a held set the adjoint's K is ih_backward_pass's K at mu = 0 bit for bit: K depends on the stage Hessians only"""
    T = 10
    F, W, Rt, gx, gu = problem(nz, T, 3)
    rng = np.random.default_rng(4)
    rc, K, _, _, _ = host_adjoint(F, W, Rt, gx, gu)
    rc2, K2, _, _, _, _ = host_pass(F, rng.normal(size=(T, 13)), W, Rt, rng.normal(size=(T, 4)), 0.0, np.zeros((nz, nz)),
                                   np.zeros(nz))
    assert rc == rc2 == 0
    assert np.array_equal(K, K2)


def test_failed_factor_is_reported():
    F, W, Rt, gx, gu = problem(13, 4, 5)
    rc, *_ = host_adjoint(F, W, np.array([0.1, np.nan, 0.1, 0.1]), gx, gu)
    assert rc == 4                                                        # the last tick, the first the pass factors


def test_abi_exports_struct_and_refusals():
    from gym_pybullet_drones_b200 import _native as N
    L = N.lib()
    for name in ("qs_ilqr_adjoint", "qs_ilqr_adjoint_rollout", "qs_sizeof_ilqr_adjoint_io"):
        assert name in N.EXPORTS
        getattr(L, name)
    assert L.qs_sizeof_ilqr_adjoint_io() == C.sizeof(N.QsIlqrAdjointIO) == 8 + 12 * 8
    P, _ = params_of("cf2x")
    buf = (C.c_double * 64)()
    a = C.addressof(buf)
    for f, outs in ((L.qs_ilqr_adjoint, ("g_states",)), (L.qs_ilqr_adjoint_rollout, ("w", "dx"))):
        io = N.QsIlqrAdjointIO()
        io.T = 2
        call = lambda io_, *args: f(C.byref(P), C.byref(io_), *args, None)
        assert f(None, C.byref(io), 1, 1, 1, 0, None) == -1
        assert f(C.byref(P), None, 1, 1, 1, 0, None) == -1
        for k in ("jac", "rpm", "weights", "K", "k", "status") + outs:
            assert call(io, 1, 1, 1, 0) == -1, k                          # each missing pointer is refused
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
        assert L.qs_last_error().startswith(f.__name__.encode() + b": ")
