"""CPU tests of the control-limited iLQR backward pass (csrc/riccati.cuh's box_qp, ric_gains_box and ric_col_K_box, built for
the host by tests/host_harness/ilqr_box_host.cpp; DESIGN.md 4.5.1):
  * the box QP alone against two independent float64 references (tests/ilqr_box_ref.py): exhaustive KKT enumeration of the 3^4
    active sets and scipy's BVLS on the Cholesky form, on random SPD matrices and boxes and on the edge cases (the minimiser
    inside the box, where the fast path must give chol4_neg_solve's bits; every dimension held; lo = hi; a minimiser on a face;
    an ill-conditioned H);
  * whole backward passes against the torch restatement, with a negative control that solves K with the full factor;
  * a pass whose bounds never bind, bit for bit the unconstrained host pass;
  * the C ABI of qs_ilqr_box_* and its refusals without a GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

import ilqr_box_ref as BR
from diff_testlib import params_of
from qs_testlib import harness

def _lib():
    L = harness("ilqr_box_host")
    for n in ("ih_box_solve", "ih_box_qp"):
        getattr(L, n).restype = C.c_int
        getattr(L, n).argtypes = [C.c_void_p] * 7
    L.ih_chol_solve.restype = C.c_int
    L.ih_chol_solve.argtypes = [C.c_void_p] * 3
    L.ih_box_backward_pass.restype = C.c_int
    L.ih_box_backward_pass.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 7 + [C.c_double] + [C.c_void_p] * 6
    return L


def _p(x):
    return x.ctypes.data_as(C.c_void_p)


def _f64(x):
    return np.ascontiguousarray(x, dtype=np.float64)


def box_solve(H, g, lo, hi, qp_only=False):
    """(rc, x, Lf [4, 4], act) of ih_box_solve (or ih_box_qp)"""
    H, g, lo, hi = (_f64(a) for a in (H, g, lo, hi))
    x, Lf, act = np.zeros(4), np.zeros(16), np.zeros(4, dtype=np.int32)
    f = _lib().ih_box_qp if qp_only else _lib().ih_box_solve
    rc = f(_p(H), _p(g), _p(lo), _p(hi), _p(x), _p(Lf), _p(act))
    return rc, x, Lf.reshape(4, 4), act


def host_box_pass(F, dx, W, Rt, du, lo, hi, mu, V, vx):
    """ih_box_backward_pass over F [T, nz, nz + 4]: (rc, K [T, 4, nz], k [T, 4], act [T, 4], V, vx, dV [2])"""
    T, nz = F.shape[0], F.shape[1]
    F, dx, W, Rt, du, lo, hi = (_f64(a) for a in (F, dx, W, Rt, du, lo, hi))
    V, vx = _f64(V).copy(), _f64(vx).copy()
    K, k, dV, act = np.zeros((T, 4, nz)), np.zeros((T, 4)), np.zeros(2), np.zeros((T, 4), dtype=np.int32)
    rc = _lib().ih_box_backward_pass(nz, T, _p(F), _p(dx), _p(W), _p(Rt), _p(du), _p(lo), _p(hi), mu, _p(V), _p(vx), _p(K), _p(k),
                                     _p(dV), _p(act))
    return rc, K, k, act, V, vx, dV


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def spd(rng, cond=1e3, scale=1.0):
    Q, _ = np.linalg.qr(rng.normal(size=(4, 4)))
    H = scale * (Q * np.exp(rng.uniform(0.0, np.log(cond), 4))) @ Q.T
    return 0.5 * (H + H.T)


def random_case(seed):
    """An SPD H (condition up to 1e4, scale 1e-9 .. 1e3: Quu in RPM^-2 units is tiny) and a box that contains 0, as the kernel's
    boxes of k do (the nominal lies in the box)"""
    rng = np.random.default_rng(seed)
    scale = 10.0 ** rng.uniform(-9, 3)
    H = spd(rng, 10.0 ** rng.uniform(0, 4), scale)
    x_unc = rng.normal(size=4) * 10.0 ** rng.uniform(-1, 3)
    g = -H @ x_unc
    lo = -np.abs(x_unc) * rng.uniform(0.0, 1.5, 4)
    hi = np.abs(x_unc) * rng.uniform(0.0, 1.5, 4)
    return H, g, lo, hi


def check_against_references(H, g, lo, hi, x, act, tol=1e-10):
    xe, ae = BR.kkt_enum(H, g, lo, hi)
    xb = BR.bvls(H, g, lo, hi)
    span = np.linalg.norm(np.maximum(np.abs(lo), np.abs(hi))) + 1e-300
    e_kkt, e_bvls = np.linalg.norm(x - xe) / span, np.linalg.norm(x - xb) / span
    assert np.all(lo <= x) and np.all(x <= hi)
    assert e_kkt <= tol, (e_kkt, x, xe)
    assert e_bvls <= 1e3 * tol, (e_bvls, x, xb)
    assert np.array_equal(act, ae), (act, ae)
    # the value: no reference point does better
    assert BR.qp_value(H, g, x) <= min(BR.qp_value(H, g, xe), BR.qp_value(H, g, xb)) + 1e-12 * abs(BR.qp_value(H, g, xe))
    return e_kkt, e_bvls


# ---- the QP alone -------------------------------------------------------------------------------------------------------------

def test_qp_random_cases_match_both_references():
    worst = [0.0, 0.0]
    held = 0
    for seed in range(300):
        H, g, lo, hi = random_case(seed)
        rc, x, Lf, act = box_solve(H, g, lo, hi)
        assert rc >= 0, seed
        e = check_against_references(H, g, lo, hi, x, act)
        worst = [max(worst[0], e[0]), max(worst[1], e[1])]
        held += int(np.any(act != 0))
        # K's factor: the free block's Cholesky factor embedded with identity on the held dimensions
        f = act == 0
        E = np.where(np.outer(f, f), H, np.eye(4))
        assert rel(np.tril(Lf) @ np.tril(Lf).T, E) <= 1e-12
    print("box QP, 300 random cases (%d with held dimensions): |x - kkt| / |box| <= %.1e, |x - bvls| / |box| <= %.1e"
          % (held, worst[0], worst[1]))
    assert held >= 150                                    # the cases exercise the QP, not only the fast path


def test_fast_path_gives_the_unconstrained_bits():
    rng = np.random.default_rng(7)
    for _ in range(50):
        H = spd(rng, 1e3, 1e-6)
        g = rng.normal(size=4) * 1e-6
        x_unc = np.zeros(4)
        assert _lib().ih_chol_solve(_p(_f64(H)), _p(_f64(g)), _p(x_unc)) == 0
        lo, hi = x_unc - np.abs(x_unc) * rng.uniform(0, 1, 4), x_unc + np.abs(x_unc) * rng.uniform(0, 1, 4)
        rc, x, Lf, act = box_solve(H, g, lo, hi)
        assert rc == 0 and np.array_equal(x, x_unc) and np.all(act == 0)
        # exactly on a face of the box: still inside, still the fast path
        lo2, hi2 = lo.copy(), hi.copy()
        lo2[0], hi2[3] = x_unc[0], x_unc[3]
        rc, x, _, act = box_solve(H, g, lo2, hi2)
        assert rc == 0 and np.array_equal(x, x_unc) and np.all(act == 0)


def test_every_dimension_held():
    # a diagonal H and the minimiser far outside a small box around 0: every gradient points out at the corner
    H = np.diag(np.diag(spd(np.random.default_rng(3), 1e2)))
    x_unc = np.array([5.0, -5.0, 5.0, -5.0])
    g = -H @ x_unc
    lo, hi = -np.ones(4), np.ones(4)
    rc, x, Lf, act = box_solve(H, g, lo, hi)
    assert rc >= 1
    assert np.array_equal(x, np.array([1.0, -1.0, 1.0, -1.0])) and np.array_equal(act, [1, -1, 1, -1])
    assert np.array_equal(Lf, np.eye(4))
    check_against_references(H, g, lo, hi, x, act)


def test_lo_equal_to_hi():
    rng = np.random.default_rng(4)
    for seed in range(20):
        H = spd(rng, 1e3)
        g = rng.normal(size=4)
        lo = rng.normal(size=4)
        hi = lo.copy()
        hi[1] = lo[1] + 1.0                                 # one free dimension, three pinned
        for l, h in ((lo, lo.copy()), (lo, hi)):
            rc, x, _, act = box_solve(H, g, l, h)
            assert rc >= 0
            assert np.all(x >= l) and np.all(x <= h)
            assert np.array_equal(x[h == l], l[h == l])      # a pinned dimension is its bound exactly
            xe, _ = BR.kkt_enum(H, g, l, h)
            assert np.linalg.norm(x - xe) <= 1e-10 * (np.linalg.norm(l) + 1.0)
            assert np.linalg.norm(x - BR.bvls(H, g, l, h)) <= 1e-8 * (np.linalg.norm(l) + 1.0)


def test_minimiser_on_a_face_with_a_zero_multiplier():
    """The constrained minimiser has x_0 = lo_0 with a zero gradient there (a degenerate face) and x_1 = hi_1 held"""
    rng = np.random.default_rng(5)
    ran = 0
    for _ in range(20):
        H = spd(rng, 1e2)
        xc = rng.normal(size=4)
        gr = np.array([0.0, -1.0, 0.0, 0.0])
        g = gr - H @ xc
        lo, hi = xc - rng.uniform(0.5, 1.0, 4), xc + rng.uniform(0.5, 1.0, 4)
        lo[0], hi[1] = xc[0], xc[1]
        lo = np.minimum(lo, 0.0)                             # keep 0 in the box, as the kernel's boxes
        hi = np.maximum(hi, 0.0)
        if lo[0] != xc[0] or hi[1] != xc[1]:
            continue
        rc, x, _, act = box_solve(H, g, lo, hi)
        assert rc >= 1
        assert np.linalg.norm(x - xc) <= 1e-10 * np.linalg.norm(xc)
        assert np.linalg.norm(x - BR.bvls(H, g, lo, hi)) <= 1e-7 * np.linalg.norm(xc)
        assert act[1] == 1 and act[2] == 0 and act[3] == 0
        ran += 1
    assert ran >= 5


@pytest.mark.parametrize("cond", [1e8, 1e12])
def test_ill_conditioned_H(cond):
    worst = 0.0
    for seed in range(40):
        rng = np.random.default_rng(100 + seed)
        H = spd(rng, 1.0, 1e-8)
        Q, _ = np.linalg.qr(rng.normal(size=(4, 4)))
        H = 1e-8 * (Q * np.array([1.0, 1.0, 1.0, 1.0 / cond])) @ Q.T
        H = 0.5 * (H + H.T)
        x_unc = rng.normal(size=4) * 100.0
        g = -H @ x_unc
        lo, hi = -np.abs(rng.normal(size=4)) * 50.0, np.abs(rng.normal(size=4)) * 50.0
        rc, x, _, act = box_solve(H, g, lo, hi)
        assert rc >= 0
        assert np.all(lo <= x) and np.all(x <= hi)
        xe, _ = BR.kkt_enum(H, g, lo, hi, tol=1e-6)
        fx, fe = BR.qp_value(H, g, x), BR.qp_value(H, g, xe)
        # an ill-conditioned H leaves x itself ill-determined along its weak direction: hold the value, not x
        worst = max(worst, (fx - fe) / abs(fe))
        assert fx <= fe + 1e-9 * abs(fe), (seed, fx, fe)
    print("ill-conditioned H (cond %.0e): worst relative value excess over the KKT point %.1e" % (cond, worst))


def test_not_positive_definite_is_a_failure():
    H = np.diag([1.0, 1.0, -1.0, 1.0])
    rc, *_ = box_solve(H, np.ones(4), -np.ones(4), np.ones(4))
    assert rc == -2                                        # the full factor, as ric_gains
    # box_qp alone: the free block fails only when a non-PD dimension is free
    rc, *_ = box_solve(H, np.array([1.0, 1.0, 0.5, 1.0]), -np.ones(4), np.ones(4), qp_only=True)
    assert rc == -1


# ---- whole backward passes ----------------------------------------------------------------------------------------------------

def _random_pass(nz, T, rng):
    F = np.zeros((T, nz, nz + 4))
    F[:, :13] = rng.normal(size=(T, 13, nz + 4)) * 0.3
    F[:, :13, :13] += np.eye(13)
    if nz == 17:
        F[:, 13:, 17:] = np.eye(4)
    G = rng.normal(size=(nz, nz))
    V = G @ G.T + np.eye(nz)
    vx = rng.normal(size=nz)
    dx, W = rng.normal(size=(T, 13)), rng.uniform(0.0, 2.0, (T, 13))
    Rt, du = rng.uniform(0.5, 2.0, 4), rng.normal(size=(T, 4))
    return F, dx, W, Rt, du, V, vx


@pytest.mark.parametrize("nz", [13, 17])
@pytest.mark.parametrize("mu", [0.0, 0.3])
def test_backward_pass_matches_restatement(nz, mu):
    rng = np.random.default_rng(nz + int(10 * mu))
    T = 6
    F, dx, W, Rt, du, V, vx = _random_pass(nz, T, rng)
    # first the unconstrained pass, to size boxes that bind at some ticks and not at others
    lo_w, hi_w = np.full((T, 4), -1e30), np.full((T, 4), 1e30)
    rc, _, k0, act0, *_ = host_box_pass(F, dx, W, Rt, du, lo_w, hi_w, mu, V, vx)
    assert rc == 0 and np.all(act0 == 0)
    lo, hi = -np.abs(k0) * rng.uniform(0.2, 2.0, (T, 4)), np.abs(k0) * rng.uniform(0.2, 2.0, (T, 4))
    rc, K, k, act, Vh, vxh, dV = host_box_pass(F, dx, W, Rt, du, lo, hi, mu, V, vx)
    assert rc == 0
    t = lambda x: torch.as_tensor(np.asarray(x, dtype=np.float64))
    r = BR.backward_pass_box(t(F), t(dx), t(W), t(Rt), t(du), t(lo), t(hi), mu, V=t(V), vx=t(vx))
    assert np.array_equal(act, r["act"].numpy())
    held = act != 0
    assert held.sum() >= 3 and (~held).sum() >= 3              # both kinds of rows occur
    errs = {"K": rel(K, r["K"]), "k": rel(k, r["k"]), "V": rel(Vh, r["V"]), "vx": rel(vxh, r["vx"]),
            "dV1": rel(dV[0], r["dV1"]), "dV2": rel(dV[1], r["dV2"])}
    print("box backward nz=%d mu=%g, %d of %d rotors held: %s" % (nz, mu, held.sum(), held.size,
                                                                  {k_: "%.1e" % v for k_, v in errs.items()}))
    for name, e in errs.items():
        assert e <= 1e-10, (name, e)
    assert np.all(K[held] == 0.0)                               # K's rows on held rotors
    assert np.all(k[act == -1] == lo[act == -1]) and np.all(k[act == 1] == hi[act == 1])
    assert np.array_equal(Vh, Vh.T)
    # the negative control: K from the full factor of Quu_mu misses
    bad = BR.backward_pass_box(t(F), t(dx), t(W), t(Rt), t(du), t(lo), t(hi), mu, V=t(V), vx=t(vx), full_factor_K=True)
    assert rel(K, bad["K"]) > 1e-3


@pytest.mark.parametrize("nz", [13, 17])
def test_bounds_that_never_bind_give_the_unconstrained_bits(nz):
    from test_ilqr_host import host_pass
    rng = np.random.default_rng(40 + nz)
    T = 8
    F, dx, W, Rt, du, V, vx = _random_pass(nz, T, rng)
    for mu in (0.0, 0.25):
        ref = host_pass(F, dx, W, Rt, du, mu, V, vx)
        assert ref[0] == 0
        k_ref = ref[2]
        lo, hi = -np.abs(k_ref) - 1.0, np.abs(k_ref) + 1.0
        lo[2], hi[5] = k_ref[2], k_ref[5]                          # on a face at two ticks: still the fast path
        rc, K, k, act, Vh, vxh, dV = host_box_pass(F, dx, W, Rt, du, lo, hi, mu, V, vx)
        assert rc == 0 and np.all(act == 0)
        for a, b in zip((K, k, Vh, vxh, dV), (ref[1], ref[2], ref[3], ref[4], ref[5])):
            assert np.array_equal(a, b)


# ---- the C ABI without a GPU ----------------------------------------------------------------------------------------------------

def test_box_abi_exports_struct_and_refusals():
    from gym_pybullet_drones_b200 import _native as N
    L = N.lib()
    for name in ("qs_ilqr_box_backward", "qs_ilqr_box_line_search", "qs_ilqr_box_commit", "qs_sizeof_ilqr_box_io"):
        assert name in N.EXPORTS
        getattr(L, name)
    assert L.qs_sizeof_ilqr_box_io() == C.sizeof(N.QsIlqrBoxIO) == C.sizeof(N.QsIlqrIO) + 4 * 8
    assert N.QsIlqrBoxIO.base.offset == 0
    P, _ = params_of("cf2x")
    buf = (C.c_double * 64)()
    a = C.addressof(buf)
    needs = [(L.qs_ilqr_box_backward, ("jac", "mu", "K", "k", "dV", "status")),
             (L.qs_ilqr_box_line_search, ("alpha", "J")),
             (L.qs_ilqr_box_commit, ("alpha", "J", "mu", "dV", "status", "converged", "cost_in", "cost_out"))]
    for f, outs in needs:
        io = N.QsIlqrBoxIO()
        io.base.T, io.base.n_alpha = 2, 1
        call = lambda *args: f(C.byref(P), C.byref(io), *args, None)
        name = f.__name__.encode()
        assert f(None, C.byref(io), 1, 1, 1, 0, None) == -1
        assert f(C.byref(P), None, 1, 1, 1, 0, None) == -1
        assert call(1, 1, 1, 0) == -1 and b"rpm_lo" in L.qs_last_error()       # NULL bounds
        io.rpm_lo = a
        assert call(1, 1, 1, 0) == -1 and b"rpm_hi" in L.qs_last_error()
        io.rpm_hi = a
        io.per_tick = 2
        assert call(1, 1, 1, 0) == -3 and b"per_tick" in L.qs_last_error()
        io.per_tick = 1
        assert call(1, 1, 1, 0) == -1                                              # today's refusals follow
        for k in ("state0", "rpm", "states", "targets", "weights", "rpm_ref"):
            setattr(io.base, k, a)
        for k in outs:
            assert call(1, 1, 1, 0) == -1, k
            assert L.qs_last_error().startswith(name + b": ")
            setattr(io.base, k, a)
        assert call(1, 1, 1, N.EFFECT_DW) == -5
        assert b"downwash" in L.qs_last_error() and L.qs_last_error().startswith(name + b": ")
        assert call(1, 1, 1, 8) == -4
        assert call(0, 1, 1, 0) == -3
        assert call(1, 0, 1, 0) == -3
        io.base.T = 0
        assert call(1, 1, 1, 0) == -3
        io.base.T = 2
        if f is not L.qs_ilqr_box_backward:
            io.base.n_alpha = 17
            assert call(1, 1, 1, 0) == -3
            io.base.n_alpha = 1
