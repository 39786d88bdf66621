"""CPU tests of the iLQR backward pass (csrc/riccati.cuh, built for the host by tests/host_harness/ilqr_host.cpp; DESIGN.md 4.5.1):
one tick against the float64 restatement tests/ilqr_ref.py for n_z = 13 and 17, a long pass with constant (A, B) from the hover
Jacobian of the reference dynamics against the discrete algebraic Riccati equation, the stage cost, a Cholesky failure, and the
C ABI's refusals of qs_ilqr_backward / qs_ilqr_line_search / qs_ilqr_commit without a GPU.  Also the restatements the device tests
use (ilqr_ref.commit, mu_ladder, rollout_cost, tick_jac) on hand-worked cases, and the host build on adversarial inputs: a
subnormal and a zero pivot, an overflowing Quu, every rotor clipped."""
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


# ---- H4: the commit rule, the restart ladder and J(alpha) of the restatement --------------------------------------------------

def test_commit_rule_by_hand():
    nan, inf = float("nan"), float("inf")
    al = [1.0, 0.5, 0.25]
    # the largest accepted alpha wins, not the first; unsorted alpha
    assert IR.commit([0.25, 1.0, 0.5], [9.0, 9.5, 8.0], 10.0, -1.0, 0.0, 0.0, 0, False)[0] == 1
    assert IR.commit([0.25, 1.0, 0.5], [9.0, 9.5, 8.0], 10.0, -1.0, 0.0, 0.0, 0, False, first_accepted=True)[0] == 0
    # a tie between equal alpha: the first index
    assert IR.commit([0.5, 0.5, 0.25], [9.0, 8.0, 7.0], 10.0, -1.0, 0.0, 0.0, 0, False)[0] == 0
    # NaN and +inf J are never accepted; with Jn = +inf only a finite J passes Ja < Jn
    assert IR.commit(al, [nan, inf, 9.0], 10.0, -1.0, 0.0, 0.0, 0, False)[0] == 2
    assert IR.commit(al, [nan, inf, nan], 10.0, -1.0, 0.0, 0.0, 0, False) == (-1, 1e-6, False)
    assert IR.commit(al, [inf, inf, inf], inf, -1.0, 0.0, 0.0, 0, False)[0] == -1
    assert IR.commit(al, [inf, 5.0, inf], inf, -1.0, 0.0, 0.0, 0, False)[0] == 1
    # Ja == Jn is rejected; Armijo at equality is accepted, one ulp short is not
    assert IR.commit([1.0], [10.0], 10.0, 0.0, 0.0, 0.0, 0, False)[0] == -1
    exp = 1e-4 * -(1.0 * -1e4 + 1.0 * 1.0 * 0.0)                 # 1.0 exactly
    assert IR.commit([1.0], [10.0 - exp], 10.0, -1e4, 0.0, 0.0, 0, False)[0] == 0
    assert IR.commit([1.0], [np.nextafter(10.0 - exp, inf)], 10.0, -1e4, 0.0, 0.0, 0, False)[0] == -1
    # a negative dV2 raises the bar: the expected decrease of alpha = 1 is -(dV1 + dV2)
    assert IR.commit([1.0], [9.99], 10.0, -1.0, -100.0, 0.0, 0, False)[0] == -1
    # mu: /10 and 0 below 1e-6 on acceptance, max(1e-6, 10 mu) on rejection
    acc = lambda mu: IR.commit([1.0], [5.0], 10.0, -1.0, 0.0, mu, 0, False)[1]
    rej = lambda mu: IR.commit([1.0], [11.0], 10.0, -1.0, 0.0, mu, 0, False)[1]
    assert acc(1e-5) == 1.0000000000000002e-06 and acc(9.999999999999999e-06) == 1e-6 and acc(1e-6) == 0.0 and acc(0.0) == 0.0
    assert acc(9.99999999999999e-06) == 0.0                       # 9.99999999999999e-07 < 1e-6
    assert rej(0.0) == 1e-6 and rej(1e-5) == 1e-4 and rej(9.999999999999999e-06) == 9.999999999999999e-05 and rej(1e-8) == 1e-6
    # converged: Jn - Jc < 1e-9 Jn, strictly
    Jn = 1.0
    Jc = IR.converged_boundary(Jn)
    assert Jn - Jc == 1e-9 * Jn or Jn - Jc > 1e-9 * Jn > Jn - np.nextafter(Jc, inf)
    assert IR.commit([1.0], [Jc], Jn, 0.0, 0.0, 0.0, 0, False) == (0, 0.0, False)
    assert IR.commit([1.0], [np.nextafter(Jc, inf)], Jn, 0.0, 0.0, 0.0, 0, False) == (0, 0.0, True)
    # status 1 and converged drones are never accepted; a converged drone keeps its mu
    assert IR.commit([1.0], [5.0], 10.0, -1.0, 0.0, 0.5, 1, False) == (-1, 5.0, False)
    assert IR.commit([1.0], [5.0], 10.0, -1.0, 0.0, 0.5, 0, True) == (-1, 0.5, True)


def test_mu_ladder():
    assert IR.mu_ladder(0.0, 0.0) == (0.0, 0)
    assert IR.mu_ladder(0.0, 5e-6) == (9.999999999999999e-06, 0)
    assert IR.mu_ladder(0.0, 5e-4) == (0.001, 0)
    assert IR.mu_ladder(0.0, lambda m: False) == (100.0, 1)
    assert IR.mu_ladder(0.37, 2.0) == (3.7, 0)
    assert IR.mu_ladder(0.37, lambda m: False)[1] == 1


def _drag_problem(T=12, B=6, seed=0, model="cf2x"):
    """A drag rollout whose nominal clips rotors at 0 and at MAX_RPM on some drones and ticks."""
    import diff_ref as DR
    from diff_testlib import aviary_rows
    P, c = params_of(model, 240, 48)
    rng = np.random.default_rng(seed)
    _, rows = aviary_rows(model, B, rng)
    hover, mx = rows[:, 12:13], rows[:, 13:14]
    rpm = hover * (1 + 0.05 * torch.as_tensor(rng.uniform(-1, 1, (T, B, 4))))
    rpm[3, 0, 1] = -50.0                                          # drone 0: a rotor below 0
    rpm[5, 1, 2] = mx[1, 0] * 1.01                               # drone 1: a rotor beyond MAX_RPM
    x0 = torch.zeros((B, 13), dtype=torch.float64)
    x0[:, 2], x0[:, 6] = 1.0, 1.0
    last = hover.expand(B, 4).clone()
    K_dyn = DR.model_constants(P)
    eff = DR.EFFECT_DRAG
    S = 5
    states = DR.rollout(K_dyn, rows, x0, rpm, last, S, eff)
    W = torch.as_tensor(rng.uniform(0.1, 2.0, (T, B, 13)))
    tg = torch.as_tensor(rng.normal(size=(T, B, 13))) * 0.1
    Rt = torch.as_tensor(rng.uniform(0.5, 2.0, (B, 4))) * 1e-2 / hover ** 2
    uref = hover.expand(B, 4) * 1.001
    return dict(K_dyn=K_dyn, rows=rows, x0=x0, last_rpm=last, rpm_nom=rpm, states_nom=states, targets=tg, W=W, Rt=Rt, uref=uref, S=S,
                effects=eff), rng


def test_rollout_cost_at_alpha_zero_is_the_nominal_cost():
    import diff_ref as DR
    a, rng = _drag_problem()
    T, B = a["rpm_nom"].shape[:2]
    want = IR.cost(a["states_nom"], a["targets"], a["W"], a["rpm_nom"], a["uref"], a["Rt"])
    for eff in (0, DR.EFFECT_DRAG):
        b = dict(a, effects=eff, states_nom=DR.rollout(a["K_dyn"], a["rows"], a["x0"], a["rpm_nom"], a["last_rpm"], a["S"], eff))
        r = IR.rollout_cost(Kfb=None, kff=None, alpha=0.0, **b)
        assert torch.equal(r["x"], b["states_nom"]) and torch.equal(r["u"], b["rpm_nom"])
        w = IR.cost(b["states_nom"], b["targets"], b["W"], b["rpm_nom"], b["uref"], b["Rt"])
        assert torch.equal(r["J"], w)
    # with gains at alpha = 0 the rollout reproduces the nominal (dz = 0 exactly) ...
    Kfb = torch.as_tensor(rng.normal(size=(T, B, 4, 17))) * 1e2
    kff = torch.as_tensor(rng.normal(size=(T, B, 4)))
    r = IR.rollout_cost(Kfb=Kfb, kff=kff, alpha=0.0, **a)
    assert torch.equal(r["J"], want)
    # ... unless the nominal's previous RPMs are taken unclipped: that changes J only on the drones whose nominal clips a rotor
    # (drones 0 and 1) before the last tick
    bad = IR.rollout_cost(Kfb=Kfb, kff=kff, alpha=0.0, drag_prev_raw=True, **a)
    changed = bad["J"] != want
    print("drag_prev_raw at alpha = 0: relative change %s" % ((bad["J"] - want).abs() / want).tolist())
    assert changed.tolist() == [True, True] + [False] * (B - 2)
    assert ((bad["J"] - want).abs() / want)[:2].min() > 1e-6
    # alpha moves J, and a per-drone alpha is the same as one alpha at a time
    al = torch.tensor([1.0, 0.5, 0.25, 0.0, 1.0, 0.125], dtype=torch.float64)
    rb = IR.rollout_cost(Kfb=Kfb, kff=kff, alpha=al, **a)
    for i in (0, 2, 3):
        one = IR.rollout_cost(Kfb=Kfb, kff=kff, alpha=float(al[i]), **a)
        assert torch.equal(one["J"][i], rb["J"][i])
    assert torch.equal(rb["J"][3], want[3]) and (rb["J"][0] != want[0])


# ---- H5: the host build of the backward pass on adversarial inputs ------------------------------------------------------------

def _adversarial(nz, seed, T=3, clipped=2):
    rng = np.random.default_rng(seed)
    F = np.concatenate([_random_tick(nz, rng, clipped) for _ in range(T)])
    F[:, :, nz + clipped] = 0.0                                   # the clipped rotor's B column is 0 (with drag too)
    dx, W = rng.normal(size=(T, 13)), rng.uniform(0.5, 2.0, (T, 13))
    Rt, du = rng.uniform(0.5, 2.0, 4), rng.normal(size=(T, 4))
    return F, dx, W, Rt, du


def _ref_pass(F, dx, W, Rt, du, mu):
    t = lambda x: torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float64)
    return IR.backward_pass(t(F), t(dx), t(W), t(Rt), t(du), mu)


@pytest.mark.parametrize("nz", [13, 17])
def test_backward_subnormal_and_zero_pivot(nz):
    F, dx, W, Rt, du = _adversarial(nz, 20 + nz)
    zero = np.zeros((nz, nz)), np.zeros(nz)
    # the smallest subnormal Rt on the clipped rotor (its B column is 0): the pivot is positive, the pass goes through
    Rt[2] = 5e-324
    rc, K, k, V, vx, dV = host_pass(F, dx, W, Rt, du, 0.0, *zero)
    r = _ref_pass(F, dx, W, Rt, du, 0.0)
    assert rc == 0 and bool(r["ok"])
    eK, ek = rel(K, r["K"]), rel(k, r["k"])
    print("subnormal Rt nz=%d: K %.1e k %.1e, k of the clipped rotor %s" % (nz, eK, ek, k[:, 2]))
    assert eK <= 1e-12 and ek <= 1e-12 and np.all(K[:, 2] == 0.0)
    # Rt = 0 there: a pivot exactly 0 at the one tick whose B column is 0; the return code names that tick
    Rt[2] = 0.0
    F2 = F.copy()
    for t in (0, 2):                                              # ticks 0 and 2 drive rotor 2 ...
        F2[t, :13, nz + 2] = np.random.default_rng(t).normal(size=13)
        if nz == 17:
            F2[t, 15, nz + 2] = 1.0
    rc = host_pass(F2, dx, W, Rt, du, 0.0, *zero)[0]
    r = _ref_pass(F2, dx, W, Rt, du, 0.0)
    assert rc == 2 and not bool(r["ok"])                          # ... tick 1 does not: 1 + 1
    assert host_pass(F2, dx, W, Rt, du, 0.5, *zero)[0] == 2        # mu diag(Quu) scales a zero pivot to zero


@pytest.mark.parametrize("nz", [13, 17])
def test_backward_overflowing_quu_is_rejected(nz):
    F, dx, W, Rt, du = _adversarial(nz, 30 + nz)
    zero = np.zeros((nz, nz)), np.zeros(nz)
    W[:] = 1e300
    F[:, :13, nz + 1] *= 1e5                                      # rotor 1: Quu_11 = +inf, every other entry finite
    rc = host_pass(F, dx, W, Rt, du, 0.0, *zero)[0]
    t = lambda x: torch.as_tensor(x, dtype=torch.float64)
    V, vx = IR.stage(t(zero[0]), t(zero[1]), t(dx[2]), t(W[2]))
    r = IR.backward_tick(t(F[2]), V, vx, t(Rt), t(du[2]), 0.0)
    B = t(F[2])[:, nz:]
    Quu = torch.diag(t(Rt)) + B.T @ V @ B
    print("overflow nz=%d: Quu diagonal %s" % (nz, torch.diagonal(Quu).tolist()))
    assert torch.isinf(Quu[1, 1]) and torch.isfinite(Quu[0]).all() and torch.isfinite(Quu[2:, 2:]).all()
    assert rc == 3 and not bool(r["ok"])                          # s = +inf fails s < INFINITY at t = T - 1
    F[:, :13, nz + 1] /= 1e5
    assert host_pass(F, dx, W, Rt, du, 0.0, *zero)[0] == 0


@pytest.mark.parametrize("nz", [13, 17])
def test_backward_all_rotors_clipped(nz):
    F, dx, W, Rt, du = _adversarial(nz, 40 + nz)
    F[:, :, nz:] = 0.0                                            # B = 0: no rotor reaches the state
    zero = np.zeros((nz, nz)), np.zeros(nz)
    rc, K, k, V, vx, dV = host_pass(F, dx, W, Rt, du, 0.3, *zero)
    r = _ref_pass(F, dx, W, Rt, du, 0.3)
    assert rc == 0 and bool(r["ok"])
    assert np.all(K == 0.0)
    ek, eV = rel(k, r["k"]), rel(V, r["V"])
    print("all rotors clipped nz=%d: k %.1e V %.1e" % (nz, ek, eV))
    assert ek <= 1e-15 and eV <= 1e-12
    assert rel(k, -du / 1.3) <= 1e-15                            # Quu = diag(Rt), Quu_mu = 1.3 Quu, Qu = Rt du


def test_tick_jac_is_jacfwd():
    import diff_ref as DR
    from diff_testlib import aviary_rows
    P, _ = params_of("cf2p", 240, 48)
    rng = np.random.default_rng(5)
    _, rows = aviary_rows("cf2p", 3, rng)
    x = torch.as_tensor(rng.normal(size=(3, 13))) * 0.1
    x[:, 2] += 0.05
    x[:, 6] += 1.0
    raw = rows[:, 12:13] * (1 + 0.2 * torch.as_tensor(rng.uniform(-1, 1, (3, 4))))
    raw[0, 1], raw[1, 2] = -1.0, rows[1, 13] * 1.5                # a rotor clipped at 0 and one at MAX_RPM
    up = raw.clamp(min=0.0) * 0.9
    for eff in (0, DR.EFFECT_GND | DR.EFFECT_DRAG):
        got = IR.tick_jac(DR.model_constants(P), rows, x, raw, up, 5, eff)
        want = ref_tick_jac(P, eff, 5, x.numpy(), raw.numpy(), up.numpy(), rows.numpy())
        w = np.concatenate([want["state"], want["rpm"]] + ([want["up"]] if eff & DR.EFFECT_DRAG else []), axis=-1)
        assert rel(got.numpy(), w) <= 1e-15
        assert np.all(got[0, :, 14].numpy() == 0.0) and np.all(got[1, :, 15].numpy() == 0.0)
