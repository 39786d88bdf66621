"""-m gpu: the iLQR kernels (ilqr_backward_kernel / ilqr_line_search_kernel / ilqr_commit_kernel, DESIGN.md 4.5.1) on the device
against float64 references at every decision of the backward pass, the line search and the commit.

E1  the backward pass bit for bit the host build of riccati.cuh (tests/host_harness/ilqr_host.cpp) on synthetic Jacobians:
    random dense F, nominal RPMs at 0, at MAX_RPM and one ulp outside each, a clipped rotor with a subnormal Rt, T = 1 and 240,
    4k + 1..3 drones (idle warps in the last CTA); and within 1e-10 of ilqr_ref.backward_pass.  The RPM edges reach the clip's
    derivative only with drag and only before the last tick: at tick 0 and T / 2 with T = 240, where flipping it changes K.
E2  the restart ladder: drones that need 0, 1, 3 and 8 restarts and one that fails 9 times, the indefinite tick last, in the
    middle and first, incoming mu 0 and 0.37: mu and status equal ilqr_ref.mu_ladder, K, k and dV the host build at that mu.
E3  J(alpha) against ilqr_ref.rollout_cost at the device's nominal and gains, per-aviary weights, targets with a time axis, a
    per-aviary phys table, RPMs clipped at 0 and MAX_RPM; the committed rpm and trajectory; the backward at forward-mode
    Jacobians of diff_ref.tick; four negative controls.
E4  the commit rule exact at each predicate's boundary and one ulp either side, against ilqr_ref.commit.
E5  six whole iterations teacher-forced on the device's nominal: the chosen alpha, mu and converged against the references.
E6  converged, failed (status 1) and zero-cost drones over 40 iterations.
E7  one iteration at 65 536 drones with drag, drones either side of every CTA boundary against E3's references."""
import time

import numpy as np
import pytest
import torch

import diff_ref as DR
import ilqr_ref as IR
from test_gpu_ilqr import _env, _vec
from test_ilqr_host import host_pass

pytestmark = pytest.mark.gpu

DEV = "cuda"
F64 = dict(dtype=torch.float64, device=DEV)


def _problem(env, T, rng, phys=None, alphas=None, rpm=None, hetero=True, **kw):
    """A Problem with per-aviary Q, Q_final, R, rpm_ref, a [T, E, D, k] target for every key, a non-zero last_rpm and `phys`."""
    from gym_pybullet_drones_b200.ilqr import ALPHAS, Problem
    E, D = env._E, env._D
    t = lambda a: torch.as_tensor(a, **F64)
    hover = env.HOVER_RPM
    if hetero:
        target = {"pos": t(rng.uniform(-0.5, 0.5, (T, E, D, 3)) + np.array([0.0, 0.0, 1.0])),
                  "quat": t(np.tile([0.0, 0.0, 0.0, 1.0], (T, E, D, 1)) + rng.uniform(-0.05, 0.05, (T, E, D, 4))),
                  "vel": t(rng.uniform(-0.3, 0.3, (T, E, D, 3))), "rpy_rates": t(rng.uniform(-0.3, 0.3, (T, E, D, 3)))}
        kw.setdefault("Q", t(rng.uniform(0.1, 2.0, (E, 13))))
        kw.setdefault("Q_final", t(rng.uniform(10.0, 200.0, (E, 13))))
        kw.setdefault("R", t(rng.uniform(1e-3, 1e-1, (E, 4))))
        kw.setdefault("rpm_ref", t(hover * (1 + 0.02 * rng.uniform(-1, 1, (E, D, 4)))))
        kw.setdefault("last_rpm", t(hover * (1 + 0.1 * rng.uniform(-1, 1, (E, D, 4)))))
    else:
        target = {"pos": t(rng.uniform(-0.5, 0.5, (E, D, 3)) + np.array([0.0, 0.0, 1.0]))}
    if rpm is None:
        rpm = t(hover * (1 + 0.03 * rng.uniform(-1, 1, (T, E, D, 4))))
    return Problem(env, target, rpm=rpm, phys=phys, alphas=ALPHAS if alphas is None else alphas, **kw)


def _phys(env, rng):
    E = env._E
    return {"m": torch.as_tensor(env.M * rng.uniform(0.8, 1.2, E), **F64), "kf": torch.as_tensor(env.KF * rng.uniform(0.8, 1.2, E), **F64)}


def _per_drone(p, idx=None):
    """The reference's inputs of a Problem per drone (drones `idx`, default all): rows, W [T, n, 13], Rt, uref, x0, last_rpm,
    the nominal states, targets and rpm, K and k."""
    E, D = p.env_shape
    T, n = p.T, p.n
    idx = torch.arange(n, device=DEV) if idx is None else torch.as_tensor(idx, device=DEV)
    rows = p.rows.repeat_interleave(D, 0)[idx]
    w = p.weights.repeat_interleave(D, 0)[idx]
    h = rows[:, 12:13]
    return dict(rows=rows, w=w, Rt=w[:, 26:30] / (h * h), W=torch.stack([w[:, :13]] * (T - 1) + [w[:, 13:26]]), uref=p.rpm_ref[idx],
                x0=_vec(p.planes0, n)[idx], last_rpm=p.last_rpm[idx], xs=_vec(p.states, n)[:, idx], tg=_vec(p.targets, n)[:, idx],
                rpm=p.rpm[:, idx], K=p.K[:, idx], k=p.k[:, idx], idx=idx)


def _consts(p):
    P, E, D, S, eff = p.cfg
    return DR.model_constants(P, DEV), S, eff


def _ref_J(p, r, alphas, feedback=True, **kw):
    """ilqr_ref.rollout_cost for every alpha at once: {J [A, n], u [T, A, n, 4], x [T, A, n, 13]}."""
    Kd, S, eff = _consts(p)
    A, n = len(alphas), r["rows"].shape[0]
    rep = lambda x, d: x.unsqueeze(d).expand(*x.shape[:d], A, *x.shape[d:]).reshape(*x.shape[:d], A * n, *x.shape[d + 1:])
    al = torch.as_tensor(alphas, **F64).repeat_interleave(n)
    W = kw.pop("W", r["W"])
    Rt = kw.pop("Rt", r["Rt"])
    out = IR.rollout_cost(Kd, rep(r["rows"], 0), rep(r["x0"], 0), rep(r["last_rpm"], 0), rep(r["rpm"], 1), rep(r["xs"], 1),
                          rep(r["K"], 1) if feedback else None, rep(r["k"], 1), al, rep(r["tg"], 1), rep(W, 1), rep(Rt, 0),
                          rep(r["uref"], 0), S, eff, **kw)
    T = r["rpm"].shape[0]
    return dict(J=out["J"].reshape(A, n), u=out["u"].reshape(T, A, n, 4), x=out["x"].reshape(T, A, n, 13))


def _ref_jac(p, r):
    """qs_dyn_tick_jac's blocks [T, n, 13, C] by forward mode of diff_ref.tick at the nominal r."""
    Kd, S, eff = _consts(p)
    T, n = r["rpm"].shape[:2]
    x = torch.cat([r["x0"][None], r["xs"][:-1]])
    mx = r["rows"][:, 13:14].expand(n, 4)
    clip = torch.clamp(r["rpm"], min=torch.zeros_like(r["rpm"]), max=mx.expand(T, n, 4))
    up = torch.cat([r["last_rpm"][None], clip[:-1]])
    rows = r["rows"].expand(T, n, 16).reshape(T * n, 16)
    return IR.tick_jac(Kd, rows, x.reshape(T * n, 13), r["rpm"].reshape(T * n, 4), up.reshape(T * n, 4), S, eff).reshape(T, n, 13, -1)


def _ref_backward(p, r, jac, mu):
    T, n = r["rpm"].shape[:2]
    F = IR.f_from_jac(jac, r["rpm"], r["rows"][:, 13].expand(T, n))
    return IR.backward_pass(F, r["xs"] - r["tg"], r["W"], r["Rt"], r["rpm"] - r["uref"], mu)


def _drone_rel(a, b):
    """[n] per-drone normwise relative errors; the drone axis is 1 for [T, n, ...] and 0 for [n, ...]."""
    a, b = a.reshape(a.shape[0], -1), b.reshape(b.shape[0], -1)
    return (a - b).norm(dim=1) / b.norm(dim=1).clamp_min(1e-300)


def _per(x, T):
    """[T, n, ...] -> [n, T * ...]"""
    return x.transpose(0, 1).reshape(x.shape[1], -1)


def _check_commit(alphas, J, Jn, cost, mu_in, dV, status, conv_in, mu_out, conv_out):
    """The commit of every drone against ilqr_ref.commit on the device's own J, dV, mu, status and converged, exactly: the new
    cost is J of the reference's choice (or Jn), and mu and converged match.  Returns (the reference's choice [n], the number of
    drones on which taking the first accepted alpha instead of the largest would have given another cost)."""
    h = lambda x: x.cpu().numpy()
    J, Jn, cost, mu_in, dV, status, conv_in, mu_out, conv_out = map(h, (J, Jn, cost, mu_in, dV, status, conv_in, mu_out, conv_out))
    best, first_differs = [], 0
    for i in range(len(Jn)):
        args = (alphas, J[:, i], Jn[i], dV[i, 0], dV[i, 1], mu_in[i], int(status[i]), bool(conv_in[i]))
        b, mu, cv = IR.commit(*args)
        want = Jn[i] if b < 0 else J[b, i]
        assert cost[i] == want and mu_out[i] == mu and bool(conv_out[i]) == cv, (i, b, cost[i], want, mu_out[i], mu)
        f = IR.commit(*args, first_accepted=True)[0]
        first_differs += int(f >= 0 and J[f, i] != want)
        best.append(b)
    return np.array(best), first_differs


# ---- E1: the backward bit for bit the host build -----------------------------------------------------------------------------

@pytest.mark.parametrize("n", [9, 10, 15])
@pytest.mark.parametrize("T", [1, 240])
@pytest.mark.parametrize("physics", ["dyn", "drag"])
def test_backward_is_the_host_build_bit_for_bit(physics, T, n):
    D = {9: 3, 10: 2, 15: 3}[n]
    env = _env(n // D, D, physics, seed=n)
    rng = np.random.default_rng(100 + T + n)
    p = _problem(env, T, rng, phys=_phys(env, rng))
    nz, C = p.nz, p.jac.shape[-1]
    rows = p.rows.repeat_interleave(D, 0)
    mx = rows[:, 13]
    # synthetic Jacobians: a dense, contracting A and a dense B
    jac = rng.normal(size=(T, n, 13, C)) * 0.05
    jac[..., :13] += 0.6 * np.eye(13)
    jac[..., 13:17] *= 1e-3
    p.jac.copy_(torch.as_tensor(jac))
    p.states.normal_()
    p.targets.normal_()
    # the RPM edges: exactly 0, exactly MAX_RPM, one ulp outside each, at tick 0 and a middle tick (and at the last tick, where
    # the value after it has no previous-RPM block, so that only du sees them), and drone 1's rotor 2 clipped at every tick (its
    # B column 0) with a subnormal Rt.  Without drag the edges reach the pass only through du; with drag the clip's derivative
    # (rpm_clip_jvp's convention at the bounds) enters F's rows 13..16, and with T = 240 it changes K (checked below).
    tm = T // 2
    edges = [(0, 0, 0.0), (0, 1, -5e-324), (2, 2, None), (3, 3, "up")]
    for t0 in {0, tm}:
        for i, j, v in edges:
            m = float(mx[i])
            p.rpm[t0, i, j] = m if v is None else (np.nextafter(m, np.inf) if v == "up" else v)
    p.rpm[T - 1, 4, 0] = float(mx[4])
    p.rpm[T - 1, 5, 1] = np.nextafter(float(mx[5]), np.inf)
    p.rpm[:, 1, 2] = -100.0
    p.jac[:, 1, :, 15] = 0.0
    e1 = 1 // D
    h = float(p.rows[e1, 12])
    p.weights[e1, 28] = 3e-310 * h * h                           # Rt of drone 1's rotor 2: subnormal
    p.mu.copy_(torch.as_tensor(rng.choice([0.0, 0.3], n), **F64))
    mu_in = p.mu.clone()
    p.backward()
    torch.cuda.synchronize()
    Rt = p.weights.repeat_interleave(D, 0)[:, 26:30] / (rows[:, 12:13] * rows[:, 12:13])
    assert 0 < float(Rt[1, 2]) < 2.2250738585072014e-308          # subnormal
    F = IR.f_from_jac(p.jac, p.rpm, mx.expand(T, n))
    if nz == 17:
        for t0 in (0, tm):
            assert float(F[t0, 0, 13, 17]) == 1.0 and float(F[t0, 0, 14, 18]) == 0.0 and float(F[t0, 2, 15, 19]) == 1.0
            assert float(F[t0, 3, 16, 20]) == 0.0
        assert float(F[T - 1, 4, 13, 17]) == 1.0 and float(F[T - 1, 5, 14, 18]) == 0.0
    r = _per_drone(p)
    dx, du = (r["xs"] - r["tg"]).cpu().numpy(), (p.rpm - p.rpm_ref).cpu().numpy()
    W, Fh, Rth = r["W"].cpu().numpy(), F.cpu().numpy(), Rt.cpu().numpy()
    assert (p.status == 0).all() and torch.equal(p.mu, mu_in)
    Kd, kd, dVd = p.K.cpu().numpy(), p.k.cpu().numpy(), p.dV.cpu().numpy()
    for i in range(n):
        rc, K, k, _, _, dV = host_pass(Fh[:, i], dx[:, i], W[:, i], Rth[i], du[:, i], float(mu_in[i]), np.zeros((nz, nz)), np.zeros(nz))
        assert rc == 0
        assert np.array_equal(Kd[:, i], K) and np.array_equal(kd[:, i], k) and np.array_equal(dVd[i], dV), i
    if nz == 17 and T > 1:
        # negative control: the other side of the clip's derivative at the middle tick's edges gives another K
        for i, j, _ in edges:
            Ff = Fh[:, i].copy()
            Ff[tm, 13 + j, 17 + j] = 1.0 - Ff[tm, 13 + j, 17 + j]
            Kf = host_pass(Ff, dx[:, i], W[:, i], Rth[i], du[:, i], float(mu_in[i]), np.zeros((nz, nz)), np.zeros(nz))[1]
            assert not np.array_equal(Kd[:tm + 1, i], Kf[:tm + 1]) and np.array_equal(Kd[tm + 1:, i], Kf[tm + 1:]), (i, j)
    ref = IR.backward_pass(F, r["xs"] - r["tg"], r["W"], Rt, p.rpm - p.rpm_ref, mu_in)
    eK, ek = _drone_rel(_per(p.K, T), _per(ref["K"], T)).max().item(), _drone_rel(_per(p.k, T), _per(ref["k"], T)).max().item()
    ed = ((p.dV - torch.stack([ref["dV1"], ref["dV2"]], 1)).abs() / torch.stack([ref["dV1"], ref["dV2"]], 1).abs()).max().item()
    print("E1 %s T=%d n=%d: bit for bit the host build; against ilqr_ref K %.1e k %.1e dV %.1e" % (physics, T, n, eK, ek, ed))
    assert max(eK, ek, ed) <= 1e-10


# ---- E2: the restart ladder ---------------------------------------------------------------------------------------------------

EPS = 1e-3                                                        # -Rt of rotors 0 and 1


def _rungs(mu0):
    out, m = [float(mu0)], float(mu0)
    for _ in range(9):
        m = max(1e-6, 10.0 * m)
        out.append(m)
    return out


def ladder_case(rng, T, k_bad, restarts, mu0, W, Rt, dx, du):
    """F [T, 13, 17] of one drone whose tick k_bad has two equal B columns (0, 1) scaled so that Quu_mu of that tick has a
    Cholesky factor from mu* on, mu* between the rungs `restarts - 1` and `restarts` of the ladder from mu0 (restarts = 9:
    beyond the last rung; 0: no such tick)."""
    F = np.zeros((T, 13, 17))
    F[:, :, :13] = 0.6 * np.eye(13) + 0.05 * rng.normal(size=(T, 13, 13))
    F[:, :, 13:] = rng.normal(size=(T, 13, 4))
    if restarts == 0:
        return F, 0.0
    rg = _rungs(mu0)
    target = rg[8] * 100.0 if restarts == 9 else np.sqrt(max(rg[restarts - 1], 1e-7) * rg[restarts])
    b0 = rng.normal(size=13)
    # V at the tick (its stage cost included), from the later ticks' pass at mu = target
    if k_bad < T - 1:
        _, _, _, V, _, _ = host_pass(F[k_bad + 1:], dx[k_bad + 1:], W[k_bad + 1:], Rt, du[k_bad + 1:], target, np.zeros((13, 13)), np.zeros(13))
    else:
        V = np.zeros((13, 13))
    V = V + np.diag(W[k_bad])
    c = EPS * (1.0 + 1.0 / target)                                # (1 + mu*) (c - eps) = c: v = (1, -1, 0, 0) is the null direction
    s = np.sqrt(c / (b0 @ V @ b0))
    F[k_bad, :, 13] = F[k_bad, :, 14] = s * b0
    return F, target


def test_restart_ladder():
    T, D = 6, 3
    cases = [(k_bad, restarts, mu0) for mu0 in (0.0, 0.37) for k_bad in (T - 1, T // 2, 0) for restarts in (0, 1, 3, 8, 9)]
    n = len(cases)
    env = _env(n // D, D, "dyn", seed=30)
    rng = np.random.default_rng(31)
    h = env.HOVER_RPM
    p = _problem(env, T, rng, hetero=False, Q=torch.ones(13, **F64), Q_final=torch.ones(13, **F64),
                 R=torch.tensor([1.0, 1.0, 1e-2 * h * h, 1e-2 * h * h], **F64))
    p.weights[:, 26:28] = -EPS * h * h                            # through the ABI: the public call refuses R <= 0
    p.states.normal_()
    p.targets.normal_()
    r = _per_drone(p)
    Rt = r["Rt"][0].cpu().numpy()
    assert np.allclose(Rt[:2], -EPS, rtol=1e-14) and (r["Rt"] == r["Rt"][0]).all()
    dx, du, W = (r["xs"] - r["tg"]).cpu().numpy(), (p.rpm - p.rpm_ref).cpu().numpy(), r["W"].cpu().numpy()
    made = [ladder_case(np.random.default_rng(i), T, kb, rs, m0, W[:, i], Rt, dx[:, i], du[:, i]) for i, (kb, rs, m0) in enumerate(cases)]
    Fs, targets = [m[0] for m in made], [m[1] for m in made]
    p.jac.copy_(torch.as_tensor(np.stack(Fs, 1)))
    p.mu.copy_(torch.as_tensor([c[2] for c in cases], **F64))
    p.backward()
    Kd, kd, dVd, mud, std = p.K.cpu().numpy(), p.k.cpu().numpy(), p.dV.cpu().numpy(), p.mu.cpu().numpy(), p.status.cpu().numpy()
    zero = np.zeros((13, 13)), np.zeros(13)
    worst_stale = np.inf
    for i, (kb, rs, m0) in enumerate(cases):
        args = (Fs[i], dx[:, i], W[:, i], Rt, du[:, i])
        ok_at = lambda m: host_pass(*args, m, *zero)[0] == 0
        mu, status = IR.mu_ladder(m0, ok_at)
        rg = _rungs(m0)
        assert (mu, status) == (rg[rs], int(rs == 9)), (i, kb, rs, m0, mu, status)     # the design: restarts as intended
        if 0 < rs < 9:                                            # mu* lies between the rungs with a margin
            assert not ok_at(max(2 * rg[rs - 1], targets[i] / 3)) and ok_at(rg[rs] / 2)
        assert mud[i] == mu and std[i] == status, (i, mud[i], mu, std[i], status)
        if status == 0:
            rc, K, k, _, _, dV = host_pass(*args, mu, *zero)
            assert np.array_equal(Kd[:, i], K) and np.array_equal(kd[:, i], k) and np.array_equal(dVd[i], dV), (i, kb, rs)
            if rs > 0 and kb < T - 1:
                # negative control: dV1 and dV2 kept across the restarts (the failed attempts' ticks after kb added in)
                stale = dV.copy()
                for m in rg[:rs]:
                    stale += host_pass(Fs[i][kb + 1:], dx[kb + 1:, i], W[kb + 1:, i], Rt, du[kb + 1:, i], m, *zero)[5]
                worst_stale = min(worst_stale, float(np.max(np.abs(stale - dVd[i]) / np.abs(dVd[i]))))
    print("E2: %d drones, restarts 0, 1, 3, 8 and 9 failures at ticks %d, %d, 0 from mu 0 and 0.37: mu, status, K, k and dV exact "
          "(device mu %s); dV kept across restarts misses by >= %.2e" % (n, T - 1, T // 2, sorted(set(mud.tolist())), worst_stale))
    assert set(std.tolist()) == {0, 1}
    assert worst_stale > 1e-3


# ---- E3: J(alpha) against the restatement --------------------------------------------------------------------------------------

CONFIGS = [("dyn", "CF2X", 48), ("gnd", "CF2P", 240), ("drag", "CF2X", 240), ("gnd_drag", "CF2P", 48),
           ("dyn", "CF2P", 240), ("drag", "CF2P", 48), ("gnd", "CF2X", 48), ("gnd_drag", "CF2X", 240)]
UNSORTED = (0.3, 1.0, 0.05, 0.5, 0.7, 0.125, 0.9, 0.01, 0.25, 0.6, 0.8, 0.4, 0.0625, 0.2, 0.15, 0.35)


def _clip_guess(p, rng):
    """The guess with rotors clipped at 0 and at MAX_RPM (drones 0 and 1 far outside, drone 2 exactly on the bounds)."""
    T, n = p.T, p.n
    mx = p.rows.repeat_interleave(p.env_shape[1], 0)[:, 13]
    p.rpm[1:T - 1, 0, 1] = -3000.0
    p.rpm[1:T - 1, 1, 3] = 1.3 * mx[1]
    p.rpm[2, 2, 0] = 0.0
    p.rpm[3, 2, 2] = mx[2]
    return mx


def _check_J(p, r, alphas, feedback, label):
    got = p.line_search(alpha=torch.as_tensor(alphas, **F64), out=torch.empty((len(alphas), p.n), **F64)).clone()
    ref = _ref_J(p, r, alphas, feedback)
    e = ((got - ref["J"]).abs() / ref["J"].abs()).max().item()
    print("E3 %s: J(alpha) %d alphas, worst relative error %.1e" % (label, len(alphas), e))
    assert e <= 1e-10
    return got, ref


@pytest.mark.parametrize("physics,model,ctrl", CONFIGS)
def test_line_search_against_rollout_cost(physics, model, ctrl):
    E, D, T = 4, 3, 12
    env = _env(E, D, physics, model, ctrl=ctrl, seed=40)
    rng = np.random.default_rng(41)
    p = _problem(env, T, rng, phys=_phys(env, rng), alphas=UNSORTED)
    mx = _clip_guess(p, rng)
    label = "%s %s 240/%d" % (physics, model, ctrl)
    p.nominal()
    Jn = torch.empty((p.n,), **F64)
    p.cost(Jn)
    p.jacobians()
    p.backward()
    assert (p.status == 0).all()
    r = _per_drone(p)
    # the backward at forward-mode Jacobians of the reference tick
    ref = _ref_backward(p, r, _ref_jac(p, r), p.mu)
    eK = _drone_rel(_per(p.K, T), _per(ref["K"], T)).max().item()
    ek = _drone_rel(_per(p.k, T), _per(ref["k"], T)).max().item()
    print("E3 %s: backward at jvp Jacobians of diff_ref.tick: K %.1e k %.1e" % (label, eK, ek))
    assert max(eK, ek) <= 1e-9
    # feedback off: n_alpha = 10 and 1
    p.feedback = False
    _check_J(p, r, tuple(2.0 ** -j for j in range(10)), False, label + " K = 0")
    _check_J(p, r, (0.75,), False, label + " K = 0")
    p.feedback = True
    _, ref = _check_J(p, r, UNSORTED, True, label)
    J = p.line_search().clone()                                   # into the Problem's J, which the commit reads
    # the clips are taken in the nominal and in the trial
    u = ref["u"]
    lo, hi = int((u < 0).sum()), int((u > mx[:, None].expand(p.n, 4)).sum())
    assert lo > 0 and hi > 0 and float(p.rpm[2, 2, 0]) == 0.0 and float(p.rpm[3, 2, 2]) == float(mx[2])
    # negative controls, each must miss
    miss = {}
    if p.nz == 17:
        bad = _ref_J(p, r, UNSORTED, True, drag_prev_raw=True)["J"]
        miss["drag_prev_raw"] = ((bad - ref["J"]).abs() / ref["J"].abs())[:, :2].max().item()
    Wq = torch.stack([r["w"][:, :13]] * T)
    miss["Q at the last tick"] = ((_ref_J(p, r, UNSORTED, True, W=Wq)["J"] - ref["J"]).abs() / ref["J"].abs()).max().item()
    wm = p.weights[torch.arange(p.n, device=DEV) % E]
    Wm = torch.stack([wm[:, :13]] * (T - 1) + [wm[:, 13:26]])
    Rtm = wm[:, 26:30] / r["rows"][:, 12:13] ** 2
    miss["aviary i % E"] = ((_ref_J(p, r, UNSORTED, True, W=Wm, Rt=Rtm)["J"] - ref["J"]).abs() / ref["J"].abs()).max().item()
    Rth = r["w"][:, 26:30] / env.HOVER_RPM ** 2
    miss["nominal HOVER_RPM"] = ((_ref_J(p, r, UNSORTED, True, Rt=Rth)["J"] - ref["J"]).abs() / ref["J"].abs()).max().item()
    print("E3 %s: negative controls miss by %s" % (label, {k: "%.1e" % v for k, v in miss.items()}))
    assert min(miss.values()) > 1e-8
    # the commit: the largest accepted alpha of ilqr_ref.commit on the device's J and dV, its rpm and its trajectory
    cost = torch.empty((p.n,), **F64)
    mu_in, conv_in = p.mu.clone(), p.converged.clone()
    p.commit(Jn, cost)
    best, first_differs = _check_commit(UNSORTED, J, Jn, cost, mu_in, p.dV, p.status, conv_in, p.mu, p.converged)
    acc = torch.as_tensor(best >= 0, device=DEV)
    assert int(acc.sum()) > 0 and first_differs > 0               # negative control: the first accepted alpha misses
    best = torch.as_tensor(np.maximum(best, 0), device=DEV)
    idx = torch.nonzero(acc)[:, 0]
    u_ref = ref["u"][:, best[idx], idx]
    eu = _drone_rel(_per(p.rpm[:, idx], T), _per(u_ref, T)).max().item()
    Kd, S, eff = _consts(p)
    x = DR.rollout(Kd, r["rows"], r["x0"], p.rpm, r["last_rpm"], S, eff)
    ex = _drone_rel(_per(_vec(p.states, p.n), T), _per(x, T)).max().item()
    print("E3 %s: committed %d / %d drones, the choice exact (the first accepted alpha would differ on %d): rpm %.1e, "
          "trajectory %.1e" % (label, int(acc.sum()), p.n, first_differs, eu, ex))
    assert eu <= 1e-12 and ex <= 1e-12


# ---- E4: the commit rule at its boundaries --------------------------------------------------------------------------------------

ALPHAS4 = (0.25, 1.0, 0.5, 1.0, 0.125)                             # unsorted, with a duplicate
NAN, INF = float("nan"), float("inf")


def _jn_boundary(c):
    """The smallest Jn with Jn - c >= 1e-9 Jn (not converged after committing c): one ulp below converges."""
    Jn = c / (1 - 1e-9)
    while Jn - c >= 1e-9 * Jn:
        Jn = np.nextafter(Jn, -np.inf)
    while not Jn - c >= 1e-9 * Jn:
        Jn = np.nextafter(Jn, np.inf)
    return float(Jn)


def _scenarios(c):
    """(name, J row, Jn, dV1, dV2, mu, status, converged) at the boundaries of every predicate, for a drone whose committed J is c."""
    up, dn = (lambda x: float(np.nextafter(x, np.inf))), (lambda x: float(np.nextafter(x, -np.inf)))
    out = []
    Jn = 2.0 * c
    for name, v in (("Ja == Jn", Jn), ("Ja one ulp below Jn", dn(Jn)), ("Ja one ulp above Jn", up(Jn))):
        out.append((name, [INF, v, INF, INF, INF], Jn, 0.0, 0.0, 0.0, 0, 0))
    for s, dv2 in ((1, 0.0), (2, -0.3 * c), (4, 0.2 * c)):        # Armijo at alpha = 1, 0.5 (negative dV2) and 0.125
        al, dv1 = ALPHAS4[s], -c * 9.0
        Ja = IR.armijo_boundary(Jn, al, dv1, dv2)
        for name, v in (("Armijo at the boundary", Ja), ("Armijo one ulp below", dn(Ja)), ("Armijo one ulp above", up(Ja))):
            row = [INF] * 5
            row[s] = v
            out.append(("%s alpha=%g dV2=%g" % (name, al, dv2), row, Jn, dv1, dv2, 0.0, 0, 0))
    Jb = _jn_boundary(c)
    for name, v in (("converged boundary", Jb), ("converged one ulp below", dn(Jb)), ("converged one ulp above", up(Jb))):
        out.append((name, [INF, c, INF, INF, INF], v, 0.0, 0.0, 0.0, 0, 0))
    for mu in (1e-5, 9.999999999999999e-06, 0.0, 1e-6):
        out.append(("mu %r accepted" % mu, [INF, c, INF, INF, INF], Jn, 0.0, 0.0, mu, 0, 0))
        out.append(("mu %r rejected" % mu, [INF, Jn, INF, INF, INF], Jn, 0.0, 0.0, mu, 0, 0))
    out += [("NaN and inf J, one finite", [NAN, INF, NAN, INF, c], Jn, 0.0, 0.0, 0.1, 0, 0),
            ("NaN J everywhere", [NAN] * 5, Jn, 0.0, 0.0, 0.1, 0, 0),
            ("Jn = inf, one finite", [INF, c, INF, INF, INF], INF, -1.0, 0.0, 0.1, 0, 0),
            ("Jn = inf, J = inf", [INF] * 5, INF, -1.0, 0.0, 0.1, 0, 0),
            ("negative dV2: alpha = 1 fails, 0.5 passes", [c] * 5, c * 1.001, -c, -10 * c, 0.1, 0, 0),
            ("duplicate alpha = 1", [INF, c, INF, c, INF], Jn, 0.0, 0.0, 0.1, 0, 0),
            ("unsorted: 0.5 over 0.25 and 0.125", [c, Jn, c, Jn, c], Jn, 0.0, 0.0, 0.1, 0, 0),
            ("status 1 with an acceptable J", [c] * 5, Jn, 0.0, 0.0, 0.37, 1, 0),
            ("converged with an acceptable J", [c] * 5, Jn, 0.0, 0.0, 0.37, 0, 1)]
    return out


def test_commit_rule_at_its_boundaries():
    n, T, n_real = 131, 8, 8
    env = _env(n, 1, "dyn", seed=50)
    rng = np.random.default_rng(51)
    p = _problem(env, T, rng, hetero=False, alphas=ALPHAS4)
    p.nominal()
    c0 = torch.empty((n,), **F64)
    p.cost(c0)
    c0h = c0.cpu().numpy()
    m = len(_scenarios(1.0))
    nb = n - n_real                                               # injected scenarios; the last n_real drones commit a real k
    pick = [_scenarios(float(c0h[i]))[i % m] for i in range(nb)]
    expect = [IR.commit(ALPHAS4, s[1], s[2], s[3], s[4], s[5], s[6], s[7], Jc=float(c0h[i])) for i, s in enumerate(pick)]
    # drones that must not commit get a non-zero k, so that a wrong commit would move their rpm; those that commit an injected J
    # keep k = 0, so that their rollout reproduces the nominal and the committed J is c0; the last n_real drones get a k of their
    # own and the J of the line search along it
    moved = torch.as_tensor([e[0] < 0 for e in expect] + [True] * n_real, device=DEV)
    p.k.copy_(torch.as_tensor(rng.normal(size=p.k.shape) * 30.0, **F64) * moved[None, :, None])
    p.k[:, nb:] *= 0.1                                            # J(alpha) then varies far less than Jn's margin of 1e-3 below
    p.status.copy_(torch.as_tensor([s[6] for s in pick] + [0] * n_real, dtype=torch.int32, device=DEV))
    p.converged.copy_(torch.as_tensor([s[7] for s in pick] + [0] * n_real, dtype=torch.uint8, device=DEV))
    # the line search skips status-1 and converged drones; the cost path (status, converged NULL) skips nothing
    Jl = p.line_search().clone()
    skip = (p.status != 0) | (p.converged != 0)
    assert torch.isinf(Jl[:, skip]).all() and torch.isfinite(Jl[:, ~skip]).all()
    cpath = torch.empty((n,), **F64)
    p.cost(cpath)
    assert torch.equal(cpath, c0)
    # the real-k drones: every alpha accepted (the first, 0.25, is not the largest, 1.0), or alpha = 1 just failing Armijo (the
    # first accepted, 0.25, is not the largest, 0.5)
    Jlh = Jl.cpu().numpy()
    for i in range(nb, n):
        row = Jlh[:, i].tolist()
        Jn = max(row) * (1 + 1e-3)
        if (i - nb) % 2 == 0:
            name, dv1 = "real k, every alpha accepted", 0.0
        else:
            name, dv1 = "real k, alpha = 1 fails Armijo", -1.01 * (Jn - row[1]) * 1e4
        pick.append((name, row, Jn, dv1, 0.0, 0.1, 0, 0))
        e = IR.commit(ALPHAS4, row, Jn, dv1, 0.0, 0.1, 0, False)
        f = IR.commit(ALPHAS4, row, Jn, dv1, 0.0, 0.1, 0, False, first_accepted=True)[0]
        assert e[0] == (1 if (i - nb) % 2 == 0 else 2) and f == 0, (i, e, f)   # the scenario as designed
        expect.append(e)
    J = torch.as_tensor(np.array([s[1] for s in pick]).T, **F64)
    Jn = torch.as_tensor([s[2] for s in pick], **F64)
    p.J.copy_(J)
    p.dV.copy_(torch.as_tensor([[s[3], s[4]] for s in pick], **F64))
    p.mu.copy_(torch.as_tensor([s[5] for s in pick], **F64))
    rpm0, st0 = p.rpm.clone(), p.states.clone()
    out = torch.full((n,), -7.0, **F64)
    p.commit(Jn, out)
    outh, muh, cvh = out.cpu().numpy(), p.mu.cpu().numpy(), p.converged.cpu().numpy()
    seen = set()
    for i, (s, (best, mu, conv)) in enumerate(zip(pick, expect)):
        want = s[2] if best < 0 else (float(c0h[i]) if i < nb else s[1][best])
        assert outh[i] == want or (np.isnan(want) and np.isnan(outh[i])), (i, s[0], outh[i], want)
        assert muh[i] == mu and bool(cvh[i]) == bool(conv), (i, s[0], muh[i], mu, cvh[i], conv)
        seen.add((s[0], best >= 0, bool(conv)))
    # rpm: untouched, except the real-k drones, which take rpm_nom + alpha k of the largest accepted alpha bit for bit (the
    # first accepted alpha's rpm differs); their new nominal's cost is the committed J
    want_rpm = rpm0.clone()
    for i in range(nb, n):
        b = expect[i][0]
        want_rpm[:, i] = rpm0[:, i] + ALPHAS4[b] * p.k[:, i]
        assert not torch.equal(p.rpm[:, i], rpm0[:, i] + ALPHAS4[0] * p.k[:, i])
    assert torch.equal(p.rpm, want_rpm)
    assert torch.equal(_vec(p.states, n)[:, :nb], _vec(st0, n)[:, :nb])
    p.cost(cpath)
    assert torch.equal(cpath[nb:], out[nb:])
    kinds = {(a, c) for _, a, c in seen}
    print("E4: %d drones, %d scenarios, every one exact; (accepted, converged) outcomes %s" % (n, m + 2, sorted(kinds)))
    for name, acc, conv in sorted(seen):
        print("   %-48s accepted=%d converged=%d" % (name, acc, conv))
    assert {(True, False), (False, False), (True, True), (False, True)} <= kinds


# ---- E5: whole iterations, teacher-forced ------------------------------------------------------------------------------------

def test_whole_iterations_teacher_forced():
    E, D, T = 16, 4, 24
    env = _env(E, D, "drag", seed=60)
    rng = np.random.default_rng(61)
    n = E * D
    tgt = rng.uniform(-2.0, 2.0, (E, D, 3)) + np.array([0.0, 0.0, 1.5])
    tgt[:2] = env.pos[:2].cpu().numpy() + rng.uniform(-1e-3, 1e-3, (2, D, 3))   # two aviaries start at their targets
    from gym_pybullet_drones_b200.ilqr import Problem
    p = Problem(env, {"pos": torch.as_tensor(tgt, **F64)}, num_steps=T)
    cost = torch.empty((7, n), **F64)
    p.nominal()
    p.cost(cost[0])
    p.jacobians()
    p.backward()
    al = p.alphas.cpu().numpy()
    chosen, rejected_all, near, checked = set(), 0, 0, 0
    for it in range(6):
        r = _per_drone(p)
        mu_in = p.mu.clone()
        ref = _ref_backward(p, r, _ref_jac(p, r), mu_in)
        J = p.line_search().clone()
        Jr = _ref_J(p, r, tuple(al), True)["J"]
        status, conv0 = p.status.cpu().numpy(), p.converged.cpu().numpy().copy()
        p.commit(cost[it], cost[it + 1])
        Jh, Jrh, Jnh, outh = J.cpu().numpy(), Jr.cpu().numpy(), cost[it].cpu().numpy(), cost[it + 1].cpu().numpy()
        d1, d2 = ref["dV1"].cpu().numpy(), ref["dV2"].cpu().numpy()
        muh, cvh, mih = p.mu.cpu().numpy(), p.converged.cpu().numpy(), mu_in.cpu().numpy()
        for i in range(n):
            if conv0[i] or status[i]:
                continue
            Jn = Jnh[i]
            best, mu, cv = IR.commit(al, Jrh[:, i], Jn, d1[i], d2[i], mih[i], 0, False)
            # the device's choice: the largest alpha whose J is the committed cost
            hit = [s for s in range(len(al)) if Jh[s, i] == outh[i]] if outh[i] != Jn else []
            dev_best = max(hit, key=lambda s: al[s]) if hit else -1
            margin = min([abs(Jrh[s, i] - Jn) for s in range(len(al))]
                         + [abs(Jn - Jrh[s, i] - 1e-4 * -(al[s] * d1[i] + al[s] * al[s] * d2[i])) for s in range(len(al))]
                         + ([abs(Jn - Jrh[best, i] - 1e-9 * Jn)] if best >= 0 else []))
            if margin <= 1e-9 * abs(Jn):
                near += 1
                continue
            checked += 1
            assert (al[dev_best] if dev_best >= 0 else -1) == (al[best] if best >= 0 else -1), (it, i, dev_best, best)
            assert muh[i] == mu and bool(cvh[i]) == cv, (it, i, muh[i], mu, cvh[i], cv)
            if best >= 0:
                chosen.add(al[best])
            else:
                rejected_all += 1
        p.jacobians()
        p.backward()
    print("E5: %d decisions checked, %d within 1e-9 of a threshold skipped; alphas chosen %s; %d rejected every alpha"
          % (checked, near, sorted(float(a) for a in chosen), rejected_all))
    assert len(chosen) >= 3 and rejected_all >= 1


# ---- E6: converged, failed and zero-cost drones over many iterations -----------------------------------------------------------

def test_converged_failed_and_zero_cost_drones():
    E, D, T, iters = 6, 4, 16, 40
    env = _env(E, D, "dyn", seed=70)
    rng = np.random.default_rng(71)
    n = E * D
    h = env.HOVER_RPM
    tgt = rng.uniform(-1.0, 1.0, (E, D, 3)) + np.array([0.0, 0.0, 1.5])
    tgt[:2] = env.pos[:2].cpu().numpy() + rng.uniform(-1e-3, 1e-3, (2, D, 3))   # aviaries 0, 1: converge early
    Q = np.tile(np.array((1.0,) * 7 + (0.1,) * 3 + (0.01,) * 3), (E, 1))
    Q[3] = 0.0                                                    # aviary 3: zero cost (and the guess is rpm_ref)
    from gym_pybullet_drones_b200.ilqr import Problem
    p = Problem(env, {"pos": torch.as_tensor(tgt, **F64)}, num_steps=T, Q=torch.as_tensor(Q, **F64), Q_final=torch.as_tensor(Q * 100, **F64))
    p.weights[2, 26:30] = -1e6                                    # aviary 2: status 1 (through the ABI)
    failed, zero = slice(2 * D, 3 * D), slice(3 * D, 4 * D)
    cost = torch.empty((iters + 1, n), **F64)
    p.nominal()
    p.cost(cost[0])
    p.jacobians()
    p.backward()
    snaps, mu_b, mu_c = [], [p.mu.clone()], []
    for it in range(iters):
        p.line_search()
        p.commit(cost[it], cost[it + 1])
        mu_c.append(p.mu.clone())
        p.jacobians()
        p.backward()
        mu_b.append(p.mu.clone())
        snaps.append((p.rpm.clone(), p.states.clone(), p.K.clone(), p.k.clone(), p.converged.clone()))
    conv = snaps[-1][4].bool()
    assert conv[:2 * D].any()
    first = {}
    for i in torch.nonzero(conv)[:, 0].tolist():
        it0 = next(it for it in range(iters) if snaps[it][4][i])
        first[i] = it0
        for it in range(it0, iters):
            assert torch.equal(snaps[it][0][:, i], snaps[it0][0][:, i]) and torch.equal(_vec(snaps[it][1], n)[:, i], _vec(snaps[it0][1], n)[:, i])
            assert torch.equal(snaps[it][2][:, i], snaps[it0][2][:, i]) and torch.equal(snaps[it][3][:, i], snaps[it0][3][:, i])
            assert torch.equal(cost[it + 1, i], cost[it0 + 1, i])
    # a fresh backward at the final trajectory gives the converged drones' K and k bit for bit
    K1, k1 = p.K.clone(), p.k.clone()
    p.jacobians()
    p.backward()
    assert torch.equal(p.K[:, conv], K1[:, conv]) and torch.equal(p.k[:, conv], k1[:, conv])
    # status 1: mu follows the ladder (nine failures per backward) and the commit's rejection
    mu = [0.0] * D
    for it in range(iters):
        mu = [IR.mu_ladder(m, lambda _: False)[0] for m in mu]
        assert mu_b[it][failed].tolist() == mu
        mu = [IR.commit((1.0,), (INF,), 0.0, 0.0, 0.0, m, 1, False)[1] for m in mu]
        assert mu_c[it][failed].tolist() == mu
    assert (p.status[failed] == 1).all() and (cost[:, failed] == cost[0, failed]).all()
    # zero cost: J(alpha) = Jn = 0, no step is ever accepted, converged is never set, and mu grows x10 per iteration
    assert (cost[:, zero] == 0).all() and not p.converged[zero].any() and (p.status[zero] == 0).all()
    mu = 0.0
    for it in range(iters):
        mu = max(1e-6, 10.0 * mu)
        assert (mu_c[it][zero] == mu).all() and (mu_b[it + 1][zero] == mu).all()
    print("E6: %d drones converged (first at iterations %s) and stayed bit-identical; status-1 mu %.3g after %d iterations; "
          "zero-cost drones never accepted, mu %.3g" % (len(first), sorted(set(first.values())), float(mu_c[-1][failed][0]), iters, mu))
    # where the zero-cost drones' mu ends: from 1e306 the commit reaches 1e308 and then +inf; Quu_mu's pivots are then +inf, so
    # the next backward fails all nine times and marks them failed (status 1) with mu = +inf, about 315 iterations from mu = 0
    p.mu[zero] = 1e306
    for it in range(3):
        p.line_search()
        p.commit(cost[-1], cost[-1].clone())
        p.jacobians()
        p.backward()
        assert bool((p.status[zero] == 1).all()) == (it == 2) and bool((p.status[zero] == 0).all()) == (it < 2)
    assert torch.isinf(p.mu[zero]).all() and (cost[-1, zero] == 0).all()


# ---- E7: size ---------------------------------------------------------------------------------------------------------------------

def test_one_iteration_at_65536_drones():
    E, D, T = 16384, 4, 8
    env = _env(E, D, "drag", seed=80)
    rng = np.random.default_rng(81)
    p = _problem(env, T, rng, phys=_phys(env, rng))
    n, na = p.n, p.alphas.numel()
    _clip_guess(p, rng)
    t0 = time.time()
    Jn = torch.empty((n,), **F64)
    p.nominal()
    p.cost(Jn)
    p.jacobians()
    p.backward()
    J = p.line_search().clone()
    cost = torch.empty((n,), **F64)
    K0, k0, xs0, rpm0 = p.K.clone(), p.k.clone(), p.states.clone(), p.rpm.clone()
    mu_b, conv_in = p.mu.clone(), p.converged.clone()            # the backward's mu, which the commit overwrites
    p.commit(Jn, cost)
    torch.cuda.synchronize()
    wall = time.time() - t0
    # the drones on either side of every CTA boundary of the three grids, the first and the last
    idx = {0, 1, n - 2, n - 1}
    for b in (1, 2, 3, 1000, 4097, (n // 4) // 2, n // 4 - 2, n // 4 - 1):   # backward: 4 drones per CTA
        idx |= {4 * b - 1, 4 * b}
    for b in (1, 2, 3, 5, 77, 1001, (n * na // 128) // 2, n * na // 128 - 2, n * na // 128 - 1):   # line search: 128 (drone, alpha)
        g = 128 * b
        idx |= {(g - 1) // na, g // na}
    for b in (1, 2, 3, 4, 100, 200, 257, 400, (n // 128) // 2, n // 128 - 2, n // 128 - 1):   # commit: 128 drones per CTA
        idx |= {128 * b - 1, 128 * b}
    idx = sorted(i for i in idx if 0 <= i < n)
    # the references at the nominal before the commit
    new = dict(states=p.states.clone(), rpm=p.rpm.clone())
    p.states.copy_(xs0)
    p.rpm.copy_(rpm0)
    r = _per_drone(p, idx)
    p.states.copy_(new["states"])
    p.rpm.copy_(new["rpm"])
    r["K"], r["k"] = K0[:, r["idx"]], k0[:, r["idx"]]
    ref = _ref_backward(p, r, _ref_jac(p, r), mu_b[r["idx"]])
    assert (p.status[r["idx"]] == 0).all()
    eK = _drone_rel(_per(K0[:, r["idx"]], T), _per(ref["K"], T)).max().item()
    Jr = _ref_J(p, r, tuple(p.alphas.tolist()), True)
    eJ = ((J[:, r["idx"]] - Jr["J"]).abs() / Jr["J"].abs()).max().item()
    # every drone's commit against ilqr_ref.commit on the device's J and dV, exactly
    best_all, _ = _check_commit(tuple(p.alphas.tolist()), J, Jn, cost, mu_b, p.dV, p.status, conv_in, p.mu, p.converged)
    best = torch.as_tensor(best_all[idx], device=DEV)
    acc = best >= 0
    best = best.clamp_min(0)
    sel = torch.nonzero(acc)[:, 0]
    eu = _drone_rel(_per(p.rpm[:, r["idx"][sel]], T), _per(Jr["u"][:, best[sel], sel], T)).max().item()
    Kd, S, eff = _consts(p)
    x = DR.rollout(Kd, r["rows"], r["x0"], p.rpm[:, r["idx"]], r["last_rpm"], S, eff)
    ex = _drone_rel(_per(_vec(p.states, n)[:, r["idx"]], T), _per(x, T)).max().item()
    print("E7: %d drones, T = %d, one iteration %.2f s (first launches included); every commit exact (%d accepted); %d drones "
          "checked (%d committed): K %.1e, J %.1e, rpm %.1e, trajectory %.1e; peak device memory of the process so far %.2f GB"
          % (n, T, wall, int((best_all >= 0).sum()), len(idx), int(acc.sum()), eK, eJ, eu, ex, torch.cuda.max_memory_allocated() / 1e9))
    assert len(idx) >= 40 and int(acc.sum()) > 0
    assert eK <= 1e-9 and eJ <= 1e-10 and eu <= 1e-12 and ex <= 1e-12
