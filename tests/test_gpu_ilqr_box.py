"""-m gpu: control-limited iLQR on the device (BaseAviary.ilqr(rpm_bounds=...), ilqr_*_kernel<EFF, true>, DESIGN.md 4.5.1).

B1  bounds that never bind (a gentle hover task): ilqr(rpm_bounds=...) is ilqr() bit for bit, every output and every iteration.
B2  the box backward bit for bit the host build (tests/host_harness/ilqr_box_host.cpp) on synthetic Jacobians, bounds binding at
    tick 0, a middle tick and the last tick, DYN and DRAG (n_z = 13 and 17), partial CTAs.
B3  a saturating task (climb 1 m and stop within 0.5 s at 48 Hz, 1 024 drones, 100 iterations): rotors reach the upper bound,
    every rpm lies in the box after every iteration, the cost never increases, the trajectory is
    differentiable_rollout(rpm=sol["rpm"]) bit for bit, and at converged drones the projected gradient of J (autograd through
    differentiable_rollout plus the R term) has the KKT signs.  The same task without bounds is reported, not asserted.
B4  tighter envelopes: a derated rotor per drone, a cap from tick T/2 on, an idle floor; each respected exactly, with the KKT check.
B5  J(alpha) of the box line search against the float64 clamped rollout (ilqr_box_ref.rollout_cost_box), the unclamped
    restatement as a negative control; dV1 against one-sided differences of J(alpha) at small alpha > 0 where the nominal sits
    on its bounds.
B6  the commit of a drone whose k is 0 at every tick, drone independence, determinism, a Morton twin, an untouched env, one
    synchronisation per solve, and the refusals."""
import warnings

import numpy as np
import pytest
import torch

import ilqr_box_ref as BR
import ilqr_ref as IR
from test_gpu_ilqr import KEYS, _env, _vec
from test_gpu_ilqr_edges import F64, _consts, _per_drone, _phys, _problem
from test_ilqr_box_host import host_box_pass

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _max_rpm(env, phys=None):
    """MAX_RPM of each aviary's row [E] (the phys table's when given), as "motor" and the bound checks take it"""
    from gym_pybullet_drones_b200.diff import _start_state
    return _start_state(env, None, None, phys)[2][:, 13].clone()


def _gentle(env, seed):
    """targets within 1 mm of each drone's start"""
    rng = np.random.default_rng(seed)
    pos = env.pos.to(torch.float64).clone()
    return {"pos": pos + torch.as_tensor(rng.uniform(-1e-3, 1e-3, tuple(pos.shape)), **F64)}


def _climb(env, height=1.0):
    """`height` m straight up from each drone's start"""
    pos = env.pos.to(torch.float64).clone()
    pos[..., 2] += height
    return {"pos": pos}


def _saturating_env(E, D, physics="dyn", seed=0):
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils.enums import Physics
    rng = np.random.default_rng(seed)
    xyz = np.stack([rng.uniform(-1, 1, D), rng.uniform(-1, 1, D), rng.uniform(0.5, 1.0, D)], 1)
    env = CtrlAviary(num_drones=D, physics=Physics.DYN if physics == "dyn" else Physics.PYB_DRAG, pyb_freq=240, ctrl_freq=48,
                     initial_xyzs=xyz, num_envs=E)
    env.reset()
    return env


def _solve_checked(env, target, T, iters, rpm_bounds, lo=None, hi=None, **kw):
    """ilqr.solve step by step, with every iteration's rpm checked against [lo, hi] ([T, n, 4] broadcastable; default the
    Problem's box)"""
    from gym_pybullet_drones_b200.ilqr import Problem
    p = Problem(env, target, num_steps=T, rpm_bounds=rpm_bounds, **kw)
    lo = p.box[0] if lo is None else lo
    hi = p.box[1] if hi is None else hi
    cost = torch.empty((iters + 1, p.n), **F64)
    inside = lambda: bool(((p.rpm >= lo) & (p.rpm <= hi)).all())
    assert inside()
    p.nominal()
    p.cost(cost[0])
    p.jacobians()
    p.backward()
    for it in range(iters):
        p.line_search()
        p.commit(cost[it], cost[it + 1])
        assert inside(), it
        p.jacobians()
        p.backward()
    return p, p.result(cost)


def _grad_J(env, p, sol):
    """dJ/du [T, n, 4] of the solution's rpm by autograd through differentiable_rollout plus the R term, with the Problem's
    weights, targets and reference (independent of the backward pass)"""
    E, D = p.env_shape
    T, n = p.T, p.n
    u = sol["rpm"].detach().clone().requires_grad_(True)
    roll = env.differentiable_rollout(rpm=u, last_rpm=p.last_rpm.view(E, D, 4), phys=None)
    x = torch.cat([roll[k].reshape(T, n, -1) for k in KEYS], dim=-1)
    r = _vec(p.targets, n)
    w = p.weights.repeat_interleave(D, 0)
    W = torch.stack([w[:, :13]] * (T - 1) + [w[:, 13:26]])
    h = p.rows.repeat_interleave(D, 0)[:, 12:13]
    Rt = w[:, 26:30] / (h * h)
    J = 0.5 * ((W * (x - r) ** 2).sum() + (Rt * (u.reshape(T, n, 4) - p.rpm_ref) ** 2).sum())
    (g,) = torch.autograd.grad(J, u)
    return g.reshape(T, n, 4)


def _kkt(env, p, sol, lo, hi, name):
    """The projected gradient at converged drones: per drone, relative to its largest |dJ/du|, the worst of |g| on free rotors,
    -g at the lower bound and g at the upper bound.  Returns (worst, converged drones)."""
    g = _grad_J(env, p, sol)
    u = sol["rpm"].reshape(p.T, p.n, 4)
    lo, hi = lo.expand_as(u), hi.expand_as(u)
    at_lo, at_hi = u == lo, u == hi
    free = ~(at_lo | at_hi)
    viol = torch.where(free, g.abs(), torch.where(at_lo, (-g).clamp_min(0), g.clamp_min(0)))
    scale = g.abs().amax(dim=(0, 2)).clamp_min(1e-300)
    per = viol.amax(dim=(0, 2)) / scale
    conv = sol["converged"].reshape(-1)
    worst = float(per[conv].max()) if bool(conv.any()) else float("nan")
    print("%s: %d of %d drones converged; projected gradient / max |dJ/du| at them <= %.1e; rotor-ticks at lo %d, at hi %d"
          % (name, int(conv.sum()), p.n, worst, int(at_lo.sum()), int(at_hi.sum())))
    return worst, int(conv.sum())


# ---- B1: bounds that never bind ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("physics", ["dyn", "drag"])
def test_never_binding_bounds_are_bit_identical(physics):
    env = _saturating_env(12, 3, physics, seed=40)                  # level starts: nothing saturates
    T = 32
    tgt = _gentle(env, 41)
    base = env.ilqr(tgt, num_steps=T, iters=8)
    h, m = float(env.HOVER_RPM), float(_max_rpm(env).min())
    bounds = ["motor", (torch.tensor([0.5 * h] * 4, **F64), torch.tensor([m] * 4, **F64)),
              (torch.full((T, 12, 3, 4), 0.3 * h, **F64), torch.full((12, 3, 4), 0.99 * m, **F64))]
    assert bool(((base["rpm"] > 0.5 * h) & (base["rpm"] < 0.99 * m)).all())
    for b in bounds:
        sol = env.ilqr(tgt, num_steps=T, iters=8, rpm_bounds=b)
        assert set(sol) == set(base) | {"active"}
        for k in base:
            assert torch.equal(sol[k], base[k]), k
        assert not bool(sol["active"].any())


# ---- B2: the box backward bit for bit the host build -------------------------------------------------------------------------

@pytest.mark.parametrize("n", [9, 10])
@pytest.mark.parametrize("physics", ["dyn", "drag"])
def test_box_backward_is_the_host_build_bit_for_bit(physics, n):
    D = {9: 3, 10: 2}[n]
    T = 48
    env = _env(n // D, D, physics, seed=50 + n)
    rng = np.random.default_rng(51 + n)
    E = env._E
    phys = _phys(env, rng)
    m = _max_rpm(env, phys).repeat_interleave(D)[:, None]              # [n, 1]
    lo0, hi0 = torch.zeros((T, E, D, 4), **F64), m.reshape(1, E, D, 1).expand(T, E, D, 4).clone()
    p = _problem(env, T, rng, phys=phys, rpm_bounds=(lo0, hi0))
    nz, C = p.nz, p.jac.shape[-1]
    jac = rng.normal(size=(T, n, 13, C)) * 0.05
    jac[..., :13] += 0.6 * np.eye(13)
    jac[..., 13:17] *= 1e-3
    p.jac.copy_(torch.as_tensor(jac))
    p.states.normal_()
    p.targets.normal_()
    p.mu.copy_(torch.as_tensor(rng.choice([0.0, 0.3], n), **F64))
    mu_in = p.mu.clone()
    # the unconstrained k, to size boxes that bind at tick 0, a middle tick and the last tick
    box = p.box
    p.box = None
    p.backward()
    p.box = box
    k0 = p.k.clone()
    p.mu.copy_(mu_in)
    lo, hi = box[0], box[1]
    lo.copy_(torch.clamp(p.rpm - 10 * k0.abs() - 1.0, min=0.0))
    hi.copy_(torch.minimum(p.rpm + 10 * k0.abs() + 1.0, m))
    tm = T // 2
    for t0 in (0, tm, T - 1):
        lo[t0] = torch.clamp(p.rpm[t0] - 0.5 * k0[t0].abs(), min=0.0)
        hi[t0] = torch.minimum(p.rpm[t0] + 0.5 * k0[t0].abs(), m)
    p.rpm[tm, 0, 0] = hi[tm, 0, 0]                                  # a nominal exactly on a bound
    p.rpm[0, 1, 1] = lo[0, 1, 1]
    p.backward()
    torch.cuda.synchronize()
    assert (p.status == 0).all() and torch.equal(p.mu, mu_in)
    act = p.active.cpu().numpy()
    for t0 in (0, tm, T - 1):
        assert np.count_nonzero(act[t0]) >= 2, t0                  # the bounds bind at these ticks
    rows = p.rows.repeat_interleave(D, 0)
    F = IR.f_from_jac(p.jac, p.rpm, rows[:, 13].expand(T, n)).cpu().numpy()
    r = _per_drone(p)
    dx, du = (r["xs"] - r["tg"]).cpu().numpy(), (p.rpm - p.rpm_ref).cpu().numpy()
    W, Rt = r["W"].cpu().numpy(), r["Rt"].cpu().numpy()
    blo, bhi = (lo - p.rpm).cpu().numpy(), (hi - p.rpm).cpu().numpy()
    Kd, kd, dVd = p.K.cpu().numpy(), p.k.cpu().numpy(), p.dV.cpu().numpy()
    held = 0
    for i in range(n):
        rc, K, k, a, _, _, dV = host_box_pass(F[:, i], dx[:, i], W[:, i], Rt[i], du[:, i], blo[:, i], bhi[:, i], float(mu_in[i]),
                                              np.zeros((nz, nz)), np.zeros(nz))
        assert rc == 0
        assert np.array_equal(Kd[:, i], K) and np.array_equal(kd[:, i], k) and np.array_equal(dVd[i], dV), i
        assert np.array_equal(act[:, i], a), i
        assert np.all(K[a != 0] == 0.0)
        held += int(np.count_nonzero(a))
    print("B2 %s n=%d: bit for bit the host build, %d of %d rotor-ticks held" % (physics, n, held, T * n * 4))


# ---- B3: a saturating task ----------------------------------------------------------------------------------------------------

def test_saturating_climb():
    E, D, T = 256, 4, 24
    env = _saturating_env(E, D, seed=60)
    tgt = _climb(env)
    before = [t.clone() for t in (env._plane, env._wz, env._last_rpm)]
    p, sol = _solve_checked(env, tgt, T, 100, "motor")
    n = p.n
    hi = p.box[1]
    rpm = sol["rpm"].reshape(T, n, 4)
    at_hi = (rpm == hi).sum().item()
    print("B3: %d of %d rotor-ticks at MAX_RPM, %d at 0" % (at_hi, rpm.numel(), int((rpm == 0).sum())))
    assert at_hi >= n                                                # rotors really saturate: the test is not vacuous
    assert bool((rpm[0] == hi).any(dim=-1).float().mean() > 0.9)      # the climb starts at full thrust
    cost = sol["cost"]
    assert (cost[1:] <= cost[:-1]).all()
    roll = env.differentiable_rollout(rpm=sol["rpm"])
    for k in KEYS:
        assert torch.equal(sol[k], roll[k]), k
    act = sol["active"].reshape(T, n, 4)
    assert bool((act != 0).any())
    assert bool((sol["K"].reshape(T, n, 4, -1)[act != 0] == 0).all())
    worst, nconv = _kkt(env, p, sol, p.box[0], hi, "B3 climb")
    assert nconv >= n // 10
    assert worst <= 2e-3                                             # measured 6.2e-4 on an H100
    for a, b in zip(before, (env._plane, env._wz, env._last_rpm)):
        assert torch.equal(a, b)
    # the same task without bounds: a measurement
    free = env.ilqr(tgt, num_steps=T, iters=100)
    over = int((free["rpm"].reshape(T, n, 4) > hi).sum()) + int((free["rpm"] < 0).sum())
    print("B3 without bounds: final cost median %.4g (bounded %.4g), max %.4g (bounded %.4g); %d rotor-ticks outside [0, MAX_RPM]"
          % (free["cost"][-1].median(), cost[-1].median(), free["cost"][-1].max(), cost[-1].max(), over))


# ---- B4: tighter envelopes ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["derated", "cap_from_half", "idle_floor"])
def test_tighter_envelopes(kind):
    E, D, T = 64, 4, 24
    env = _saturating_env(E, D, "drag" if kind == "cap_from_half" else "dyn", seed=70)
    n, m, h = E * D, float(_max_rpm(env).min()), float(env.HOVER_RPM)
    tgt = _climb(env, 3.0 if kind == "cap_from_half" else 1.0)      # out of reach: thrust past T/2
    lo = torch.zeros((T, E, D, 4), **F64)
    hi = torch.full((T, E, D, 4), m, **F64)
    if kind == "derated":
        rotor = torch.arange(n, device=DEV) % 4
        hi.view(T, n, 4)[:, torch.arange(n, device=DEV), rotor] = 0.7 * m
        b = (lo[0], hi[0])                                           # [E, D, 4]: no time axis
    elif kind == "cap_from_half":
        hi[T // 2:] = 0.8 * m
        b = (lo, hi)
    else:
        lo.fill_(0.9 * h)
        b = (torch.full((4,), 0.9 * h, **F64), torch.full((E, D, 4), m, **F64))
    lo_n, hi_n = lo.reshape(T, n, 4), hi.reshape(T, n, 4)
    p, sol = _solve_checked(env, tgt, T, 100, b, lo=lo_n, hi=hi_n)
    rpm = sol["rpm"].reshape(T, n, 4)
    assert bool(((rpm >= lo_n) & (rpm <= hi_n)).all())
    tight = (hi_n < m) if kind != "idle_floor" else (lo_n > 0)
    on = (rpm == (hi_n if kind != "idle_floor" else lo_n)) & tight
    print("B4 %s: %d rotor-ticks on the tightened bound" % (kind, int(on.sum())))
    assert int(on.sum()) >= n // 4                                   # the tightened bound binds
    assert (sol["cost"][1:] <= sol["cost"][:-1]).all()
    worst, nconv = _kkt(env, p, sol, lo_n, hi_n, "B4 " + kind)
    assert nconv >= n // 10
    assert worst <= 2e-3                                             # measured <= 4.9e-4 on an H100


# ---- B5: the line search ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("physics", ["dyn", "drag"])
def test_line_search_against_the_clamped_rollout(physics):
    E, D, T = 8, 4, 24
    env = _saturating_env(E, D, physics, seed=80)
    p, _ = _solve_checked(env, _climb(env), T, 3, "motor")          # a nominal with saturated rotors
    assert bool((p.active != 0).any())
    n = p.n
    alphas = [1.0, 0.5, 0.25, 1e-3, 0.125]
    J = p.line_search(alpha=torch.tensor(alphas, **F64), out=torch.empty((len(alphas), n), **F64)).clone()
    r = _per_drone(p)
    Kd, S, eff = _consts(p)
    A = len(alphas)
    rep = lambda x, d: x.unsqueeze(d).expand(*x.shape[:d], A, *x.shape[d:]).reshape(*x.shape[:d], A * n, *x.shape[d + 1:])
    al = torch.tensor(alphas, **F64).repeat_interleave(n)
    lo, hi = p.box[0].expand(T, n, 4), p.box[1].expand(T, n, 4)
    args = (Kd, rep(r["rows"], 0), rep(r["x0"], 0), rep(r["last_rpm"], 0), rep(r["rpm"], 1), rep(r["xs"], 1), rep(r["K"], 1),
            rep(r["k"], 1), al, rep(r["tg"], 1), rep(r["W"], 1), rep(r["Rt"], 0), rep(r["uref"], 0), S, eff, rep(lo, 1), rep(hi, 1))
    ref = BR.rollout_cost_box(*args)["J"].reshape(A, n)
    bad = BR.rollout_cost_box(*args, clamp=False)["J"].reshape(A, n)
    e = ((J - ref).abs() / ref.abs()).max().item()
    e_bad = ((J - bad).abs() / bad.abs()).max().item()
    print("B5 %s: J(alpha) against the clamped restatement %.1e; unclamped %.1e" % (physics, e, e_bad))
    assert e <= 1e-10
    assert e_bad > 1e-6
    # dV1 = dJ/dalpha at 0+ (one-sided differences, Richardson-corrected for the alpha^2 term), at mu = 0 as for the
    # unconstrained pass.  Tassa's value update carries the k of held rotors into V_x, so dV1 is the slope where that k is 0
    # (the nominal on its bound); farther from the bound it is the model's, not the rollout's, first-order decrease.
    cost = torch.empty((2, n), **F64)
    p.cost(cost[0])
    for _ in range(60):                                              # near the solution: the nominal on its bounds
        p.line_search()
        p.commit(cost[0], cost[1])
        cost[0].copy_(cost[1])
        p.jacobians()
        p.backward()
    p.converged.zero_()                                              # the line search skips converged drones
    p.mu.zero_()
    p.backward()
    hs = torch.tensor([0.0, 1e-5, 2e-5], **F64)
    Jh = p.line_search(alpha=hs, out=torch.empty((3, n), **F64))
    slope = 2 * (Jh[1] - Jh[0]) / 1e-5 - (Jh[2] - Jh[0]) / 2e-5
    es = (slope - p.dV[:, 0]).abs() / p.dV[:, 0].abs()
    on_bound = ~((p.active != 0) & (p.k != 0)).any(dim=2).any(dim=0) & (p.status == 0) & (p.dV[:, 0] < 0)
    off = ~on_bound & (p.status == 0)
    print("B5 %s: dV1 against one-sided differences of J(alpha): %d drones with held k = 0, max %.1e; %d others, max %.1e"
          % (physics, int(on_bound.sum()), es[on_bound].max().item() if bool(on_bound.any()) else float("nan"), int(off.sum()),
             es[off].max().item() if bool(off.any()) else float("nan")))
    assert int(on_bound.sum()) >= 1
    assert es[on_bound].max().item() <= 1e-4


# ---- B6: the rest --------------------------------------------------------------------------------------------------------------

def test_drones_are_independent_and_deterministic():
    E, D, T = 21, 3, 20
    env = _saturating_env(E, D, "drag", seed=90)
    rng = np.random.default_rng(91)
    phys = _phys(env, rng)
    m = _max_rpm(env, phys).reshape(E, 1, 1)
    lo = torch.as_tensor(rng.uniform(0.0, 0.3, (E, D, 4)), **F64) * m
    hi = torch.as_tensor(rng.uniform(0.75, 1.0, (E, D, 4)), **F64) * m
    tgt = _climb(env)
    before = [t.clone() for t in (env._plane, env._wz, env._last_rpm, env.pos, env.vel)]
    sol = env.ilqr(tgt, num_steps=T, iters=6, phys=phys, rpm_bounds=(lo, hi))
    again = env.ilqr(tgt, num_steps=T, iters=6, phys=phys, rpm_bounds=(lo, hi))
    for k in sol:
        assert torch.equal(sol[k], again[k]), k
    for a, b in zip(before, (env._plane, env._wz, env._last_rpm, env.pos, env.vel)):
        assert torch.equal(a, b)
    assert bool((sol["active"] != 0).any())
    one = _saturating_env(1, 1, "drag", seed=90)
    for e, d in ((0, 0), (10, 2), (20, 1)):
        state = {k: getattr(env, k)[e:e + 1, d:d + 1].clone().to(torch.float64) for k in KEYS}
        alone = one.ilqr({"pos": tgt["pos"][e:e + 1, d:d + 1]}, num_steps=T, iters=6, state=state,
                         last_rpm=torch.zeros((1, 1, 4), **F64),
                         phys={k: v[e:e + 1] for k, v in phys.items()},
                         rpm_bounds=(lo[e:e + 1, d:d + 1].contiguous(), hi[e:e + 1, d:d + 1].contiguous()))
        for k in sol:
            got = sol[k][:, e, d] if sol[k].dim() >= 4 or k == "cost" else sol[k][e, d]
            want = alone[k][:, 0, 0] if alone[k].dim() >= 4 or k == "cost" else alone[k][0, 0]
            assert torch.equal(got, want), (k, e, d)


def test_morton_twin_matches_in_drone_id_order():
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils.enums import Physics
    from test_gpu_formation import stacks
    xyz = stacks(10, 9)[:333]
    xyz = xyz[np.random.default_rng(6).permutation(len(xyz))]
    a = CtrlAviary(num_drones=len(xyz), initial_xyzs=xyz, physics=Physics.PYB_DW, num_envs=1)
    b = CtrlAviary(num_drones=len(xyz), initial_xyzs=xyz, physics=Physics.DYN, num_envs=1)
    a.reset(); b.reset()
    order = a.reorder_by_morton().cpu().numpy()
    assert np.count_nonzero(order == np.arange(len(order))) < len(order) // 10
    a._effects = 0
    m = float(_max_rpm(b).min())
    hi = torch.as_tensor(np.random.default_rng(7).uniform(0.6, 1.0, (1, len(xyz), 4)) * m, **F64)
    lo = torch.zeros_like(hi)
    tgt = {"pos": torch.tensor(xyz + np.array([0.3, -0.2, 0.8]), device=DEV)[None]}
    sa = a.ilqr(tgt, num_steps=16, iters=4, rpm_bounds=(lo, hi))
    sb = b.ilqr(tgt, num_steps=16, iters=4, rpm_bounds=(lo, hi))
    assert bool((sa["active"] != 0).any())
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k


def test_commit_converges_a_drone_whose_k_is_zero():
    """The box commit sets converged (cost kept, mu unchanged) when dV1 = dV2 = 0, i.e. k = 0 at every tick, instead of raising
    mu: with every rotor held at a bound no step lowers J"""
    env = _saturating_env(4, 4, seed=97)
    p = _problem(env, 12, np.random.default_rng(98), rpm_bounds="motor")
    n = p.n
    cost = torch.empty((2, n), **F64)
    p.nominal()
    p.cost(cost[0])
    p.jacobians()
    p.backward()
    p.mu.fill_(0.5)
    p.dV[:3] = 0.0                                                   # drones 0..2: a stationary point
    p.dV[3, 1] = 0.0                                                 # drone 3: dV1 alone is not enough
    p.status[2] = 1                                                  # drone 2: a failed pass is never converged
    p.line_search()
    p.commit(cost[0], cost[1])
    conv, mu = p.converged.cpu().tolist(), p.mu.cpu().tolist()
    assert conv[:4] == [1, 1, 0, 0] and mu[:2] == [0.5, 0.5] and mu[2] == 5.0
    assert torch.equal(cost[1, :2], cost[0, :2])
    assert not any(conv[4:])


def test_one_synchronisation_per_solve():
    env = _saturating_env(4, 2, seed=95)
    tgt = _climb(env)
    counts = []
    for b in (None, "motor"):
        env.ilqr(tgt, num_steps=8, iters=2, rpm_bounds=b)         # warm: lazy initialisation outside the count
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("warn")
        try:
            with warnings.catch_warnings(record=True) as w:
                warnings.simplefilter("always")
                env.ilqr(tgt, num_steps=8, iters=2, rpm_bounds=b)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        counts.append(sum("synchroniz" in str(x.message) for x in w))
    print("synchronising calls per solve: without bounds %d, with bounds %d" % tuple(counts))
    assert counts[0] == counts[1] >= 1


def test_refusals():
    env = _saturating_env(2, 2, seed=96)
    E, D, T = 2, 2, 6
    m, h = float(_max_rpm(env).min()), float(env.HOVER_RPM)
    tgt = _climb(env)
    f = lambda v, shape=(4,): torch.full(shape, v, **F64)
    bad = [
        ((f(float("nan")), f(m)), "NaN"),
        ((f(0.0), f(float("nan"), (E, D, 4))), "NaN"),
        ((f(0.6 * m), f(0.5 * m)), "lo <= hi"),
        ((f(-1.0), f(m)), "0 <= lo"),
        ((f(0.0), f(m * (1 + 1e-12))), "MAX_RPM"),
        ((f(0.0, (T + 1, E, D, 4)), f(m)), "horizon"),
        ((f(0.0).float(), f(m)), "float64"),
        ((f(0.0).cpu(), f(m)), "must be on"),
        ((f(0.0, (E, 4)), f(m)), "rpm_bounds"),
        ((f(0.0, (E, D + 1, 4)), f(m)), "shape"),
        ((f(0.0),), "pair"),
        ("full", "pair"),
        ((0.0, m), "rpm_bounds"),
    ]
    for b, match in bad:
        with pytest.raises(ValueError, match=match):
            env.ilqr(tgt, num_steps=T, iters=1, rpm_bounds=b)
    # "motor" and the MAX_RPM check take each aviary's row: a larger kf lowers aviary 1's MAX_RPM
    phys = {"kf": torch.as_tensor([env.KF, env.KF * 1.2], **F64)}
    from gym_pybullet_drones_b200.ilqr import Problem
    p = Problem(env, tgt, num_steps=T, phys=phys, rpm_bounds="motor")
    assert torch.equal(p.box[1].view(E, D, 4)[:, 0, 0], p.rows[:, 13])
    with pytest.raises(ValueError, match="MAX_RPM"):
        env.ilqr(tgt, num_steps=T, iters=1, phys=phys, rpm_bounds=(f(0.0), f(float(p.rows[:, 13].max()))))
