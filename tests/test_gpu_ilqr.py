"""-m gpu: batched iLQR on the device (BaseAviary.ilqr, ilqr_backward_kernel / ilqr_line_search_kernel / ilqr_commit_kernel,
DESIGN.md 4.5.1).

Covered: the backward pass's predicted first-order decrease dV1 against central differences of the line search's J(alpha)
(with mu > 0 as the negative control); the backward pass against the float64 restatement tests/ilqr_ref.py at the device's own
Jacobians for DYN, GND, DRAG and GND|DRAG, CF2X and CF2P; the returned trajectory against differentiable_rollout bit for bit, the
commit's J against the line search's and the alpha = 0 rollout against the nominal; non-increasing cost; a formation task with
K = 0 as the negative control; independence of the drones, a Morton-reordered twin, partial CTAs, determinism and an untouched
env; and the refusals."""
import numpy as np
import pytest
import torch

import ilqr_ref as IR

pytestmark = pytest.mark.gpu

DEV = "cuda"
KEYS = ("pos", "quat", "vel", "rpy_rates")
PHYSICS = {"dyn": ("DYN", None), "gnd": ("PYB_GND", None), "drag": ("PYB_DRAG", None), "gnd_drag": ("PYB_GND_DRAG_DW", 3)}


def _imports():
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils.enums import DroneModel, Physics
    return CtrlAviary, DroneModel, Physics


def _env(E, D, physics="dyn", model="CF2X", pyb=240, ctrl=48, seed=0, **kw):
    CtrlAviary, DroneModel, Physics = _imports()
    name, effects = PHYSICS[physics]
    rng = np.random.default_rng(seed)
    xyz = np.stack([rng.uniform(-1, 1, D), rng.uniform(-1, 1, D), rng.uniform(0.3, 1.5, D)], 1)
    env = CtrlAviary(drone_model=getattr(DroneModel, model), num_drones=D, physics=getattr(Physics, name), pyb_freq=pyb, ctrl_freq=ctrl,
                     initial_xyzs=xyz, initial_rpys=rng.uniform(-0.3, 0.3, (D, 3)), num_envs=E, **kw)
    env.reset()
    if effects is not None:
        env._effects = effects                       # GND|DRAG without the downwash of PYB_GND_DRAG_DW
    return env


def _targets(env, seed, spread=0.5):
    rng = np.random.default_rng(seed)
    E, D = env._E, env._D
    return {"pos": torch.tensor(rng.uniform(-spread, spread, (E, D, 3)) + np.array([0.0, 0.0, 1.0]), device=DEV)}


def _guess(env, T, seed, spread=0.03):
    rng = np.random.default_rng(seed)
    return torch.tensor(env.HOVER_RPM * (1 + spread * rng.uniform(-1, 1, (T, env._E, env._D, 4))), device=DEV)


def _problem(env, T, seed, **kw):
    from gym_pybullet_drones_b200.ilqr import Problem
    return Problem(env, _targets(env, seed), rpm=_guess(env, T, seed + 1), **kw)


def _vec(planes, n):
    from gym_pybullet_drones_b200.diff import unpack_states
    u = unpack_states(planes, n)
    return torch.cat([u[k] for k in KEYS], dim=-1)


# ---- G1: dV1 is dJ/dalpha at alpha = 0 --------------------------------------------------------------------------------------

@pytest.mark.parametrize("physics", ["dyn", "drag"])
def test_dV1_is_the_line_search_slope(physics):
    env = _env(16, 4, physics, seed=1)
    h = 1e-6
    slopes = {}
    for mu in (0.0, 1.0):
        p = _problem(env, 24, 2)
        p.nominal()
        p.jacobians()
        p.mu.fill_(mu)
        p.backward()
        assert int(p.status.sum()) == 0
        J = p.line_search(alpha=torch.tensor([h, -h], dtype=torch.float64, device=DEV), out=torch.empty((2, p.n), dtype=torch.float64, device=DEV))
        fd = (J[0] - J[1]) / (2 * h)
        slopes[mu] = ((fd - p.dV[:, 0]).abs() / p.dV[:, 0].abs()).max().item()
        assert (p.dV[:, 0] < 0).all()                  # a descent direction
    print("dV1 against dJ/dalpha (%s): mu = 0 %.1e, mu = 1 %.1e" % (physics, slopes[0.0], slopes[1.0]))
    assert slopes[0.0] <= 1e-6
    assert slopes[1.0] > 1e-4                          # negative control: Tassa's update with a regularised K is not the slope


# ---- G2: the backward pass against the float64 restatement ------------------------------------------------------------------

@pytest.mark.parametrize("model", ["CF2X", "CF2P"])
@pytest.mark.parametrize("physics", list(PHYSICS))
def test_backward_matches_reference(model, physics):
    env = _env(8, 4, physics, model, seed=3)
    p = _problem(env, 16, 4)
    p.nominal()
    p.jacobians()
    p.backward()
    T, n, D = p.T, p.n, env._D
    rows = p.rows.repeat_interleave(D, dim=0)
    raw = p.rpm
    F = IR.f_from_jac(p.jac, raw, rows[:, 13].expand(T, n))
    dx = _vec(p.states, n) - _vec(p.targets, n)
    w = p.weights.repeat_interleave(D, dim=0)
    W = torch.stack([w[:, :13]] * (T - 1) + [w[:, 13:26]])
    Rt = w[:, 26:30] / rows[:, 12:13] ** 2
    ref = IR.backward_pass(F, dx, W, Rt, raw - p.rpm_ref, p.mu)
    rel = lambda a, b: ((a - b).flatten(2).norm(dim=-1) / b.flatten(2).norm(dim=-1).clamp_min(1e-300)).max().item()
    eK, ek = rel(p.K, ref["K"]), rel(p.k[..., None], ref["k"][..., None])
    e1 = ((p.dV[:, 0] - ref["dV1"]).abs() / ref["dV1"].abs()).max().item()
    e2 = ((p.dV[:, 1] - ref["dV2"]).abs() / ref["dV2"].abs()).max().item()
    print("backward %s %s: K %.1e k %.1e dV1 %.1e dV2 %.1e" % (model, physics, eK, ek, e1, e2))
    assert int(p.status.sum()) == 0 and bool(ref["ok"].all())
    assert max(eK, ek, e1, e2) <= 1e-10


# ---- G3 / G4: bits of the result, monotone cost -----------------------------------------------------------------------------

@pytest.mark.parametrize("physics", list(PHYSICS))
def test_result_is_differentiable_rollout_and_cost_decreases(physics):
    env = _env(12, 3, physics, seed=5)
    tgt, guess = _targets(env, 6), _guess(env, 32, 7)
    sol = env.ilqr(tgt, rpm=guess, iters=6)
    roll = env.differentiable_rollout(rpm=sol["rpm"])
    for k in KEYS:
        assert torch.equal(sol[k], roll[k]), k
    cost = sol["cost"]
    assert cost.shape == (7, 12, 3)
    assert (cost[1:] <= cost[:-1]).all()
    assert (cost[-1] < cost[0]).all()
    assert sol["K"].shape == (32, 12, 3, 4, 17 if "drag" in physics else 13) and sol["k"].shape == (32, 12, 3, 4)
    assert sol["rpm"].grad_fn is None and not sol["K"].requires_grad


@pytest.mark.parametrize("physics", ["dyn", "gnd_drag"])
def test_commit_takes_the_line_search_bits(physics):
    env = _env(10, 5, physics, seed=8)
    p = _problem(env, 20, 9)
    f64 = dict(dtype=torch.float64, device=DEV)
    cost = torch.empty((3, p.n), **f64)
    p.nominal()
    p.cost(cost[0])
    p.jacobians()
    p.backward()
    # alpha = 0 with the feedback applied reproduces the nominal: its J has the nominal's bits
    J0 = p.line_search(alpha=torch.zeros((1,), **f64), out=torch.empty((1, p.n), **f64))
    assert torch.equal(J0[0], cost[0])
    states0 = p.states.clone()
    J = p.line_search().clone()
    p.commit(cost[0], cost[1])
    moved = cost[1] < cost[0]
    assert moved.float().mean().item() > 0.9
    assert ((J == cost[1]).any(dim=0) | ~moved).all()  # a committed J is one of the line search's, bit for bit
    # the nominal's own J after the commit: the rollout of the committed rpm
    p.cost(cost[2])
    assert torch.equal(cost[2], cost[1])
    assert not torch.equal(states0, p.states)


# ---- G5: a formation task ----------------------------------------------------------------------------------------------------

def _task(feedback):
    from gym_pybullet_drones_b200.ilqr import Problem, solve
    from gym_pybullet_drones_b200.params import quaternion_from_euler
    E, D = 1024, 4
    env = _env(E, D, "dyn", ctrl=48, seed=10)
    rng = np.random.default_rng(11)
    n = E * D
    start = np.array([0.0, 0.0, 1.0]) + rng.uniform(-0.5, 0.5, (n, 3)) / np.sqrt(3)
    quat = np.stack([quaternion_from_euler(r) for r in rng.uniform(-0.3, 0.3, (n, 3)) / np.sqrt(3)])
    state = {"pos": torch.tensor(start, device=DEV).reshape(E, D, 3), "quat": torch.tensor(quat, device=DEV).reshape(E, D, 4),
             "vel": torch.zeros((E, D, 3), dtype=torch.float64, device=DEV), "rpy_rates": torch.zeros((E, D, 3), dtype=torch.float64, device=DEV)}
    goal = np.array([0.0, 0.0, 1.0]) + rng.uniform(-0.5, 0.5, (n, 3)) / np.sqrt(3)
    target = {"pos": torch.tensor(goal, device=DEV).reshape(E, D, 3)}
    p = Problem(env, target, num_steps=96, state=state)
    p.feedback = feedback
    sol = solve(p, 30)
    err = (sol["pos"][-1] - target["pos"]).norm(dim=-1)
    speed = sol["vel"][-1].norm(dim=-1)
    return sol, err, speed


def test_formation_task_reaches_every_target():
    sol, err, speed = _task(True)
    print("task: worst final position error %.2e m, worst final speed %.2e m/s, converged %d / %d, worst mu %.1e"
          % (err.max().item(), speed.max().item(), int(sol["converged"].sum()), sol["converged"].numel(), sol["mu"].max().item()))
    assert err.max().item() <= 0.01
    assert speed.max().item() <= 0.05
    assert (sol["cost"][1:] <= sol["cost"][:-1]).all()
    _, err0, speed0 = _task(False)
    print("task with K = 0: worst final position error %.2e m, worst final speed %.2e m/s" % (err0.max().item(), speed0.max().item()))
    assert err0.max().item() > 0.01 or speed0.max().item() > 0.05


# ---- G6: independence, layout, determinism -----------------------------------------------------------------------------------

def _phys(env, seed):
    rng = np.random.default_rng(seed)
    E = env._E
    return {"m": torch.tensor(env.M * rng.uniform(0.8, 1.2, E), device=DEV), "kf": torch.tensor(env.KF * rng.uniform(0.8, 1.2, E), device=DEV)}


def _snapshot(env):
    return [t.clone() for t in (env._plane, env._wz, env._last_rpm, env.pos, env.vel)]


def test_drones_are_independent_and_deterministic():
    E, D, T = 37, 3, 20
    env = _env(E, D, "drag", seed=12)
    phys = _phys(env, 13)
    tgt, guess = _targets(env, 14), _guess(env, T, 15)
    before = _snapshot(env)
    sol = env.ilqr(tgt, rpm=guess, iters=5, phys=phys)
    again = env.ilqr(tgt, rpm=guess, iters=5, phys=phys)
    for k in sol:
        assert torch.equal(sol[k], again[k]), k
    for a, b in zip(before, _snapshot(env)):
        assert torch.equal(a, b)
    one = _env(1, 1, "drag", seed=12)
    for e, d in ((0, 0), (17, 2), (36, 1)):
        state = {k: getattr(env, k)[e:e + 1, d:d + 1].clone() for k in KEYS}
        alone = one.ilqr({"pos": tgt["pos"][e:e + 1, d:d + 1]}, rpm=guess[:, e:e + 1, d:d + 1].contiguous(), iters=5, state=state,
                         last_rpm=torch.zeros((1, 1, 4), dtype=torch.float64, device=DEV),
                         phys={k: v[e:e + 1] for k, v in phys.items()})
        for k in sol:
            got = sol[k][:, e, d] if sol[k].dim() >= 4 or k == "cost" else sol[k][e, d]
            want = alone[k][:, 0, 0] if alone[k].dim() >= 4 or k == "cost" else alone[k][0, 0]
            assert torch.equal(got, want), (k, e, d)


def test_morton_twin_matches_in_drone_id_order():
    CtrlAviary, _, Physics = _imports()
    from test_gpu_formation import stacks
    xyz = stacks(10, 9)[:333]
    xyz = xyz[np.random.default_rng(5).permutation(len(xyz))]
    a = CtrlAviary(num_drones=len(xyz), initial_xyzs=xyz, physics=Physics.PYB_DW, num_envs=1)
    b = CtrlAviary(num_drones=len(xyz), initial_xyzs=xyz, physics=Physics.DYN, num_envs=1)
    a.reset(); b.reset()
    order = a.reorder_by_morton().cpu().numpy()          # a formation large enough to re-bin is a downwash formation
    assert np.count_nonzero(order == np.arange(len(order))) < len(order) // 10
    with pytest.raises(ValueError, match="downwash"):
        a.ilqr({"pos": torch.tensor(xyz, device=DEV)[None]}, num_steps=4)
    a._effects = 0
    tgt = {"pos": torch.tensor(xyz + np.array([0.3, -0.2, 0.4]), device=DEV)[None]}
    sa, sb = a.ilqr(tgt, num_steps=16, iters=4), b.ilqr(tgt, num_steps=16, iters=4)
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k


# ---- G7: refusals -------------------------------------------------------------------------------------------------------------

def test_refusals():
    CtrlAviary, _, Physics = _imports()
    env = _env(2, 2, "dyn", seed=16)
    tgt = {"pos": torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64, device=DEV)}
    dw = CtrlAviary(num_drones=2, physics=Physics.PYB_DW, num_envs=2)
    with pytest.raises(ValueError, match="downwash"):
        dw.ilqr(tgt, num_steps=4)
    bad = [
        (dict(target=tgt), "horizon"),
        (dict(target=tgt, num_steps=0), "T must be > 0"),
        (dict(target=tgt, num_steps=4, iters=-1), "iters"),
        (dict(target=tgt, num_steps=4, rpm=torch.zeros((5, 2, 2, 4), dtype=torch.float64, device=DEV)), "disagree"),
        (dict(target={"pos": torch.zeros((6, 2, 2, 3), dtype=torch.float64, device=DEV)}, num_steps=4), "disagree"),
        (dict(target={"quat": tgt["pos"]}, num_steps=4), "pos"),
        (dict(target={"pos": tgt["pos"], "acc": tgt["pos"]}, num_steps=4), "unknown target"),
        (dict(target={"pos": torch.zeros((2, 3), dtype=torch.float64, device=DEV)}, num_steps=4), "shape"),
        (dict(target={"pos": tgt["pos"].float()}, num_steps=4), "float64"),
        (dict(target={"pos": tgt["pos"].cpu()}, num_steps=4), "cuda"),
        (dict(target=tgt, num_steps=4, Q=-torch.ones(13, dtype=torch.float64, device=DEV)), ">= 0"),
        (dict(target=tgt, num_steps=4, Q_final=torch.full((13,), float("nan"), dtype=torch.float64, device=DEV)), ">= 0"),
        (dict(target=tgt, num_steps=4, R=torch.zeros(4, dtype=torch.float64, device=DEV)), "R finite and > 0"),
        (dict(target=tgt, num_steps=4, R=torch.ones((3, 4), dtype=torch.float64, device=DEV)), "shape"),
        (dict(target=tgt, num_steps=4, rpm_ref=torch.ones(3, dtype=torch.float64, device=DEV)), "shape"),
    ]
    for kw, msg in bad:
        with pytest.raises(ValueError, match=msg):
            env.ilqr(**kw)
    sol = env.ilqr(tgt, num_steps=4, iters=0)           # iters = 0: the guess, its cost and its gains
    assert sol["cost"].shape == (1, 2, 2) and sol["K"].shape == (4, 2, 2, 4, 13)


def test_indefinite_quu_sets_the_status():
    """Through the ABI (the public call refuses R <= 0): a negative R makes Quu indefinite at every tick; the backward raises mu
    8 times, marks the drone failed, and the line search and the commit leave it alone."""
    env = _env(1, 4, "dyn", seed=17)
    p = _problem(env, 8, 18)
    p.weights[:, 26:30] = -1e6
    f64 = dict(dtype=torch.float64, device=DEV)
    cost = torch.empty((2, p.n), **f64)
    p.nominal()
    p.cost(cost[0])
    p.jacobians()
    p.backward()
    assert (p.status == 1).all()
    assert torch.allclose(p.mu, torch.full_like(p.mu, 1e-6 * 10.0 ** 8), rtol=1e-12)
    rpm0 = p.rpm.clone()
    assert torch.isinf(p.line_search()).all()
    p.commit(cost[0], cost[1])
    assert torch.equal(cost[1], cost[0]) and torch.equal(p.rpm, rpm0)
