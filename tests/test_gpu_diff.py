"""-m gpu: BaseAviary.differentiable_rollout (qs_dyn_traj / qs_dyn_traj_vjp, DESIGN.md 4.5).

The forward is held to T CtrlAviary.step() calls and to CtrlAviary.rollout() bit for bit, the env to its own bits afterwards;
the gradients to the autograd of the float64 torch reference tests/diff_ref.py on the same device (normwise relative per input
block), to torch.autograd.gradcheck, to themselves (determinism) and, through a Morton-reordered formation, to a twin that was
never reordered.  A system-identification fit recovers per-aviary mass and motor constant from recorded flights."""
import numpy as np
import pytest
import torch

import diff_ref as R

pytestmark = pytest.mark.gpu

GRAD_TOL = 1e-9


def _imports():
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.params import PHYS_KEYS, physical_rows
    from gym_pybullet_drones_b200.utils.enums import DroneModel, Physics
    return CtrlAviary, Physics, DroneModel, PHYS_KEYS, physical_rows


def _env(E, D, physics, model, pyb=240, ctrl=240, **kw):
    CtrlAviary, Physics, DroneModel, _, _ = _imports()
    rng = np.random.default_rng(E * 1000 + D)
    xyz = np.stack([rng.uniform(-1, 1, D), rng.uniform(-1, 1, D), rng.uniform(0.02, 1.0, D)], 1)
    rpy = rng.uniform(-0.3, 0.3, (D, 3))
    env = CtrlAviary(drone_model=getattr(DroneModel, model), num_drones=D, physics=getattr(Physics, physics), pyb_freq=pyb,
                     ctrl_freq=ctrl, initial_xyzs=xyz, initial_rpys=rpy, num_envs=E, **kw)
    env.reset()
    return env


def _rpm(env, T, rng, spread=0.05, clip=True):
    r = env.HOVER_RPM * (1 + spread * rng.uniform(-1, 1, (T, env._E, env._D, 4)))
    if clip:                                             # commands beyond the clip on both sides, in the last two ticks (sustained,
        r[-2:, :, 0, 0] = env.MAX_RPM * 1.2              # they would tumble the drone within a second)
        r[-2:, :, -1, 3] = -100.0
    return torch.tensor(r, device=env.device)


def _snapshot(env):
    t = [env._planes, env._last_rpm, env._step_counter, env._obs_buf[0], env._obs_buf[1], env._reward]
    if env._phys is not None:
        t += [env._phys, env._phys_props]
    return [x.clone() for x in t] + [env._cur]


def _same(a, b):
    for x, y in zip(a, b):
        assert (x == y) if not isinstance(x, torch.Tensor) else torch.equal(x, y)


FWD_CASES = [("DYN", "CF2X", 240, 48), ("PYB", "CF2P", 240, 240), ("PYB_GND", "RACE", 240, 30), ("PYB_DRAG", "CF2X", 240, 30),
             ("PYB_GND", "CF2X", 240, 48), ("PYB_DRAG", "RACE", 240, 240), ("DYN", "CF2P", 240, 30), ("PYB_GND", "CF2P", 240, 240)]


@pytest.mark.parametrize("physics,model,pyb,ctrl", FWD_CASES)
@pytest.mark.parametrize("table", [False, True])
@pytest.mark.parametrize("T", [1, 6])
def test_forward_bit_identical_to_step_and_rollout(physics, model, pyb, ctrl, table, T):
    E, D = 3, 11                                           # 33 drones: not a multiple of 32
    env = _env(E, D, physics, model, pyb, ctrl)
    rng = np.random.default_rng(T)
    if table:
        env.set_physical_params(m=env.M * rng.uniform(0.8, 1.2, E), kf=env.KF * rng.uniform(0.8, 1.2, E),
                                ixx=env.J[0, 0] * rng.uniform(0.8, 1.2, E))
    for _ in range(2):                                     # a non-trivial start (and last_clipped_action)
        env.step(_rpm(env, 1, rng)[0])
    rpm = _rpm(env, T, rng)
    before = _snapshot(env)
    out = env.differentiable_rollout(rpm)
    _same(before, _snapshot(env))
    twin_state = [t.clone() for t in (env.pos, env.quat, env.vel, env.rpy_rates)]
    for k in range(T):
        env.step(rpm[k])
        assert torch.equal(out["pos"][k], env.pos) and torch.equal(out["quat"][k], env.quat)
        assert torch.equal(out["vel"][k], env.vel) and torch.equal(out["rpy_rates"][k], env.rpy_rates)
    env.set_state(*twin_state)
    env._last_rpm.copy_(before[1])
    env.rollout(actions=rpm, record=False)
    for key in ("pos", "quat", "vel", "rpy_rates"):
        assert torch.equal(out[key][-1], getattr(env, key)), key


def _ref_grads(env, rpm, state, last, props, g, effects):
    """diff_ref on the device: the reference gradients for the inputs of differentiable_rollout."""
    _, _, _, PHYS_KEYS, physical_rows = _imports()
    E, D, n, T = env._E, env._D, env._N, rpm.shape[0]
    leaves = [rpm] + [state[k] for k in ("pos", "quat", "vel", "rpy_rates")] + [last] + [props[k] for k in PHYS_KEYS]
    leaves = [x.detach().clone().requires_grad_(True) for x in leaves]
    r, pos, quat, vel, w, lr = leaves[:6]
    pr = dict(zip(PHYS_KEYS, leaves[6:]))
    rows = physical_rows(env.DRONE_MODEL, pr, env.G).repeat_interleave(D, dim=0)
    x0 = torch.cat([pos.reshape(n, 3), quat.reshape(n, 4), vel.reshape(n, 3), w.reshape(n, 3)], 1)
    out = R.rollout(R.model_constants(env._P, env.device), rows, x0, r.reshape(T, n, 4), lr.reshape(n, 4), env.PYB_STEPS_PER_CTRL, effects)
    loss = (out * torch.cat([g[k].reshape(T, n, -1) for k in ("pos", "quat", "vel", "rpy_rates")], 2)).sum()
    gs = torch.autograd.grad(loss, leaves, allow_unused=True)          # last_rpm is unused without drag
    return [torch.zeros_like(x) if g is None else g for g, x in zip(gs, leaves)]


@pytest.mark.parametrize("physics,model,effects", [("DYN", "CF2X", 0), ("PYB_GND", "CF2P", 1), ("PYB_DRAG", "RACE", 2)])
def test_gradients_match_reference_4096_drones(physics, model, effects):
    _, _, _, PHYS_KEYS, _ = _imports()
    E, D, T = 2048, 2, 32
    env = _env(E, D, physics, model, 240, 30)
    rng = np.random.default_rng(11)
    dev = env.device
    props = {k: v * torch.tensor(rng.uniform(0.8, 1.2, E), device=dev) for k, v in env.physical_params().items()}
    state = {"pos": env.pos.clone(), "quat": env.quat.clone(), "vel": torch.tensor(rng.uniform(-1, 1, (E, D, 3)), device=dev),
             "rpy_rates": torch.tensor(rng.uniform(-2, 2, (E, D, 3)), device=dev)}
    last = torch.tensor(env.HOVER_RPM * rng.uniform(0.9, 1.1, (E, D, 4)), device=dev)
    rpm = _rpm(env, T, rng)
    leaves = [rpm] + [state[k] for k in ("pos", "quat", "vel", "rpy_rates")] + [last] + [props[k] for k in PHYS_KEYS]
    leaves = [x.clone().requires_grad_(True) for x in leaves]
    st = dict(zip(("pos", "quat", "vel", "rpy_rates"), leaves[1:5]))
    out = env.differentiable_rollout(leaves[0], state=st, last_rpm=leaves[5], phys=dict(zip(PHYS_KEYS, leaves[6:])))
    g = {k: torch.tensor(rng.standard_normal(tuple(v.shape)), device=dev) for k, v in out.items()}
    got = torch.autograd.grad(sum((out[k] * g[k]).sum() for k in out), leaves)
    want = _ref_grads(env, rpm, state, last, props, g, effects)
    names = ["rpm", "pos", "quat", "vel", "rpy_rates", "last_rpm"] + list(PHYS_KEYS)
    worst = {}
    for name, a, b in zip(names, got, want):
        worst[name] = R.relerr(a, b)
    print("worst normwise relative error per block (%s %s): %s" % (physics, model, {k: "%.1e" % v for k, v in worst.items()}))
    for name, e in worst.items():
        if name == "last_rpm" and not effects & 2:          # only drag reads it
            assert float(got[5].abs().max()) == 0.0
        else:
            assert e <= GRAD_TOL, (name, e)


def test_gradcheck_tumbling():
    env = _env(2, 2, "PYB_DRAG", "CF2X", 240, 48)
    rng = np.random.default_rng(3)
    dev = env.device
    w = np.concatenate([rng.uniform(-5, 5, (2, 2, 2)), rng.uniform(250, 300, (2, 2, 1))], 2)
    x = [_rpm(env, 3, rng, 0.05, clip=False), env.pos.clone(), env.quat.clone(), torch.tensor(rng.uniform(-1, 1, (2, 2, 3)), device=dev),
         torch.tensor(w, device=dev), torch.tensor(env.HOVER_RPM * rng.uniform(0.9, 1.1, (2, 2, 4)), device=dev),
         torch.ones(2, dtype=torch.float64, device=dev), torch.ones(2, dtype=torch.float64, device=dev)]
    x = [t.detach().clone().requires_grad_(True) for t in x]

    def f(rpm, pos, quat, vel, rates, last, m_scale, kf_scale):      # gradcheck's absolute eps: the constants as O(1) factors
        o = env.differentiable_rollout(rpm, state=dict(pos=pos, quat=quat, vel=vel, rpy_rates=rates), last_rpm=last,
                                       phys=dict(m=env.M * m_scale, kf=env.KF * kf_scale))
        return o["pos"], o["quat"], o["vel"], o["rpy_rates"]

    assert torch.autograd.gradcheck(f, tuple(x), eps=1e-6, atol=1e-5, rtol=1e-4)


def test_backward_is_deterministic():
    env = _env(64, 4, "PYB_DRAG", "CF2X", 240, 48)
    rng = np.random.default_rng(4)
    rpm = _rpm(env, 8, rng).requires_grad_(True)
    m = env.physical_params()["m"].requires_grad_(True)
    out = env.differentiable_rollout(rpm, phys={"m": m})
    loss = out["pos"].square().sum() + out["quat"][..., 0].sum()
    a = torch.autograd.grad(loss, (rpm, m), retain_graph=True)
    b = torch.autograd.grad(loss, (rpm, m))
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_morton_reordered_formation_gradients_in_drone_id_order():
    """reorder_by_morton() needs a downwash formation; the rollout refuses downwash, so the reordered env's effects are switched
    to plain DYN after the reorder (the id mapping is what is under test) and compared with a DYN twin never reordered."""
    CtrlAviary, Physics, _, _, _ = _imports()
    from test_gpu_formation import stacks
    xyz = stacks(10, 9)[:333]
    xyz = xyz[np.random.default_rng(5).permutation(len(xyz))]
    a = CtrlAviary(num_drones=len(xyz), initial_xyzs=xyz, physics=Physics.PYB_DW, num_envs=1)
    b = CtrlAviary(num_drones=len(xyz), initial_xyzs=xyz, physics=Physics.DYN, num_envs=1)
    a.reset(); b.reset()
    order = a.reorder_by_morton().cpu().numpy()
    assert np.count_nonzero(order == np.arange(len(order))) < len(order) // 10
    with pytest.raises(ValueError, match="downwash"):
        a.differentiable_rollout(_rpm(a, 2, np.random.default_rng(0)))
    a._effects = 0
    rng = np.random.default_rng(6)
    rpm = _rpm(b, 4, rng)
    grads = []
    for env in (a, b):
        r = rpm.clone().requires_grad_(True)
        v = env.vel.clone().requires_grad_(True)
        out = env.differentiable_rollout(r, state={"vel": v})
        loss = (out["pos"] * torch.arange(1, out["pos"].numel() + 1, device=r.device, dtype=torch.float64).view_as(out["pos"])).sum()
        grads.append(torch.autograd.grad(loss, (r, v)) + (out["pos"].detach(),))
    for x, y in zip(grads[0], grads[1]):
        assert torch.equal(x, y)


def test_system_identification_recovers_mass_and_motor_constant():
    """256 aviaries with m and kf within +-30 % fly recorded random-RPM flights with step(); fitting log-ratios from the nominal
    values with L-BFGS on differentiable_rollout gradients recovers both to 1e-3 relative within a fixed iteration budget."""
    E, T = 256, 24
    env = _env(E, 1, "DYN", "CF2X", 240, 48)
    rng = np.random.default_rng(7)
    dev = env.device
    m_true = torch.tensor(env.M * rng.uniform(0.7, 1.3, E), device=dev)
    kf_true = torch.tensor(env.KF * rng.uniform(0.7, 1.3, E), device=dev)
    env.set_physical_params(m=m_true, kf=kf_true)
    start = {k: getattr(env, k).clone() for k in ("pos", "quat", "vel", "rpy_rates")}
    last = env.last_clipped_action.clone()
    rpm = _rpm(env, T, rng, 0.1, clip=False)
    rec = {k: [] for k in start}
    for k in range(T):
        env.step(rpm[k])
        for key in rec:
            rec[key].append(getattr(env, key).clone())
    rec = {k: torch.stack(v) for k, v in rec.items()}
    env.set_physical_params(m=env.M, kf=env.KF)              # the fit starts from the nominal model
    theta = torch.zeros((2, E), dtype=torch.float64, device=dev, requires_grad=True)
    opt = torch.optim.LBFGS([theta], lr=1, max_iter=200, history_size=20, tolerance_grad=1e-14, tolerance_change=1e-20,
                            line_search_fn="strong_wolfe")

    def closure():
        opt.zero_grad()
        out = env.differentiable_rollout(rpm, state=start, last_rpm=last,
                                         phys={"m": env.M * torch.exp(theta[0]), "kf": env.KF * torch.exp(theta[1])})
        loss = ((out["pos"] - rec["pos"]) / 1e-3).square().sum() + ((out["quat"] - rec["quat"]) / 1e-3).square().sum()
        loss.backward()
        return loss

    for _ in range(3):
        opt.step(closure)
    m_fit, kf_fit = env.M * torch.exp(theta[0].detach()), env.KF * torch.exp(theta[1].detach())
    em = float(((m_fit - m_true) / m_true).abs().max())
    ek = float(((kf_fit - kf_true) / kf_true).abs().max())
    print("system identification: worst relative error m %.1e, kf %.1e" % (em, ek))
    assert em < 1e-3 and ek < 1e-3


def test_refusals():
    CtrlAviary, Physics, _, _, _ = _imports()
    env = _env(2, 2, "DYN", "CF2X")
    rng = np.random.default_rng(8)
    rpm = _rpm(env, 2, rng)
    with pytest.raises(ValueError, match="float64"):
        env.differentiable_rollout(rpm.float())
    with pytest.raises(ValueError, match="shape"):
        env.differentiable_rollout(rpm[:, :, :1])
    with pytest.raises(ValueError):
        env.differentiable_rollout(rpm[0])
    with pytest.raises(ValueError, match="cuda|cpu"):
        env.differentiable_rollout(rpm.cpu())
    with pytest.raises(ValueError, match="shape"):
        env.differentiable_rollout(rpm, state={"pos": torch.zeros((2, 2, 4), dtype=torch.float64, device=env.device)})
    with pytest.raises(ValueError, match="unknown"):
        env.differentiable_rollout(rpm, state={"position": env.pos})
    with pytest.raises(ValueError, match="float64"):
        env.differentiable_rollout(rpm, phys={"m": env.physical_params()["m"].float()})
    with pytest.raises(ValueError, match="unknown"):
        env.differentiable_rollout(rpm, phys={"mass": env.physical_params()["m"]})
    with pytest.raises(ValueError, match="cuda|cpu"):
        env.differentiable_rollout(rpm, last_rpm=torch.zeros((2, 2, 4), dtype=torch.float64))
    dw = CtrlAviary(num_drones=2, physics=Physics.PYB_DW, num_envs=2)
    with pytest.raises(ValueError, match="downwash"):
        dw.differentiable_rollout(rpm)
    r = rpm.clone().requires_grad_(True)
    out = env.differentiable_rollout(r)
    with pytest.raises(ValueError, match="double backward"):
        torch.autograd.grad(out["pos"].sum(), r, create_graph=True)
