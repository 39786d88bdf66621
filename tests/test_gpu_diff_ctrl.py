"""-m gpu: BaseAviary.differentiable_rollout(controller=DSLPIDControl) (qs_dyn_ctrl_traj / qs_dyn_ctrl_traj_vjp, DESIGN.md 4.5).

The forward is held to CtrlAviary.rollout(controller=...) and to T x (computeControlFromEnv + step) bit for bit, the env and the
controller to their own bits afterwards; the gradients to the autograd of the float64 torch reference tests/diff_pid_ref.py on the
same device (normwise relative per input block), to torch.autograd.gradcheck, to themselves (determinism) and, through a
Morton-reordered formation, to a twin that was never reordered.  A gain-identification fit recovers per-aviary position-loop P
and D gains from recorded closed-loop flights."""

import numpy as np
import pytest
import torch

import diff_pid_ref as PR
import diff_ref as R

pytestmark = pytest.mark.gpu

GRAD_TOL = 1e-9
STATE_KEYS = ("pos", "quat", "vel", "rpy_rates")
GAIN_KEYS = ("P_COEFF_FOR", "I_COEFF_FOR", "D_COEFF_FOR", "P_COEFF_TOR", "I_COEFF_TOR", "D_COEFF_TOR")
PID_KEYS = ("integral_pos_e", "last_rpy", "integral_rpy_e")


def _imports():
    from gym_pybullet_drones_b200.control import DSLPIDControl
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils.enums import DroneModel, Physics
    return DSLPIDControl, CtrlAviary, DroneModel, Physics


def _env(E, D, physics="DYN", model="CF2X", pyb=240, ctrl=48, seed=0, **kw):
    DSLPIDControl, CtrlAviary, DroneModel, Physics = _imports()
    rng = np.random.default_rng(seed)
    xyz = np.stack([rng.uniform(-1, 1, D), rng.uniform(-1, 1, D), rng.uniform(0.05, 1.0, D)], 1)
    env = CtrlAviary(drone_model=DroneModel[model], num_drones=D, physics=Physics[physics], pyb_freq=pyb, ctrl_freq=ctrl,
                     initial_xyzs=xyz, initial_rpys=rng.uniform(-0.1, 0.1, (D, 3)), num_envs=E, **kw)
    env.reset()
    ctl = DSLPIDControl(DroneModel[model], num_drones=E * D, device=env.device)
    return env, ctl


def _circle(W, E, D, per_drone, rng, dev):
    i = np.arange(W)
    c = np.stack([0.3 * np.cos(2 * np.pi * i / W), 0.3 * np.sin(2 * np.pi * i / W), 0.2 * np.sin(4 * np.pi * i / W)], 1)
    if per_drone:
        c = c[:, None, None, :] + rng.uniform(-0.05, 0.05, (1, E, D, 3))
    return torch.tensor(c, device=dev)


def _snapshot(env, ctl):
    t = [env._planes, env._last_rpm, env._step_counter, env._obs_buf[0], env._obs_buf[1], env._reward, ctl._state]
    if env._phys is not None:
        t += [env._phys, env._phys_props]
    return [x.clone() for x in t] + [env._cur, ctl.control_counter]


def _same(a, b):
    for x, y in zip(a, b):
        assert (x == y) if not isinstance(x, torch.Tensor) else torch.equal(x, y)


def _restore(env, ctl, state, last, pid, cc):
    env.set_state(*state)
    env._last_rpm.copy_(last)
    ctl._state.copy_(pid)
    ctl.control_counter = cc


FWD = [("DYN", "CF2X", 240, 240), ("PYB_GND", "CF2P", 240, 48), ("PYB_DRAG", "CF2X", 240, 30), ("DYN", "CF2P", 240, 48),
       ("PYB_DRAG", "CF2P", 240, 240), ("PYB_GND", "CF2X", 240, 30)]


@pytest.mark.parametrize("physics,model,pyb,ctrl", FWD)
@pytest.mark.parametrize("table", [False, True])
@pytest.mark.parametrize("per_drone", [False, True])
def test_forward_bit_identical_to_rollout_and_loop(physics, model, pyb, ctrl, table, per_drone):
    E, D, T, W = 3, 11, 7, 5                                # 33 drones: not a multiple of 32; T > W wraps the schedule
    env, ctl = _env(E, D, physics, model, pyb, ctrl)
    rng = np.random.default_rng(hash((physics, model, ctrl, table, per_drone)) % 2 ** 32)
    dev = env.device
    if table:
        env.set_physical_params(m=env.M * rng.uniform(0.8, 1.2, E), kf=env.KF * rng.uniform(0.9, 1.1, E),
                                ixx=env.J[0, 0] * rng.uniform(0.8, 1.2, E))
    wp = _circle(W, E, D, per_drone, rng, dev)
    start = torch.tensor(rng.integers(-3, 9, (E, D)), device=dev)
    offset = torch.tensor(np.concatenate([rng.uniform(-1, 1, (E, D, 2)), rng.uniform(0.5, 1.0, (E, D, 1))], -1), device=dev)
    tvel = torch.tensor(rng.uniform(-0.1, 0.1, (E, D, 3)), device=dev)
    trpy = torch.tensor([0.0, 0.0, 0.3], device=dev, dtype=torch.float64)
    sched = dict(waypoints=wp, start=start, offset=offset, target_vel=tvel, target_rpy=trpy)
    for k in range(2):                                      # a non-trivial start: controller state, last_clipped_action
        env.step(ctl.computeControlFromEnv(env, (wp[k] if not per_drone else wp[k]).expand(E, D, 3).reshape(-1, 3) + offset.reshape(-1, 3)))
    before = _snapshot(env, ctl)
    out = env.differentiable_rollout(controller=ctl, num_steps=T, **sched)
    _same(before, _snapshot(env, ctl))
    saved = ([t.clone() for t in (env.pos, env.quat, env.vel, env.rpy_rates)], env._last_rpm.clone(), ctl._state.clone(), ctl.control_counter)
    # the pid.py loop
    n = E * D
    wpn = wp.reshape(W, -1, 3).expand(W, n, 3)
    for k in range(T):
        rows = torch.remainder(start.reshape(-1) + k, W)
        tp = wpn[rows, torch.arange(n, device=dev)] + offset.reshape(n, 3)
        rpm = ctl.computeControlFromEnv(env, tp, target_rpy=trpy.expand(n, 3), target_vel=tvel.reshape(n, 3))
        env.step(rpm)
        for key in STATE_KEYS:
            assert torch.equal(out[key][k], getattr(env, key)), (key, k)
        assert torch.equal(out["rpm"][k], env.last_clipped_action), k
    # CtrlAviary.rollout
    _restore(env, ctl, *saved)
    ro = env.rollout(controller=ctl, num_steps=T, record=False, **sched)
    assert torch.equal(ro["rpm"], out["rpm"])
    for key in STATE_KEYS:
        assert torch.equal(out[key][-1], getattr(env, key)), key


def _leaves(env, ctl, rng, W, per_drone):
    """Every differentiable input of the closed loop, as fresh leaves."""
    E, D, dev = env._E, env._D, env.device
    t = lambda a: torch.tensor(a, device=dev)
    L = {"waypoints": _circle(W, E, D, per_drone, rng, dev),
         "offset": t(np.concatenate([rng.uniform(-1, 1, (E, D, 2)), rng.uniform(0.5, 1.0, (E, D, 1))], -1)),
         "target_vel": t(rng.uniform(-0.1, 0.1, (E, D, 3))), "target_rpy": t(rng.uniform(-0.5, 0.5, (E, D, 3))),
         "target_rpy_rates": t(rng.uniform(-0.1, 0.1, (E, D, 3)))}
    L.update({k: env_v.clone() for k, env_v in zip(STATE_KEYS, (env.pos, env.quat, env.vel, env.rpy_rates))})
    L["vel"] = t(rng.uniform(-0.5, 0.5, (E, D, 3)))
    L["rpy_rates"] = t(rng.uniform(-1, 1, (E, D, 3)))
    L.update({k: t(rng.uniform(-0.02, 0.02, (E, D, 3))) for k in PID_KEYS})
    L["last_rpm"] = t(env.HOVER_RPM * rng.uniform(0.9, 1.1, (E, D, 4)))
    co = PR.gains_of(ctl._P, dev).reshape(6, 3)
    L.update({k: co[j] * t(rng.uniform(0.8, 1.2, (E, 3))) for j, k in enumerate(GAIN_KEYS)})
    L.update({k: v * t(rng.uniform(0.8, 1.2, E)) for k, v in env.physical_params().items()})
    return {k: v.detach().clone().requires_grad_(True) for k, v in L.items()}


def _call(env, ctl, L, T, start, **kw):
    from gym_pybullet_drones_b200.params import PHYS_KEYS
    return env.differentiable_rollout(controller=ctl, num_steps=T, start=start, waypoints=L["waypoints"], offset=L["offset"],
                                      target_vel=L["target_vel"], target_rpy=L["target_rpy"], target_rpy_rates=L["target_rpy_rates"],
                                      state={k: L[k] for k in STATE_KEYS}, pid_state={k: L[k] for k in PID_KEYS},
                                      last_rpm=L["last_rpm"], gains={k: L[k] for k in GAIN_KEYS}, phys={k: L[k] for k in PHYS_KEYS}, **kw)


def _ref(env, ctl, L, T, start, effects):
    """diff_pid_ref's closed loop on the device from the same leaves: {state keys, rpm} [T, E, D, k]."""
    from gym_pybullet_drones_b200.diff import schedule_targets
    from gym_pybullet_drones_b200.params import PHYS_KEYS, physical_rows
    E, D, n, dev = env._E, env._D, env._N, env.device
    rows = physical_rows(env.DRONE_MODEL, {k: L[k] for k in PHYS_KEYS}, env.G).repeat_interleave(D, dim=0)
    gains = torch.cat([L[k] for k in GAIN_KEYS], dim=1).repeat_interleave(D, dim=0)
    x0 = torch.cat([L[k].reshape(n, -1) for k in STATE_KEYS], 1)
    pid0 = torch.cat([L[k].reshape(n, 3) for k in PID_KEYS], 1)
    tpos = schedule_targets(L["waypoints"], start, L["offset"], T, E, D, dev)
    xs, us = PR.closed_loop(R.model_constants(env._P, dev), PR.controller_constants(ctl._P, dev), rows, gains, x0, pid0, tpos,
                            L["target_rpy"].reshape(n, 3)[:, 2], L["target_vel"].reshape(n, 3), L["target_rpy_rates"].reshape(n, 3),
                            L["last_rpm"].reshape(n, 4), env.CTRL_TIMESTEP, env.PYB_STEPS_PER_CTRL, effects)
    out = {k: xs[..., a:b].reshape(T, E, D, b - a) for k, (a, b) in zip(STATE_KEYS, ((0, 3), (3, 7), (7, 10), (10, 13)))}
    out["rpm"] = us.reshape(T, E, D, 4)
    return out


def _grads(out, L, g):
    loss = sum((out[k] * g[k]).sum() for k in g)
    gs = torch.autograd.grad(loss, list(L.values()), allow_unused=True)
    return {k: torch.zeros_like(v) if x is None else x for (k, v), x in zip(L.items(), gs)}


@pytest.mark.parametrize("physics,model,effects,per_drone", [("DYN", "CF2X", 0, False), ("PYB_GND", "CF2P", 1, True),
                                                             ("PYB_DRAG", "CF2X", 2, False)])
def test_gradients_match_reference_4096_drones(physics, model, effects, per_drone):
    E, D, T, W = 2048, 2, 24, 16
    env, ctl = _env(E, D, physics, model, 240, 48)
    rng = np.random.default_rng(5)
    L = _leaves(env, ctl, rng, W, per_drone)
    start = torch.tensor(rng.integers(0, W, (E, D)), device=env.device)
    out = _call(env, ctl, L, T, start)
    g = {k: torch.tensor(rng.standard_normal(tuple(v.shape)), device=env.device) for k, v in out.items()}
    got = _grads(out, L, g)
    ref = _ref(env, ctl, L, T, start, effects)
    for k in out:
        assert R.relerr(out[k], ref[k]) < 1e-10, k
    want = _grads(ref, L, g)
    worst = {}
    for k in L:
        worst[k] = R.relerr(got[k], want[k])
        assert worst[k] <= GRAD_TOL, (k, worst[k])
    print("worst block %s: %.2e" % (max(worst, key=worst.get), max(worst.values())))


def test_gnd_drag_through_the_abi():
    """GND|DRAG has no Physics mode: qs_dyn_ctrl_traj / _vjp through the C ABI against the reference."""
    from gym_pybullet_drones_b200 import _native as N
    from gym_pybullet_drones_b200.diff import DynCtrlTrajectory, pack_state
    env, ctl = _env(64, 3, "DYN", "CF2X", 240, 48)
    E, D, n, T, dev = env._E, env._D, env._N, 12, env.device
    rng = np.random.default_rng(6)
    L = _leaves(env, ctl, rng, 8, True)
    from gym_pybullet_drones_b200.params import PHYS_KEYS, physical_rows
    start = torch.tensor(rng.integers(0, 8, (E, D)), device=dev)
    from gym_pybullet_drones_b200.diff import schedule_targets
    rows = physical_rows(env.DRONE_MODEL, {k: L[k] for k in PHYS_KEYS}, env.G)
    planes0 = pack_state(*[L[k].reshape(n, -1) for k in STATE_KEYS])
    pid0 = torch.cat([L[k].reshape(n, 3).t() for k in PID_KEYS])
    tpos = schedule_targets(L["waypoints"], start, L["offset"], T, E, D, dev)
    cfg = (env._P, ctl._P, env.CTRL_TIMESTEP, E, D, env.PYB_STEPS_PER_CTRL, N.EFFECT_GND | N.EFFECT_DRAG)
    states, rpm = DynCtrlTrajectory.apply(planes0, pid0, tpos, L["target_vel"].reshape(n, 3), L["target_rpy"].reshape(n, 3),
                                          L["target_rpy_rates"].reshape(n, 3), L["last_rpm"].reshape(n, 4), rows,
                                          torch.cat([L[k] for k in GAIN_KEYS], 1), cfg)
    from gym_pybullet_drones_b200.diff import unpack_states
    out = {k: v.reshape(T, E, D, -1) for k, v in unpack_states(states, n).items()}
    out["rpm"] = rpm.reshape(T, E, D, 4)
    ref = _ref(env, ctl, L, T, start, 3)
    g = {k: torch.tensor(rng.standard_normal(tuple(v.shape)), device=dev) for k, v in out.items()}
    got, want = _grads(out, L, g), _grads(ref, L, g)
    for k in L:
        assert R.relerr(got[k], want[k]) <= GRAD_TOL, k


def test_gradcheck_tiny():
    env, ctl = _env(1, 2, "PYB_DRAG", "CF2X", 240, 48)
    rng = np.random.default_rng(7)
    L = _leaves(env, ctl, rng, 3, False)
    sub = ("pos", "vel", "P_COEFF_FOR", "D_COEFF_FOR", "waypoints", "offset")
    fixed = {k: v.detach() for k, v in L.items()}

    def f(*xs):
        M = dict(fixed, **dict(zip(sub, xs)))
        out = _call(env, ctl, M, 3, None)
        return tuple(out[k] for k in ("pos", "vel", "rpm"))
    assert torch.autograd.gradcheck(f, tuple(L[k] for k in sub), eps=1e-7, atol=1e-5, rtol=1e-4)


def test_deterministic_gradients():
    env, ctl = _env(512, 4, "PYB_GND", "CF2X", 240, 48)
    rng = np.random.default_rng(8)
    L = _leaves(env, ctl, rng, 6, False)
    start = torch.tensor(rng.integers(0, 6, (512, 4)), device=env.device)
    g = None
    runs = []
    for _ in range(2):
        out = _call(env, ctl, L, 20, start)
        g = g or {k: torch.tensor(rng.standard_normal(tuple(v.shape)), device=env.device) for k, v in out.items()}
        runs.append(_grads(out, L, g))
    for k in L:
        assert torch.equal(runs[0][k], runs[1][k]), k


def test_morton_order_same_gradients():
    """A Morton-reordered formation and a twin that was never reordered give the same trajectory and gradients (drone-id
    indices).  reorder_by_morton() needs a downwash formation and the adjoint refuses downwash, so the reordered env's effects are
    switched to plain DYN after the reorder, as in the open-loop test."""
    DSLPIDControl, CtrlAviary, DroneModel, Physics = _imports()
    from test_gpu_formation import stacks
    xyz = stacks(10, 9)[:333]
    xyz = xyz[np.random.default_rng(5).permutation(len(xyz))]
    a = CtrlAviary(num_drones=len(xyz), initial_xyzs=xyz, physics=Physics.PYB_DW, ctrl_freq=48, num_envs=1)
    b = CtrlAviary(num_drones=len(xyz), initial_xyzs=xyz, physics=Physics.DYN, ctrl_freq=48, num_envs=1)
    a.reset(); b.reset()
    order = a.reorder_by_morton().cpu().numpy()
    assert np.count_nonzero(order == np.arange(len(order))) < len(order) // 10
    a._effects = 0
    ca, cb = (DSLPIDControl(DroneModel.CF2X, num_drones=len(xyz), device=e.device) for e in (a, b))
    rng = np.random.default_rng(9)
    La = _leaves(a, ca, rng, 8, True)
    Lb = {k: v.detach().clone().requires_grad_(True) for k, v in La.items()}
    start = torch.tensor(rng.integers(0, 8, (1, len(xyz))), device=a.device)
    oa, ob = _call(a, ca, La, 10, start), _call(b, cb, Lb, 10, start)
    g = {k: torch.tensor(rng.standard_normal(tuple(v.shape)), device=a.device) for k, v in oa.items()}
    ga, gb = _grads(oa, La, g), _grads(ob, Lb, g)
    for k in oa:
        assert torch.equal(oa[k], ob[k]), k
    for k in La:
        assert torch.equal(ga[k], gb[k]), k


def test_gain_identification():
    """256 aviaries whose position-loop P and D gains are within +-30 % of the defaults fly half of pid.py's circle; L-BFGS on the
    closed-loop trajectory recovers those gains.  At 240 Hz control: at 48 Hz the attitude loop's saturated limit cycles make the
    trajectory's sensitivities over two seconds grow far beyond what central differences of the same function show (DESIGN.md 4.5)."""
    E, D, T, W = 256, 1, 240, 480
    env, ctl = _env(E, D, "DYN", "CF2X", 240, 240)
    dev = env.device
    rng = np.random.default_rng(10)
    co = PR.gains_of(ctl._P, dev).reshape(6, 3)
    true_p = co[0] * torch.tensor(rng.uniform(0.7, 1.3, (E, 3)), device=dev)
    true_d = co[2] * torch.tensor(rng.uniform(0.7, 1.3, (E, 3)), device=dev)
    wp = _circle(W, E, D, False, rng, dev)
    wp = wp - wp[0]                                          # the circle starts where each drone hovers
    offset = env.pos.clone()
    # the recorded flights: the closed loop's forward, which is CtrlAviary.rollout(controller=...)'s bits (the forward test
    # above), with each aviary's own gain set (one DSLPIDControl holds a single one)
    rec = env.differentiable_rollout(controller=ctl, waypoints=wp, offset=offset, num_steps=T,
                                     gains={"P_COEFF_FOR": true_p, "D_COEFF_FOR": true_d})
    rec = {k: v.detach() for k, v in rec.items()}
    theta = torch.zeros((2, E, 3), dtype=torch.float64, device=dev, requires_grad=True)     # log-ratios from the defaults
    opt = torch.optim.LBFGS([theta], lr=1, max_iter=200, history_size=20, tolerance_grad=1e-14, tolerance_change=1e-20,
                            line_search_fn="strong_wolfe")

    def closure():
        opt.zero_grad()
        out = env.differentiable_rollout(controller=ctl, waypoints=wp, offset=offset, num_steps=T,
                                         gains={"P_COEFF_FOR": co[0] * torch.exp(theta[0]), "D_COEFF_FOR": co[2] * torch.exp(theta[1])})
        loss = sum(((out[k] - rec[k]) / 1e-3).square().sum() for k in ("pos", "quat", "vel"))
        loss.backward()
        return loss
    for _ in range(4):
        opt.step(closure)
    p, d = co[0] * torch.exp(theta[0].detach()), co[2] * torch.exp(theta[1].detach())
    err = max(float(((p - true_p) / true_p).abs().max()), float(((d - true_d) / true_d).abs().max()))
    print("gain identification: worst relative error %.2e" % err)
    assert err <= 1e-3


def test_refusals():
    from gym_pybullet_drones_b200.control import MRAC
    DSLPIDControl, CtrlAviary, DroneModel, Physics = _imports()
    env, ctl = _env(2, 2)
    dev = env.device
    wp = torch.zeros((4, 3), dtype=torch.float64, device=dev)
    rpm = torch.full((2, 2, 2, 4), env.HOVER_RPM, dtype=torch.float64, device=dev)
    with pytest.raises(ValueError, match="MRAC"):
        env.differentiable_rollout(controller=MRAC(DroneModel.CF2X, num_drones=4, device=dev), waypoints=wp)
    with pytest.raises(ValueError, match="num_drones"):
        env.differentiable_rollout(controller=DSLPIDControl(DroneModel.CF2X, num_drones=3, device=dev), waypoints=wp)
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError, match="state is on"):
            env.differentiable_rollout(controller=DSLPIDControl(DroneModel.CF2X, num_drones=4, device="cuda:1"), waypoints=wp)
    with pytest.raises(ValueError, match="exactly one"):
        env.differentiable_rollout(rpm, controller=ctl, waypoints=wp)
    with pytest.raises(ValueError, match="exactly one"):
        env.differentiable_rollout()
    with pytest.raises(ValueError, match="float64"):
        env.differentiable_rollout(controller=ctl, waypoints=wp.float())
    with pytest.raises(ValueError, match="shape"):
        env.differentiable_rollout(controller=ctl, waypoints=wp, offset=torch.zeros((3, 3), dtype=torch.float64, device=dev))
    with pytest.raises(ValueError, match="unknown gains"):
        env.differentiable_rollout(controller=ctl, waypoints=wp, gains={"P_COEFF": torch.zeros(3, dtype=torch.float64, device=dev)})
    with pytest.raises(ValueError, match="unknown pid_state"):
        env.differentiable_rollout(controller=ctl, waypoints=wp, pid_state={"integral": torch.zeros((2, 2, 3), dtype=torch.float64, device=dev)})
    with pytest.raises(ValueError, match="controller rollout only"):
        env.differentiable_rollout(rpm, waypoints=wp)
    with pytest.raises(ValueError, match="needs waypoints"):
        env.differentiable_rollout(controller=ctl)
    kp = torch.ones((2, 3), dtype=torch.float64, device=dev, requires_grad=True)
    out = env.differentiable_rollout(controller=ctl, waypoints=wp, gains={"P_COEFF_FOR": kp})
    with pytest.raises(ValueError, match="double backward"):
        torch.autograd.grad(out["pos"].sum(), kp, create_graph=True)
    dw, cdw = _env(1, 2, "PYB_DW")
    with pytest.raises(ValueError, match="downwash"):
        dw.differentiable_rollout(controller=cdw, waypoints=wp)
