"""-m gpu: BaseAviary.differentiable_rollout(downwash=True) (qs_dyn_traj_dw / qs_dyn_ctrl_traj_dw and their VJPs, DESIGN.md 4.5,
downwash adjoint).

The forward is held to T CtrlAviary.step() calls, to CtrlAviary.rollout() and to mppi()'s committed trajectory bit for bit; the
gradients to the autograd of the float64 reference tests/diff_dw_ref.py on the same device (per drone and per input block), the
cross-drone term and each pair decision included; the invariants (batch independence, determinism, gradcheck); the refusals;
and a system identification through downwash that its downwash-blind twin cannot do."""
import numpy as np
import pytest
import torch

import diff_dw_ref as DW
import diff_pid_ref as PR
import diff_ref as R
from diff_testlib import per_drone_relerr

pytestmark = pytest.mark.gpu

GRAD_TOL = 1e-9
STATE_KEYS = ("pos", "quat", "vel", "rpy_rates")
PID_KEYS = ("integral_pos_e", "last_rpy", "integral_rpy_e")
GAIN_KEYS = ("P_COEFF_FOR", "I_COEFF_FOR", "D_COEFF_FOR", "P_COEFF_TOR", "I_COEFF_TOR", "D_COEFF_TOR")


def _imports():
    from gym_pybullet_drones_b200.control import DSLPIDControl
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils.enums import DroneModel, Physics
    return DSLPIDControl, CtrlAviary, DroneModel, Physics


def stack_xyz(D, rng, spacing=0.9):
    """D drones in columns of up to 4, `spacing` apart in z, the columns 0.3 m apart on a grid (every pair within 10 m in xy)"""
    k = np.arange(D)
    cols = int(np.ceil(np.sqrt((D + 3) // 4)))
    col = k // 4
    xy = 0.3 * np.stack([col % cols, col // cols], 1) + rng.uniform(-0.02, 0.02, (D, 2))
    return np.concatenate([xy, (0.5 + spacing * (k % 4))[:, None]], 1)


def _env(E, D, physics="PYB_DW", model="CF2X", pyb=240, ctrl=48, seed=0, xyz=None, controller=False):
    DSLPIDControl, CtrlAviary, DroneModel, Physics = _imports()
    rng = np.random.default_rng(seed)
    xyz = stack_xyz(D, rng) if xyz is None else xyz
    env = CtrlAviary(drone_model=DroneModel[model], num_drones=D, physics=Physics[physics], pyb_freq=pyb, ctrl_freq=ctrl,
                     initial_xyzs=xyz, initial_rpys=rng.uniform(-0.1, 0.1, (D, 3)), num_envs=E)
    env.reset()
    if not controller:
        return env
    return env, DSLPIDControl(DroneModel[model], num_drones=E * D, device=env.device)


def _rpm(env, T, rng, spread=0.05, clip=True):
    r = env.HOVER_RPM * (1 + spread * rng.uniform(-1, 1, (T, env._E, env._D, 4)))
    if clip:
        r[-1:, :, 0, 0] = env.MAX_RPM * 1.2
        r[-1:, :, -1, 3] = -100.0
    return torch.tensor(r, device=env.device)


def _snapshot(env, ctl=None):
    t = [env._planes, env._last_rpm, env._step_counter, env._obs_buf[0], env._obs_buf[1], env._reward]
    if env._phys is not None:
        t += [env._phys, env._phys_props]
    if ctl is not None:
        t += [ctl._state]
    return [x.clone() for x in t] + [env._cur] + ([ctl.control_counter] if ctl is not None else [])


def _same(a, b):
    for x, y in zip(a, b):
        assert (x == y) if not isinstance(x, torch.Tensor) else torch.equal(x, y)


def _cases():
    out = []
    for j, D in enumerate((1, 2, 3, 5, 32, 33, 127, 128)):
        out.append((D, ("PYB_DW", "PYB_GND_DRAG_DW")[j % 2], ("CF2X", "CF2P")[(j // 2) % 2], (240, 48)[(j // 4) % 2 ^ j % 2],
                    j % 3 != 0))
    return out


@pytest.mark.parametrize("D,physics,model,ctrl,table", _cases())
def test_forward_bit_identical_to_step_and_rollout(D, physics, model, ctrl, table):
    per_cta = 128 // D
    E = 2 * per_cta + 1 if per_cta > 1 else 3                # the last CTA holds fewer aviaries than the others
    env = _env(E, D, physics, model, 240, ctrl, seed=D)
    rng = np.random.default_rng(D)
    if table:
        env.set_physical_params(m=env.M * rng.uniform(0.8, 1.2, E), kf=env.KF * rng.uniform(0.9, 1.1, E),
                                ixx=env.J[0, 0] * rng.uniform(0.8, 1.2, E))
    for _ in range(2):                                        # a non-trivial start and last_clipped_action
        env.step(_rpm(env, 1, rng, clip=False)[0])
    T = 5
    rpm = _rpm(env, T, rng)
    before = _snapshot(env)
    out = env.differentiable_rollout(rpm, downwash=True)
    _same(before, _snapshot(env))
    again = env.differentiable_rollout(rpm, downwash=True, last_rpm=env.last_clipped_action.reshape(E, D, 4).clone())
    for key in STATE_KEYS:
        assert torch.equal(out[key], again[key]), key
    twin = [t.clone() for t in (env.pos, env.quat, env.vel, env.rpy_rates)]
    for k in range(T):
        env.step(rpm[k])
        for key in STATE_KEYS:
            assert torch.equal(out[key][k], getattr(env, key)), (key, k)
    env.set_state(*twin)
    env._last_rpm.copy_(before[1])
    env.rollout(actions=rpm, record=False)
    for key in STATE_KEYS:
        assert torch.equal(out[key][-1], getattr(env, key)), key


def test_mppi_committed_trajectory_is_the_rollout():
    env = _env(6, 3, "PYB_DW", seed=1)
    rng = np.random.default_rng(1)
    tgt = {"pos": torch.tensor(stack_xyz(3, rng)[None].repeat(6, 0) + rng.uniform(-0.2, 0.2, (6, 3, 3)), device=env.device)}
    sol = env.mppi(tgt, num_steps=8, iters=3, samples=16)
    out = env.differentiable_rollout(sol["rpm"], downwash=True)
    for key in STATE_KEYS:
        assert torch.equal(out[key], sol[key]), key


def _crossing(E):
    """downwash.py: two drones crossing 0.5 m apart in z, 240/48 Hz, each flying to the other's x and back"""
    W = 48
    xyz = np.array([[0.5, 0.0, 1.0], [-0.5, 0.0, 0.5]])
    s = 0.5 * (1 - np.cos(2 * np.pi * np.arange(W) / W))      # 0 -> 1 -> 0
    wp = np.zeros((W, E, 2, 3))
    wp[:, :, 0] = np.stack([0.5 - s, 0 * s, 1.0 + 0 * s], 1)[:, None]
    wp[:, :, 1] = np.stack([-0.5 + s, 0 * s, 0.5 + 0 * s], 1)[:, None]
    return xyz, wp


@pytest.mark.parametrize("D", [2, 3, 128])
def test_closed_loop_forward_bit_identical_to_rollout_and_loop(D):
    E = 5 if D < 128 else 3
    rng = np.random.default_rng(D)
    if D == 2:
        xyz, wp = _crossing(E)
    else:
        xyz = stack_xyz(D, rng)
        wp = xyz[None, None] + 0.2 * np.sin(np.linspace(0, 3, 16))[:, None, None, None] * rng.uniform(-1, 1, (1, E, D, 3))
    env, ctl = _env(E, D, "PYB_GND_DRAG_DW" if D == 3 else "PYB_DW", xyz=xyz, controller=True)
    dev = env.device
    wp = torch.tensor(wp, device=dev)
    T = wp.shape[0]
    before = _snapshot(env, ctl)
    out = env.differentiable_rollout(controller=ctl, waypoints=wp, num_steps=T, downwash=True)
    _same(before, _snapshot(env, ctl))
    saved = ([t.clone() for t in (env.pos, env.quat, env.vel, env.rpy_rates)], env._last_rpm.clone(), ctl._state.clone(),
             ctl.control_counter)
    n = E * D
    for k in range(T):                                        # the downwash.py loop
        env.step(ctl.computeControlFromEnv(env, wp[k].reshape(n, 3)))
        for key in STATE_KEYS:
            assert torch.equal(out[key][k], getattr(env, key)), (key, k)
        assert torch.equal(out["rpm"][k], env.last_clipped_action), k
    env.set_state(*saved[0])
    env._last_rpm.copy_(saved[1])
    ctl._state.copy_(saved[2])
    ctl.control_counter = saved[3]
    ro = env.rollout(controller=ctl, waypoints=wp, num_steps=T, record=False)
    assert torch.equal(ro["rpm"], out["rpm"])
    for key in STATE_KEYS:
        assert torch.equal(out[key][-1], getattr(env, key)), key


# ---- gradients against the reference on the device ------------------------------------------------------------------------

def _stacks(E, D, rng, dev, spacing=0.9):
    """per-aviary start states: stack_xyz moved and jittered per aviary, tilted, moving and turning"""
    pos = stack_xyz(D, rng, spacing)[None] + np.concatenate([rng.uniform(-0.02, 0.02, (E, D, 2)), rng.uniform(-0.05, 0.05, (E, D, 1))], 2)
    from diff_testlib import quat_from_rpy
    quat = quat_from_rpy(rng.uniform(-0.2, 0.2, (E * D, 3))).reshape(E, D, 4)
    t = lambda a: torch.tensor(a, device=dev)
    return {"pos": t(pos), "quat": t(quat), "vel": t(rng.uniform(-0.3, 0.3, (E, D, 3))), "rpy_rates": t(rng.uniform(-1, 1, (E, D, 3)))}


def _open_leaves(env, rng):
    E, D, dev = env._E, env._D, env.device
    L = {"rpm": _rpm(env, 32, rng)}
    L.update(_stacks(E, D, rng, dev))
    L["last_rpm"] = torch.tensor(env.HOVER_RPM * rng.uniform(0.9, 1.1, (E, D, 4)), device=dev)
    L.update({k: v * torch.tensor(rng.uniform(0.8, 1.2, E), device=dev) for k, v in env.physical_params().items()})
    return {k: v.detach().clone().requires_grad_(True) for k, v in L.items()}


def _open_call(env, L, **kw):
    from gym_pybullet_drones_b200.params import PHYS_KEYS
    return env.differentiable_rollout(L["rpm"], state={k: L[k] for k in STATE_KEYS}, last_rpm=L["last_rpm"],
                                      phys={k: L[k] for k in PHYS_KEYS}, downwash=True, **kw)


def _open_ref(env, L, **kw):
    from gym_pybullet_drones_b200.params import PHYS_KEYS, physical_rows
    E, D, n, dev = env._E, env._D, env._N, env.device
    T = L["rpm"].shape[0]
    rows = physical_rows(env.DRONE_MODEL, {k: L[k] for k in PHYS_KEYS}, env.G).repeat_interleave(D, dim=0)
    x0 = torch.cat([L[k].reshape(n, -1) for k in STATE_KEYS], 1)
    xs = DW.rollout(R.model_constants(env._P, dev), env._P, rows, x0, L["rpm"].reshape(T, n, 4), L["last_rpm"].reshape(n, 4),
                    env.PYB_STEPS_PER_CTRL, env._effects, D, **kw)
    return {k: xs[..., a:b].reshape(T, E, D, b - a) for k, (a, b) in zip(STATE_KEYS, ((0, 3), (3, 7), (7, 10), (10, 13)))}


def _grads(out, L, g):
    loss = sum((out[k] * g[k]).sum() for k in g)
    gs = torch.autograd.grad(loss, list(L.values()), allow_unused=True)
    return {k: torch.zeros_like(v) if x is None else x for (k, v), x in zip(L.items(), gs)}


def _worst_per_drone(got, want, E, D):
    """{block: the worst per-drone relative error}: per drone for blocks with a drone axis ([E, D, ...] or [T, E, D, ...]), per
    aviary for per-aviary blocks ([E] or [E, 3])"""
    worst = {}
    for k in got:
        a, b = (x.detach().cpu().numpy() for x in (got[k], want[k]))
        if a.shape[0] != E:                                   # [T or W, E, D, k] -> [E, D, T or W, k]
            a, b = np.moveaxis(a, 0, 2), np.moveaxis(b, 0, 2)
        units = E * D if a.ndim > 2 and a.shape[1] == D else E
        worst[k] = float(np.max(per_drone_relerr(a.reshape(units, -1), b.reshape(units, -1))))
    return worst


@pytest.mark.parametrize("physics,model", [("PYB_DW", "CF2X"), ("PYB_GND_DRAG_DW", "CF2P")])
def test_open_loop_gradients_match_reference_4096_drones(physics, model):
    E, D = 2048, 2
    env = _env(E, D, physics, model, 240, 48)
    rng = np.random.default_rng(11)
    L = _open_leaves(env, rng)
    out = _open_call(env, L)
    ref = _open_ref(env, L)
    for k in out:
        assert R.relerr(out[k], ref[k]) < 1e-12, k
    g = {k: torch.tensor(rng.standard_normal(tuple(v.shape)), device=env.device) for k, v in out.items()}
    got, want = _grads(out, L, g), _grads(ref, L, g)
    worst = _worst_per_drone(got, want, E, D)
    print("worst per-drone relative error per block (%s %s): %s" % (physics, model, {k: "%.1e" % v for k, v in worst.items()}))
    for k, e in worst.items():
        if k == "last_rpm" and not env._effects & 2:
            assert float(got[k].abs().max()) == 0.0
        else:
            assert e <= GRAD_TOL, (k, e)


def _circle(W, E, D, rng, dev, centre):
    i = np.arange(W)
    c = np.stack([0.2 * np.cos(2 * np.pi * i / W), 0.2 * np.sin(2 * np.pi * i / W), 0.1 * np.sin(4 * np.pi * i / W)], 1)
    return torch.tensor(c[:, None, None, :] + centre[None] + rng.uniform(-0.02, 0.02, (1, E, D, 3)), device=dev)


def _closed_leaves(env, ctl, rng, W):
    """every differentiable input of the closed loop, as fresh leaves: stacks 1.5 m apart, tracking their start positions"""
    E, D, dev = env._E, env._D, env.device
    t = lambda a: torch.tensor(a, device=dev)
    st = _stacks(E, D, rng, dev, spacing=1.5)
    L = {"waypoints": _circle(W, E, D, rng, dev, np.zeros((E, D, 3))), "offset": st["pos"].clone(),
         "target_vel": t(rng.uniform(-0.1, 0.1, (E, D, 3))), "target_rpy": t(rng.uniform(-0.5, 0.5, (E, D, 3))),
         "target_rpy_rates": t(rng.uniform(-0.1, 0.1, (E, D, 3)))}
    L.update(st)
    L.update({k: t(rng.uniform(-0.02, 0.02, (E, D, 3))) for k in PID_KEYS})
    L["last_rpm"] = t(env.HOVER_RPM * rng.uniform(0.9, 1.1, (E, D, 4)))
    co = PR.gains_of(ctl._P, dev).reshape(6, 3)
    L.update({k: co[j] * t(rng.uniform(0.8, 1.2, (E, 3))) for j, k in enumerate(GAIN_KEYS)})
    L.update({k: v * t(rng.uniform(0.8, 1.2, E)) for k, v in env.physical_params().items()})
    return {k: v.detach().clone().requires_grad_(True) for k, v in L.items()}


def _closed_call(env, ctl, L, T, start):
    from gym_pybullet_drones_b200.params import PHYS_KEYS
    return env.differentiable_rollout(controller=ctl, num_steps=T, start=start, waypoints=L["waypoints"], offset=L["offset"],
                                      target_vel=L["target_vel"], target_rpy=L["target_rpy"], target_rpy_rates=L["target_rpy_rates"],
                                      state={k: L[k] for k in STATE_KEYS}, pid_state={k: L[k] for k in PID_KEYS},
                                      last_rpm=L["last_rpm"], gains={k: L[k] for k in GAIN_KEYS}, phys={k: L[k] for k in PHYS_KEYS},
                                      downwash=True)


def _closed_ref(env, ctl, L, T, start):
    from gym_pybullet_drones_b200.diff import schedule_targets
    from gym_pybullet_drones_b200.params import PHYS_KEYS, physical_rows
    E, D, n, dev = env._E, env._D, env._N, env.device
    rows = physical_rows(env.DRONE_MODEL, {k: L[k] for k in PHYS_KEYS}, env.G).repeat_interleave(D, dim=0)
    gains = torch.cat([L[k] for k in GAIN_KEYS], dim=1).repeat_interleave(D, dim=0)
    x0 = torch.cat([L[k].reshape(n, -1) for k in STATE_KEYS], 1)
    pid0 = torch.cat([L[k].reshape(n, 3) for k in PID_KEYS], 1)
    tpos = schedule_targets(L["waypoints"], start, L["offset"], T, E, D, dev)
    xs, us = DW.closed_loop(R.model_constants(env._P, dev), env._P, PR.controller_constants(ctl._P, dev), rows, gains, x0, pid0, tpos,
                            L["target_rpy"].reshape(n, 3)[:, 2], L["target_vel"].reshape(n, 3), L["target_rpy_rates"].reshape(n, 3),
                            L["last_rpm"].reshape(n, 4), env.CTRL_TIMESTEP, env.PYB_STEPS_PER_CTRL, env._effects, D)
    out = {k: xs[..., a:b].reshape(T, E, D, b - a) for k, (a, b) in zip(STATE_KEYS, ((0, 3), (3, 7), (7, 10), (10, 13)))}
    out["rpm"] = us.reshape(T, E, D, 4)
    return out


@pytest.mark.parametrize("physics", ["PYB_DW", "PYB_GND_DRAG_DW"])
def test_closed_loop_gradients_match_reference_4096_drones(physics):
    """Normwise per block to GRAD_TOL, per drone to 1e-7, at T = 24 ticks: the stacked closed loop is ill-conditioned (in the
    reference alone, a relative perturbation of 1e-15 in the start state moves the worst drone's trajectory by 1e-10 after 24
    ticks and by 2e-9 after 32), so two correct float64 implementations part per drone by more than GRAD_TOL."""
    E, D, T, W = 2048, 2, 24, 16
    env, ctl = _env(E, D, physics, "CF2X", 240, 48, controller=True)
    rng = np.random.default_rng(5)
    L = _closed_leaves(env, ctl, rng, W)
    start = torch.tensor(rng.integers(0, W, (E, D)), device=env.device)
    out = _closed_call(env, ctl, L, T, start)
    ref = _closed_ref(env, ctl, L, T, start)
    for k in out:
        assert R.relerr(out[k], ref[k]) < 1e-10, k
    g = {k: torch.tensor(rng.standard_normal(tuple(v.shape)), device=env.device) for k, v in out.items()}
    got, want = _grads(out, L, g), _grads(ref, L, g)
    norm = {k: R.relerr(got[k], want[k]) for k in L}
    worst = _worst_per_drone(got, want, E, D)
    print("closed loop %s: normwise relative error per block %s; worst per drone %s" % (
        physics, {k: "%.1e" % v for k, v in norm.items()}, {k: "%.1e" % v for k, v in worst.items()}))
    for k in L:
        if k == "last_rpm" and not env._effects & 2:
            assert float(got[k].abs().max()) == 0.0
        else:
            assert norm[k] <= GRAD_TOL and worst[k] <= 1e-7, (k, norm[k], worst[k])


def _pair_env(D=2):
    env = _env(1, D, "PYB_DW", xyz=stack_xyz(D, np.random.default_rng(0)))
    return env


def _level_pair_state(env, lo, hi):
    """one aviary, level and at rest, drone 0 at lo and drone 1 at hi"""
    dev = env.device
    pos = torch.tensor([[lo, hi]], dtype=torch.float64, device=dev)
    quat = torch.tensor([[[0.0, 0.0, 0.0, 1.0]] * 2], dtype=torch.float64, device=dev)
    z = torch.zeros((1, 2, 3), dtype=torch.float64, device=dev)
    return {"pos": pos, "quat": quat, "vel": z.clone(), "rpy_rates": z.clone()}


def _pair_grad(env, st, rpm, **ref_kw):
    """(kernel, reference) gradients of the lower drone's final z w.r.t. the rpm and the start state"""
    L = {"rpm": rpm.clone().requires_grad_(True)}
    L.update({k: v.clone().requires_grad_(True) for k, v in st.items()})
    L["last_rpm"] = torch.full((1, 2, 4), env.HOVER_RPM, dtype=torch.float64, device=env.device, requires_grad=True)
    L.update({k: v.clone().requires_grad_(True) for k, v in env.physical_params().items()})
    out = _open_call(env, L)
    ref = _open_ref(env, L, **ref_kw)
    g = {k: torch.zeros_like(v) for k, v in out.items()}
    g["pos"][-1, 0, 0, 2] = 1.0
    return _grads(out, L, g), _grads(ref, L, g)


def test_cross_drone_gradient():
    """The lower drone's height after 4 ticks depends on the upper drone's RPMs only through downwash: nonzero, the reference's,
    and missed by a reference without the source term."""
    env = _pair_env()
    st = _level_pair_state(env, [0.0, 0.0, 1.0], [0.02, -0.01, 2.0])
    rpm = torch.full((4, 1, 2, 4), 1.02 * env.HOVER_RPM, dtype=torch.float64, device=env.device)
    got, want = _pair_grad(env, st, rpm)
    _, blind = _pair_grad(env, st, rpm, source=False)
    cross = got["rpm"][:, 0, 1]
    assert float(cross.abs().max()) > 0
    e = R.relerr(cross, want["rpm"][:, 0, 1])
    print("cross-drone gradient: relative error %.1e" % e)
    assert e <= GRAD_TOL
    assert float(blind["rpm"][:, 0, 1].abs().max()) == 0.0 and R.relerr(blind["rpm"][:, 0, 1], cross) > 1e-3


def test_pair_decisions_on_the_device():
    """Level pairs at rest (their xy stay exact over the substeps): dxy2 = 100 - 2 ulp acts, 100 - 1 ulp and 100 do not, equal
    heights do not; each matches the reference on the kernel's side and a reference that takes dxy2 < 100 misses at
    100 - 1 ulp.  Stacked drones get finite gradients."""
    env = _pair_env()
    rpm = torch.full((1, 1, 2, 4), 1.01 * env.HOVER_RPM, dtype=torch.float64, device=env.device)
    below = lambda v, k: [v := float(np.nextafter(v, 0.0)) for _ in range(k)][-1] if k else v
    for k, acts in ((2, True), (1, False), (0, False)):
        dx, dy = DW.pair_offset_for(below(100.0, k))
        st = _level_pair_state(env, [0.0, 0.0, 1.0], [dx, dy, 21.0])
        got, want = _pair_grad(env, st, rpm)
        upper = got["pos"][0, 1]
        assert bool((upper != 0).any()) == acts, k
        for key in got:
            assert R.relerr(got[key], want[key]) <= GRAD_TOL, (k, key)
        if k == 1:
            _, flipped = _pair_grad(env, st, rpm, lt100=True)
            assert bool((flipped["pos"][0, 1] != 0).any())
    st = _level_pair_state(env, [0.0, 0.0, 1.0], [0.3, -0.2, 1.0])          # dz = 0: no pair either way
    got, want = _pair_grad(env, st, rpm)
    assert float(got["pos"][0, 1].abs().max()) == 0.0 and float(got["rpm"][0, 0, 1].abs().max()) == 0.0
    for key in got:
        assert R.relerr(got[key], want[key]) <= GRAD_TOL, key
    st = _level_pair_state(env, [0.1, 0.2, 1.0], [0.1, 0.2, 2.0])           # exactly stacked
    got, want = _pair_grad(env, st, rpm)
    assert all(bool(torch.isfinite(v).all()) for v in got.values())
    assert float(got["pos"][0, 1, 2].abs()) > 0
    for key in got:
        assert R.relerr(got[key], want[key]) <= GRAD_TOL, key


# ---- invariants -----------------------------------------------------------------------------------------------------------

def test_batch_independence_and_determinism():
    E, D, e = 37, 5, 17
    env = _env(E, D, "PYB_GND_DRAG_DW")
    one = _env(1, D, "PYB_GND_DRAG_DW")
    rng = np.random.default_rng(3)
    L = _open_leaves(env, rng)
    L["rpm"] = L["rpm"][:6].detach().clone().requires_grad_(True)
    sub = {k: (v[:, e:e + 1] if k == "rpm" else v[e:e + 1]).detach().clone().requires_grad_(True) for k, v in L.items()}
    out = _open_call(env, L)
    g = {k: torch.tensor(rng.standard_normal(tuple(v.shape)), device=env.device) for k, v in out.items()}
    a = _grads(out, L, g)
    b = _grads(_open_call(env, L), L, g)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    out1 = _open_call(one, sub)
    c = _grads(out1, sub, {k: v[:, e:e + 1] for k, v in g.items()})
    for k in c:
        mine = a[k][:, e:e + 1] if k == "rpm" else a[k][e:e + 1]
        assert torch.equal(mine, c[k]), k


def test_gradcheck_small():
    env = _env(2, 3, "PYB_GND_DRAG_DW", seed=4)
    rng = np.random.default_rng(4)
    dev = env.device
    st = _stacks(2, 3, rng, dev)
    x = [_rpm(env, 2, rng, clip=False), st["pos"], st["vel"], torch.ones(2, dtype=torch.float64, device=dev)]
    x = [t.detach().clone().requires_grad_(True) for t in x]

    def f(rpm, pos, vel, m_scale):
        o = env.differentiable_rollout(rpm, state=dict(pos=pos, quat=st["quat"], vel=vel, rpy_rates=st["rpy_rates"]),
                                       phys=dict(m=env.M * m_scale), downwash=True)
        return o["pos"], o["quat"], o["vel"], o["rpy_rates"]

    assert torch.autograd.gradcheck(f, tuple(x), eps=1e-6, atol=1e-5, rtol=1e-4)


def test_refusals():
    DSLPIDControl, CtrlAviary, DroneModel, Physics = _imports()
    from gym_pybullet_drones_b200.ilqr import Tracker
    env = _env(2, 2, "PYB_DW")
    dev = env.device
    rng = np.random.default_rng(8)
    rpm = _rpm(env, 2, rng)
    with pytest.raises(ValueError, match="downwash couples|pairwise term has no adjoint"):
        env.differentiable_rollout(rpm)                       # the default keeps today's refusal
    with pytest.raises(ValueError, match="pairwise term has no tangent"):
        env.linearise(rpm)
    plain = _env(2, 2, "PYB_DRAG")
    with pytest.raises(ValueError, match="no downwash to differentiate"):
        plain.differentiable_rollout(rpm, downwash=True)
    big = CtrlAviary(num_drones=129, physics=Physics.PYB_DW, num_envs=1, initial_xyzs=stack_xyz(129, rng))
    big.reset()
    with pytest.raises(ValueError, match="at most 128"):
        big.differentiable_rollout(_rpm(big, 1, rng), downwash=True)
    env._EXTERNAL_DOWNWASH = True
    try:
        with pytest.raises(ValueError, match="sharded"):
            env.differentiable_rollout(rpm, downwash=True)
    finally:
        del env._EXTERNAL_DOWNWASH
    with pytest.raises(ValueError, match="policy and tracker"):
        env.differentiable_rollout(policy=object(), num_steps=2, downwash=True)
    with pytest.raises(ValueError, match="policy and tracker"):
        env.differentiable_rollout(controller=Tracker.__new__(Tracker), downwash=True)
    import torch.autograd.forward_ad as fwAD
    with fwAD.dual_level():
        dual = fwAD.make_dual(rpm, torch.ones_like(rpm))
        with pytest.raises(ValueError, match="reverse mode only"):
            env.differentiable_rollout(dual, downwash=True)
    ctl = DSLPIDControl(DroneModel.CF2X, num_drones=4, device=dev)
    wp = torch.tensor(stack_xyz(2, rng)[None, None].repeat(2, 1), device=dev).expand(3, 2, 2, 3).contiguous()
    with fwAD.dual_level():
        with pytest.raises(ValueError, match="reverse mode only"):
            env.differentiable_rollout(controller=ctl, waypoints=fwAD.make_dual(wp, torch.ones_like(wp)), downwash=True)
    r = rpm.clone().requires_grad_(True)
    out = env.differentiable_rollout(r, downwash=True)
    with pytest.raises(ValueError, match="double backward"):
        torch.autograd.grad(out["pos"].sum(), r, create_graph=True)


# ---- a use: system identification through downwash ----------------------------------------------------------------------

def _fit(env, rpm, start, last, rec, downwash, iters=3):
    theta = torch.zeros((2, env._E), dtype=torch.float64, device=env.device, requires_grad=True)
    opt = torch.optim.LBFGS([theta], lr=1, max_iter=200, history_size=20, tolerance_grad=1e-14, tolerance_change=1e-20,
                            line_search_fn="strong_wolfe")

    def closure():
        opt.zero_grad()
        out = env.differentiable_rollout(rpm, state=start, last_rpm=last, downwash=downwash,
                                         phys={"m": env.M * torch.exp(theta[0]), "kf": env.KF * torch.exp(theta[1])})
        loss = ((out["pos"] - rec["pos"]) / 1e-3).square().sum() + ((out["quat"] - rec["quat"]) / 1e-3).square().sum()
        loss.backward()
        return loss

    for _ in range(iters):
        opt.step(closure)
    return env.M * torch.exp(theta[0].detach()), env.KF * torch.exp(theta[1].detach())


def test_system_identification_through_downwash():
    """256 two-drone stacks 0.8 m apart (the lower drone loses over a third of its weight to downwash) fly recorded random-RPM
    flights with step(); fitting per-aviary m and kf from the nominal values with differentiable_rollout(downwash=True)
    recovers both to 1e-3 relative.  The downwash-blind twin (effects switched off: the per-drone adjoint) cannot."""
    E, T = 256, 24
    xyz = np.array([[0.0, 0.0, 1.0], [0.01, 0.0, 1.8]])
    env = _env(E, 2, "PYB_DW", xyz=xyz)
    rng = np.random.default_rng(7)
    dev = env.device
    m_true = torch.tensor(env.M * rng.uniform(0.7, 1.3, E), device=dev)
    kf_true = torch.tensor(env.KF * rng.uniform(0.7, 1.3, E), device=dev)
    env.set_physical_params(m=m_true, kf=kf_true)
    start = {k: getattr(env, k).clone() for k in STATE_KEYS}
    last = env.last_clipped_action.clone().reshape(E, 2, 4)
    rpm = _rpm(env, T, rng, 0.1, clip=False)
    rec = {k: [] for k in ("pos", "quat")}
    for k in range(T):
        env.step(rpm[k])
        for key in rec:
            rec[key].append(getattr(env, key).clone())
    rec = {k: torch.stack(v) for k, v in rec.items()}
    env.set_physical_params(m=env.M, kf=env.KF)
    m_fit, kf_fit = _fit(env, rpm, start, last, rec, True)
    em = float(((m_fit - m_true) / m_true).abs().max())
    ek = float(((kf_fit - kf_true) / kf_true).abs().max())
    print("system identification through downwash: worst relative error m %.1e, kf %.1e" % (em, ek))
    assert em < 1e-3 and ek < 1e-3
    env._effects = 0                                          # the downwash-blind twin
    m_b, kf_b = _fit(env, rpm, start, last, rec, False)
    eb = max(float(((m_b - m_true) / m_true).abs().max()), float(((kf_b - kf_true) / kf_true).abs().max()))
    print("downwash-blind twin: worst relative error %.1e" % eb)
    assert eb > 1e-3
