"""-m gpu: the LQR tracker of an iLQR plan flown by CtrlAviary.rollout(controller=ilqr.Tracker(sol)) (qs_ctrl_rollout_lqr,
DESIGN.md 4.1e).

Covered: sol["z"] against the solve's start and states; from the solve's own start on its own plant the tracker is
rollout(actions=sol["rpm"]) bit for bit, every output and the Logger ring included; from perturbed starts, on every Physics mode
(downwash up to 128 drones per aviary), three drone models, two control rates, n_z 13 and 17, plans flown on another plant, a
phys table on the plant only and partial CTAs, the launch equals a per-tick loop of tests/ilqr_tracker_ref.py and
rollout(actions=u, 1 tick), with a reversed summation and an omitted clamp as negative controls that miss; continuation; the
reordered-formation refusal; three tasks with bounds that open loop misses; and the refusals."""
import numpy as np
import pytest
import torch

import ilqr_tracker_ref as TR

pytestmark = pytest.mark.gpu

DEV = "cuda"
KEYS = ("pos", "quat", "vel", "rpy_rates")
F64 = torch.float64


def _imports():
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.ilqr import Tracker
    from gym_pybullet_drones_b200.utils.enums import DroneModel, Physics
    return CtrlAviary, Tracker, DroneModel, Physics


def _env(E, D, physics="DYN", model="CF2X", pyb=240, ctrl=48, seed=0, xyz=None, rpy=0.3):
    """physics "gnd_drag": GND|DRAG without the downwash of PYB_GND_DRAG_DW (what ilqr plans on)"""
    CtrlAviary, _, DroneModel, Physics = _imports()
    rng = np.random.default_rng(seed)
    if xyz is None:
        xyz = np.stack([rng.uniform(-1, 1, D), rng.uniform(-1, 1, D), rng.uniform(0.3, 1.5, D)], 1)
    name = "PYB_GND_DRAG_DW" if physics == "gnd_drag" else physics
    env = CtrlAviary(drone_model=getattr(DroneModel, model), num_drones=D, physics=getattr(Physics, name), pyb_freq=pyb, ctrl_freq=ctrl,
                     initial_xyzs=xyz, initial_rpys=rng.uniform(-rpy, rpy, (D, 3)), num_envs=E)
    env.reset()
    if physics == "gnd_drag":
        env._effects = 3
    return env


def _phys(env, seed, lo=0.8, hi=1.2):
    rng = np.random.default_rng(seed)
    E = env._E
    env.set_physical_params(m=env.M * rng.uniform(lo, hi, E), kf=env.KF * rng.uniform(lo, hi, E))


def _targets(env, seed, spread=0.5):
    rng = np.random.default_rng(seed)
    return {"pos": torch.tensor(rng.uniform(-spread, spread, (env._E, env._D, 3)) + np.array([0.0, 0.0, 1.0]), device=DEV)}


def _state(env):
    return torch.cat([getattr(env, k) for k in KEYS], dim=-1)


def _assert_same_env(a, b):
    for name in ("_planes", "_last_rpm", "_step_counter"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name
    assert torch.equal(a._obs_buf[a._cur], b._obs_buf[b._cur])


def _perturb(envs, seed, dp=0.03, dv=0.1, dw=0.2):
    rng = np.random.default_rng(seed)
    e = envs[0]
    shp = (e._E, e._D, 3)
    pos = e.pos.cpu().numpy() + rng.uniform(-dp, dp, shp)
    vel, w = rng.uniform(-dv, dv, shp), rng.uniform(-dw, dw, shp)
    for env in envs:
        env.set_state(pos=pos, vel=vel, rpy_rates=w)


def _bounds(kind, sol, env):
    if kind is None:
        return None
    if kind == "const":
        h = env.HOVER_RPM
        return (torch.full((4,), 0.97 * h, dtype=F64, device=DEV), torch.full((env._E, env._D, 4), 1.03 * h, dtype=F64, device=DEV))
    return (sol["rpm"] - 30.0, sol["rpm"] + 30.0)                                     # per tick, tight around the plan


# ---- 1: sol["z"] ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("physics", ["DYN", "PYB_DRAG"])
def test_loop_states_are_the_solves_start_and_states(physics):
    E, D, T = 9, 3, 12
    env = _env(E, D, physics, seed=1)
    env.rollout(actions=torch.full((1, E, D, 4), env.HOVER_RPM * 1.01, dtype=F64, device=DEV))      # last_rpm != 0
    start, last = _state(env).clone(), env._last_rpm.view(E, D, 4).clone()
    sol = env.ilqr(_targets(env, 2), num_steps=T, iters=2)
    nz = 17 if physics == "PYB_DRAG" else 13
    z = sol["z"]
    assert z.shape == (T, E, D, nz) and z.dtype == F64 and z.is_contiguous()
    assert torch.equal(z[0, ..., :13], start)
    assert torch.equal(z[1:, ..., :13], torch.cat([sol[k][:-1] for k in KEYS], dim=-1))
    if nz == 17:
        assert torch.equal(z[0, ..., 13:], last)
        mr = torch.tensor(env.MAX_RPM, dtype=F64, device=DEV)
        assert torch.equal(z[1:, ..., 13:], TR.clampd(sol["rpm"][:-1], torch.zeros_like(mr), mr))


# ---- 2: zero perturbation ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("phys", [False, True], ids=["nominal", "phys"])
@pytest.mark.parametrize("bounds", [None, "motor", "const", "per_tick"])
@pytest.mark.parametrize("physics", ["DYN", "PYB_GND", "PYB_DRAG"])
def test_zero_perturbation_is_the_open_loop_plan(tmp_path, physics, bounds, phys):
    from gym_pybullet_drones_b200.utils.Logger import Logger
    _, Tracker, _, _ = _imports()
    E, D, T = 6, 5, 16
    a, b = _env(E, D, physics, seed=3), _env(E, D, physics, seed=3)
    if phys:
        _phys(a, 4)
        _phys(b, 4)
    if bounds == "per_tick":
        h = a.HOVER_RPM
        g = np.random.default_rng(5)
        rb = (torch.tensor(h * g.uniform(0.85, 0.9, (T, E, D, 4)), device=DEV), torch.tensor(h * g.uniform(1.1, 1.15, (T, E, D, 4)), device=DEV))
    elif bounds == "const":
        rb = (torch.full((4,), 0.9 * a.HOVER_RPM, dtype=F64, device=DEV), torch.full((4,), 1.1 * a.HOVER_RPM, dtype=F64, device=DEV))
    else:
        rb = bounds
    sol = a.ilqr(_targets(a, 6), num_steps=T, iters=3, rpm_bounds=rb)
    logs = [Logger(logging_freq_hz=48, output_folder=str(tmp_path / s), num_drones=D).attach(e, aviary=2, capacity=32)
            for s, e in (("a", a), ("b", b))]
    trk = Tracker(sol, rpm_bounds=rb)
    ra = a.rollout(controller=trk)
    rb_ = b.rollout(actions=sol["rpm"])
    assert trk.tick == T
    for k in ("obs", "rpm"):
        assert torch.equal(ra[k], rb_[k]), k
    _assert_same_env(a, b)
    assert torch.equal(logs[0]._ring, logs[1]._ring) and torch.equal(logs[0]._head, logs[1]._head)
    assert torch.equal(_state(a), torch.cat([sol[k][-1] for k in KEYS], dim=-1))


# ---- 3: the law, teacher-forced ------------------------------------------------------------------------------------------------

LAW = [
    # id, plant, planner, model, (pyb, ctrl), E, D, phys table on the plant, bounds
    ("dyn-cf2x", "DYN", "DYN", "CF2X", (240, 48), 37, 3, False, None),
    ("pyb-cf2p-240hz", "PYB", "DYN", "CF2P", (240, 240), 5, 7, False, "per_tick"),
    ("gnd-race-phys", "PYB_GND", "PYB_GND", "RACE", (240, 48), 10, 3, True, "const"),
    ("drag-nz17-240hz", "PYB_DRAG", "PYB_DRAG", "CF2X", (240, 240), 13, 5, False, "per_tick"),
    ("dw-128", "PYB_DW", "DYN", "CF2X", (240, 48), 2, 128, False, None),
    ("all-dw-nz17-phys", "PYB_GND_DRAG_DW", "gnd_drag", "CF2P", (240, 48), 3, 100, True, "per_tick"),
    ("plan-dyn-fly-drag", "PYB_DRAG", "DYN", "RACE", (240, 48), 7, 9, False, None),
    ("plan-nz17-fly-dyn", "DYN", "PYB_DRAG", "CF2X", (240, 48), 9, 4, True, None),
    ("one-drone", "DYN", "DYN", "CF2X", (240, 48), 1, 1, False, "const"),
]


@pytest.mark.parametrize("case", LAW, ids=[c[0] for c in LAW])
def test_the_law_teacher_forced(case):
    _, Tracker, _, _ = _imports()
    _, plant, planner, model, (pyb, ctrl), E, D, phys, kind = case
    T, n = 12, E * D
    a, b = _env(E, D, plant, model, pyb, ctrl, seed=7), _env(E, D, plant, model, pyb, ctrl, seed=7)
    p = _env(E, D, planner, model, pyb, ctrl, seed=7)
    if phys:
        _phys(a, 8, 0.9, 1.1)
        _phys(b, 8, 0.9, 1.1)
    sol = p.ilqr(_targets(p, 9), num_steps=T, iters=3)
    nz = sol["K"].shape[-1]
    bounds = _bounds(kind, sol, p)
    _perturb([a, b], 10)
    trk = Tracker(sol, rpm_bounds=bounds)
    ra = a.rollout(controller=trk)
    zt, Kt, rt = sol["z"].reshape(T, n, nz), sol["K"].reshape(T, n, 4, nz), sol["rpm"].reshape(T, n, 4)
    rpm, obs, miss_order, miss_clamp, bound = [], [], 0, 0, 0
    for k in range(T):
        x, prev = TR.drone_vec(b._planes, n), b._last_rpm.clone()
        lo = hi = None
        if bounds is not None:
            lo, hi = (t.expand(T, E, D, 4)[k].reshape(n, 4) if t.dim() == 4 else t.expand(E, D, 4).reshape(n, 4) for t in bounds)
        u = TR.control(x, prev, zt[k], Kt[k], rt[k], lo, hi)
        out = b.rollout(actions=u.view(1, E, D, 4))
        rpm.append(out["rpm"][0])
        obs.append(out["obs"][0])
        got = ra["rpm"][k].reshape(n, 4)
        miss_order += int((TR.control(x, prev, zt[k], Kt[k], rt[k], lo, hi, order=range(nz - 1, -1, -1)) != got).sum())
        if lo is not None:
            free = TR.control(x, prev, zt[k], Kt[k], rt[k])
            miss_clamp += int((free != got).sum())
            bound += int(((free < lo) | (free > hi)).sum())
    assert torch.equal(ra["rpm"], torch.stack(rpm))
    assert torch.equal(ra["obs"], torch.stack(obs))
    _assert_same_env(a, b)
    print("%s: n_z %d, reversed summation misses %d of %d commands; clamp binds %d, omitting it misses %d"
          % (case[0], nz, miss_order, 4 * n * T, bound, miss_clamp))
    assert miss_order > 0 or n == 1                        # one drone's few commands can round alike in either order
    if bounds is not None:
        assert miss_clamp >= bound > 0                     # every clamped command, and those the motor clip also holds


# ---- 4: continuation -----------------------------------------------------------------------------------------------------------

def test_continuation_and_suppressed_outputs():
    _, Tracker, _, _ = _imports()
    E, D, T, R = 11, 3, 20, 7
    a, b, p = _env(E, D, "PYB_DRAG", seed=11), _env(E, D, "PYB_DRAG", seed=11), _env(E, D, "PYB_DRAG", seed=11)
    sol = p.ilqr(_targets(p, 12), num_steps=T, iters=3)
    _perturb([a, b], 13)
    ta, tb = Tracker(sol), Tracker(sol)
    first = a.rollout(controller=ta, num_steps=R)
    assert ta.tick == R
    sentinel = torch.full((T - R, E, D, 20), 7.0, dtype=torch.float32, device=DEV)
    rpm_buf = torch.empty((T - R, E, D, 4), dtype=F64, device=DEV)
    rest = a.rollout(controller=ta, record=False, out={"obs": sentinel, "rpm": rpm_buf})
    assert ta.tick == T and "obs" not in rest and rest["rpm"] is rpm_buf
    assert (sentinel == 7.0).all()
    whole = b.rollout(controller=tb)
    assert torch.equal(torch.cat([first["rpm"], rest["rpm"]]), whole["rpm"])
    assert torch.equal(first["obs"], whole["obs"][:R])
    _assert_same_env(a, b)
    tb.tick = 3                                            # the caller may set it
    c = _env(E, D, "PYB_DRAG", seed=11)
    c.set_state(**{k: getattr(b, k) for k in KEYS}, step_counter=0)
    c._last_rpm.copy_(b._last_rpm)
    assert c.rollout(controller=tb, num_steps=2)["rpm"].shape == (2, E, D, 4) and tb.tick == 5


def test_a_plan_of_any_strides_flies_the_same():
    _, Tracker, _, _ = _imports()
    E, D, T = 5, 3, 10
    a, b, p = _env(E, D, "PYB_DRAG", seed=14), _env(E, D, "PYB_DRAG", seed=14), _env(E, D, "PYB_DRAG", seed=14)
    sol = p.ilqr(_targets(p, 15), num_steps=T, iters=2)
    _perturb([a, b], 16)
    # the same values through per-drone [E, D, T, ...] storage: non-contiguous [T, E, D, ...] views
    strided = {k: sol[k].permute(1, 2, 0, *range(3, sol[k].dim())).contiguous().permute(2, 0, 1, *range(3, sol[k].dim()))
               for k in ("rpm", "K", "z")}
    assert not any(v.is_contiguous() for v in strided.values())
    ts = Tracker(strided)
    assert ts.K.is_contiguous() and ts.z_nom.is_contiguous() and ts.rpm_nom.is_contiguous()
    ra, rb = a.rollout(controller=ts), b.rollout(controller=Tracker(sol))
    assert torch.equal(ra["rpm"], rb["rpm"])
    _assert_same_env(a, b)


# ---- 5: a reordered formation --------------------------------------------------------------------------------------------------

def test_reordered_formation_is_refused():
    CtrlAviary, Tracker, _, Physics = _imports()
    from test_gpu_formation import stacks
    xyz = stacks(10, 9)[:333]
    xyz = xyz[np.random.default_rng(5).permutation(len(xyz))]
    a = CtrlAviary(num_drones=len(xyz), initial_xyzs=xyz, physics=Physics.PYB_DW, num_envs=1)
    p = CtrlAviary(num_drones=len(xyz), initial_xyzs=xyz, physics=Physics.DYN, num_envs=1)
    a.reset(); p.reset()
    a.reorder_by_morton()
    sol = p.ilqr({"pos": torch.tensor(xyz + np.array([0.3, -0.2, 0.4]), device=DEV)[None]}, num_steps=8, iters=2)
    trk = Tracker(sol)
    with pytest.raises(ValueError):
        a.rollout(actions=sol["rpm"])                      # rollout(actions=) refuses the formation too
    with pytest.raises(ValueError, match="reorder_by_morton"):
        a.rollout(controller=trk)
    a._effects = 0                                         # even without the downwash that makes it a formation
    with pytest.raises(ValueError, match="reorder_by_morton"):
        a.rollout(controller=trk)
    assert trk.tick == 0


# ---- 6: tasks ------------------------------------------------------------------------------------------------------------------

def _quat_small(rng, n, tilt):
    from gym_pybullet_drones_b200.params import quaternion_from_euler
    rp = rng.uniform(-1, 1, (n, 2))
    rp = rp / np.maximum(np.linalg.norm(rp, axis=1, keepdims=True), 1e-12) * rng.uniform(0, tilt, (n, 1))
    return np.stack([quaternion_from_euler(np.array([r, q, 0.0])) for r, q in rp])


def _ball(rng, n, r):
    v = rng.normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True) * r * rng.uniform(0, 1, (n, 1)) ** (1 / 3)


def test_task_formation_from_perturbed_starts():
    """The formation task of test_gpu_ilqr.py, flown from perturbed starts.  The solve ends with mu up to 1e5 on some drones,
    which shrinks their K by about 1 / (1 + mu) (Kmax 0.1 against 1.8e5 elsewhere) and left them near the open loop's error (2.08
    m worst); the gains are therefore recomputed at mu = 0 at the returned trajectory before flying (Tracker's docstring)."""
    _, Tracker, _, _ = _imports()
    from gym_pybullet_drones_b200.ilqr import Problem, solve
    from gym_pybullet_drones_b200.params import quaternion_from_euler
    E, D, T = 1024, 4, 96
    n = E * D
    a, b = _env(E, D, "DYN", seed=10), _env(E, D, "DYN", seed=10)
    rng = np.random.default_rng(11)
    start = np.array([0.0, 0.0, 1.0]) + rng.uniform(-0.5, 0.5, (n, 3)) / np.sqrt(3)
    quat = np.stack([quaternion_from_euler(r) for r in rng.uniform(-0.3, 0.3, (n, 3)) / np.sqrt(3)])
    state = {"pos": torch.tensor(start, device=DEV).reshape(E, D, 3), "quat": torch.tensor(quat, device=DEV).reshape(E, D, 4),
             "vel": torch.zeros((E, D, 3), dtype=F64, device=DEV), "rpy_rates": torch.zeros((E, D, 3), dtype=F64, device=DEV)}
    goal = torch.tensor(np.array([0.0, 0.0, 1.0]) + rng.uniform(-0.5, 0.5, (n, 3)) / np.sqrt(3), device=DEV).reshape(E, D, 3)
    p = Problem(a, {"pos": goal}, num_steps=T, state=state)
    sol = solve(p, 30)
    print("task a: drones ending the solve with mu > 0: %d of %d" % (int((sol["mu"] > 0).sum()), n))
    p.mu.zero_()
    p.backward()                                           # the tracker's gains at mu = 0, at the returned trajectory
    assert int(p.status.sum()) == 0
    sol = p.result(sol["cost"])
    # perturbed starts: up to 5 cm, 0.05 rad of tilt (composed with the planned attitude) and 0.1 rad/s of rates
    from scipy.spatial.transform import Rotation
    dq = Rotation.from_quat(_quat_small(rng, n, 0.05))
    q = (Rotation.from_quat(quat) * dq).as_quat()
    pert = dict(pos=start + _ball(rng, n, 0.05), quat=q, vel=np.zeros((n, 3)), rpy_rates=_ball(rng, n, 0.1))
    for env in (a, b):
        env.set_state(**{k: v.reshape(E, D, -1) for k, v in pert.items()})
    a.rollout(controller=Tracker(sol), record=False)
    b.rollout(actions=sol["rpm"], record=False)
    err, err_ol = ((x.pos - goal).norm(dim=-1) for x in (a, b))
    print("task a: worst / mean final position error %.3e / %.3e m with the tracker, %.3e / %.3e m open loop (plan %.3e m)"
          % (err.max().item(), err.mean().item(), err_ol.max().item(), err_ol.mean().item(),
             (sol["pos"][-1] - goal).norm(dim=-1).max().item()))
    # measured on an H100: 4.86e-3 m worst with the tracker (the plan's own 4.84e-3 m), 2.26 m open loop; bound 2x the former
    assert err.max().item() <= TASK_A_BOUND
    assert err_ol.max().item() > TASK_A_BOUND


TASK_A_BOUND = 0.01      # m
TASK_B_BOUND = 0.035     # m
TASK_C_BOUND = 0.25      # m


def _stacked(E, physics, seed, dz=1.5):
    """E aviaries of 4 drones stacked dz apart, each 3 cm off the axis of the one below.  At dz = 1.5 m the drones above push a
    lower one down with up to about 0.045 N, 17 % of a CF2X's weight, which the DYN plan does not model.  (At 0.4 m it is 0.38 N
    on the next drone alone, more than the 0.6 N of full thrust leaves after the weight: no controller can hold that stack.)"""
    xyz = np.array([[0.0, 0.0, 0.5], [0.03, 0.0, 0.5 + dz], [0.0, 0.03, 0.5 + 2 * dz], [0.03, 0.03, 0.5 + 3 * dz]])
    return _env(E, 4, physics, seed=seed, xyz=xyz, rpy=0.0)


def test_tasks_on_an_unmodelled_plant_and_receding_horizon():
    """(b) planned with DYN and nominal constants under the motor box, flown with ground effect, drag, downwash and masses
    scaled by 0.9-1.1; (c) the same plant with the plan replanned from the plant's state every R ticks (2 iterations, the previous
    plan shifted by R and padded with hover), each piece flown by its own Tracker."""
    _, Tracker, _, _ = _imports()
    E, T, R = 256, 96, 16
    p = _stacked(E, "DYN", 20)
    goal = p.pos.clone() + torch.tensor([0.3, -0.2, 0.2], dtype=F64, device=DEV)
    sol = p.ilqr({"pos": goal}, num_steps=T, iters=30, rpm_bounds="motor")
    a, b, c = (_stacked(E, "PYB_GND_DRAG_DW", 20) for _ in range(3))
    m = p.M * np.random.default_rng(21).uniform(0.9, 1.1, E)
    for env in (a, b, c):
        env.set_physical_params(m=m)
    a.rollout(controller=Tracker(sol, rpm_bounds="motor"), record=False)
    b.rollout(actions=sol["rpm"], record=False)
    rpm = sol["rpm"]
    hover = torch.full((R, E, 4, 4), p.HOVER_RPM, dtype=F64, device=DEV)
    for r in range(T // R):
        s = sol
        if r > 0:
            rpm = torch.cat([rpm[R:], hover]).clamp(0.0, p.MAX_RPM)
            s = p.ilqr({"pos": goal}, rpm=rpm, iters=2, state={k: getattr(c, k).clone() for k in KEYS}, rpm_bounds="motor")
        rpm = s["rpm"]
        c.rollout(controller=Tracker(s, rpm_bounds="motor"), num_steps=R, record=False)
    err, err_ol, err_rh = ((x.pos - goal).norm(dim=-1) for x in (a, b, c))
    print("task b: worst / mean final position error %.3e / %.3e m with the tracker, %.3e / %.3e m open loop"
          % (err.max().item(), err.mean().item(), err_ol.max().item(), err_ol.mean().item()))
    print("task c: worst / mean final position error %.3e / %.3e m, receding horizon (R = %d, iters = 2)"
          % (err_rh.max().item(), err_rh.mean().item(), R))
    # measured on an H100: (b) 1.69e-2 m worst, open loop 366 m; (c) 0.113 m worst.  Bounds: about 2x the measured worst.
    # (c) does not end closer than (b): at the end of the flight its latest plan is R ticks into a 96-tick horizon, its terminal
    # weight Q_final = 100 Q still 80 ticks away, while (b) ends on its plan's terminal tick; and 2 iterations from the shifted
    # guess leave part of the horizon unconverged (DESIGN.md 4.1e).
    assert err.max().item() <= TASK_B_BOUND
    assert err_ol.max().item() > TASK_C_BOUND
    assert err_rh.max().item() <= TASK_C_BOUND


# ---- 7: refusals ---------------------------------------------------------------------------------------------------------------

def test_refusals():
    CtrlAviary, Tracker, _, Physics = _imports()
    E, D, T = 2, 3, 6
    env = _env(E, D, "DYN", seed=30)
    sol = env.ilqr(_targets(env, 31), num_steps=T, iters=1)
    trk = Tracker(sol)
    with pytest.raises(ValueError, match="plan is for"):
        _env(E, D + 1, "DYN", seed=30).rollout(controller=trk)
    with pytest.raises(ValueError, match="plan is for"):
        _env(E + 1, D, "DYN", seed=30).rollout(controller=trk)
    with pytest.raises(ValueError, match="do not fit"):
        env.rollout(controller=trk, num_steps=T + 1)
    trk.tick = 4
    with pytest.raises(ValueError, match="do not fit"):
        env.rollout(controller=trk, num_steps=3)
    trk.tick = -1
    with pytest.raises(ValueError, match="tick must be an integer >= 0"):
        env.rollout(controller=trk)
    trk.tick = T
    with pytest.raises(ValueError, match="do not fit"):
        env.rollout(controller=trk)                        # nothing left of the plan
    trk.tick = 0
    cpu = dict(sol)
    cpu.update(rpm=sol["rpm"].cpu(), K=sol["K"].cpu(), z=sol["z"].cpu())
    with pytest.raises(ValueError):
        Tracker(cpu)
    other = Tracker(sol)
    other.device = torch.device("cpu")
    with pytest.raises(ValueError, match="plan is on"):
        env.rollout(controller=other)
    drag = _env(E, D, "PYB_DRAG", seed=30)
    sol17 = drag.ilqr(_targets(drag, 31), num_steps=T, iters=1)
    nolast = CtrlAviary(num_drones=D, physics=Physics.DYN, num_envs=E, track_last_action=False)
    nolast.reset()
    with pytest.raises(ValueError, match="last_clipped_action"):
        nolast.rollout(controller=Tracker(sol17))
    single = CtrlAviary(num_drones=1, physics=Physics.DYN)
    single.reset()
    one = _env(1, 1, "DYN", seed=32)
    with pytest.raises(ValueError, match="vector API"):
        single.rollout(controller=Tracker(one.ilqr(_targets(one, 33), num_steps=T, iters=1)))
    big = CtrlAviary(num_drones=129, physics=Physics.PYB_DW, num_envs=1)
    big.reset()
    twin = CtrlAviary(num_drones=129, physics=Physics.DYN, num_envs=1)
    twin.reset()
    with pytest.raises(ValueError, match="drones_per_env <= 128"):
        big.rollout(controller=Tracker(twin.ilqr({"pos": torch.tensor([0.0, 0.0, 1.0], dtype=F64, device=DEV)}, num_steps=T, iters=1)))
    gd = _env(E, D, "gnd_drag", seed=30)
    with pytest.raises(ValueError, match="GND\\|DRAG"):
        gd.rollout(controller=Tracker(gd.ilqr(_targets(gd, 31), num_steps=T, iters=1)))
    with pytest.raises(ValueError, match="takes no waypoints"):
        env.rollout(controller=trk, waypoints=np.zeros((4, 3)))
    with pytest.raises(ValueError, match="errors=True"):
        env.rollout(controller=trk, errors=True)
    with pytest.raises(ValueError, match="log_targets"):
        env.rollout(controller=trk, log_targets=True)
    with pytest.raises(ValueError, match="either actions or a controller"):
        env.rollout(actions=sol["rpm"], controller=trk)
    with pytest.raises(ValueError, match="lo <= hi"):
        Tracker(sol, rpm_bounds=(torch.full((4,), 2.0e4, dtype=F64, device=DEV), torch.full((4,), 1.0e4, dtype=F64, device=DEV)))
    with pytest.raises(ValueError, match="K"):
        Tracker(dict(sol, K=sol["K"][..., :12]))
    with pytest.raises(ValueError, match="z"):
        Tracker(dict(sol, z=sol["z"][:-1]))
    assert trk.tick == 0 and int(env._step_counter[0]) == 0
