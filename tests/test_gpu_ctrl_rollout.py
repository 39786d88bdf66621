"""rollout() of the control envs (qs_ctrl_rollout): T control ticks of CtrlAviary / VelocityAviary in one launch.

* Twins: two envs (and controllers) built alike from the same seeds; one runs rollout(), the other the per-tick loop it
  replaces -- T x step(actions[k]) for RAW (float32 and float64 RPMs) and VEL, and the pid.py loop
  `rpm = ctrl.computeControlFromEnv(env, wp[(start + k) % W] + offset, ...); env.step(rpm)` for a controller.  Every output
  and all end state (planes, last_rpm, step counters, current observation, embedded / external controller state, reward,
  control_counter) must be the same bits.  Every Physics mode, downwash at D = 3 and D = 128, a per-aviary constants table,
  CF2X and CF2P, 240/48 and 240/240 Hz, CTAs that end part-way, and one run above a million drones.
* Continuation: split rollouts, rollout then step() and step() then rollout equal the pure loop.
* The reference's goldens: the pid.py circle (CF2X, CF2P) free-running for its first 8 ticks at test_pid_circle_workload's
  tolerances, and velocity_aviary_480 through VelocityAviary.rollout.
* An attached Logger, suppressed outputs, and the refusals through the env."""
import numpy as np
import pytest
import torch

from qs_testlib import RTOL, quat_err, relerr

pytestmark = pytest.mark.gpu


def _imports():
    from gym_pybullet_drones_b200.control import DSLPIDControl
    from gym_pybullet_drones_b200.envs import CtrlAviary, VelocityAviary
    from gym_pybullet_drones_b200.utils.enums import DroneModel, Physics
    return DSLPIDControl, CtrlAviary, VelocityAviary, DroneModel, Physics


def _bits(t):
    return t.contiguous().view(torch.int64 if t.dtype == torch.float64 else torch.int32)


def _same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    assert torch.equal(_bits(a), _bits(b)), what


def _stack(D):
    """Drones stacked in a narrow column so that downwash acts on most pairs."""
    i = np.arange(D)
    return np.stack([0.01 * (i % 8), 0.01 * ((i // 8) % 4), 0.2 + 0.02 * i], axis=1)


def _pair(cls, E, D, physics="DYN", model="CF2X", pyb=240, ctrl=48, init=None, table=None, seed=0):
    """Two identical envs (same constructor, same perturbed start state, same per-aviary constants)."""
    _, CtrlAviary, VelocityAviary, DroneModel, Physics = _imports()
    klass = {"ctrl": CtrlAviary, "vel": VelocityAviary}[cls]
    envs = []
    for _ in range(2):
        env = klass(drone_model=DroneModel[model], num_drones=D, physics=Physics[physics], pyb_freq=pyb, ctrl_freq=ctrl,
                    initial_xyzs=init, num_envs=E)
        env.reset()
        envs.append(env)
    rng = np.random.default_rng(seed)
    pos = envs[0].pos.cpu().numpy() + rng.uniform(-0.02, 0.02, (E, D, 3))
    q = np.concatenate([rng.uniform(-0.05, 0.05, (E, D, 3)), np.ones((E, D, 1))], axis=-1)
    q /= np.linalg.norm(q, axis=-1, keepdims=True)
    vel, rates = rng.uniform(-0.2, 0.2, (E, D, 3)), rng.uniform(-0.5, 0.5, (E, D, 3))
    sc = rng.integers(0, 1000) * envs[0].PYB_STEPS_PER_CTRL
    for env in envs:
        env.set_state(pos=pos, quat=q, vel=vel, rpy_rates=rates, step_counter=sc)
        if table is not None:
            r = np.random.default_rng(table)
            env.set_physical_params(m=env.M * r.uniform(0.8, 1.2, E), kf=env.KF * r.uniform(0.9, 1.1, E),
                                    km=env.KM * r.uniform(0.9, 1.1, E), ixx=env.J[0, 0] * r.uniform(0.8, 1.2, E),
                                    thrust2weight=env.THRUST2WEIGHT_RATIO * r.uniform(0.9, 1.1, E))
    return envs


def _state(env):
    out = dict(planes=env._planes, last_rpm=env._last_rpm, step_counter=env._step_counter, obs=env._obs_buf[env._cur], reward=env._reward)
    if env._pid is not None:
        out["pid"] = env._pid
    return out


def _assert_same_state(env, twin):
    sa, sb = _state(env), _state(twin)
    assert sa.keys() == sb.keys()
    for k in sa:
        _same(sa[k], sb[k], k)


def _raw_actions(env, T, seed, f64):
    rng = np.random.default_rng(seed)
    E, D = env._E, env._D
    a = env.HOVER_RPM * (1 + 0.05 * rng.uniform(-1, 1, (T, E, D, 4)))
    m = rng.uniform(size=a.shape)
    a[m < 0.03] = -100.0                                         # clipped to 0
    a[m > 0.97] = 1.5 * env.MAX_RPM                               # clipped to MAX_RPM (the aviary's own with a table)
    return torch.from_numpy(a if f64 else a.astype(np.float32)).cuda()


def _vel_actions(env, T, seed):
    rng = np.random.default_rng(seed)
    a = np.concatenate([rng.uniform(-1, 1, (T, env._E, env._D, 3)), rng.uniform(0, 1, (T, env._E, env._D, 1))], axis=-1)
    return torch.from_numpy(a.astype(np.float32)).cuda()


def _replay_actions(out, twin, actions):
    for k in range(actions.shape[0]):
        obs, rew, _, _, _ = twin.step(actions[k])
        _same(out["obs"][k], obs, ("obs", k))
        _same(out["rpm"][k], twin.last_clipped_action, ("rpm", k))
        assert float(rew[0]) == -1.0


def _circle(W, seed):
    """pid.py's circle of W waypoints (z = 0: the height comes from each drone's offset)."""
    i = np.arange(W)
    r = 0.3 + 0.05 * seed
    return np.stack([r * np.cos(2 * np.pi * i / W + np.pi / 2), r * np.sin(2 * np.pi * i / W + np.pi / 2) - r, np.zeros(W)], axis=1)


def _track_inputs(env, W, seed, extras=False):
    rng = np.random.default_rng(seed)
    n = env._N
    wp = _circle(W, seed)
    start = rng.integers(0, W, n).astype(np.int32)
    offset = np.zeros((n, 3))
    offset[:, 2] = env.pos.reshape(n, 3)[:, 2].cpu().numpy() + 0.1
    kw = dict(waypoints=wp, start=start, offset=offset, target_rpy=np.concatenate([np.zeros((n, 2)), rng.uniform(-0.5, 0.5, (n, 1))], axis=1))
    if extras:
        kw.update(target_vel=rng.uniform(-0.1, 0.1, (n, 3)), target_rpy_rates=rng.uniform(-0.1, 0.1, (n, 3)))
    return kw


def _track_loop(twin, ctrl, kw, T, k0=0, out=None, logger=None):
    """The pid.py loop on the twin for ticks k0 .. k0+T-1 of the schedule; checks `out` tick by tick when given."""
    from gym_pybullet_drones_b200.envs import CtrlAviary
    E, D, n = twin._E, twin._D, twin._N
    tp = CtrlAviary.schedule_targets(kw["waypoints"], kw["start"], kw.get("offset"), k0 + T)[k0:]
    for k in range(T):
        if logger is not None:
            c = np.zeros((n, 12))
            c[:, 0:3] = tp[k]
            for j, key in ((3, "target_rpy"), (6, "target_vel"), (9, "target_rpy_rates")):
                if kw.get(key) is not None:
                    c[:, j:j + 3] = kw[key]
            logger.set_controls(c.reshape(E, D, 12)[logger._rg.first_drone // D])
        rpm = ctrl.computeControlFromEnv(twin, tp[k], target_rpy=kw.get("target_rpy"), target_vel=kw.get("target_vel"),
                                         target_rpy_rates=kw.get("target_rpy_rates"))
        obs, rew, _, _, _ = twin.step(rpm)
        if out is not None:
            _same(out["obs"][k], obs, ("obs", k))
            _same(out["rpm"][k], twin.last_clipped_action, ("rpm", k))
            if "pos_e" in out:
                _same(out["pos_e"][k], ctrl._pos_e.view(E, D, 3), ("pos_e", k))
                _same(out["yaw_e"][k], ctrl._yaw_e.view(E, D), ("yaw_e", k))
            assert float(rew[0]) == -1.0


def _controllers(env, model):
    DSLPIDControl, _, _, DroneModel, _ = _imports()
    return [DSLPIDControl(DroneModel[model], num_drones=env._N, device=env.device) for _ in range(2)]


# (name, E, D, physics, model, pyb/ctrl, init, table)
CASES = [
    ("dyn", 100, 3, "DYN", "CF2X", (240, 48), None, None),
    ("gnd", 100, 3, "PYB_GND", "CF2X", (240, 48), None, None),
    ("drag", 100, 3, "PYB_DRAG", "CF2X", (240, 48), None, None),
    ("dw-d3", 100, 3, "PYB_DW", "CF2X", (240, 48), "stack", None),
    ("all-d3", 100, 3, "PYB_GND_DRAG_DW", "CF2X", (240, 48), "stack", None),
    ("dw-d128", 3, 128, "PYB_DW", "CF2X", (240, 48), "stack", None),
    ("all-d128-cf2p", 3, 128, "PYB_GND_DRAG_DW", "CF2P", (240, 48), "stack", None),
    ("table-all", 77, 2, "PYB_GND_DRAG_DW", "CF2X", (240, 48), "stack", 5),
    ("table-dyn-cf2p", 333, 1, "DYN", "CF2P", (240, 48), None, 6),
    ("cf2p-240", 50, 5, "PYB_DRAG", "CF2P", (240, 240), None, None),
    ("dyn-240", 129, 1, "DYN", "CF2X", (240, 240), None, None),
]


def _make(cls, case, seed=0):
    name, E, D, physics, model, (pyb, ctrl), init, table = case
    return _pair(cls, E, D, physics, model, pyb, ctrl, _stack(D) if init == "stack" else None, table, seed)


@pytest.mark.parametrize("f64", [False, True], ids=["f32", "f64"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_raw_rollout_equals_steps(case, f64):
    env, twin = _make("ctrl", case, 1)
    T = 13
    acts = _raw_actions(env, T, 3, f64)
    out = env.rollout(acts)
    assert set(out) == {"obs", "rpm"} and out["obs"].shape == (T, env._E, env._D, 20)
    _replay_actions(out, twin, acts)
    _assert_same_state(env, twin)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_vel_rollout_equals_steps(case):
    env, twin = _make("vel", case, 2)
    T = 11
    acts = _vel_actions(env, T, 4)
    out = env.rollout(acts)
    _replay_actions(out, twin, acts)
    _assert_same_state(env, twin)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_track_rollout_equals_control_loop(case):
    env, twin = _make("ctrl", case, 3)
    c1, c2 = _controllers(env, case[4])
    T, W = 14, 9
    kw = _track_inputs(env, W, 5, extras=case[0] in ("drag", "table-all"))
    out = env.rollout(controller=c1, errors=True, num_steps=T, **kw)
    assert set(out) == {"obs", "rpm", "pos_e", "yaw_e"}
    _track_loop(twin, c2, kw, T, out=out)
    _assert_same_state(env, twin)
    _same(c1._state, c2._state, "controller state")
    assert c1.control_counter == c2.control_counter == T


def test_track_full_schedule_per_drone_paths():
    """M = N, W = T: a full per-drone schedule (downwash.py-like, D = 3 with downwash)."""
    case = ("all-d3", 40, 3, "PYB_GND_DRAG_DW", "CF2X", (240, 48), "stack", None)
    env, twin = _make("ctrl", case, 7)
    c1, c2 = _controllers(env, "CF2X")
    T, n = 10, env._N
    rng = np.random.default_rng(9)
    wp = env.pos.cpu().numpy()[None] + np.cumsum(rng.uniform(-0.02, 0.02, (T, env._E, env._D, 3)), axis=0)
    kw = dict(waypoints=wp, start=np.zeros(n, np.int32), offset=None)
    out = env.rollout(controller=c1, errors=True, **kw)                 # num_steps defaults to W = T
    assert out["rpm"].shape[0] == T
    _track_loop(twin, c2, dict(kw, waypoints=wp.reshape(T, n, 3)), T, out=out)
    _assert_same_state(env, twin)
    _same(c1._state, c2._state, "controller state")


def test_million_drones():
    case = ("big", 1 << 20, 1, "DYN", "CF2X", (240, 48), None, None)
    env, twin = _make("ctrl", case, 11)
    c1, c2 = _controllers(env, "CF2X")
    T = 4
    kw = _track_inputs(env, 48, 13)
    out = env.rollout(controller=c1, errors=True, num_steps=T, **kw)
    _track_loop(twin, c2, kw, T, out=out)
    _assert_same_state(env, twin)
    _same(c1._state, c2._state, "controller state")


def test_continuation():
    """A rollout split in two calls equals one call; rollout then the per-tick loop, and the loop then a rollout, equal the
    pure loop (drag carries last_rpm, downwash couples the drones, the controller state crosses every boundary)."""
    case = ("all-d3", 60, 3, "PYB_GND_DRAG_DW", "CF2X", (240, 48), "stack", None)
    T1, T2, W = 5, 8, 7
    envs = _make("ctrl", case, 21) + _make("ctrl", case, 21)
    ctrls = [_controllers(envs[0], "CF2X")[0] for _ in range(4)]
    kw = _track_inputs(envs[0], W, 17)
    one, split, mix1, mix2 = envs
    ref_twin = _make("ctrl", case, 21)[0]
    ref_ctrl = _controllers(envs[0], "CF2X")[0]
    out = one.rollout(controller=ctrls[0], num_steps=T1 + T2, **kw)
    _track_loop(ref_twin, ref_ctrl, kw, T1 + T2, out=out)
    a = split.rollout(controller=ctrls[1], num_steps=T1, **kw)
    b = split.rollout(controller=ctrls[1], num_steps=T2, **dict(kw, start=kw["start"] + T1))
    _same(torch.cat([a["obs"], b["obs"]]), out["obs"], "split obs")
    _same(torch.cat([a["rpm"], b["rpm"]]), out["rpm"], "split rpm")
    a = mix1.rollout(controller=ctrls[2], num_steps=T1, **kw)
    _track_loop(mix1, ctrls[2], kw, T2, k0=T1)
    _track_loop(mix2, ctrls[3], kw, T1)
    b = mix2.rollout(controller=ctrls[3], num_steps=T2, **dict(kw, start=kw["start"] + T1))
    _same(b["obs"], out["obs"][T1:], "step then rollout")
    for env, c in ((one, ctrls[0]), (split, ctrls[1]), (mix1, ctrls[2]), (mix2, ctrls[3])):
        _assert_same_state(env, ref_twin)
        _same(c._state, ref_ctrl._state, "controller state")
        assert c.control_counter == T1 + T2


@pytest.mark.parametrize("model", ["cf2x", "cf2p"])
def test_pid_circle_golden_free_running(golden, model):
    """examples/pid.py through rollout(controller=...): the shared circle with per-drone phases and INIT_XYZS' z as the offset,
    free-running for the first 8 ticks at test_pid_circle_workload's tolerances (beyond them the reference itself amplifies
    perturbations ~1.5x per tick; the twins above carry the rest)."""
    DSLPIDControl, CtrlAviary, _, DroneModel, Physics = _imports()
    g = golden("pid_circle_" + model)
    dm = DroneModel[model.upper()]
    nd, cf = 3, 48
    W = cf * 10
    i = np.arange(W)
    x0, y0 = g["INIT_XYZS"][0, 0], g["INIT_XYZS"][0, 1]
    tpos = np.stack([0.3 * np.cos((i / W) * (2 * np.pi) + np.pi / 2) + x0, 0.3 * np.sin((i / W) * (2 * np.pi) + np.pi / 2) - 0.3 + y0,
                     np.zeros(W)], axis=1)
    start = np.array([int((j * W / 6) % W) for j in range(nd)])
    offset = np.zeros((nd, 3))
    offset[:, 2] = g["INIT_XYZS"][:, 2]
    T = 8
    assert np.array_equal(CtrlAviary.schedule_targets(tpos, start, offset, T), g["target"][:T])     # the schedule is pid.py's
    env = CtrlAviary(drone_model=dm, num_drones=nd, initial_xyzs=g["INIT_XYZS"], initial_rpys=g["INIT_RPYS"], physics=Physics.DYN,
                     pyb_freq=240, ctrl_freq=cf, num_envs=1)
    ctrl = DSLPIDControl(dm, num_drones=nd)
    env.reset()
    env.step(torch.zeros((1, nd, 4), dtype=torch.float64, device="cuda"))          # pid.py's first step: zero RPMs
    obs0 = env._obs_buf[env._cur].double().cpu().numpy()
    assert relerr(obs0[:, 0:3], g["obs"][0][:, 0:3]) < RTOL
    out = env.rollout(controller=ctrl, waypoints=tpos, start=start, offset=offset, target_rpy=g["INIT_RPYS"], num_steps=T, errors=True)
    obs, rpm = out["obs"][:, 0].double().cpu().numpy(), out["rpm"][:, 0].cpu().numpy()
    for k in range(T):
        ref = g["obs"][k + 1]
        assert relerr(obs[k][:, 0:3], ref[:, 0:3]) < RTOL and quat_err(obs[k][:, 3:7], ref[:, 3:7]) < RTOL, k
        assert relerr(obs[k][:, 7:16], ref[:, 7:16]) < RTOL, k
        if k > 0:
            assert relerr(rpm[k], g["action"][k]) < 1e-6, k                # free-running: 1e-12 x 1.5^k x the D-gain
            assert relerr(out["pos_e"][k, 0].double().cpu().numpy(), g["pos_e"][k]) < 1e-6, k
    assert ctrl.control_counter == T


def test_velocity_aviary_golden(golden):
    _, _, VelocityAviary, _, Physics = _imports()
    g = golden("velocity_aviary_480")
    env = VelocityAviary(num_drones=2, physics=Physics.DYN, pyb_freq=240, ctrl_freq=240, num_envs=1)
    obs, _ = env.reset()
    assert relerr(obs[0].cpu().numpy(), g["obs0"]) < 1e-6
    acts = torch.from_numpy(g["actions"].astype(np.float32)[:, None]).cuda()
    out = env.rollout(acts)
    o = out["obs"][:, 0].double().cpu().numpy()
    for t in range(acts.shape[0]):
        ref = g["obs"][t]
        assert relerr(o[t][:, 0:3], ref[:, 0:3]) < RTOL and quat_err(o[t][:, 3:7], ref[:, 3:7]) < RTOL, t
        assert relerr(o[t][:, 7:16], ref[:, 7:16]) < RTOL and relerr(o[t][:, 16:20], ref[:, 16:20]) < RTOL, t
    assert int(env._step_counter[0]) == acts.shape[0] * env.PYB_STEPS_PER_CTRL


@pytest.mark.parametrize("mode", ["track-targets", "vel"])
def test_logger_ring_equals_the_loop(tmp_path, mode):
    from gym_pybullet_drones_b200.utils.Logger import Logger
    case = ("all-d3", 20, 3, "PYB_GND_DRAG_DW", "CF2X", (240, 48), "stack", None)
    env, twin = _make("vel" if mode == "vel" else "ctrl", case, 31)
    T = 9
    logs = [Logger(logging_freq_hz=48, output_folder=str(tmp_path / s), num_drones=3).attach(e, aviary=7, capacity=16)
            for s, e in (("a", env), ("b", twin))]
    for lg in logs:
        lg.set_controls(np.arange(36, dtype=np.float32).reshape(3, 12) * 0.5)
    if mode == "vel":
        acts = _vel_actions(env, T, 8)
        env.rollout(acts, record=False)
        for k in range(T):
            twin.step(acts[k])
    else:
        c1, c2 = _controllers(env, "CF2X")
        kw = _track_inputs(env, 5, 41, extras=True)
        env.rollout(controller=c1, num_steps=T, log_targets=True, record=False, **kw)
        _track_loop(twin, c2, kw, T, logger=logs[1])
    _same(logs[0]._head, logs[1]._head, "head")
    _same(logs[0]._ring, logs[1]._ring, "ring")
    _assert_same_state(env, twin)
    paths = [lg.save() for lg in logs]
    a, b = np.load(paths[0]), np.load(paths[1])
    assert a.files == b.files
    for k in a.files:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), k


def test_suppressed_outputs_stay_untouched():
    case = ("drag", 70, 3, "PYB_DRAG", "CF2X", (240, 48), None, None)
    env, twin = _make("ctrl", case, 51)
    c1, c2 = _controllers(env, "CF2X")
    T = 6
    E, D = env._E, env._D
    kw = _track_inputs(env, 4, 53)
    sentinel = dict(obs=torch.full((T, E, D, 20), -7.25, device="cuda"), pos_e=torch.full((T, E, D, 3), 3.5, device="cuda"),
                    yaw_e=torch.full((T, E, D), 1.75, device="cuda"), rpm=torch.full((T, E, D, 4), 2.0, dtype=torch.float64, device="cuda"))
    keep = {k: v.clone() for k, v in sentinel.items()}
    out = env.rollout(controller=c1, num_steps=T, record=False, errors=False, out=sentinel, **kw)
    assert set(out) == {"rpm"} and out["rpm"] is sentinel["rpm"]
    for k in ("obs", "pos_e", "yaw_e"):
        _same(sentinel[k], keep[k], k)
    _track_loop(twin, c2, kw, T)
    _assert_same_state(env, twin)
    _same(c1._state, c2._state, "controller state")
    # RAW without rows: the env's current observation still receives the last tick
    env2, twin2 = _make("ctrl", case, 52)
    acts = _raw_actions(env2, T, 54, False)
    out = env2.rollout(acts, record=False)
    assert set(out) == {"rpm"}
    for k in range(T):
        twin2.step(acts[k])
    _assert_same_state(env2, twin2)


def test_refusals_through_the_env():
    DSLPIDControl, CtrlAviary, VelocityAviary, DroneModel, Physics = _imports()
    big = CtrlAviary(num_drones=129, physics=Physics.PYB_DW, num_envs=1)
    with pytest.raises(ValueError, match="drones_per_env <= 128"):
        big.rollout(torch.zeros((2, 1, 129, 4), device="cuda"))
    env = CtrlAviary(num_drones=2, physics=Physics.DYN, num_envs=4)
    wp = np.zeros((3, 3))
    with pytest.raises(ValueError, match="num_drones"):
        env.rollout(controller=DSLPIDControl(DroneModel.CF2X, num_drones=7), waypoints=wp)
    wrong = DSLPIDControl(DroneModel.CF2X, num_drones=8)
    wrong.device = torch.device("cuda", env.device.index + 1)
    with pytest.raises(ValueError, match="state is on"):
        env.rollout(controller=wrong, waypoints=wp)
    ok = DSLPIDControl(DroneModel.CF2X, num_drones=8)
    with pytest.raises(ValueError, match="either actions or a controller"):
        env.rollout(torch.zeros((2, 4, 2, 4), device="cuda"), controller=ok, waypoints=wp)
    with pytest.raises(ValueError, match="needs actions"):
        env.rollout()
    with pytest.raises(ValueError, match="waypoints"):
        env.rollout(controller=ok)
    with pytest.raises(ValueError, match="needs a controller rollout"):
        env.rollout(torch.zeros((2, 4, 2, 4), device="cuda"), errors=True)
    assert ok.control_counter == 0 and int(env._step_counter.sum()) == 0
    with pytest.raises(ValueError, match="vector API"):
        CtrlAviary(num_drones=2, physics=Physics.DYN).rollout(torch.zeros((2, 1, 2, 4), device="cuda"))
    with pytest.raises(ValueError, match="vector API"):
        VelocityAviary(num_drones=2, physics=Physics.DYN).rollout(torch.zeros((2, 1, 2, 4), device="cuda"))
