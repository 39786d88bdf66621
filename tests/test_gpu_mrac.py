"""MRAC on the device (qs_mrac_control, qs_mrac_control_state, qs_ctrl_rollout_mrac).

* KAT: computeControl against the reference's fixture for CF2X, CF2P and RACE, fed the reference's inputs, at TF_TOL.
* Env loop: computeControlFromEnv + step at 4096 random states, each call teacher-forced against the tier-2 oracle.
* Rollout = loop: `CtrlAviary.rollout(controller=MRAC(...))` against its twin running computeControlFromEnv + step, every output
  and all end state the same bits; every Physics mode, downwash at D = 3 and 128, a per-aviary table, partial CTAs, continuation
  across two calls, the Logger ring with log_targets, suppressed outputs and a million drones.
* The fixture's closed loops (mrac.py's CF2X loop, the CF2P offset case) free-running against the reference for the horizon
  derived by free_running_horizon (tier 2 against a twin with a one-ulp perturbation per tick).
* reset() keeps Kx / Kr and re-initialises Xm; refusals."""
import numpy as np
import pytest
import torch

from mrac_testlib import DT, MODELS, TF_TOL, TOL, drone_model, err, free_running_horizon, gains_of, kat_worst, loop_inputs, loop_worst
from test_gpu_ctrl_rollout import _assert_same_state, _pair, _same, _track_inputs

pytestmark = pytest.mark.gpu
F32_TOL = 2.0 ** -23          # pos_e / rpy_e are float32: one rounding of the float64 value


def _mrac(m, n):
    from gym_pybullet_drones_b200.control import MRAC
    return MRAC(drone_model(m), num_drones=n)


def _dev(x):
    return torch.as_tensor(np.ascontiguousarray(x, dtype=np.float64), device="cuda")


class _Device:
    """MRAC.computeControl behind the interface of mrac_testlib.kat_worst / loop_worst."""

    def __init__(self, m, n):
        self.c = _mrac(m, n)

    def call(self, pos, quat, vel, angv, t):
        rpm, pe, re = self.c.computeControl(DT, _dev(pos), _dev(quat), _dev(vel), _dev(angv), _dev(t[:, 0:3]), _dev(t[:, 3:6]),
                                            _dev(t[:, 6:9]), _dev(t[:, 9:12]))
        return rpm.cpu().numpy(), pe.cpu().numpy(), re.cpu().numpy()

    def state(self):
        return self.c.Kx, self.c.Kr, self.c.Xm


@pytest.mark.parametrize("m", MODELS)
def test_kat_compute_control(golden, m):
    """computeControl fed the reference's inputs, the three calls of every controller chained (and, for CF2X, the 600 calls of
    mrac.py's loop): rpm and the controller state at TF_TOL, the float32 pos_e / rpy_e to their rounding."""
    g = golden("mrac")
    d = _Device(m, 256)
    worst = kat_worst(d, g, m)
    assert d.c.control_counter == 3
    if m == "cf2x":
        for k, v in loop_worst(_Device(m, 1), g).items():
            worst[k] = max(worst.get(k, 0.0), v)
    print(m, {k: "%.1e" % v for k, v in worst.items()})
    assert max(worst[k] for k in ("rpm", "Kx", "Kr", "Xm")) <= TF_TOL, worst
    assert max(worst["pos_e"], worst["rpy_e"]) <= F32_TOL, worst


def _oracle_from(c, m, G):
    """A tier-2 controller holding the device controller's current state."""
    from oracle.mrac_oracle import OracleMRAC
    o = OracleMRAC(c.num_drones, m, gains_=G)
    o.Kx, o.Kr, o.Xm, o.control_counter = c.Kx.copy(), c.Kr.copy(), c.Xm.copy(), c.control_counter
    return o


def test_env_loop_teacher_forced(golden):
    """computeControlFromEnv + step at 4096 random states: each call against tier 2 fed the env's float64 state and the device
    controller's state; ang_v is rebuilt from the planes on both sides."""
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils.enums import Physics
    from oracle.mrac_oracle import ang_v_from_state
    E = 4096
    env = CtrlAviary(num_drones=1, physics=Physics.DYN, pyb_freq=240, ctrl_freq=120, num_envs=E)
    env.reset()
    rng = np.random.default_rng(7)
    q = np.concatenate([rng.normal(0, 0.1, (E, 1, 3)), np.ones((E, 1, 1))], axis=-1)
    env.set_state(pos=rng.uniform(-1, 1, (E, 1, 3)) + [0, 0, 1], quat=q / np.linalg.norm(q, axis=-1, keepdims=True),
                  vel=rng.uniform(-0.5, 0.5, (E, 1, 3)), rpy_rates=rng.uniform(-1, 1, (E, 1, 3)))
    c = _mrac("cf2x", E)
    G = gains_of(golden("mrac"), "cf2x")
    tgt = np.concatenate([rng.uniform(-1, 1, (E, 2)), rng.uniform(0.5, 1.5, (E, 1))], axis=1)
    trpy = np.concatenate([np.zeros((E, 2)), rng.uniform(-0.3, 0.3, (E, 1))], axis=1)
    worst = 0.0
    for k in range(4):
        o = _oracle_from(c, "cf2x", G)
        pos, quat = env.pos.reshape(E, 3).cpu().numpy(), env.quat.reshape(E, 4).cpu().numpy()
        vel, w = env.vel.reshape(E, 3).cpu().numpy(), env.rpy_rates.reshape(E, 3).cpu().numpy()
        rpm_o, pe_o, re_o = o.compute(DT, pos, quat, vel, ang_v_from_state(quat, w), tgt, trpy)
        rpm = c.computeControlFromEnv(env, tgt, target_rpy=trpy)
        got = rpm.reshape(E, 4).cpu().numpy()
        worst = max(worst, err(got, np.clip(rpm_o, 0, env.MAX_RPM)), err(c.Kx, o.Kx), err(c.Kr, o.Kr), err(c.Xm, o.Xm))
        assert err(c.last_pos_e.cpu().numpy(), pe_o) <= F32_TOL and err(c.last_rpy_e.cpu().numpy(), re_o) <= F32_TOL
        env.step(rpm)
    print("env loop worst %.1e" % worst)
    assert worst <= TF_TOL


def _mrac_loop(twin, ctrl, kw, T, k0=0, logger=None):
    """mrac.py's loop on the twin for ticks k0 .. k0+T-1 of the schedule: (rpm, pos_e, rpy_e) per tick, stacked."""
    from gym_pybullet_drones_b200.envs import CtrlAviary
    E, D, n = twin._E, twin._D, twin._N
    tp = CtrlAviary.schedule_targets(kw["waypoints"], kw["start"], kw.get("offset"), k0 + T)[k0:]
    out = {k: [] for k in ("obs", "rpm", "pos_e", "rpy_e")}
    for k in range(T):
        if logger is not None:
            c = np.zeros((n, 12))
            c[:, 0:3] = tp[k]
            for j, key in ((3, "target_rpy"), (6, "target_vel"), (9, "target_rpy_rates")):
                if kw.get(key) is not None:
                    c[:, j:j + 3] = kw[key]
            logger.set_controls(c.reshape(E, D, 12)[logger._rg.first_drone // D])
        rpm = ctrl.computeControlFromEnv(twin, tp[k], kw.get("target_rpy"), kw.get("target_vel"), kw.get("target_rpy_rates"))
        out["pos_e"].append(ctrl.last_pos_e.clone().view(E, D, 3))
        out["rpy_e"].append(ctrl.last_rpy_e.clone().view(E, D, 3))
        obs, _, _, _, _ = twin.step(rpm)
        out["obs"].append(obs.clone())
        out["rpm"].append(twin.last_clipped_action.clone())
    return {k: torch.stack(v) for k, v in out.items()}


def _check_rollout(envs, m, T, W, extras=False, seed=0, split=None, record=True):
    env, twin = envs
    c1, c2 = _mrac(m, env._N), _mrac(m, env._N)
    kw = _track_inputs(env, W, seed, extras)
    if split is None:
        res = env.rollout(controller=c1, num_steps=T, errors=True, record=record, **kw)
        parts = [res]
    else:
        kw1 = dict(kw)
        parts = [env.rollout(controller=c1, num_steps=split, errors=True, **kw1)]
        kw2 = dict(kw, start=np.asarray(kw["start"]) + split)
        parts.append(env.rollout(controller=c1, num_steps=T - split, errors=True, **kw2))
        res = {k: torch.cat([p[k] for p in parts]) for k in parts[0]}
    ref = _mrac_loop(twin, c2, kw, T)
    keys = ("rpm", "pos_e", "rpy_e") + (("obs",) if record else ())
    for k in keys:
        _same(res[k], ref[k].reshape(res[k].shape), k)
    _assert_same_state(env, twin)
    _same(c1._state, c2._state, "mrac state")
    assert c1.control_counter == c2.control_counter == T


@pytest.mark.parametrize("physics", ["DYN", "PYB_GND", "PYB_DRAG", "PYB_DW", "PYB_GND_DRAG_DW"])
def test_rollout_equals_loop_every_physics(physics):
    _check_rollout(_pair("ctrl", 37, 3, physics=physics, ctrl=120, seed=1), "cf2x", T=24, W=16)    # 111 drones: one partial CTA


@pytest.mark.parametrize("m", ["cf2p", "race"])
def test_rollout_equals_loop_models(m):
    _check_rollout(_pair("ctrl", 50, 2, model=m.upper(), ctrl=120, seed=2), m, T=12, W=12, extras=True)


def test_rollout_equals_loop_downwash_128_and_table():
    _check_rollout(_pair("ctrl", 3, 128, physics="PYB_DW", ctrl=120, seed=3), "cf2x", T=8, W=8)
    _check_rollout(_pair("ctrl", 41, 4, physics="PYB_GND_DRAG_DW", ctrl=48, table=11, seed=4), "cf2x", T=10, W=7, extras=True)


def test_rollout_continues_across_calls_and_records_nothing():
    _check_rollout(_pair("ctrl", 64, 3, ctrl=120, seed=5), "cf2x", T=20, W=9, split=7)
    _check_rollout(_pair("ctrl", 64, 3, ctrl=120, seed=6), "cf2x", T=6, W=9, record=False)


def test_rollout_logger_with_targets(tmp_path):
    from gym_pybullet_drones_b200.utils.Logger import Logger
    env, twin = _pair("ctrl", 8, 2, ctrl=120, seed=8)
    logs = [Logger(logging_freq_hz=120, output_folder=str(tmp_path / s), num_drones=2).attach(e, aviary=3, capacity=16)
            for s, e in (("a", env), ("b", twin))]
    c1, c2 = _mrac("cf2x", 16), _mrac("cf2x", 16)
    kw = _track_inputs(env, 6, 8, extras=True)
    env.rollout(controller=c1, num_steps=6, log_targets=True, record=False, **kw)
    _mrac_loop(twin, c2, kw, 6, logger=logs[1])
    _same(logs[0]._head, logs[1]._head, "head")
    _same(logs[0]._ring, logs[1]._ring, "ring")
    _assert_same_state(env, twin)
    _same(c1._state, c2._state, "mrac state")


def test_rollout_a_million_drones():
    _check_rollout(_pair("ctrl", 1 << 20, 1, ctrl=120, seed=9), "cf2x", T=2, W=4, record=False)


@pytest.mark.parametrize("case", ["cf2x", "cf2p"])
def test_golden_loop_free_running(golden, case):
    """The fixture's closed loops: examples/mrac.py (CF2X from (0,0,0) to (0,0,1)) and the CF2P offset case (CtrlAviary DYN,
    240/120 Hz): one step(zeros), then computeControlFromEnv + step, free-running against the reference for the horizon that
    free_running_horizon derives (93 of mrac.py's ticks, all 1800 of the CF2P case)."""
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils.enums import Physics
    from mrac_testlib import LOOPS
    g = golden("mrac")
    model, init, target, _ = LOOPS[case]
    _, H = free_running_horizon(case)
    pre, every = ("loop_", 1) if case == "cf2x" else ("p_", 10)                # the fixture keeps every 10th CF2P call
    env = CtrlAviary(drone_model=drone_model(model), num_drones=1, initial_xyzs=np.array([init]), initial_rpys=np.zeros((1, 3)),
                     physics=Physics.DYN, pyb_freq=240, ctrl_freq=120, num_envs=1)
    env.reset()
    c = _mrac(model, 1)
    env.step(torch.zeros((1, 1, 4), dtype=torch.float64, device="cuda"))
    pos, quat, vel, _ = loop_inputs(g[pre + "state"])
    tgt = torch.tensor([target], dtype=torch.float64, device="cuda")
    states, rpms, ctrl = [], [], {}
    for k in range(H):
        if k % every == 0:
            states.append(torch.cat([env.pos.reshape(3), env.quat.reshape(4), env.vel.reshape(3)]).clone())
        rpm = c.computeControlFromEnv(env, tgt)
        if k % every == 0:
            rpms.append(rpm.reshape(4).clone())
        if k % 100 == 99:
            ctrl[k // 100] = (c.Kx[0], c.Kr[0], c.Xm[0])
        env.step(rpm)
    s, r = torch.stack(states).cpu().numpy(), torch.stack(rpms).cpu().numpy()
    worst = max(err(s, np.concatenate([pos, quat, vel], axis=1)[:len(s)]), err(r, g[pre + "rpm"][:len(r)]))
    for j, (Kx, Kr, Xm) in ctrl.items():
        worst = max(worst, err(Kx, g[pre + "Kx"][j]), err(Kr, g[pre + "Kr"][j]), err(Xm, g[pre + "Xm"][j]))
    print("%s free-running: %d ticks, worst %.1e" % (case, H, worst))
    assert worst <= TOL


def test_reset_keeps_gains_and_reinitialises_xm(golden):
    from oracle.mrac_oracle import OracleMRAC
    g = golden("mrac")
    G = gains_of(g, "cf2x")
    n = 64
    rng = np.random.default_rng(12)
    c, o = _mrac("cf2x", n), OracleMRAC(n, "cf2x", gains_=G)
    tgt = rng.uniform(-1, 1, (n, 3))

    def call():
        q = np.concatenate([rng.normal(0, 0.05, (n, 3)), np.ones((n, 1))], axis=1)
        q /= np.linalg.norm(q, axis=1, keepdims=True)
        x = (rng.uniform(-1, 1, (n, 3)), q, rng.uniform(-0.3, 0.3, (n, 3)), rng.uniform(-0.5, 0.5, (n, 3)))
        o.Kx, o.Kr, o.Xm = c.Kx.copy(), c.Kr.copy(), c.Xm.copy()
        ro, _, _ = o.compute(DT, *x, tgt)
        r, _, _ = c.computeControl(DT, *(_dev(v) for v in x), _dev(tgt))
        assert err(r.cpu().numpy(), ro) <= TF_TOL and err(c.Kx, o.Kx) <= TF_TOL and err(c.Xm, o.Xm) <= TF_TOL
        return x
    for _ in range(3):
        call()
    Kx, Kr = c.Kx.copy(), c.Kr.copy()
    c.reset()
    o.reset()
    assert c.control_counter == 0 and np.array_equal(c.Kx, Kx) and np.array_equal(c.Kr, Kr)
    x = call()
    from oracle.mrac_oracle import body_rates
    from oracle.dyn_oracle import quat_to_euler
    rpy = quat_to_euler(x[1])
    X = np.concatenate([x[0], rpy, x[2], body_rates(rpy, x[3])], axis=1)
    # Xm was set to X, then advanced by one model step from there: the error e of the call was zero, so Kx moved by 0
    assert np.array_equal(c.Kx, Kx) and np.array_equal(c.Kr, Kr)
    assert err(c.Xm, X + (X @ G["Am"].T + (G["Bm"] @ (-G["Kr_ref_gain"] @ np.concatenate([tgt, np.zeros((n, 9))], axis=1).T)).T) * DT) <= TF_TOL


def test_refusals():
    from gym_pybullet_drones_b200.control import MRAC
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils.enums import DroneModel, Physics
    with pytest.raises(ValueError, match="MRAC requires"):
        MRAC("cf2x")
    env = CtrlAviary(num_drones=2, physics=Physics.DYN, num_envs=4)
    wp = np.zeros((3, 3))
    with pytest.raises(ValueError, match="num_drones"):
        env.rollout(controller=MRAC(DroneModel.CF2X, num_drones=7), waypoints=wp)
    ok = MRAC(DroneModel.CF2X, num_drones=8)
    with pytest.raises(ValueError, match="either actions or a controller"):
        env.rollout(torch.zeros((2, 4, 2, 4), device="cuda"), controller=ok, waypoints=wp)
    with pytest.raises(ValueError, match="controller for 8 drones"):
        MRAC(DroneModel.CF2X, num_drones=8).computeControlFromEnv(CtrlAviary(num_drones=3, physics=Physics.DYN, num_envs=1), np.zeros((3, 3)))
    with pytest.raises(ValueError, match="expected shape"):
        ok.computeControl(DT, np.zeros((7, 3)), np.zeros((7, 4)), np.zeros((7, 3)), np.zeros((7, 3)), np.zeros((7, 3)))
    big = CtrlAviary(num_drones=129, physics=Physics.PYB_DW, num_envs=1)
    with pytest.raises(ValueError, match="drones_per_env <= 128"):
        big.rollout(controller=MRAC(DroneModel.CF2X, num_drones=129), waypoints=wp)
    with pytest.raises(ValueError, match="vector API"):
        CtrlAviary(num_drones=2, physics=Physics.DYN).rollout(controller=MRAC(DroneModel.CF2X, num_drones=2), waypoints=wp)
    assert ok.control_counter == 0
