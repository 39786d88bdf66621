"""Pins the tier-2 oracle (oracle/dyn_oracle.py) against golden vectors produced by the
UNMODIFIED reference (tests/golden/make_golden.py).  CPU only."""
import numpy as np
import pytest

from oracle import dyn_oracle as O

TOL = 1e-10


def relerr(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1.0))) if a.size else 0.0


FIELDS = ("pos", "quat", "rpy", "vel", "ang_v", "rpy_rates")


def replay(env, g, key, obs_every, tol=TOL, steps=None):
    acts = g[key + "_actions"][:steps]
    o0 = env.reset()
    assert relerr(o0[0], g[key + "_obs0"]) < 1e-6
    for t in range(acts.shape[0]):
        obs, r, te, tr = env.step(acts[t][None])
        for f in FIELDS:
            assert relerr(getattr(env, f)[0], g[key + "_" + f][t]) < tol, (key, f, t)
        assert abs(r[0] - g[key + "_reward"][t]) < 1e-9
        assert bool(te[0]) == bool(g[key + "_terminated"][t]) and bool(tr[0]) == bool(g[key + "_truncated"][t]), (key, t)
        if t % obs_every == 0:
            assert relerr(obs[0], g[key + "_obs"][t // obs_every]) < 1e-6, (key, t)


def test_constants(golden):
    g = golden("constants")
    for model in ("cf2x", "cf2p", "racer"):
        P = O.OracleParams(model)
        ref = dict(zip(g[model + "_names"], g[model + "_values"]))
        for name, mine in (("M", P.M), ("L", P.L), ("KF", P.KF), ("KM", P.KM), ("GRAVITY", P.GRAVITY), ("HOVER_RPM", P.HOVER_RPM),
                           ("MAX_RPM", P.MAX_RPM), ("MAX_THRUST", P.MAX_THRUST), ("MAX_XY_TORQUE", P.MAX_XY_TORQUE),
                           ("MAX_Z_TORQUE", P.MAX_Z_TORQUE), ("GND_EFF_H_CLIP", P.GND_EFF_H_CLIP), ("GND_EFF_COEFF", P.GND_EFF_COEFF),
                           ("PROP_RADIUS", P.PROP_RADIUS), ("DW_COEFF_1", P.DW[0]), ("DW_COEFF_2", P.DW[1]), ("DW_COEFF_3", P.DW[2]),
                           ("MAX_SPEED_KMH", P.MAX_SPEED_KMH), ("COLLISION_H", P.COLLISION_H)):
            assert mine == ref[name], (model, name)
        assert np.array_equal(P.J, g[model + "_J"]) and np.array_equal(P.DRAG_COEFF, g[model + "_DRAG_COEFF"])
        assert np.array_equal(P.default_init_xyzs(3), g[model + "_INIT_XYZS3"])


@pytest.mark.parametrize("cf", [240, 30])
@pytest.mark.parametrize("stream", ["zeros", "const", "rand", "sine"])
def test_hover_rpm_1000(golden, cf, stream):
    g = golden("hover_rpm_1000")
    replay(O.OracleAviary("hover", 1, 1, ctrl_freq=cf, act="rpm"), g, "cf%d_%s" % (cf, stream), 50)


def test_learn_config_episode(golden):
    """learn.py config: time-out truncation fires on env step 242, return 333.8626 (SURVEY 8c KAT-episode)."""
    g = golden("hover_one_d_rpm_episode")
    env = O.OracleAviary("hover", 1, 1, act="one_d_rpm")
    env.reset()
    ret, n = 0.0, 0
    for t in range(250):
        obs, r, te, tr = env.step(np.zeros((1, 1, 1), np.float32))
        assert abs(r[0] - g["reward"][t]) < 1e-12 and bool(tr[0]) == bool(g["truncated"][t])
        if n == 0:
            ret += r[0]
            if te[0] or tr[0]:
                n = t + 1
    assert n == 242 and abs(ret - 333.862626904298) < 1e-9


@pytest.mark.parametrize("key,nd,act", [("d2_one_d_rpm", 2, "one_d_rpm"), ("d2_rpm", 2, "rpm"), ("d3_rpm", 3, "rpm")])
def test_multihover(golden, key, nd, act):
    g = golden("multihover_rand_300")
    env = O.OracleAviary("multihover", 1, nd, act=act)
    assert relerr(env.TARGET_POS[0], g[key + "_TARGET_POS"]) == 0
    replay(env, g, key, 10)


PID_CASES = [("hover_d1_pid", "hover", 1, "pid"), ("hover_d1_vel", "hover", 1, "vel"),
             ("hover_d1_one_d_pid", "hover", 1, "one_d_pid"), ("multi_d2_pid", "multihover", 2, "pid")]


@pytest.mark.parametrize("key,kind,nd,act", PID_CASES)
def test_rl_env_with_embedded_pid_trajectory(golden, key, kind, nd, act):
    """240/120 Hz: the closed loop is contractive, whole trajectories are comparable."""
    replay(O.OracleAviary(kind, 1, nd, act=act, ctrl_freq=120), golden("rl_pid_cf120"), key, 10, tol=1e-9)


def force_state(env, g, key, t):
    """Teacher forcing: load the reference's state after step t (t=-1: reset state)."""
    if t < 0:
        env.reset()
        if hasattr(env, "ctrl"):
            env.ctrl.reset()
        return
    for f in FIELDS:
        getattr(env, f)[0] = g[key + "_" + f][t]
    env.step_counter[:] = (t + 1) * env.P.S
    if hasattr(env, "ctrl"):
        env.ctrl.integral_pos_e = g[key + "_pid_integral_pos_e"][t].copy()
        env.ctrl.integral_rpy_e = g[key + "_pid_integral_rpy_e"][t].copy()
        env.ctrl.last_rpy = g[key + "_pid_last_rpy"][t].copy()


@pytest.mark.parametrize("key,kind,nd,act", PID_CASES)
def test_rl_env_with_embedded_pid_teacher_forced(golden, key, kind, nd, act):
    """240/30 Hz (the RL default): the reference's PID chatters chaotically (1e-12 -> 1e-2 in 3 s), so every
    step is checked from the reference's own previous state instead of as a free-running trajectory."""
    g = golden("rl_pid_cf30")
    env = O.OracleAviary(kind, 1, nd, act=act)
    acts = g[key + "_actions"]
    env.reset()
    for t in range(acts.shape[0]):
        force_state(env, g, key, t - 1)
        obs, r, te, tr = env.step(acts[t][None])
        for f in FIELDS:
            assert relerr(getattr(env, f)[0], g[key + "_" + f][t]) < 1e-11, (key, f, t)
        assert relerr(env.ctrl.integral_rpy_e, g[key + "_pid_integral_rpy_e"][t]) < 1e-11
        assert abs(r[0] - g[key + "_reward"][t]) < 1e-10
        assert bool(tr[0]) == bool(g[key + "_truncated"][t])


def rl_config_cases(g):
    import json
    return {c["key"]: c for c in json.loads(str(g["cases"]))}


def rl_config_oracle(c, num_envs=1):
    return O.OracleAviary(c["kind"], num_envs, c.get("nd", 1), drone_model=c["model"], pyb_freq=c["pyb"], ctrl_freq=c["ctrl"],
                          act=c["act"], initial_rpys=c.get("rpys"))


RL_CONFIG_FREE = ["race_500_50_rpm", "cf2p_240_16_one_d_rpm", "multi3_race_240_80_rpm_rpys", "cf2x_1000_50_one_d_rpm_timeout",
                  "cf2x_240_1_one_d_rpm_b0", "cf2x_240_30_rpm_x30"]


@pytest.mark.parametrize("key", RL_CONFIG_FREE)
def test_rl_configs(golden, key):
    """Other drone models, rates, initial attitudes, B = 0 and out-of-range actions: whole trajectories at TOL."""
    g = golden("rl_configs")
    c = rl_config_cases(g)[key]
    env = rl_config_oracle(c)
    if c["kind"] == "multihover":
        assert relerr(env.TARGET_POS[0], g[key + "_TARGET_POS"]) == 0
    assert env.B == c["ctrl"] // 2 and env.P.S == c["pyb"] // c["ctrl"]
    replay(env, g, key, c["obs_every"])
    assert g[key + "_obs"].shape[-1] == 12 + env.B * env.A


def test_rl_configs_time_out_ticks(golden):
    """The time-out tick follows pyb_freq: step_counter / PYB_FREQ > EPISODE_LEN_SEC first holds on tick 402 at 1000/50
    (step counter 8020 before the tick's increment) and on tick 10 at 240/1."""
    g = golden("rl_configs")
    for key, first in (("cf2x_1000_50_one_d_rpm_timeout", 402), ("cf2x_240_1_one_d_rpm_b0", 10)):
        tr = g[key + "_truncated"]
        assert int(np.argmax(tr)) + 1 == first and tr[first - 1:].all(), key


def test_rl_configs_pid_60hz_teacher_forced(golden):
    """CF2P 240/60 with the embedded PID: every tick from the reference's previous state and controller integrals."""
    key = "cf2p_240_60_pid"
    g = golden("rl_configs")
    c = rl_config_cases(g)[key]
    env = rl_config_oracle(c)
    acts = g[key + "_actions"]
    env.reset()
    for t in range(acts.shape[0]):
        force_state(env, g, key, t - 1)
        obs, r, te, tr = env.step(acts[t][None])
        for f in FIELDS:
            assert relerr(getattr(env, f)[0], g[key + "_" + f][t]) < 1e-11, (key, f, t)
        assert relerr(env.ctrl.integral_rpy_e, g[key + "_pid_integral_rpy_e"][t]) < 1e-11
        assert relerr(env.ctrl.integral_pos_e, g[key + "_pid_integral_pos_e"][t]) < 1e-11
        assert abs(r[0] - g[key + "_reward"][t]) < 1e-10
        assert bool(tr[0]) == bool(g[key + "_truncated"][t])
        if t % c["obs_every"] == 0:
            assert relerr(obs[0], g[key + "_obs"][t // c["obs_every"]]) < 1e-6, t


def test_oracle_without_action_buffer():
    """ctrl_freq = 1: B = 0, the observation is the 12-column kinematic head and stepping keeps no buffer."""
    env = O.OracleAviary("hover", 2, 1, ctrl_freq=1, act="one_d_rpm")
    assert env.B == 0 and env.reset().shape == (2, 1, 12)
    for _ in range(3):
        obs, r, te, tr = env.step(np.zeros((2, 1, 1), np.float32))
        assert obs.shape == (2, 1, 12) and env.action_buffer == []


@pytest.mark.parametrize("model", ["cf2x", "cf2p"])
def test_pid_circle(golden, model):
    """examples/pid.py workload: CtrlAviary(DYN, 240/48) x 3 drones tracked by DSLPIDControl.  Free-running for the
    first 30 ticks, then teacher-forced tick by tick (at 48 Hz the loop amplifies 1e-16 noise to 1e-8 in ~40 ticks)."""
    g = golden("pid_circle_" + model)
    env = O.OracleAviary("ctrl", 1, 3, drone_model=model, ctrl_freq=48, initial_xyzs=g["INIT_XYZS"], initial_rpys=g["INIT_RPYS"])
    ctrl = O.OraclePID(3, model)
    env.reset()
    action = np.zeros((1, 3, 4))
    for t in range(g["obs"].shape[0]):
        if t > 30:      # teacher forcing: state after tick t-1 from the reference
            st = g["obs"][t - 1]
            env.pos[0], env.quat[0], env.rpy[0], env.vel[0] = st[:, 0:3], st[:, 3:7], st[:, 7:10], st[:, 10:13]
            env.last_clipped_action[0] = st[:, 16:20]
            env.rpy_rates[0] = g["rpy_rates"][t - 1]
            ctrl.integral_pos_e, ctrl.integral_rpy_e = g["pid_integral_pos_e"][t - 1].copy(), g["pid_integral_rpy_e"][t - 1].copy()
            ctrl.last_rpy = g["pid_last_rpy"][t - 1].copy()
            action = g["action"][t - 1][None]
        obs, _, _, _ = env.step(action)
        assert relerr(obs[0], g["obs"][t]) < 1e-9, t
        st = obs[0]
        rpm, pe, ye = ctrl.compute(env.P.CTRL_TIMESTEP, st[:, 0:3], st[:, 3:7], st[:, 10:13], g["target"][t], target_rpy=g["INIT_RPYS"])
        assert relerr(rpm, g["action"][t]) < 1e-9 and relerr(pe, g["pos_e"][t]) < 1e-10 and relerr(ye, g["yaw_e"][t]) < 1e-9
        assert relerr(ctrl.integral_rpy_e, g["pid_integral_rpy_e"][t]) < 1e-10
        action = rpm[None]


@pytest.mark.parametrize("model", ["cf2x", "cf2p"])
def test_pid_known_answers(golden, model):
    g = golden("pid_kat")
    k = model + "_"
    n = g[k + "pos"].shape[0]
    ctrl = O.OraclePID(n, model)
    for call in range(3):
        rpm, pe, ye = ctrl.compute(1 / 48, g[k + "pos"] + 0.01 * call, g[k + "quat"], g[k + "vel"], g[k + "target_pos"],
                                   g[k + "target_rpy"], g[k + "target_vel"], g[k + "target_rpy_rates"])
        assert relerr(rpm, g[k + "rpm"][call]) < 1e-9
        assert relerr(pe, g[k + "pos_e"][call]) < 1e-12 and relerr(ye, g[k + "yaw_e"][call]) < 1e-10
        assert relerr(ctrl.integral_pos_e, g[k + "integral_pos_e"][call]) < 1e-12
        assert relerr(ctrl.integral_rpy_e, g[k + "integral_rpy_e"][call]) < 1e-10
        assert relerr(ctrl.last_rpy, g[k + "last_rpy"][call]) < 1e-12


@pytest.mark.parametrize("model", ["cf2p", "racer"])
def test_ctrl_other_models(golden, model):
    g = golden("ctrl_models_300")
    env = O.OracleAviary("ctrl", 1, 2, drone_model=model, ctrl_freq=120)
    acts = g[model + "_actions"]
    env.reset()
    for t in range(acts.shape[0]):
        obs, r, te, tr = env.step(acts[t][None])
        assert relerr(obs[0], g[model + "_obs"][t]) < 1e-9, t
        assert relerr(env.rpy_rates[0], g[model + "_rpy_rates"][t]) < 1e-9


def test_velocity_aviary(golden):
    g = golden("velocity_aviary_480")
    env = O.OracleAviary("velocity", 1, 2)
    acts = g["actions"]
    o0 = env.reset()
    assert relerr(o0[0], g["obs0"]) < 1e-12
    for t in range(acts.shape[0]):
        obs, r, te, tr = env.step(acts[t][None])
        assert relerr(obs[0], g["obs"][t]) < 1e-9, t
        assert r[0] == -1 and not te[0] and not tr[0]


@pytest.mark.parametrize("model", ["cf2x", "cf2p"])
def test_effect_formulas(golden, model):
    """_groundEffect/_drag/_downwash exist only on the reference's PYB_* branches: pinned at force level."""
    g = golden("effects_formula")
    k = model + "_"
    P = O.OracleParams(model)
    pos, quat, rpy, vel, rpm = (g[k + n] for n in ("pos", "quat", "rpy", "vel", "rpm"))
    R = O.quat_to_matrix(quat)
    assert relerr(O.ground_effect_thrust(P, rpm, pos, R, rpy), g[k + "gnd_thrust"]) < 1e-12
    assert np.count_nonzero(g[k + "gnd_thrust"].sum(1) == 0) >= 1      # the tilted-over drones get none
    fw = O.drag_force_world(P, rpm, vel)
    body = np.einsum("nji,nj->ni", R, fw)                               # reference applies R^T (f) in LINK_FRAME
    assert relerr(body * 1e3, g[k + "drag_body"] * 1e3) < 1e-10
    dw = O.downwash_body_z(P, pos[None])[0]
    assert relerr(dw, g[k + "downwash_body_z"]) < 1e-10
    assert np.count_nonzero(g[k + "downwash_body_z"]) > 10


def test_adjacency_matrix(golden):
    g = golden("adjacency")
    for k in range(3):
        adj = O.adjacency_matrix(g["case%d_pos" % k][None], float(g["case%d_radius" % k]))[0]
        assert np.array_equal(adj, g["case%d_adjacency" % k])


def test_quaternion_helpers_against_scipy():
    """Bullet's helpers are restated from its published algorithm (library absent): cross-check with scipy."""
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(3)
    q = rng.normal(size=(500, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    assert relerr(O.quat_to_matrix(q), Rotation.from_quat(q).as_matrix()) < 1e-13
    assert relerr(O.quat_to_matrix(3.0 * q), Rotation.from_quat(q).as_matrix()) < 1e-13      # implicit normalisation
    e = O.quat_to_euler(q)
    ok = np.abs(e[:, 1]) < 1.5
    assert relerr(e[ok], Rotation.from_quat(q[ok]).as_euler("xyz")) < 1e-9
    rpy = rng.uniform(-1.5, 1.5, (500, 3))
    q2 = O.euler_to_quat(rpy)
    q3 = Rotation.from_euler("xyz", rpy).as_quat()
    sgn = np.sign(np.sum(q2 * q3, axis=1, keepdims=True))
    assert relerr(q2, sgn * q3) < 1e-13
    assert relerr(O.quat_to_euler(q2), rpy) < 1e-12
    # gimbal guard
    qg = O.euler_to_quat(np.array([[0.3, np.pi / 2, -0.2], [0.1, -np.pi / 2, 0.4]]))
    eg = O.quat_to_euler(qg)
    assert np.all(eg[:, 0] == 0) and np.allclose(np.abs(eg[:, 1]), np.pi / 2)


def test_integrate_q_properties():
    rng = np.random.default_rng(4)
    q = rng.normal(size=(200, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    w = rng.normal(size=(200, 3)) * 5
    q1 = O.integrate_q(q, w, 1 / 240)
    assert np.max(np.abs(np.linalg.norm(q1, axis=1) - 1)) < 1e-14
    assert np.array_equal(O.integrate_q(q, np.zeros((200, 3)), 1 / 240), q)
    assert np.array_equal(O.integrate_q(q, np.full((200, 3), 5e-9), 1 / 240), q)             # np.isclose(|w|,0) branch
    from scipy.spatial.transform import Rotation
    ref = (Rotation.from_quat(q) * Rotation.from_rotvec(w / 240)).as_quat()
    sgn = np.sign(np.sum(q1 * ref, axis=1, keepdims=True))
    assert relerr(q1, sgn * ref) < 1e-12                                                    # body-rate exponential map
