"""Parity tests proper (-m gpu): the CUDA path, called through the C ABI via the product env/controller classes,
against (a) golden vectors of the unmodified reference, (b) the float64 NumPy oracle on seeded inputs at sizes it
finishes in seconds, (c) size-independent properties at BASELINE.json's full sizes.

Tolerance (north star): |a - b| <= 1e-5 * max(|b|, 1) element-wise on the kinematic state over 1000 physics steps
(RTOL).  Quaternions are compared up to sign.  The state planes are float64 since round 2, so pos/quat/vel/rpy_rates
are held to TIGHT (1e-9) wherever the reference trajectory itself is not chaotic; rpy and ang_v are read back from the
float32 observation (the reference casts its observations to float32 too) and get OBS_TOL = 2e-6."""
import numpy as np
import pytest
import torch

from qs_testlib import FIELDS, RTOL, TIGHT, quat_err, relerr

OBS_TOL = 2e-6          # float32 cast of the observation (6e-8 rel) + atan2f/asinf on float32-rounded arguments (measured worst
                        # case over 4096 tumbling drones x 1000 steps: 9e-7); five times inside the north-star bound
OBS_FIELDS = ("rpy", "ang_v")

pytestmark = pytest.mark.gpu


def _imports():
    from gym_pybullet_drones_b200.control import DSLPIDControl
    from gym_pybullet_drones_b200.envs import CtrlAviary, HoverAviary, MultiHoverAviary
    from gym_pybullet_drones_b200.utils.enums import ActionType, DroneModel, Physics
    from oracle import dyn_oracle as O
    return DSLPIDControl, CtrlAviary, HoverAviary, MultiHoverAviary, ActionType, DroneModel, Physics, O


def state_of(env):
    """float64 host copies of the kinematic state [E,D,.] + the derived rpy/ang_v of the last observation."""
    obs = env._obs_buf[env._cur].view(env._E, env._D, env._obs_dim).double().cpu().numpy()
    assert env._planes.dtype == torch.float64
    out = dict(pos=env.pos.cpu().numpy(), quat=env.quat.cpu().numpy(), vel=env.vel.cpu().numpy(), rpy_rates=env.rpy_rates.cpu().numpy())
    if env._state20_obs():          # (not the width: a KIN row is 20 floats wide at ONE_D_RPM / ctrl_freq 16)
        out["rpy"], out["ang_v"] = obs[..., 7:10], obs[..., 13:16]
    else:
        out["rpy"], out["ang_v"] = obs[..., 3:6], obs[..., 9:12]
    return out


def check_fields(st, g, key, t, tol=TIGHT, env_idx=0):
    for f in FIELDS:
        ref = g[key + "_" + f][t]
        mine = st[f][env_idx]
        e = quat_err(mine, ref) if f == "quat" else relerr(mine, ref)
        assert e <= (max(tol, OBS_TOL) if f in OBS_FIELDS else tol), (key, f, t, e)


# ---------------------------------------------------------------------------------------------------------------
# (a) golden vectors of the reference
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cf,steps", [(240, 1000), (30, 125)])
@pytest.mark.parametrize("stream", ["zeros", "rand", "sine", "const"])
def test_config1_hover_1000_physics_steps(golden, cf, steps, stream):
    """BASELINE config 1 on the GPU: every element of pos/quat/rpy/vel/ang_v/rpy_rates within 1e-5 rel for 1000 physics
    steps; E=3 identical aviaries also checks that lanes do not interact."""
    _, _, HoverAviary, _, ActionType, _, Physics, _ = _imports()
    g = golden("hover_rpm_1000")
    key = "cf%d_%s" % (cf, stream)
    env = HoverAviary(physics=Physics.DYN, pyb_freq=240, ctrl_freq=cf, act=ActionType.RPM, num_envs=3)
    obs, _ = env.reset()
    assert relerr(obs[0].cpu().numpy(), g[key + "_obs0"]) < 1e-6
    acts = g[key + "_actions"]
    tol = TIGHT
    for t in range(min(steps, acts.shape[0])):
        a = torch.from_numpy(np.broadcast_to(acts[t], (3, 1, 4)).copy()).cuda()
        obs, rew, term, trunc, _ = env.step(a)
        st = state_of(env)
        check_fields(st, g, key, t, tol, 0)
        check_fields(st, g, key, t, tol, 2)
        assert abs(float(rew[0]) - g[key + "_reward"][t]) < 1e-5
        assert bool(term[0]) == bool(g[key + "_terminated"][t]) and bool(trunc[0]) == bool(g[key + "_truncated"][t]), t
        if t % 50 == 0:
            assert relerr(obs[0].cpu().numpy(), g[key + "_obs"][t // 50]) < OBS_TOL


def test_learn_config_episode_single_env_api(golden):
    """learn.py's config through the reference's single-env API: time-out on env step 242, return 333.8626."""
    _, _, HoverAviary, _, ActionType, _, Physics, _ = _imports()
    g = golden("hover_one_d_rpm_episode")
    env = HoverAviary(physics=Physics.DYN, act=ActionType.ONE_D_RPM)
    obs, info = env.reset(seed=42, options={})
    assert isinstance(obs, np.ndarray) and obs.shape == (1, 27) and obs.dtype == np.float32 and info == {"answer": 42}
    assert env.action_space.shape == (1, 1) and env.observation_space.shape == (1, 27)
    ret, n = 0.0, 0
    for t in range(250):
        obs, r, te, tr, info = env.step(np.zeros((1, 1), np.float32))
        assert isinstance(r, float) and isinstance(te, bool) and isinstance(tr, bool)
        assert abs(r - g["reward"][t]) < 1e-5 and tr == bool(g["truncated"][t])
        if n == 0:
            ret += r
            if te or tr:
                n = t + 1
    assert n == 242 and abs(ret - 333.862626904298) < 1e-2
    assert env.step_counter == 250 * 8 and env.CTRL_FREQ == 30 and env.EPISODE_LEN_SEC == 8


@pytest.mark.parametrize("key,nd,act", [("d2_one_d_rpm", 2, "ONE_D_RPM"), ("d2_rpm", 2, "RPM"), ("d3_rpm", 3, "RPM")])
def test_multihover_golden(golden, key, nd, act):
    _, _, _, MultiHoverAviary, ActionType, _, Physics, _ = _imports()
    g = golden("multihover_rand_300")
    env = MultiHoverAviary(num_drones=nd, physics=Physics.DYN, act=ActionType[act], num_envs=2)
    assert relerr(env.TARGET_POS, g[key + "_TARGET_POS"]) == 0
    obs, _ = env.reset()
    acts = g[key + "_actions"]
    for t in range(125):      # 1000 physics steps
        a = torch.from_numpy(np.broadcast_to(acts[t], (2,) + acts[t].shape).copy()).cuda()
        obs, rew, term, trunc, _ = env.step(a)
        check_fields(state_of(env), g, key, t, TIGHT, 1)
        assert abs(float(rew[1]) - g[key + "_reward"][t]) < 5e-7 * max(1.0, abs(g[key + "_reward"][t]))
        assert bool(term[1]) == bool(g[key + "_terminated"][t]) and bool(trunc[1]) == bool(g[key + "_truncated"][t]), t
        if t % 10 == 0:
            assert relerr(obs[1].cpu().numpy(), g[key + "_obs"][t // 10]) < OBS_TOL


@pytest.mark.parametrize("model", ["CF2P", "RACE"])
def test_ctrl_aviary_other_models(golden, model):
    _, CtrlAviary, _, _, _, DroneModel, Physics, _ = _imports()
    g = golden("ctrl_models_300")
    dm = DroneModel[model]
    key = dm.value
    env = CtrlAviary(drone_model=dm, num_drones=2, physics=Physics.DYN, pyb_freq=240, ctrl_freq=120)
    obs, _ = env.reset()
    assert obs.shape == (2, 20) and relerr(obs, g[key + "_obs0"]) < 1e-6
    acts = g[key + "_actions"]
    for t in range(acts.shape[0]):
        obs, r, te, tr, _ = env.step(acts[t])
        ref = g[key + "_obs"][t]
        assert r == -1 and te is False and tr is False
        # the raw RPM enter the ABI as float32 (the golden used float64 rpm): 6e-8 relative on the thrust, integrated twice
        assert relerr(obs[:, 0:3], ref[:, 0:3]) < RTOL and quat_err(obs[:, 3:7], ref[:, 3:7]) < RTOL, t
        assert relerr(obs[:, 7:16], ref[:, 7:16]) < RTOL and relerr(obs[:, 16:20], ref[:, 16:20]) < 1e-7, t


@pytest.mark.parametrize("model", ["CF2X", "CF2P"])
def test_pid_known_answers(golden, model):
    """DSLPIDControl.computeControl on 256 random states x 3 stateful calls (float32 inputs: 1e-5 on rpm)."""
    DSLPIDControl, _, _, _, _, DroneModel, _, _ = _imports()
    g = golden("pid_kat")
    dm = DroneModel[model]
    k = dm.value + "_"
    n = g[k + "pos"].shape[0]
    ctrl = DSLPIDControl(dm, num_drones=n)
    for call in range(3):
        rpm, pe, ye = ctrl.computeControl(1 / 48, g[k + "pos"] + 0.01 * call, g[k + "quat"], g[k + "vel"], None, g[k + "target_pos"],
                                          g[k + "target_rpy"], g[k + "target_vel"], g[k + "target_rpy_rates"])
        assert relerr(rpm, g[k + "rpm"][call]) < 2e-5, call
        assert relerr(pe, g[k + "pos_e"][call]) < 1e-6 and relerr(ye, g[k + "yaw_e"][call]) < 1e-5
        assert relerr(ctrl.integral_pos_e, g[k + "integral_pos_e"][call]) < 1e-6
        assert relerr(ctrl.last_rpy, g[k + "last_rpy"][call]) < 1e-6
        assert relerr(ctrl.integral_rpy_e, g[k + "integral_rpy_e"][call]) < 1e-5
    one = DSLPIDControl(dm)
    r1, p1, y1 = one.computeControl(1 / 48, g[k + "pos"][0], g[k + "quat"][0], g[k + "vel"][0], np.zeros(3), g[k + "target_pos"][0])
    assert r1.shape == (4,) and p1.shape == (3,) and isinstance(y1, float)


PID_CASES = [("hover_d1_pid", 1, "PID"), ("hover_d1_vel", 1, "VEL"), ("hover_d1_one_d_pid", 1, "ONE_D_PID"), ("multi_d2_pid", 2, "PID")]


def _pid_env(nd, act, cf):
    _, _, HoverAviary, MultiHoverAviary, ActionType, _, Physics, _ = _imports()
    kw = dict(physics=Physics.DYN, act=ActionType[act], pyb_freq=240, ctrl_freq=cf, num_envs=1)
    return HoverAviary(**kw) if nd == 1 else MultiHoverAviary(num_drones=nd, **kw)


@pytest.mark.parametrize("key,nd,act", PID_CASES)
def test_rl_pid_teacher_forced_30hz(golden, key, nd, act):
    g = golden("rl_pid_cf30")
    env = _pid_env(nd, act, 30)
    env.reset()
    acts = g[key + "_actions"]
    for t in range(acts.shape[0]):
        if t > 0:
            env.set_state(pos=g[key + "_pos"][t - 1], quat=g[key + "_quat"][t - 1], vel=g[key + "_vel"][t - 1],
                          rpy_rates=g[key + "_rpy_rates"][t - 1], step_counter=t * 8)
            env._pid[0:3] = torch.from_numpy(g[key + "_pid_integral_pos_e"][t - 1].T.copy()).cuda()
            env._pid[3:6] = torch.from_numpy(g[key + "_pid_last_rpy"][t - 1].T.copy()).cuda()
            env._pid[6:9] = torch.from_numpy(g[key + "_pid_integral_rpy_e"][t - 1].T.copy()).cuda()
        obs, rew, term, trunc, _ = env.step(torch.from_numpy(acts[t][None]).cuda())
        check_fields(state_of(env), g, key, t, 1e-7)
        assert abs(float(rew[0]) - g[key + "_reward"][t]) < 1e-6 and bool(trunc[0]) == bool(g[key + "_truncated"][t])


@pytest.mark.parametrize("key,nd,act", PID_CASES)
def test_rl_pid_trajectory_120hz(golden, key, nd, act):
    g = golden("rl_pid_cf120")
    env = _pid_env(nd, act, 120)
    env.reset()
    acts = g[key + "_actions"]
    for t in range(acts.shape[0]):
        obs, rew, term, trunc, _ = env.step(torch.from_numpy(acts[t][None]).cuda())
        check_fields(state_of(env), g, key, t, RTOL)
        if t % 10 == 0:
            assert relerr(obs[0].cpu().numpy(), g[key + "_obs"][t // 10]) < RTOL


def test_pid_circle_workload(golden):
    """examples/pid.py: CtrlAviary(DYN, 240/48) x 3 + DSLPIDControl; free-running for 8 ticks, then teacher-forced (the
    48 Hz loop amplifies any perturbation ~1.5x per tick in the reference itself).  The controller reads the env's float64
    state on the device (computeControlFromEnv) and the env takes its float64 RPMs: no float32 rounding in the loop."""
    DSLPIDControl, CtrlAviary, _, _, _, DroneModel, Physics, _ = _imports()
    g = golden("pid_circle_cf2x")
    env = CtrlAviary(num_drones=3, initial_xyzs=g["INIT_XYZS"], initial_rpys=g["INIT_RPYS"], physics=Physics.DYN, pyb_freq=240, ctrl_freq=48)
    ctrl = DSLPIDControl(DroneModel.CF2X, num_drones=3)
    env.reset()
    action = np.zeros((3, 4))
    for t in range(g["obs"].shape[0]):
        if t > 8:
            st = g["obs"][t - 1]
            env.set_state(pos=st[:, 0:3], quat=st[:, 3:7], vel=st[:, 10:13], rpy_rates=g["rpy_rates"][t - 1])
            ctrl.set_state(g["pid_integral_pos_e"][t - 1], g["pid_last_rpy"][t - 1], g["pid_integral_rpy_e"][t - 1])
            action = g["action"][t - 1]
        obs, _, _, _, _ = env.step(action)
        ref = g["obs"][t]
        tol = RTOL              # (the observation is float32; the float64 state is checked through the next tick's RPMs)
        assert relerr(obs[:, 0:3], ref[:, 0:3]) < tol and quat_err(obs[:, 3:7], ref[:, 3:7]) < tol and relerr(obs[:, 7:16], ref[:, 7:16]) < tol, t
        rpm = ctrl.computeControlFromEnv(env, g["target"][t], target_rpy=g["INIT_RPYS"])
        if t > 8:
            assert relerr(rpm.cpu().numpy(), g["action"][t]) < 1e-7, t
        elif t > 0:
            assert relerr(rpm.cpu().numpy(), g["action"][t]) < 1e-6, t          # free-running: 1e-12 x 1.5^t x the D-gain
        action = rpm


def test_velocity_aviary_golden(golden):
    """VelocityAviary (SURVEY 8f rank 2): act VEL through the embedded PID, 20-float state vectors out, 240/240 Hz."""
    from gym_pybullet_drones_b200.envs import VelocityAviary
    from gym_pybullet_drones_b200.utils.enums import Physics
    g = golden("velocity_aviary_480")
    env = VelocityAviary(num_drones=2, physics=Physics.DYN, pyb_freq=240, ctrl_freq=240)
    assert env.action_space.shape == (2, 4) and env.observation_space.shape == (2, 20) and abs(env.SPEED_LIMIT - 0.25) < 1e-12
    obs, _ = env.reset()
    assert relerr(obs, g["obs0"]) < 1e-6
    acts = g["actions"]
    for t in range(acts.shape[0]):
        obs, r, te, tr, _ = env.step(acts[t])
        ref = g["obs"][t]
        assert r == -1 and te is False and tr is False
        assert relerr(obs[:, 0:3], ref[:, 0:3]) < RTOL and quat_err(obs[:, 3:7], ref[:, 3:7]) < RTOL, t
        assert relerr(obs[:, 7:16], ref[:, 7:16]) < RTOL and relerr(obs[:, 16:20], ref[:, 16:20]) < RTOL, t


# ---------------------------------------------------------------------------------------------------------------
# (b) seeded inputs against the float64 oracle
# ---------------------------------------------------------------------------------------------------------------
BORDERLINE = {"ticks": 0, "old": 0, "new": 0}     # aviary-ticks seen, and excluded by the former fixed 1e-4 window and by this one


def _borderline(ora, tol):
    """[E] bool: some truncation test of the oracle state sits so close to its threshold that the kernel's state may lie on the
    other side.  The caller holds that state to `tol`: positions relative to max(|x|, 1) (<= 2 at the bounds), the unit quaternion
    absolutely, so |d(roll)|, |d(pitch)| <= 6 tol / cos(pitch) (test_gpu_configs._rpy_bound).  The window is 10x those.  The
    kernel decides on float64 angles (quad_core.cuh, qs::tilted), so nothing wider is needed; test_gpu_thresholds.py pins the
    decisions themselves to the ulp.  Callers that assert the state only at the end of a rollout (and the observations, at
    OBS_TOL, on the way) rely on the state error not shrinking over the rollout, which holds for these runs: the state
    differs from the oracle's by rounding that accumulates.  Each caller starts with _reset_borderline()."""
    cosp = np.maximum(np.abs(np.cos(ora.rpy[..., 1])), 0.02)
    wp, wa = 10.0 * tol * 2.0, 10.0 * 6.0 * tol / cosp
    dp = np.minimum.reduce([np.abs(np.abs(ora.pos[..., 0]) - ora.xy_bound), np.abs(np.abs(ora.pos[..., 1]) - ora.xy_bound),
                            np.abs(ora.pos[..., 2] - 2.0)])
    da = np.minimum(np.abs(np.abs(ora.rpy[..., 0]) - 0.4), np.abs(np.abs(ora.rpy[..., 1]) - 0.4))
    near = np.any((dp < wp) | (da < wa), axis=1)
    BORDERLINE["ticks"] += near.size
    BORDERLINE["old"] += int(np.any(np.minimum(dp, da) < 1e-4, axis=1).sum())
    BORDERLINE["new"] += int(near.sum())
    return near


def _reset_borderline():
    BORDERLINE.update(ticks=0, old=0, new=0)


def _report_borderline(name):
    """Prints and clears the counts of _borderline since the last report."""
    print("[borderline] %s: %d aviary-ticks, truncation unchecked on %d (fixed 1e-4 window: %d)"
          % (name, BORDERLINE["ticks"], BORDERLINE["new"], BORDERLINE["old"]))
    BORDERLINE.update(ticks=0, old=0, new=0)


def _compare_with_oracle(env, ora, acts, tol, check_obs_every=5):
    _reset_borderline()
    obs, _ = env.reset()
    o_obs = ora.reset()
    assert relerr(obs.cpu().numpy(), o_obs) < 1e-6
    for t in range(acts.shape[0]):
        obs, rew, term, trunc, _ = env.step(torch.from_numpy(acts[t]).cuda())
        o_obs, o_rew, o_term, o_trunc = ora.step(acts[t])
        st = state_of(env)
        # roll/yaw are ill-conditioned near pitch = +-90 deg (d(roll) ~ d(q)/cos(pitch)); tumbling drones get there,
        # so the Euler-angle (and only the Euler-angle) tolerance is scaled by 1/cos(pitch)
        cosp = np.maximum(np.abs(np.cos(ora.rpy[..., 1:2])), 0.02)
        for f in FIELDS:
            ref = getattr(ora, f)
            if f == "quat":
                e = quat_err(st[f], ref)
            elif f == "rpy":
                e = float(np.max(np.abs(st[f] - ref) * cosp / np.maximum(np.abs(ref), 1.0)))
            else:
                e = relerr(st[f], ref)
            assert e <= (max(tol, OBS_TOL) if f in OBS_FIELDS else tol), (f, t, e)
        assert relerr(rew.cpu().numpy(), o_rew) < max(tol, OBS_TOL)
        assert np.array_equal(term.cpu().numpy(), o_term), t
        # a truncation bound crossed within the state tolerance of the threshold may legitimately flip: skip those envs
        clear = ~_borderline(ora, tol)
        assert np.array_equal(trunc.cpu().numpy()[clear], o_trunc[clear]), t
        if t % check_obs_every == 0:
            assert relerr(obs.cpu().numpy(), o_obs) < max(tol, OBS_TOL)
    _report_borderline("compare_with_oracle tol=%g" % tol)


@pytest.mark.parametrize("act,A", [("RPM", 4), ("ONE_D_RPM", 1)])
def test_config3_multihover_4096_vs_oracle(act, A):
    """MultiHover, E=2048 x D=2 (4096 drones), random actions, 125 ticks x 8 substeps = 1000 physics steps of tumbling
    flight (|v| up to 20 m/s): with float64 state planes the kernel stays within 1e-9 of the float64 oracle (round 1,
    float32 planes: 5e-5, all of it the rounding of the stored quaternion)."""
    _, _, _, MultiHoverAviary, ActionType, _, Physics, O = _imports()
    E, D, T = 2048, 2, 125
    rng = np.random.default_rng(123)
    acts = rng.uniform(-1, 1, (T, E, D, A)).astype(np.float32)
    env = MultiHoverAviary(num_drones=D, physics=Physics.DYN, act=ActionType[act], num_envs=E)
    ora = O.OracleAviary("multihover", E, D, act=act.lower())
    _compare_with_oracle(env, ora, acts, TIGHT)


def test_config2_pid_4096_fixed_setpoints_vs_oracle():
    """BASELINE config 2 shape: 4096 x HoverAviary with the embedded DSLPIDControl (act=PID).  At the RL default 30 Hz the
    loop is chaotic in the reference itself, so the free-running comparison uses 240/120 Hz (S=2) for 250 ticks."""
    _, _, HoverAviary, _, ActionType, _, Physics, O = _imports()
    E, T = 4096, 250
    g = torch.Generator().manual_seed(0)
    sp = (torch.tensor([-0.5, -0.5, 0.5]) + torch.rand((E, 1, 3), generator=g) * torch.tensor([1.0, 1.0, 1.0])).numpy().astype(np.float32)
    acts = np.broadcast_to(sp, (T, E, 1, 3)).copy()
    env = HoverAviary(physics=Physics.DYN, act=ActionType.PID, pyb_freq=240, ctrl_freq=120, num_envs=E)
    ora = O.OracleAviary("hover", E, 1, act="pid", ctrl_freq=120)
    _compare_with_oracle(env, ora, acts, RTOL, check_obs_every=25)


@pytest.mark.parametrize("phys,eff", [("PYB_GND", 1), ("PYB_DRAG", 2), ("PYB_DW", 4), ("PYB_GND_DRAG_DW", 7)])
def test_dynplus_effects_vs_oracle(phys, eff):
    """DYN+ terms (ground effect, drag, in-CTA downwash): 64 aviaries x 4 drones stacked 1.5 m apart, 60 ticks x 8
    substeps.  (The reference's downwash term ~ 1/dz^2 is singular for dz -> 0+: drones at nearly equal heights make any
    comparison meaningless, so the stack keeps them apart.)"""
    _, _, _, MultiHoverAviary, ActionType, _, Physics, O = _imports()
    E, D, T = 64, 4, 60
    xyz = np.array([[0.0, 0.0, 0.06], [0.05, 0.02, 1.6], [0.1, -0.03, 3.1], [-0.05, 0.05, 4.6]])
    rng = np.random.default_rng(5)
    acts = (0.3 * rng.uniform(-1, 1, (T, E, D, 4))).astype(np.float32)
    env = MultiHoverAviary(num_drones=D, initial_xyzs=xyz, physics=Physics[phys], act=ActionType.RPM, num_envs=E)
    ora = O.OracleAviary("multihover", E, D, act="rpm", initial_xyzs=xyz, effects=eff)
    _compare_with_oracle(env, ora, acts, 1e-7)


def test_config4_big_formation_downwash_vs_oracle():
    """Config 4 shape at oracle-sized N: ONE aviary of 1024 drones = 256 stacks (1.6 m pitch) x 4 layers 1.5 m apart with
    small lateral offsets, ground effect + drag + downwash: the tiled pairwise kernel + split-substep protocol against the
    O(N^2) NumPy oracle.  (Well-conditioned geometry: the model's 1/dz^2 singularity makes dense same-height formations
    diverge between float32 and float64 pair evaluation within a few substeps -- in the reference as well.)"""
    _, CtrlAviary, _, _, _, _, Physics, O = _imports()
    D, T = 1024, 10
    i = np.arange(D)
    st_, ly = i // 4, i % 4
    xyz = np.stack([1.6 * (st_ % 16) + 0.04 * ly, 1.6 * (st_ // 16) - 0.03 * ly, 0.5 + 1.5 * ly], axis=1)
    env = CtrlAviary(num_drones=D, initial_xyzs=xyz, physics=Physics.PYB_GND_DRAG_DW, pyb_freq=240, ctrl_freq=48, num_envs=1)
    ora = O.OracleAviary("ctrl", 1, D, ctrl_freq=48, initial_xyzs=xyz, effects=7)
    rng = np.random.default_rng(9)
    env.reset(); ora.reset()
    # the pair term itself at step 0
    import ctypes as C
    from gym_pybullet_drones_b200 import _native as N
    fz = torch.zeros(D, device="cuda")
    N.check(N.lib().qs_downwash(C.byref(env._P), C.byref(env._st), 1, D, fz.data_ptr(), torch.cuda.current_stream().cuda_stream), "qs_downwash")
    ref_fz = O.downwash_body_z(ora.P, ora.pos)[0]
    assert np.count_nonzero(ref_fz) > 700 and relerr(fz.cpu().numpy(), ref_fz) < 1e-5
    for t in range(T):
        a = (ora.P.HOVER_RPM * (1 + 0.05 * rng.uniform(-1, 1, (1, D, 4)))).astype(np.float32)
        obs, _, _, _, _ = env.step(torch.from_numpy(a).cuda())
        o_obs, _, _, _ = ora.step(a)
        o = obs.cpu().numpy()
        assert relerr(o[..., 0:3], o_obs[..., 0:3]) < RTOL and quat_err(o[..., 3:7], o_obs[..., 3:7]) < RTOL, t
        assert relerr(o[..., 7:16], o_obs[..., 7:16]) < RTOL, t


# ---------------------------------------------------------------------------------------------------------------
# autoreset / vector-env semantics
# ---------------------------------------------------------------------------------------------------------------
def test_autoreset_same_step_matches_manual_reset_loop():
    """SB3 VecEnv semantics: done envs return the reset observation, the terminal one lands in info['final_obs'];
    compared with an oracle loop that resets done envs by hand (the reference's reset keeps the action buffer)."""
    _, _, HoverAviary, _, ActionType, _, Physics, O = _imports()
    E, T = 512, 300
    rng = np.random.default_rng(77)
    acts = rng.uniform(-1, 1, (T, E, 1, 4)).astype(np.float32)
    env = HoverAviary(physics=Physics.DYN, act=ActionType.RPM, num_envs=E, autoreset="same_step")
    ora = O.OracleAviary("hover", E, 1, act="rpm")
    env.reset(); ora.reset()
    n_done = 0
    for t in range(T):
        obs, rew, term, trunc, info = env.step(torch.from_numpy(acts[t]).cuda())
        o_obs, o_rew, o_term, o_trunc = ora.step(acts[t])
        done = o_term | o_trunc
        assert np.array_equal((term | trunc).cpu().numpy(), done), t
        assert np.array_equal(info["_final_obs"].cpu().numpy(), done)
        if done.any():
            n_done += int(done.sum())
            assert relerr(info["final_obs"].cpu().numpy()[done], o_obs[done]) < OBS_TOL
            o_obs2 = ora.reset(mask=done)
            o_obs = o_obs2
        assert relerr(obs.cpu().numpy(), o_obs) < OBS_TOL, t
        assert np.array_equal(env.step_counter.cpu().numpy(), ora.step_counter), t
    assert n_done > E // 2      # random +-5 % RPM tips the drone past 0.4 rad quickly: plenty of resets exercised


def test_autoreset_next_step_semantics():
    _, _, HoverAviary, _, ActionType, _, Physics, O = _imports()
    E, T = 256, 200
    rng = np.random.default_rng(78)
    acts = rng.uniform(-1, 1, (T, E, 1, 4)).astype(np.float32)
    env = HoverAviary(physics=Physics.DYN, act=ActionType.RPM, num_envs=E, autoreset="next_step")
    ora = O.OracleAviary("hover", E, 1, act="rpm")
    env.reset(); ora.reset()
    pending = np.zeros(E, bool)
    saw = 0
    for t in range(T):
        obs, rew, term, trunc, _ = env.step(torch.from_numpy(acts[t]).cuda())
        # oracle: envs that finished last step are reset now (their action is ignored, the buffer is untouched)
        buf_before = [b.copy() for b in ora.action_buffer]
        snap = {f: getattr(ora, f).copy() for f in ("pos", "quat", "vel", "rpy_rates", "ang_v", "rpy", "last_clipped_action")}
        sc = ora.step_counter.copy()
        o_obs, o_rew, o_term, o_trunc = ora.step(acts[t])
        if pending.any():
            saw += int(pending.sum())
            for f, v in snap.items():
                getattr(ora, f)[pending] = v[pending]
            ora.step_counter[pending] = sc[pending]
            for b_new, b_old in zip(ora.action_buffer, buf_before):
                b_new[pending] = b_old[pending]
            o_obs_r = ora.reset(mask=pending)
            o_obs[pending] = o_obs_r[pending]
            o_rew[pending] = 0; o_term[pending] = False; o_trunc[pending] = False
        assert relerr(obs.cpu().numpy(), o_obs) < OBS_TOL, t
        assert relerr(rew.cpu().numpy(), o_rew) < OBS_TOL
        assert np.array_equal((term | trunc).cpu().numpy(), o_term | o_trunc), t
        pending = o_term | o_trunc
    assert saw > E // 4


def test_numpy_vector_api_roundtrip_equals_tensor_api():
    """NumPy in / NumPy out (pinned staging, compact final_obs rows) returns exactly what the tensor API returns."""
    _, _, _, MultiHoverAviary, ActionType, _, Physics, _ = _imports()
    E, D = 128, 2
    rng = np.random.default_rng(3)
    kw = dict(num_drones=D, physics=Physics.DYN, act=ActionType.RPM, num_envs=E, autoreset="same_step")
    e1, e2 = MultiHoverAviary(**kw), MultiHoverAviary(**kw)
    o1, _ = e1.reset(); o2, _ = e2.reset()
    seen = 0
    for t in range(120):
        a = rng.uniform(-1, 1, (E, D, 4)).astype(np.float32)
        o1, r1, te1, tr1, i1 = e1.step(torch.from_numpy(a).cuda())
        o2, r2, te2, tr2, i2 = e2.step(a)
        assert isinstance(o2, np.ndarray) and o2.dtype == np.float32 and r2.shape == (E,) and te2.dtype == bool
        assert np.array_equal(o1.cpu().numpy(), o2) and np.array_equal(r1.cpu().numpy(), r2)
        assert np.array_equal(te1.cpu().numpy(), te2) and np.array_equal(tr1.cpu().numpy(), tr2)
        done = te2 | tr2
        assert np.array_equal(i1["_final_obs"].cpu().numpy(), done) and np.array_equal(i2["_final_obs"], done)
        if done.any():
            seen += int(done.sum())
            assert np.array_equal(i2["final_obs_env"], np.flatnonzero(done))
            assert np.array_equal(i2["final_obs"], i1["final_obs"].cpu().numpy()[done])
    assert seen > 20


@pytest.mark.parametrize("act,E,D,chunks,autoreset", [("RPM", 128, 2, "3", "same_step"), ("ONE_D_RPM", 1024, 4, "8", "same_step"),
                                                     ("RPM", 8192, 2, None, "same_step"), ("RPM", 1000, 1, "4", None),
                                                     ("RPM", 96, 32, "5", "same_step")])
def test_numpy_vector_api_chunked_pipeline_equals_tensor_api(act, E, D, chunks, autoreset, monkeypatch):
    """qs_step_host cuts the batch into chunks of whole warps and pipelines H2D(actions) -> tick -> D2H(observations) chunk by
    chunk (default: 4 chunks from 16 384 drones up; QS_HOST_CHUNKS forces a count): what comes back is exactly what the
    tensor API returns -- observations, rewards, flags, indices and rows of the terminal observations -- for chunk counts
    that do not divide the number of warps, a ragged last warp (1000 drones), aviaries of 32 drones, and without autoreset."""
    _, _, _, MultiHoverAviary, ActionType, _, Physics, _ = _imports()
    if chunks is None:
        monkeypatch.delenv("QS_HOST_CHUNKS", raising=False)
    else:
        monkeypatch.setenv("QS_HOST_CHUNKS", chunks)
    A = 4 if act == "RPM" else 1
    rng = np.random.default_rng(8)
    kw = dict(num_drones=D, physics=Physics.DYN, act=getattr(ActionType, act), num_envs=E, autoreset=autoreset)
    e1, e2 = MultiHoverAviary(**kw), MultiHoverAviary(**kw)
    e1.reset(); e2.reset()
    seen = 0
    for t in range(100 if E <= 1024 else 30):
        a = rng.uniform(-1, 1, (E, D, A)).astype(np.float32)
        o1, r1, te1, tr1, i1 = e1.step(torch.from_numpy(a).cuda())
        o2, r2, te2, tr2, i2 = e2.step(a)
        assert np.array_equal(o1.cpu().numpy(), o2) and np.array_equal(r1.cpu().numpy(), r2)
        assert np.array_equal(te1.cpu().numpy(), te2) and np.array_equal(tr1.cpu().numpy(), tr2)
        done = te2 | tr2
        if autoreset and done.any():
            seen += int(done.sum())
            assert np.array_equal(i2["final_obs_env"], np.flatnonzero(done))
            assert np.array_equal(i2["final_obs"], i1["final_obs"].cpu().numpy()[done])
    assert seen > 0 or not autoreset or act == "ONE_D_RPM"      # (collective thrust only: nothing finishes within 100 ticks)


# ---------------------------------------------------------------------------------------------------------------
# (c) size-independent properties at BASELINE.json's full sizes
# ---------------------------------------------------------------------------------------------------------------
def test_full_size_65536_properties():
    """65536 drones (32768 x MultiHover D=2), 100 random ticks: unit quaternions, finite state, every aviary that received
    the same action stream has bit-identical state (position in the batch does not matter), reset is idempotent."""
    _, _, _, MultiHoverAviary, ActionType, _, Physics, _ = _imports()
    E, D, T = 32768, 2, 100
    env = MultiHoverAviary(num_drones=D, physics=Physics.DYN, act=ActionType.RPM, num_envs=E, autoreset="same_step")
    env.reset()
    gen = torch.Generator(device="cuda").manual_seed(5)
    base = torch.rand((T, 64, D, 4), device="cuda", generator=gen) * 2 - 1
    for t in range(T):
        a = base[t].repeat(E // 64, 1, 1)           # aviary e gets stream e % 64
        obs, rew, term, trunc, _ = env.step(a)
    torch.cuda.synchronize()
    q = env.quat
    assert torch.all(torch.isfinite(env._planes)) and torch.all(torch.isfinite(obs))
    assert float((q.norm(dim=-1) - 1).abs().max()) < 1e-15
    pl = env._plane.view(3, E // 64, 64, D, 4)
    assert torch.equal(pl[:, 0], pl[:, 1]) and torch.equal(pl[:, 0], pl[:, -1])
    wz = env._wz.view(E // 64, 64, D)
    assert torch.equal(wz[0], wz[1]) and torch.equal(wz[0], wz[-1])
    ob = obs.view(E // 64, 64, D, -1)
    assert torch.equal(ob[0], ob[-1]) and torch.equal(rew.view(-1, 64)[0], rew.view(-1, 64)[-1])
    o1, _ = env.reset(); p1 = env._planes.clone()
    o2, _ = env.reset()
    assert torch.equal(p1, env._planes) and torch.equal(o1[..., :12], o2[..., :12])
    assert int(env.step_counter.max()) == 0


def test_history_shift_is_exact():
    """The observation tail is the last B actions oldest -> newest, bit-exact (BaseRLAviary.py:316-319)."""
    _, _, HoverAviary, _, ActionType, _, Physics, _ = _imports()
    for act, A in (("RPM", 4), ("PID", 3), ("ONE_D_RPM", 1)):
        E = 333
        env = HoverAviary(physics=Physics.DYN, act=ActionType[act], num_envs=E)
        env.reset()
        rng = np.random.default_rng(1)
        hist = [np.zeros((E, 1, A), np.float32) for _ in range(15)]
        for t in range(40):
            a = rng.uniform(-1, 1, (E, 1, A)).astype(np.float32)
            if act == "PID":
                a = (a * 0.1 + np.array([0, 0, 0.5], np.float32)).astype(np.float32)
            obs, *_ = env.step(a)
            hist = hist[1:] + [a]
            assert np.array_equal(obs[..., 12:], np.concatenate(hist, axis=-1)), (act, t)


def test_abi_argument_errors():
    import ctypes as C
    from gym_pybullet_drones_b200 import _native as N
    _, _, HoverAviary, _, ActionType, _, Physics, _ = _imports()
    env = HoverAviary(physics=Physics.DYN, act=ActionType.RPM, num_envs=4)
    L = N.lib()
    io = env._io
    io.action = env._action_dev.data_ptr(); io.obs_prev = env._obs_buf[0].data_ptr(); io.obs = env._obs_buf[1].data_ptr()
    s = torch.cuda.current_stream().cuda_stream
    assert L.qs_step(C.byref(env._P), C.byref(env._st), C.byref(io), 99, 1, 4, 1, 8, 0, 0, s) == -4
    assert L.qs_step(C.byref(env._P), C.byref(env._st), C.byref(io), 0, 1, 0, 1, 8, 0, 0, s) == -3
    assert L.qs_step(None, C.byref(env._st), C.byref(io), 0, 1, 4, 1, 8, 0, 0, s) == -1
    io.action = env._action_dev.data_ptr() + 4
    assert L.qs_step(C.byref(env._P), C.byref(env._st), C.byref(io), 0, 1, 4, 1, 8, 0, 0, s) == -2
    assert b"aligned" in L.qs_last_error()
    with pytest.raises(ValueError):
        N.check(-2, "x")


@pytest.mark.parametrize("D,E,phys,eff", [(100, 7, "DYN", 0), (128, 3, "DYN", 0), (5, 103, "PYB_GND_DRAG_DW", 7)])
def test_ragged_aviary_sizes_vs_oracle(D, E, phys, eff):
    """Aviary sizes that do not divide the CTA (D=100 -> 100 live threads of 128; D=5 -> 125), a last CTA that is only
    partly full, and the in-CTA downwash over D drones: 40 ticks against the oracle."""
    _, _, _, MultiHoverAviary, ActionType, _, Physics, O = _imports()
    T = 40
    i = np.arange(D)
    xyz = np.stack([0.4 * (i % 10) + 0.03 * (i // 10), 0.4 * ((i // 10) % 10), 0.3 + 1.5 * (i // 100) + 0.013 * i], axis=1) if eff == 0 else \
        np.stack([0.05 * i, -0.03 * i, 0.3 + 1.5 * i], axis=1)
    rng = np.random.default_rng(17)
    acts = (0.5 * rng.uniform(-1, 1, (T, E, D, 4))).astype(np.float32)
    env = MultiHoverAviary(num_drones=D, initial_xyzs=xyz, physics=Physics[phys], act=ActionType.RPM, num_envs=E)
    ora = O.OracleAviary("multihover", E, D, act="rpm", initial_xyzs=xyz, effects=eff)
    _compare_with_oracle(env, ora, acts, 1e-7)


def test_set_pid_coefficients_changes_the_controller():
    """BaseControl.setPIDCoefficients (BaseControl.py:138-177): new gains reach the kernel and match the oracle."""
    DSLPIDControl, _, _, _, _, DroneModel, _, O = _imports()
    n = 64
    rng = np.random.default_rng(2)
    pos, vel, tp = rng.uniform(-1, 1, (n, 3)), rng.uniform(-1, 1, (n, 3)), rng.uniform(-1, 1, (n, 3))
    q = rng.normal(size=(n, 4)); q[:, 3] = np.abs(q[:, 3]) + 2; q /= np.linalg.norm(q, axis=1, keepdims=True)
    ctrl = DSLPIDControl(DroneModel.CF2X, num_drones=n)
    ora = O.OraclePID(n, "cf2x")
    r0, _, _ = ctrl.computeControl(1 / 240, pos, q, vel, None, tp)
    ctrl.reset()
    ctrl.setPIDCoefficients(p_coeff_pos=np.array([.8, .8, 2.0]), d_coeff_att=np.array([10000., 10000., 6000.]))
    ora.P_FOR = np.array([.8, .8, 2.0]); ora.D_TOR = np.array([10000., 10000., 6000.])
    r1, pe, ye = ctrl.computeControl(1 / 240, pos, q, vel, None, tp)
    o1, ope, oye = ora.compute(1 / 240, pos, q, vel, tp)
    assert relerr(r1, o1) < 2e-5 and relerr(pe, ope) < 1e-6 and np.abs(r1 - r0).max() > 1.0


@pytest.mark.parametrize("mode", ["same_step", "next_step"])
def test_autoreset_can_clear_action_buffer_and_controllers(mode):
    """The reference's reset() keeps the action buffer and the embedded PID state (SURVEY.md 3.3); the opt-in flags clear
    them when an aviary auto-resets.  Oracle loop with the same clearing done by hand."""
    _, _, HoverAviary, _, ActionType, _, Physics, O = _imports()
    E, T = 256, 420
    rng = np.random.default_rng(91)
    # one fixed far-away set-point per aviary: the drone flies out of the |x|,|y| <= 1.5 box, is truncated, resets, flies again
    sp = (np.array([0, 0, 1.0], np.float32) + rng.choice([-1.0, 1.0], (E, 1, 3)).astype(np.float32) * np.array([3.0, 3.0, 0.3], np.float32)).astype(np.float32)
    acts = np.broadcast_to(sp, (T, E, 1, 3)).copy()
    env = HoverAviary(physics=Physics.DYN, act=ActionType.PID, pyb_freq=240, ctrl_freq=120, num_envs=E, autoreset=mode,
                      autoreset_clears_action_buffer=True, autoreset_clears_controllers=True)
    ora = O.OracleAviary("hover", E, 1, act="pid", ctrl_freq=120)
    env.reset(); ora.reset()
    pending = np.zeros(E, bool)
    n_resets = 0

    def clear(mask):
        for b in ora.action_buffer:
            b[mask] = 0
        ora.ctrl.reset(mask=mask)

    for t in range(T):
        obs, rew, term, trunc, info = env.step(torch.from_numpy(acts[t]).cuda())
        if mode == "next_step" and pending.any():
            snap = {f: getattr(ora, f).copy() for f in ("pos", "quat", "vel", "rpy_rates", "ang_v", "rpy", "last_clipped_action")}
            sc, buf = ora.step_counter.copy(), [b.copy() for b in ora.action_buffer]
            pid = [a.copy() for a in (ora.ctrl.integral_pos_e, ora.ctrl.last_rpy, ora.ctrl.integral_rpy_e)]
            o_obs, o_rew, o_term, o_trunc = ora.step(acts[t])
            for f, v in snap.items():
                getattr(ora, f)[pending] = v[pending]
            ora.step_counter[pending] = sc[pending]
            for bn, bo in zip(ora.action_buffer, buf):
                bn[pending] = bo[pending]
            for a_new, a_old in zip((ora.ctrl.integral_pos_e, ora.ctrl.last_rpy, ora.ctrl.integral_rpy_e), pid):
                a_new[pending] = a_old[pending]
            clear(pending)
            o_obs[pending] = ora.reset(mask=pending)[pending]
            o_rew[pending] = 0; o_term[pending] = False; o_trunc[pending] = False
        else:
            o_obs, o_rew, o_term, o_trunc = ora.step(acts[t])
        done = o_term | o_trunc
        assert np.array_equal((term | trunc).cpu().numpy(), done), t
        if mode == "same_step" and done.any():
            assert relerr(info["final_obs"].cpu().numpy()[done], o_obs[done]) < RTOL
            clear(done)
            o_obs = ora.reset(mask=done)
            assert np.all(obs.cpu().numpy()[done][..., 12:] == 0)
        n_resets += int(done.sum())
        assert relerr(obs.cpu().numpy(), o_obs) < RTOL, t
        pending = done if mode == "next_step" else pending
    assert n_resets > E // 2
    pid_dev = env._pid.view(9, E).cpu().numpy()
    assert relerr(pid_dev[0:3].T, ora.ctrl.integral_pos_e) < RTOL and relerr(pid_dev[6:9].T, ora.ctrl.integral_rpy_e) < 1e-4


# ---------------------------------------------------------------------------------------------------------------
# (d) BASELINE configs at their full sizes against the oracle (VERDICT round 1, item 2)
# ---------------------------------------------------------------------------------------------------------------
def test_config3_full_size_65536_drones_125_ticks_vs_oracle():
    """BASELINE configs[2] at size: 32768 x MultiHover D=2 = 65536 drones, random actions, 125 ticks x 8 substeps = 1000
    physics steps, every element of the kinematic state against the float64 oracle (the port needs ~20 s for this)."""
    _, _, _, MultiHoverAviary, ActionType, _, Physics, O = _imports()
    E, D, T = 32768, 2, 125
    rng = np.random.default_rng(2024)
    env = MultiHoverAviary(num_drones=D, physics=Physics.DYN, act=ActionType.RPM, num_envs=E)
    ora = O.OracleAviary("multihover", E, D, act="rpm")
    env.reset(); ora.reset()
    for t in range(T):
        a = rng.uniform(-1, 1, (E, D, 4)).astype(np.float32)
        obs, rew, term, trunc, _ = env.step(torch.from_numpy(a).cuda())
        o_obs, o_rew, o_term, o_trunc = ora.step(a)
        if t % 25 == 24 or t == T - 1:
            st = state_of(env)
            assert relerr(st["pos"], ora.pos) < TIGHT and quat_err(st["quat"], ora.quat) < TIGHT, t
            assert relerr(st["vel"], ora.vel) < TIGHT and relerr(st["rpy_rates"], ora.rpy_rates) < TIGHT, t
            assert relerr(obs.cpu().numpy()[..., 6:], o_obs[..., 6:]) < OBS_TOL and relerr(rew.cpu().numpy(), o_rew) < OBS_TOL, t
            assert np.array_equal(term.cpu().numpy(), o_term)
            clear = ~_borderline(ora, TIGHT)
            assert np.array_equal(trunc.cpu().numpy()[clear], o_trunc[clear]), t
    _report_borderline("65536 drones")


def test_config2_pid_4096_30hz_teacher_forced_vs_oracle():
    """BASELINE configs[1] as written: 4096 x HoverAviary with the embedded DSLPIDControl (act=PID) at the RL default
    240/30 Hz (S=8).  The 30 Hz loop is chaotic in the reference itself, so every tick restarts from the ORACLE's previous
    state (kinematics + controller integrals), exactly like the reference-golden teacher-forced test, but at E=4096."""
    _, _, HoverAviary, _, ActionType, _, Physics, O = _imports()
    E, T = 4096, 40
    g = torch.Generator().manual_seed(0)
    sp = (torch.tensor([-0.5, -0.5, 0.5]) + torch.rand((E, 1, 3), generator=g)).numpy().astype(np.float32)
    env = HoverAviary(physics=Physics.DYN, act=ActionType.PID, pyb_freq=240, ctrl_freq=30, num_envs=E)
    ora = O.OracleAviary("hover", E, 1, act="pid", ctrl_freq=30)
    env.reset(); ora.reset()
    for t in range(T):
        if t > 0:
            env.set_state(pos=ora.pos, quat=ora.quat, vel=ora.vel, rpy_rates=ora.rpy_rates, step_counter=ora.step_counter)
            env._pid[0:3] = torch.from_numpy(ora.ctrl.integral_pos_e.T.copy()).cuda()
            env._pid[3:6] = torch.from_numpy(ora.ctrl.last_rpy.T.copy()).cuda()
            env._pid[6:9] = torch.from_numpy(ora.ctrl.integral_rpy_e.T.copy()).cuda()
        obs, rew, term, trunc, _ = env.step(torch.from_numpy(sp).cuda())
        o_obs, o_rew, o_term, o_trunc = ora.step(sp)
        st = state_of(env)
        for f in ("pos", "quat", "vel", "rpy_rates"):
            e = quat_err(st[f], getattr(ora, f)) if f == "quat" else relerr(st[f], getattr(ora, f))
            assert e < 1e-7, (f, t, e)
        pid = env._pid.cpu().numpy()
        assert relerr(pid[0:3].T, ora.ctrl.integral_pos_e) < 1e-9 and relerr(pid[3:6].T, ora.ctrl.last_rpy) < 1e-9, t
        assert relerr(pid[6:9].T, ora.ctrl.integral_rpy_e) < 1e-7, t


def _chunked_downwash(O, xyz, chunk=1024):
    P = O.OracleParams()
    out = np.zeros(len(xyz))
    pos = xyz[None]
    for s in range(0, len(xyz), chunk):                     # rows [s, s+chunk) against every source: O(N^2) in pieces
        rows = pos[:, s:s + chunk]
        dz = pos[:, None, :, 2] - rows[:, :, None, 2]
        dxy = np.sqrt((pos[:, None, :, 0] - rows[:, :, None, 0]) ** 2 + (pos[:, None, :, 1] - rows[:, :, None, 1]) ** 2)
        act = (dz > 0) & (dxy < 10)
        dzs = np.where(act, dz, 1.0)
        alpha = P.DW[0] * (P.PROP_RADIUS / (4 * dzs)) ** 2
        beta = P.DW[1] * dzs + P.DW[2]
        with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
            f = -alpha * np.exp(-0.5 * (dxy / beta) ** 2)
        out[s:s + chunk] = np.sum(np.where(act, f, 0.0), axis=2)[0]
    return out


def test_config4_full_size_16384_static_downwash_vs_oracle():
    """BASELINE configs[3] geometry at size: 128 x 128 grid, 0.15 m pitch, 16 height levels (SURVEY 8d), one aviary of 16384
    drones.  The pairwise force of qs_downwash, qs_downwash_boxed and the row-sharded qs_downwash_rows (two halves against
    the gathered array) against BaseAviary._downwash restated in float64 (evaluated in row chunks)."""
    import ctypes as C
    from gym_pybullet_drones_b200 import _native as N
    _, CtrlAviary, _, _, _, _, Physics, O = _imports()
    k = np.arange(128 * 128)
    j, i = np.divmod(k, 128)
    xyz = np.stack([0.15 * i, 0.15 * j, 0.1 + 0.05 * (k % 16)], axis=1).astype(np.float32).astype(np.float64)
    D = len(xyz)
    ref = _chunked_downwash(O, xyz)
    assert np.count_nonzero(ref) > 0.9 * D
    env = CtrlAviary(num_drones=D, initial_xyzs=xyz, physics=Physics.PYB_DW, num_envs=1)
    env.reset()
    L, sp = N.lib(), torch.cuda.current_stream().cuda_stream
    fz = torch.zeros(D, device="cuda")
    N.check(L.qs_downwash(C.byref(env._P), C.byref(env._st), 1, D, fz.data_ptr(), sp), "qs_downwash")
    a = fz.cpu().numpy().astype(np.float64)
    assert relerr(a, ref) < RTOL
    ws = torch.zeros((1, D // 32, 8), device="cuda")
    fz2 = torch.zeros(D, device="cuda")
    N.check(L.qs_downwash_boxed(C.byref(env._P), C.byref(env._st), 1, D, ws.data_ptr(), fz2.data_ptr(), sp), "qs_downwash_boxed")
    assert np.array_equal(fz2.cpu().numpy(), fz.cpu().numpy())                 # same chunks, same order: same bits
    # row-sharded: the gathered array holds every position + the chunk boxes; each half evaluates its own rows
    nf = int(L.qs_dw_gathered_floats(D))
    gathered = torch.zeros(nf, device="cuda")
    gathered[:4 * D] = env._pos_f32.reshape(-1)
    N.check(L.qs_dw_boxes(gathered.data_ptr(), D, sp), "qs_dw_boxes")
    fz3 = torch.zeros(D, device="cuda")
    half = D // 2
    for r in range(2):
        rows = env._pos_f32[r * half:(r + 1) * half]
        N.check(L.qs_downwash_rows(C.byref(env._P), rows.data_ptr(), half, gathered.data_ptr(), D, None, 0, 0, None,
                                   fz3[r * half:].data_ptr(), sp), "qs_downwash_rows")
    assert np.array_equal(fz3.cpu().numpy(), fz.cpu().numpy())


def test_rollout_vs_oracle_directly():
    """qs_rollout (T fused ticks, state in registers, history in a sliding shared-memory window) against the float64 oracle
    itself -- not only against T calls of qs_step: observations, rewards and flags of every tick, state after the last."""
    _, _, _, MultiHoverAviary, ActionType, _, Physics, O = _imports()
    E, D, T = 512, 2, 60
    rng = np.random.default_rng(31)
    acts = (0.6 * rng.uniform(-1, 1, (T, E, D, 4))).astype(np.float32)
    env = MultiHoverAviary(num_drones=D, physics=Physics.DYN, act=ActionType.RPM, num_envs=E)
    ora = O.OracleAviary("multihover", E, D, act="rpm")
    env.reset(); ora.reset()
    out = env.rollout(torch.from_numpy(acts).cuda())
    obs, rew = out["obs"].cpu().numpy(), out["rewards"].cpu().numpy()
    te, tr = out["terminated"].cpu().numpy(), out["truncated"].cpu().numpy()
    for t in range(T):
        o_obs, o_rew, o_term, o_trunc = ora.step(acts[t])
        assert relerr(obs[t], o_obs) < OBS_TOL and relerr(rew[t], o_rew) < OBS_TOL, t
        clear = ~_borderline(ora, TIGHT)       # the end state is held to TIGHT below
        assert np.array_equal(te[t], o_term) and np.array_equal(tr[t][clear], o_trunc[clear]), t
    _report_borderline("rollout")
    st = state_of(env)
    assert relerr(st["pos"], ora.pos) < TIGHT and quat_err(st["quat"], ora.quat) < TIGHT
    assert relerr(st["vel"], ora.vel) < TIGHT and relerr(st["rpy_rates"], ora.rpy_rates) < TIGHT
