"""Per-aviary physical constants on the device (-m gpu): env.set_physical_params / QsState.phys in the fast and general step
kernels, qs_step_host, qs_dyn_substeps and qs_rollout (with and without the on-device policy).

  (a) a table of nominal rows gives the bytes of the env without a table, on every kernel family
  (b) random constants per aviary against the float64 oracle flying the same drones (tests/dyn_params_lib.py), CF2X / CF2P / RACE
  (c) rollout(T) == T x step() with the same table; the policy rollout equals the action rollout fed its clipped actions
  (d) per-episode re-randomisation with same-step autoreset, and a table switched on between readiness-ordered fast steps
  (e) a negative control (one aviary's kf moved by 1e-6) and the refusals"""
import numpy as np
import pytest
import torch

from dyn_params_lib import PerAviaryOracle, merge, random_properties, set_oracle_properties
from qs_testlib import FIELDS, TIGHT, quat_err, relerr
from test_gpu_configs import PID_TF_TOL, _force_from_snapshot, _ran_fast, _snapshot, _state_ratio
from test_gpu_parity import state_of

pytestmark = pytest.mark.gpu

MODELS = {"cf2x": "CF2X", "cf2p": "CF2P", "racer": "RACE"}


def _imports():
    from gym_pybullet_drones_b200.envs import CtrlAviary, HoverAviary, MultiHoverAviary
    from gym_pybullet_drones_b200.params import PHYS_KEYS
    from gym_pybullet_drones_b200.utils.enums import ActionType, DroneModel, Physics
    from oracle import dyn_oracle as O
    return CtrlAviary, HoverAviary, MultiHoverAviary, ActionType, DroneModel, Physics, PHYS_KEYS, O


def make(kind, E, D=1, model="cf2x", act="rpm", physics="DYN", pyb=240, ctrl=None, **kw):
    CtrlAviary, HoverAviary, MultiHoverAviary, ActionType, DroneModel, Physics, _, _ = _imports()
    args = dict(drone_model=DroneModel[MODELS[model]], physics=Physics[physics], pyb_freq=pyb, num_envs=E, **kw)
    if kind == "ctrl":
        return CtrlAviary(num_drones=D, ctrl_freq=ctrl or 240, **args)
    args.update(act=ActionType[act.upper()], ctrl_freq=ctrl or 30)
    return HoverAviary(**args) if kind == "hover" else MultiHoverAviary(num_drones=D, **args)


def oracle(kind, E, D=1, model="cf2x", act="rpm", effects=0, pyb=240, ctrl=None):
    return PerAviaryOracle(kind, E, D, drone_model=model, pyb_freq=pyb, ctrl_freq=ctrl, act=act, effects=effects)


def set_env(env, props):
    env.set_physical_params(**{k: torch.as_tensor(v, device=env.device) for k, v in props.items()})


def actions(env, T, seed):
    rng = np.random.default_rng(seed)
    if env._act_type() == 5:                                    # CtrlAviary: 0.6-1.2 x the nominal MAX_RPM, so the clip binds often
        return (env.MAX_RPM * rng.uniform(0.6, 1.2, (T, env._E, env._D, 4))).astype(np.float32)
    a = rng.uniform(-1, 1, (T, env._E, env._D, env._A)).astype(np.float32)
    if env._act_type() == 1:                                    # PID: waypoints near the start
        a = (0.3 * a + np.array([0, 0, 1], np.float32)).astype(np.float32)
    return a


def outputs(env, info):
    out = dict(obs=env._obs_buf[env._cur], rew=env._reward, te=env._terminated, tr=env._truncated, planes=env._planes,
               sc=env._step_counter)
    if env._track_last_action:
        out["last"] = env._last_rpm
    if env._pid is not None:
        out["pid"] = env._pid
    if info and "final_obs" in info and isinstance(info["final_obs"], torch.Tensor):
        out["final"] = info["final_obs"]
    return {k: v.detach().cpu().numpy().copy() for k, v in out.items()}


def assert_same(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), (what, k)


# ---------------------------------------------------------------------------------------------------------------
# (a) nominal table == no table, byte for byte
# ---------------------------------------------------------------------------------------------------------------
NOMINAL_ROWS = [
    # name, kind, E, D, act, physics, ctrl, extra kwargs, expected kernel
    ("hover_rpm", "hover", 512, 1, "rpm", "DYN", 30, {}, "fast"),
    ("hover_one_d_rpm", "hover", 512, 1, "one_d_rpm", "DYN", 30, {}, "fast"),
    ("multi2_same_step", "multi", 1024, 2, "rpm", "DYN", 30, dict(autoreset="same_step"), "fast"),
    ("multi3", "multi", 512, 3, "rpm", "DYN", 30, dict(autoreset="same_step"), "general"),
    ("pid48", "hover", 256, 1, "pid", "DYN", 48, {}, "general"),
    ("vel", "hover", 256, 1, "vel", "DYN", 30, {}, "general"),
    ("ctrl", "ctrl", 256, 2, "rpm", "DYN", 240, {}, "general"),
    ("gnd_drag_dw4", "multi", 256, 4, "rpm", "PYB_GND_DRAG_DW", 30, {}, "general"),
]


@pytest.mark.parametrize("row", NOMINAL_ROWS, ids=[r[0] for r in NOMINAL_ROWS])
def test_nominal_table_gives_the_bytes_of_no_table(row):
    name, kind, E, D, act, physics, ctrl, kw, kernel = row
    a, b = make(kind, E, D, act=act, physics=physics, ctrl=ctrl, **kw), make(kind, E, D, act=act, physics=physics, ctrl=ctrl, **kw)
    b.set_physical_params()
    assert b._st.phys and not a._st.phys
    a.reset(); b.reset()
    acts = actions(a, 120, seed=11)
    for t in range(120):
        act_t = torch.from_numpy(acts[t]).cuda()
        ra, rb = a.step(act_t), b.step(act_t)
        assert_same(outputs(a, ra[4]), outputs(b, rb[4]), (name, t))
    assert _ran_fast(b) == (kernel == "fast"), name             # CtrlAviary: qs_dyn_substeps, the general kernel


def test_nominal_table_numpy_path_chunked():
    """qs_step_host in chunks (16 384 drones): NumPy actions in, host arrays out, same bytes with the nominal table."""
    E, D = 8192, 2
    a, b = make("multi", E, D, autoreset="same_step"), make("multi", E, D, autoreset="same_step")
    b.set_physical_params()
    a.reset(); b.reset()
    acts = actions(a, 100, seed=12)
    for t in range(100):
        oa, ob = a.step(acts[t]), b.step(acts[t])
        for x, y in zip(oa[:4], ob[:4]):
            assert np.asarray(x).tobytes() == np.asarray(y).tobytes(), t
    assert _ran_fast(b)
    assert a._planes.cpu().numpy().tobytes() == b._planes.cpu().numpy().tobytes()


@pytest.mark.parametrize("policy", [False, True])
def test_nominal_table_rollout(policy):
    E, D = 1024, 2
    a, b = make("multi", E, D, autoreset="same_step"), make("multi", E, D, autoreset="same_step")
    b.set_physical_params()
    a.reset(); b.reset()
    if policy:
        pol = _policy(D * a._obs_dim, D * 4, critic=True)
        noise = torch.randn((100, E, D * 4), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
        oa, ob = a.rollout(policy=pol, noise=noise), b.rollout(policy=pol, noise=noise)
    else:
        acts = torch.from_numpy(actions(a, 100, seed=13)).cuda()
        oa, ob = a.rollout(acts), b.rollout(acts)
    for k in oa:
        assert oa[k].cpu().numpy().tobytes() == ob[k].cpu().numpy().tobytes(), k
    assert outputs(a, None)["planes"].tobytes() == outputs(b, None)["planes"].tobytes()


def _policy(in_dim, out_dim, critic=False, seed=0):
    from gym_pybullet_drones_b200.policy import MlpPolicy
    g = torch.Generator(device="cuda").manual_seed(seed)

    def lin(i, o):
        return (torch.randn((i, o), device="cuda", generator=g) / i ** 0.5, 0.05 * torch.randn((o,), device="cuda", generator=g))
    net = lambda o: [lin(in_dim, 64), lin(64, 64), lin(64, o)]     # noqa: E731
    return MlpPolicy(net(out_dim), torch.full((out_dim,), -1.0, device="cuda"), net(1) if critic else None)


# ---------------------------------------------------------------------------------------------------------------
# (b) random constants per aviary against the oracle
# ---------------------------------------------------------------------------------------------------------------
ORACLE_ROWS = [
    # name, env kind, oracle kind, D, act, physics, effects, ctrl, kernel
    ("fast_hover", "hover", "hover", 1, "rpm", "DYN", 0, 30, "fast"),
    ("fast_multi2_one_d", "multi", "multihover", 2, "one_d_rpm", "DYN", 0, 30, "fast"),
    ("general_multi3", "multi", "multihover", 3, "rpm", "DYN", 0, 30, "general"),
    ("general_ctrl_clip", "ctrl", "ctrl", 1, "rpm", "DYN", 0, 240, "general"),
    ("general_dynplus4", "multi", "multihover", 4, "rpm", "PYB_GND_DRAG_DW", 7, 30, "general"),
]


@pytest.mark.parametrize("model", list(MODELS))
@pytest.mark.parametrize("row", ORACLE_ROWS, ids=[r[0] for r in ORACLE_ROWS])
def test_random_constants_match_the_oracle(row, model):
    name, kind, okind, D, act, physics, eff, ctrl, kernel = row
    _, _, _, _, DroneModel, _, _, _ = _imports()
    E = 4096 // D
    env = make(kind, E, D, model=model, act=act, physics=physics, ctrl=ctrl)
    ora = oracle(okind, E, D, model=model, act=act, effects=eff, ctrl=ctrl)
    props = random_properties(DroneModel[MODELS[model]], E, seed=21)
    set_env(env, props)
    set_oracle_properties(ora, props)
    env.reset(); ora.reset()
    acts = actions(env, 40, seed=22)
    if kind == "ctrl":
        assert np.mean(acts[..., :] > ora.P.MAX_RPM) > 0.2          # the per-aviary MAX_RPM clip binds
    worst = 0.0
    for t in range(40):
        env.step(torch.from_numpy(acts[t]).cuda())
        ora.step(acts[t].astype(np.float64) if kind == "ctrl" else acts[t])
        worst = max(worst, _state_ratio(state_of(env), ora, TIGHT))
    assert worst <= 1.0, (name, model, worst)
    assert _ran_fast(env) == (kernel == "fast"), name


@pytest.mark.parametrize("model", ["cf2x", "cf2p"])
def test_random_constants_pid_teacher_forced(model):
    """PID at 48 Hz (general kernel): the drone's constants vary, the embedded controller stays the nominal CF2X one."""
    _, _, _, _, DroneModel, _, _, _ = _imports()
    E = 1024
    env = make("hover", E, model=model, act="pid", ctrl=48)
    ora = oracle("hover", E, model=model, act="pid", ctrl=48)
    props = random_properties(DroneModel[MODELS[model]], E, seed=31)
    set_env(env, props)
    set_oracle_properties(ora, props)
    env.reset(); ora.reset()
    acts = actions(env, 30, seed=32)
    worst = 0.0
    for t in range(30):
        _force_from_snapshot(env, _snapshot(ora))
        env.step(torch.from_numpy(acts[t]).cuda())
        ora.step(acts[t])
        worst = max(worst, _state_ratio(state_of(env), ora, PID_TF_TOL))
    assert worst <= 1.0, worst
    assert not _ran_fast(env)


@pytest.mark.parametrize("model", list(MODELS))
def test_rollout_random_constants(model):
    """rollout(T) with a random table: the oracle at TIGHT, and T x step() on a twin bit for bit."""
    _, _, _, _, DroneModel, _, _, _ = _imports()
    E, D, T = 2048, 2, 40
    a, b = make("multi", E, D, model=model), make("multi", E, D, model=model)
    ora = oracle("multihover", E, D, model=model)
    props = random_properties(DroneModel[MODELS[model]], E, seed=41)
    set_env(a, props); set_env(b, props); set_oracle_properties(ora, props)
    a.reset(); b.reset(); ora.reset()
    acts = actions(a, T, seed=42)
    out = a.rollout(torch.from_numpy(acts).cuda())
    for t in range(T):
        b.step(torch.from_numpy(acts[t]).cuda())
        ora.step(acts[t])
        assert out["obs"][t].cpu().numpy().tobytes() == b._obs_buf[b._cur].view(E, D, -1).cpu().numpy().tobytes(), t
    assert a._planes.cpu().numpy().tobytes() == b._planes.cpu().numpy().tobytes()
    assert _state_ratio(state_of(a), ora, TIGHT) <= 1.0


def test_policy_rollout_physics_equals_the_action_rollout():
    """Random table: the policy rollout's physics is the action rollout's, fed the policy's clipped actions."""
    _, _, _, _, DroneModel, _, _, _ = _imports()
    E, D, T = 1024, 2, 32
    a, b = make("multi", E, D, autoreset="same_step"), make("multi", E, D, autoreset="same_step")
    props = random_properties(DroneModel.CF2X, E, seed=51)
    set_env(a, props); set_env(b, props)
    a.reset(); b.reset()
    pol = _policy(D * a._obs_dim, D * 4, critic=True, seed=5)
    noise = torch.randn((T, E, D * 4), device="cuda", generator=torch.Generator(device="cuda").manual_seed(6))
    oa = a.rollout(policy=pol, noise=noise)
    ob = b.rollout(oa["actions"].clamp(-1, 1).clone())
    for k in ("obs", "rewards", "terminated", "truncated"):
        assert oa[k].cpu().numpy().tobytes() == ob[k].cpu().numpy().tobytes(), k
    assert a._planes.cpu().numpy().tobytes() == b._planes.cpu().numpy().tobytes()


# ---------------------------------------------------------------------------------------------------------------
# (d) re-randomisation at episode boundaries; a table switched on between readiness-ordered steps
# ---------------------------------------------------------------------------------------------------------------
def test_rerandomise_finished_aviaries_with_same_step_autoreset():
    _, _, _, _, DroneModel, _, PHYS_KEYS, _ = _imports()
    E, D = 2048, 2
    env = make("multi", E, D, autoreset="same_step")
    ora = oracle("multihover", E, D)
    props = random_properties(DroneModel.CF2X, E, seed=61)
    set_env(env, props); set_oracle_properties(ora, props)
    env.reset(); ora.reset()
    acts = actions(env, 120, seed=62)
    g = torch.Generator(device="cuda").manual_seed(63)
    nom = env.physical_params()
    resets = 0
    for t in range(120):
        _, _, _, _, info = env.step(torch.from_numpy(acts[t]).cuda())
        _, _, term, trunc = ora.step(acts[t])
        done_o = term | trunc
        done = info["_final_obs"]
        assert np.array_equal(done.cpu().numpy(), done_o), t
        # fresh CUDA-tensor constants for the aviaries that start a new episode (no host synchronisation in the setter)
        new = {k: nom[k] * (0.8 + 0.4 * torch.rand((E,), device="cuda", dtype=torch.float64, generator=g)) for k in PHYS_KEYS}
        env.set_physical_params(**new, envs=done)
        if done_o.any():
            resets += int(done_o.sum())
            ora.reset(mask=done_o)
            props = merge(props, {k: v.cpu().numpy() for k, v in new.items()}, done_o)
            set_oracle_properties(ora, props)
        assert _state_ratio(state_of(env), ora, TIGHT) <= 1.0, t
    assert resets > 0 and _ran_fast(env) and int(env._ready_err.item()) == 0
    got = env.physical_params()
    assert all(np.array_equal(got[k].cpu().numpy(), props[k]) for k in PHYS_KEYS)


def test_table_switched_on_between_readiness_ordered_steps():
    _, _, _, _, DroneModel, _, _, _ = _imports()
    E, D = 4096, 2
    env = make("multi", E, D)
    ora = oracle("multihover", E, D)
    env.reset(); ora.reset()
    acts = actions(env, 40, seed=71)
    props = random_properties(DroneModel.CF2X, E, seed=72)
    for t in range(40):
        if t == 15:
            set_env(env, props)                                  # between two fast steps of the same stream
            set_oracle_properties(ora, props)
        env.step(torch.from_numpy(acts[t]).cuda())
        ora.step(acts[t])
        assert _state_ratio(state_of(env), ora, TIGHT) <= 1.0, t
    assert _ran_fast(env) and int(env._ready_err.item()) == 0


# ---------------------------------------------------------------------------------------------------------------
# (e) negative control, refusals
# ---------------------------------------------------------------------------------------------------------------
def test_negative_control_one_aviarys_kf():
    _, _, _, _, DroneModel, _, _, _ = _imports()
    E, k = 256, 7
    a, b = make("hover", E), make("hover", E)
    ora = oracle("hover", E)
    props = random_properties(DroneModel.CF2X, E, seed=81)
    moved = dict(props, kf=props["kf"].copy())
    moved["kf"][k] *= 1 + 1e-6
    set_env(a, props); set_env(b, moved); set_oracle_properties(ora, props)
    a.reset(); b.reset(); ora.reset()
    acts = actions(a, 50, seed=82)
    for t in range(50):
        a.step(torch.from_numpy(acts[t]).cuda()); b.step(torch.from_numpy(acts[t]).cuda()); ora.step(acts[t])
    sa, sb = state_of(a), state_of(b)
    others = np.arange(E) != k
    for f in FIELDS:
        assert sa[f][others].tobytes() == sb[f][others].tobytes(), f
    assert relerr(sb["pos"][k], ora.pos[k]) > 10 * TIGHT                  # the moved aviary leaves TIGHT ...
    assert _state_ratio(sa, ora, TIGHT) <= 1.0                             # ... the unmoved env stays inside it
    assert quat_err(sa["quat"], ora.quat) <= TIGHT


def test_refusals():
    CtrlAviary, _, _, _, _, Physics, _, _ = _imports()
    env = make("multi", 8, 2)
    env.set_physical_params()                                    # allocates the table, all rows nominal
    for bad in (dict(m=np.full(7, 0.03)), dict(kf=-3e-10), dict(km=0.0), dict(ixx=np.full(8, np.nan)), dict(arm=np.inf)):
        with pytest.raises(ValueError):
            env.set_physical_params(**bad)
    with pytest.raises(ValueError):
        env.set_physical_params(m=0.03, envs=np.ones(7, bool))
    assert env._phys is not None and int(env.physical_params_rejected.item()) == 0
    # CUDA tensors are screened on the device: the aviary keeps its row, the refusal is counted
    before = env._phys.clone()
    m = torch.full((8,), 0.03, dtype=torch.float64, device="cuda")
    m[3] = float("nan")
    env.set_physical_params(m=m)
    assert int(env.physical_params_rejected.item()) == 1
    assert torch.equal(env._phys[3], before[3]) and not torch.equal(env._phys[2], before[2])
    # aviaries larger than one CTA with downwash take the split-substep kernels: refused in Python and in the C ABI
    big = CtrlAviary(num_drones=130, physics=Physics.PYB_DW, num_envs=1)
    with pytest.raises(ValueError):
        big.set_physical_params(m=0.03)
    big._st.phys = env._phys.data_ptr()
    with pytest.raises(ValueError, match="QS_ERR -5"):
        big.step(np.full((1, 130, 4), 14000.0, np.float32))
    big._st.phys = None
    # FormationShard (one formation, here world 1 with the in-process exchange) takes the same external-downwash kernels
    from gym_pybullet_drones_b200.formation import FormationShard
    xyz = np.stack([np.arange(64) * 0.3, np.zeros(64), np.full(64, 1.0)], axis=1)
    shard = FormationShard(xyz, physics=Physics.PYB_DW, exchange="local")
    with pytest.raises(ValueError, match="external downwash"):
        shard.set_physical_params(m=0.03)
    assert shard._phys is None and not shard._st.phys
    # the opt-in check reads CUDA tensors back and raises like the host inputs
    bad = torch.full((8,), 0.03, dtype=torch.float64, device="cuda")
    bad[5] = -1.0
    before = env._phys.clone()
    with pytest.raises(ValueError):
        env.set_physical_params(m=bad, check=True)
    assert torch.equal(env._phys, before) and int(env.physical_params_rejected.item()) == 1


# ---------------------------------------------------------------------------------------------------------------
# (f) the unmodified reference with overwritten constants (tests/golden/dyn_params.npz) on the device
# ---------------------------------------------------------------------------------------------------------------
GOLDEN_KEYS = ["cf2x_heavy_rpm", "cf2p_light_one_d_rpm", "race_long_arm_rpm", "multi3_rpm", "ctrl_low_t2w_clip", "pid_48"]
# E = 3, ONE_D_RPM at 30 Hz: od = 27 and 3 x 27 floats in the ragged last warp are not a 16-byte multiple -> general kernel
GOLDEN_KERNEL = {"cf2x_heavy_rpm": "fast", "cf2p_light_one_d_rpm": "general", "race_long_arm_rpm": "fast", "multi3_rpm": "general",
                 "ctrl_low_t2w_clip": "general", "pid_48": "general"}


@pytest.mark.parametrize("key", GOLDEN_KEYS)
def test_dyn_params_golden_on_device(golden, key):
    """E = 3 aviaries with the fixture's constants: state within TIGHT of the reference, observations within OBS_TOL, reward and
    flags on every tick, in aviaries 0 and 2.  PID at 48 Hz is teacher-forced (as every device PID golden) at PID_TF_TOL."""
    import json
    from test_gpu_parity import OBS_TOL, check_fields
    _, _, _, _, _, _, PHYS_KEYS, _ = _imports()
    g = golden("dyn_params")
    c = {c["key"]: c for c in json.loads(str(g["cases"]))}[key]
    E, D = 3, c["nd"]
    env = make("ctrl" if c["kind"] == "ctrl" else ("hover" if c["kind"] == "hover" else "multi"), E, D, model=c["model"],
               act="rpm" if c["act"] == "raw" else c["act"], pyb=c["pyb"], ctrl=c["ctrl"])
    p = g[key + "_props"]
    env.set_physical_params(**{k: np.full(E, float(p[j])) for j, k in enumerate(PHYS_KEYS)})
    obs, _ = env.reset()
    assert relerr(obs[0].cpu().numpy(), g[key + "_obs0"]) < 1e-6
    acts = g[key + "_actions"]
    pid = c["act"] == "pid"
    S = c["pyb"] // c["ctrl"]
    tol = PID_TF_TOL if pid else TIGHT
    for t in range(acts.shape[0]):
        if pid and t > 0:
            env.set_state(pos=np.broadcast_to(g[key + "_pos"][t - 1], (E, D, 3)), quat=np.broadcast_to(g[key + "_quat"][t - 1], (E, D, 4)),
                          vel=np.broadcast_to(g[key + "_vel"][t - 1], (E, D, 3)),
                          rpy_rates=np.broadcast_to(g[key + "_rpy_rates"][t - 1], (E, D, 3)), step_counter=t * S)
            for k, name in enumerate(("pid_integral_pos_e", "pid_last_rpy", "pid_integral_rpy_e")):
                env._pid[3 * k:3 * k + 3] = torch.from_numpy(np.repeat(g[key + "_" + name][t - 1].T, E, axis=1).copy()).cuda()
        a = np.broadcast_to(acts[t], (E,) + acts[t].shape).copy()
        # CtrlAviary: float64 RPMs, as the reference got them (QS_FLAG_ACTION_F64)
        out = env.step(a if c["kind"] == "ctrl" else torch.from_numpy(a).cuda())
        obs, rew, term, trunc = (x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x) for x in out[:4])
        st = state_of(env)
        for e in (0, 2):
            check_fields(st, g, key, t, tol, e)
            ref_r = g[key + "_reward"][t]
            assert abs(float(rew[e]) - ref_r) <= OBS_TOL * max(1.0, abs(ref_r)), (t, float(rew[e]), ref_r)
            assert bool(term[e]) == bool(g[key + "_terminated"][t]) and bool(trunc[e]) == bool(g[key + "_truncated"][t]), (e, t)
            assert relerr(obs[e], g[key + "_obs"][t]) < OBS_TOL, t
    assert _ran_fast(env) == (GOLDEN_KERNEL[key] == "fast")
    assert int(env._ready_err.item()) == 0
