"""The on-device policy of qs_rollout with the embedded DSLPID controller (PID, VEL, ONE_D_PID actions) and with the DYN+ effects
(ground effect, drag, downwash): rollout_kernel<EFF, PIDACT, kNetClassic, PHYS>.

Every case runs the two checks of test_gpu_policy.py, with episodes started near their time limit so that same-step autoresets
happen inside the rollout:
* MLP, teacher-forced per tick against the float64 tests/qs_testlib.PolicyRef: worst error / tolerance <= 1.
* Physics, bit for bit: a twin env replays `out["actions"].clamp(-1, 1)` through the action rollout from the same state;
  observations, rewards, flags, state planes, last RPMs, PID states and step counters are equal.
The oracle cases replay one policy rollout of each new family through the float64 OracleAviary, teacher-forced where
test_gpu_configs.py's matrix is, at that matrix's tolerances.  The refusals need no GPU.

Set QS_POLICY_REPORT=1 to print every case's worst error / tolerance."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from qs_testlib import RTOL, PolicyRef, relerr

_STACK4 = np.array([[0.0, 0.0, 0.06], [0.05, 0.02, 1.6], [0.1, -0.03, 3.1], [-0.05, 0.05, 4.6]])   # as test_gpu_api / test_gpu_configs


def _report(name, r):
    if os.environ.get("QS_POLICY_REPORT"):
        print("policy-ratio %-44s %s" % (name, " ".join("%s=%.3g" % kv for kv in sorted(r.items()))))


def _make(cls, act, D, E, physics="DYN", autoreset="same_step", **kw):
    import gym_pybullet_drones_b200.envs as envs
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    args = dict(physics=Physics[physics], act=ActionType[act], num_envs=E, autoreset=autoreset, track_last_action=True, **kw)
    if cls == "MultiHoverAviary":
        args["num_drones"] = D
    return getattr(envs, cls)(**args)


def _state(env):
    out = dict(planes=env._planes, last_rpm=env._last_rpm, step_counter=env._step_counter, obs_buf=env._obs_buf[env._cur])
    if env._pid is not None:
        out["pid"] = env._pid
    return {k: v.clone() for k, v in out.items()}


def _assert_same_physics(out, twin_out, env, twin):
    for k in ("obs", "rewards", "terminated", "truncated"):
        a, b = out[k], twin_out[k]
        assert a.shape == b.shape and torch.equal(a, b), k
    sa, sb = _state(env), _state(twin)
    assert sa.keys() == sb.keys()
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k


def _teacher_forced(ref, obs0, out, noise):
    """Worst error / tolerance over the ticks of `out`, the reference evaluated on the kernel's observation before each tick as
    the kernel's saturating fp16 split sees it (PolicyRef.OBS_SATURATION; test_gpu_policy.py pins that point).  The largest
    observation magnitude is reported too: where two drones of an aviary pass close above each other, the reference's
    downwash model (proportional to 1 / dz^2) can throw them to speeds past the saturation point."""
    worst = {"obs_max": 0.0}
    for t in range(out["obs"].shape[0]):
        x = ref.flat(obs0 if t == 0 else out["obs"][t - 1])
        r = ref.check(x, None if noise is None else noise[t], out["actions"][t], out["log_probs"][t], out.get("values", [None] * (t + 1))[t],
                      ref_obs=PolicyRef.saturate(x).astype(np.float32))
        for k, v in r.items():
            worst[k] = max(worst.get(k, 0.0), v)
        worst["obs_max"] = max(worst["obs_max"], float(np.abs(x).max()))
    return worst


def _ratio(worst):
    return max(v for k, v in worst.items() if k != "obs_max")


def _physical_table(env, seed):
    """A random per-aviary table (set_physical_params) around the env's drone; returns it to be given to the twin."""
    from dyn_params_lib import random_properties
    props = random_properties(env.DRONE_MODEL, env._E, seed)
    env.set_physical_params(**props)
    return props


# (name, cls, act, D, E, physics, T, options): E leaves the last CTA partial (a policy CTA holds 64 // D aviaries); D = 3 and 10
# leave idle threads (63 and 60 drones in a 64-thread CTA)
CASES = [
    ("pid-hover", "HoverAviary", "PID", 1, 200, "DYN", 10, {}),                # in_dim 57: the scalar layer-1 path
    ("pid-multi2", "MultiHoverAviary", "PID", 2, 150, "DYN", 10, {}),
    ("pid-multi3", "MultiHoverAviary", "PID", 3, 100, "DYN", 10, {}),         # 21 aviaries per CTA, partial CTA
    ("pid-multi10", "MultiHoverAviary", "PID", 10, 20, "DYN", 10, {}),        # out_dim 30, nt3 = 4
    ("vel-hover", "HoverAviary", "VEL", 1, 200, "DYN", 10, {}),
    ("vel-multi2", "MultiHoverAviary", "VEL", 2, 150, "DYN", 10, {}),
    ("vel-multi8", "MultiHoverAviary", "VEL", 8, 20, "DYN", 10, {}),          # out_dim 32
    ("one_d_pid-hover", "HoverAviary", "ONE_D_PID", 1, 200, "DYN", 12, {}),
    ("one_d_pid-multi4", "MultiHoverAviary", "ONE_D_PID", 4, 37, "DYN", 12, {}),
    ("one_d_pid-multi32", "MultiHoverAviary", "ONE_D_PID", 32, 5, "DYN", 12, {}),   # in_dim 864, 2 aviaries per CTA
    ("rpm-gnd-multi2", "MultiHoverAviary", "RPM", 2, 150, "PYB_GND", 10, {}),
    ("rpm-drag-multi2", "MultiHoverAviary", "RPM", 2, 150, "PYB_DRAG", 10, {}),
    ("rpm-dw-multi2", "MultiHoverAviary", "RPM", 2, 150, "PYB_DW", 10, {}),
    ("rpm-all-multi2", "MultiHoverAviary", "RPM", 2, 150, "PYB_GND_DRAG_DW", 10, {}),
    ("rpm-dw-stack4", "MultiHoverAviary", "RPM", 4, 50, "PYB_DW", 10, {"initial_xyzs": _STACK4}),
    ("rpm-all-stack4", "MultiHoverAviary", "RPM", 4, 50, "PYB_GND_DRAG_DW", 10, {"initial_xyzs": _STACK4}),
    ("pid-all-multi2", "MultiHoverAviary", "PID", 2, 150, "PYB_GND_DRAG_DW", 10, {}),
    ("pid-clears-multi2", "MultiHoverAviary", "PID", 2, 150, "DYN", 10,
     {"autoreset_clears_controllers": True, "autoreset_clears_action_buffer": True}),
    ("pid-phys-multi2", "MultiHoverAviary", "PID", 2, 150, "DYN", 10, {"table": 71}),
    ("rpm-all-phys-stack4", "MultiHoverAviary", "RPM", 4, 50, "PYB_GND_DRAG_DW", 10, {"initial_xyzs": _STACK4, "table": 72}),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_policy_rollout_with_controller_and_effects(case):
    from gym_pybullet_drones_b200.policy import MlpPolicy
    name, cls, act, D, E, physics, T, opts = case
    opts = dict(opts)
    table = opts.pop("table", None)
    env, twin = _make(cls, act, D, E, physics, **opts), _make(cls, act, D, E, physics, **opts)
    if table is not None:
        props = _physical_table(env, table)
        twin.set_physical_params(**props)
    A, od = env._A, env._obs_dim
    pol = MlpPolicy.random(D * od, D * A, seed=5 + D + A, critic=True, log_std=-1.0)
    ref = PolicyRef(pol)
    noise = torch.randn((T, E, D * A), device="cuda", generator=torch.Generator(device="cuda").manual_seed(9))
    obs0 = env.reset()[0].clone()
    twin.reset()
    # episodes near their time limit, ending at different ticks: the rollout autoresets aviaries on the way
    sc = np.random.default_rng(1).integers(1880, 1960, E)
    env.set_state(step_counter=sc); twin.set_state(step_counter=sc)
    out = env.rollout(policy=pol, noise=noise)
    assert out["actions"].shape == (T, E, D, A) and out["log_probs"].shape == (T, E) and out["values"].shape == (T, E)
    twin_out = twin.rollout(actions=out["actions"].clamp(-1, 1))
    torch.cuda.synchronize()
    _assert_same_physics(out, twin_out, env, twin)
    assert int((out["terminated"] | out["truncated"]).sum()) > 0
    worst = _teacher_forced(ref, obs0, out, noise)
    _report(name, worst)
    assert _ratio(worst) <= 1.0, worst


@pytest.mark.gpu
def test_policy_rollout_with_controller_across_the_launch_split():
    """PID at 440/44 Hz (B = 22, obs 78 floats) allows 84 ticks per launch: T = 100 takes two launches, and a second rollout()
    continues from the first one's last observation."""
    from gym_pybullet_drones_b200.policy import MlpPolicy
    E, D, T, T2 = 90, 2, 100, 20
    kw = dict(pyb_freq=440, ctrl_freq=44)
    env, twin = _make("MultiHoverAviary", "PID", D, E, **kw), _make("MultiHoverAviary", "PID", D, E, **kw)
    tmax = env._lib.qs_rollout_max_ticks(env._act_type(), env._B, D)
    assert 0 < tmax < T, tmax
    pol = MlpPolicy.random(D * env._obs_dim, D * 3, seed=8, critic=True, log_std=-1.0)
    ref = PolicyRef(pol)
    g = torch.Generator(device="cuda").manual_seed(4)
    noise, noise2 = torch.randn((T, E, D * 3), device="cuda", generator=g), torch.randn((T2, E, D * 3), device="cuda", generator=g)
    obs0 = env.reset()[0].clone()
    twin.reset()
    sc = np.random.default_rng(2).integers(3300, 3520, E)        # 8 s at 440 Hz = 3520 physics steps
    env.set_state(step_counter=sc); twin.set_state(step_counter=sc)
    out = env.rollout(policy=pol, noise=noise)
    twin_out = twin.rollout(actions=out["actions"].clamp(-1, 1))
    torch.cuda.synchronize()
    _assert_same_physics(out, twin_out, env, twin)
    assert int((out["terminated"] | out["truncated"]).sum()) > 0
    worst = _teacher_forced(ref, obs0, out, noise)
    last = out["obs"][-1].clone()
    out2 = env.rollout(policy=pol, noise=noise2)
    twin_out2 = twin.rollout(actions=out2["actions"].clamp(-1, 1))
    torch.cuda.synchronize()
    _assert_same_physics(out2, twin_out2, env, twin)
    w2 = _teacher_forced(ref, last, out2, noise2)
    worst = {k: max(v, w2[k]) for k, v in worst.items()}
    _report("pid-split-T100+20", worst)
    assert _ratio(worst) <= 1.0, worst


# ---------------------------------------------------------------------------------------------------------------
# the float64 oracle: one case per new family, at the tolerances of test_gpu_configs.py's matrix (rows 13-16); the rates are
# the rollout's (rows 13, 14 and 16 have observations too wide for its shared-memory window), models and modes are the rows'
# ---------------------------------------------------------------------------------------------------------------
# (name, kind, D, model, pyb, ctrl, act, E, ticks, teacher-forced, tol, options)
ORACLE_CASES = [
    ("pid", "hover", 1, "cf2p", 240, 30, "pid", 256, 40, True, 1e-7, {}),
    ("vel", "multihover", 2, "cf2p", 240, 30, "vel", 128, 60, True, RTOL, {}),
    ("one_d_pid", "hover", 1, "cf2x", 480, 60, "one_d_pid", 256, 60, False, RTOL, {}),
    ("dynplus", "multihover", 4, "racer", 240, 30, "rpm", 64, 60, False, 1e-7, {"physics": "PYB_GND_DRAG_DW", "xyzs": _STACK4}),
]


def _small_policy(in_dim, out_dim, seed, scale):
    """A random actor whose means stay within about +-scale, with std e^-3: gentle actions keep the free-running rows
    non-chaotic over the whole replay (test_gpu_configs.py scales row 16's actions by 0.3 for the same reason)."""
    from gym_pybullet_drones_b200.policy import MlpPolicy
    base = MlpPolicy.random(in_dim, out_dim, seed=seed, critic=True, log_std=-3.0, device="cpu")
    actor = [(w, b) for w, b in base.actor]
    actor[2] = (actor[2][0] * scale, actor[2][1] * scale)
    return MlpPolicy(actor, base.log_std, base.critic)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ORACLE_CASES, ids=[c[0] for c in ORACLE_CASES])
def test_policy_rollout_vs_oracle(case):
    from test_gpu_configs import _force_from_snapshot, _snapshot, _state_ratio, make_env, make_oracle
    from test_gpu_parity import OBS_TOL, _borderline, _report_borderline, state_of
    name, kind, D, model, pyb, ctrl, act, E, T, teacher, tol, opts = case
    kw = {"initial_xyzs": opts["xyzs"]} if "xyzs" in opts else {}
    env = make_env(kind, D, model, pyb, ctrl, act, E, physics=opts.get("physics", "DYN"), **kw)
    ora = make_oracle(kind, D, model, pyb, ctrl, act, E, effects=7 if "physics" in opts else 0, **kw)
    A = env._A
    pol = _small_policy(D * env._obs_dim, D * A, seed=21, scale=0.3 if "physics" in opts else 1.0)
    noise = torch.randn((T, E, D * A), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    obs, _ = env.reset()
    assert relerr(obs.cpu().numpy(), ora.reset()) < 1e-6
    worst = 0.0

    def compare(t, obs, rew, term, trunc):
        o_obs, o_rew, o_term, o_trunc = ora.step(out_actions[t])
        r = max(relerr(rew.cpu().numpy(), o_rew) / max(tol, OBS_TOL), relerr(obs.cpu().numpy(), o_obs) / max(tol, OBS_TOL))
        assert np.array_equal(term.cpu().numpy(), o_term), t
        clear = ~_borderline(ora, tol)
        assert np.array_equal(trunc.cpu().numpy()[clear], o_trunc[clear]), t
        return r

    if teacher:
        # one launch per tick, the device forced onto the oracle's state before each (the matrix's teacher forcing)
        out_actions = []
        for t in range(T):
            if t > 0:
                _force_from_snapshot(env, _snapshot(ora))
            out = env.rollout(policy=pol, noise=noise[t:t + 1])
            out_actions.append(out["actions"][0].clamp(-1, 1).cpu().numpy())
            r = compare(t, out["obs"][0], out["rewards"][0], out["terminated"][0], out["truncated"][0])
            r = max(r, _state_ratio(state_of(env), ora, tol))
            assert r <= 1.0, (name, t, r)
            worst = max(worst, r)
    else:
        # one launch for all ticks: every observation and reward on the way, the state at the end
        out = env.rollout(policy=pol, noise=noise)
        out_actions = out["actions"].clamp(-1, 1).cpu().numpy()
        for t in range(T):
            r = compare(t, out["obs"][t], out["rewards"][t], out["terminated"][t], out["truncated"][t])
            assert r <= 1.0, (name, t, r)
            worst = max(worst, r)
        r = _state_ratio(state_of(env), ora, tol)
        assert r <= 1.0, (name, "final state", r)
        worst = max(worst, r)
    _report_borderline("policy " + name)
    _report("oracle-" + name, {"state": worst})


# ---------------------------------------------------------------------------------------------------------------
# refusals (no GPU): what stays unsupported comes back as QS_ERR_* with a message before any launch
# ---------------------------------------------------------------------------------------------------------------
def _rollout_call(lib, act_type, D, effects, pol, st_extra=()):
    from gym_pybullet_drones_b200 import _native as N
    buf = (C.c_char * 8192)()
    base = (C.addressof(buf) + 63) & ~63
    P, st, rio = N.QsParams(), N.QsState(), N.QsRolloutIO()
    st.planes, st.step_counter, st.target_pos, st.pid, st.last_rpm = base, base + 2048, base + 1024, base + 3072, base + 4096
    rio.obs_init, rio.obs, rio.reward, rio.terminated, rio.truncated = base + 512, base + 768, base + 1280, base + 1536, base + 1600
    rio.T, rio.act_buffer_size = 4, 15
    rio.policy = C.addressof(pol)
    rc = lib.qs_rollout(C.byref(P), C.byref(st), C.byref(rio), act_type, 1, 4, D, 8, effects, 0, None)
    return rc, lib.qs_last_error().decode()


def _complete_policy(in_dim, out_dim, buf):
    """A QsPolicy whose arrays all point into `buf` (16-byte aligned, never read: the calls below are refused first)."""
    from gym_pybullet_drones_b200 import _native as N
    q = N.QsPolicy()
    base = (C.addressof(buf) + 63) & ~63
    for f in ("w1", "b1", "w2", "b2", "w3", "b3", "log_std"):
        setattr(q, f, base)
    q.in_dim, q.out_dim, q.nt3 = in_dim, out_dim, 1 if out_dim <= 8 else (2 if out_dim <= 16 else 4)
    return q


@pytest.mark.parametrize("effects,what", [(3, "GND|DRAG"), (5, "GND|DW"), (6, "DRAG|DW")])
def test_policy_refuses_effect_sets_the_envs_cannot_produce(effects, what):
    from gym_pybullet_drones_b200 import _native as N
    lib = N.lib()
    buf = (C.c_char * 256)()
    pol = _complete_policy(2 * 57, 2 * 3, buf)
    rc, msg = _rollout_call(lib, N.ACT_PID, 2, effects, pol)
    assert rc == -5 and what in msg and "policy" in msg and msg.startswith("qs_rollout: "), (rc, msg)


def test_policy_refusals_before_launch():
    """The checks that remain for the new variants: more than 64 drones per aviary, actions and a policy at once, widths."""
    from gym_pybullet_drones_b200 import _native as N
    lib = N.lib()
    buf = (C.c_char * 256)()
    # PID, D = 2: obs 12 + 15 * 3 = 57
    rc, msg = _rollout_call(lib, N.ACT_PID, 2, 7, _complete_policy(2 * 57, 2 * 4, buf))
    assert rc == -3 and "in_dim/out_dim" in msg and msg.startswith("qs_rollout: "), (rc, msg)
    rc, msg = _rollout_call(lib, N.ACT_ONE_D_PID, 65, 0, _complete_policy(65 * 27, 65, buf))
    assert rc == -5 and "drones_per_env <= 64" in msg and msg.startswith("qs_rollout: "), (rc, msg)
    pol = N.QsPolicy()                                   # empty: NULL weights
    rc, msg = _rollout_call(lib, N.ACT_VEL, 2, 4, pol)
    assert rc == -1 and "policy" in msg and msg.startswith("qs_rollout: "), (rc, msg)


@pytest.mark.gpu
def test_env_rollout_reports_a_refused_policy_configuration():
    """An effect set the Physics enum cannot produce (forced onto the env here) makes rollout(policy=...) raise ValueError
    naming it, before anything is launched."""
    from gym_pybullet_drones_b200 import _native as N
    from gym_pybullet_drones_b200.policy import MlpPolicy
    env = _make("MultiHoverAviary", "PID", 2, 8, "PYB_GND_DRAG_DW")
    env.reset()
    env._effects = N.EFFECT_GND | N.EFFECT_DW
    pol = MlpPolicy.random(2 * env._obs_dim, 2 * 3, seed=1)
    with pytest.raises(ValueError, match=r"GND\|DW"):
        env.rollout(policy=pol, num_steps=2)
