"""Terminal observations and their critic values from rollout() under same-step autoreset (QsRolloutIO.final_obs / final_values).

Episodes start near their time limit (set_state(step_counter=...)), so aviaries finish inside the rollout; every case asserts
that some did.
* Action rollouts: a twin env steps the same actions one tick at a time; per tick its info["_final_obs"] is the rollout's
  terminated | truncated and its info["final_obs"] rows are the rollout's final_obs rows, bit for bit.
* Policy rollouts: final_obs against the twin fed out["actions"].clamp(-1, 1); final_values teacher-forced against the float64
  PolicyRef critic on the terminal rows, with PolicyRef's criterion.
* Entries of aviaries that did not finish are left untouched; asking for the outputs changes no other output or state.
* Refusals: at the C ABI without a GPU, and as the env's ValueErrors.

Set QS_POLICY_REPORT=1 to print every policy case's worst final_values error / tolerance."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from qs_testlib import PolicyRef

_STACK4 = np.array([[0.0, 0.0, 0.06], [0.05, 0.02, 1.6], [0.1, -0.03, 3.1], [-0.05, 0.05, 4.6]])
_NAN_BITS = 0x7FC0DEAD                                    # a quiet NaN no kernel produces: marks entries that must stay untouched


def _make(cls, act, D, E, physics="DYN", autoreset="same_step", **kw):
    import gym_pybullet_drones_b200.envs as envs
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    args = dict(physics=Physics[physics], act=ActionType[act], num_envs=E, autoreset=autoreset, track_last_action=True, **kw)
    if cls == "MultiHoverAviary":
        args["num_drones"] = D
    return getattr(envs, cls)(**args)


def _pair(cls, act, D, E, physics, opts, sc):
    """Two envs in the same state, episodes near their time limit (`sc`: step counters)."""
    opts = dict(opts)
    table = opts.pop("table", None)
    env, twin = _make(cls, act, D, E, physics, **opts), _make(cls, act, D, E, physics, **opts)
    if table is not None:
        from dyn_params_lib import random_properties
        props = random_properties(env.DRONE_MODEL, E, table)
        env.set_physical_params(**props)
        twin.set_physical_params(**props)
    obs0 = env.reset()[0].clone()
    twin.reset()
    env.set_state(step_counter=sc)
    twin.set_state(step_counter=sc)
    return env, twin, obs0


def _bits(x):
    return x.contiguous().view(torch.int32)


def _nan_filled(shape):
    return torch.full(shape, _NAN_BITS, dtype=torch.int32, device="cuda").view(torch.float32)


def _actions(act, T, E, D, A, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.rand((T, E, D, A), device="cuda", generator=g) * 2 - 1
    if act == "PID":                                     # as test_gpu_api.py: targets around the hover point
        a = a * 0.3 + torch.tensor([0.0, 0.0, 0.8], device="cuda")
    return a.contiguous()


def _replay(out, twin, actions):
    """Steps the twin through `actions` ([T, E, D, A], CUDA) and checks final_obs against its info, tick by tick.  Returns the
    number of finished aviaries."""
    n_fin = 0
    for k in range(actions.shape[0]):
        _, _, term, trunc, info = twin.step(actions[k].contiguous())
        done = out["terminated"][k] | out["truncated"][k]
        assert torch.equal(term, out["terminated"][k]) and torch.equal(trunc, out["truncated"][k]), k
        assert torch.equal(info["_final_obs"], done), k
        assert torch.equal(_bits(info["final_obs"][done]), _bits(out["final_obs"][k][done])), k
        n_fin += int(done.sum())
    return n_fin


# (name, cls, act, D, E, physics, T, options)
ACTION_CASES = [
    ("rpm-multi2", "MultiHoverAviary", "RPM", 2, 300, "DYN", 12, {}),
    ("one_d_rpm-hover", "HoverAviary", "ONE_D_RPM", 1, 300, "DYN", 12, {}),
    ("pid-clears-multi2", "MultiHoverAviary", "PID", 2, 300, "DYN", 12,
     {"autoreset_clears_controllers": True, "autoreset_clears_action_buffer": True}),
    ("rpm-all-stack4", "MultiHoverAviary", "RPM", 4, 100, "PYB_GND_DRAG_DW", 12, {"initial_xyzs": _STACK4}),
    ("rpm-phys-multi2", "MultiHoverAviary", "RPM", 2, 300, "DYN", 12, {"table": 81}),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ACTION_CASES, ids=[c[0] for c in ACTION_CASES])
def test_action_rollout_final_obs_equals_step(case):
    name, cls, act, D, E, physics, T, opts = case
    sc = np.random.default_rng(3).integers(1880, 1960, E)              # 8 s at 240 Hz = 1920 physics steps
    env, twin, _ = _pair(cls, act, D, E, physics, opts, sc)
    actions = _actions(act, T, E, D, env._A, seed=5)
    out = env.rollout(actions=actions, final_obs=True)
    assert out["final_obs"].shape == (T, E, D, env._obs_dim) and out["final_obs"].dtype == torch.float32
    assert _replay(out, twin, actions) > 0
    if opts.get("autoreset_clears_action_buffer"):
        # the terminal row keeps its action history, the reset row that follows it has none
        done = out["terminated"] | out["truncated"]
        assert bool((out["final_obs"][done][..., 12:] != 0).any(dim=-1).all())
        assert bool((out["obs"][done][..., 12:] == 0).all())


@pytest.mark.gpu
def test_action_rollout_final_obs_across_the_launch_split():
    """PID at 440/44 Hz allows 84 ticks per launch: T = 100 takes two launches.  A group of aviaries times out on tick 83, the
    last tick of the first launch (8 s = 3520 physics steps, 10 per tick: 2700 + 830 > 3520 >= 2700 + 820)."""
    E, D, T = 90, 2, 100
    kw = dict(pyb_freq=440, ctrl_freq=44)
    sc = np.random.default_rng(4).integers(3300, 3520, E)
    sc[:12] = 2700
    env, twin, _ = _pair("MultiHoverAviary", "PID", D, E, "DYN", kw, sc)
    tmax = env._lib.qs_rollout_max_ticks(env._act_type(), env._B, D)
    assert tmax == 84, tmax
    actions = _actions("PID", T, E, D, 3, seed=6)
    out = env.rollout(actions=actions, final_obs=True)
    assert bool(out["truncated"][tmax - 1, :12].any())
    assert _replay(out, twin, actions) > 0


@pytest.mark.gpu
def test_entries_of_unfinished_aviaries_are_untouched():
    from gym_pybullet_drones_b200.policy import MlpPolicy
    E, D, T = 200, 2, 10
    sc = np.random.default_rng(5).integers(1880, 1960, E)
    env, _, _ = _pair("MultiHoverAviary", "RPM", D, E, "DYN", {}, sc)
    od = env._obs_dim
    actions = _actions("RPM", T, E, D, 4, seed=7)
    out = dict(obs=torch.empty((T, E, D, od), device="cuda"), actions=actions, rewards=torch.empty((T, E), device="cuda"),
               terminated=torch.empty((T, E), dtype=torch.bool, device="cuda"), truncated=torch.empty((T, E), dtype=torch.bool, device="cuda"),
               final_obs=_nan_filled((T, E, D, od)))
    out = env.rollout(actions=actions, out=out, final_obs=True)
    done = out["terminated"] | out["truncated"]
    assert 0 < int(done.sum()) < done.numel()
    assert bool((_bits(out["final_obs"][~done]) == _NAN_BITS).all())
    assert not bool((_bits(out["final_obs"][done]) == _NAN_BITS).any())
    # the policy rollout: final_obs and final_values
    pol = MlpPolicy.random(D * od, D * 4, seed=3, critic=True, log_std=-1.0)
    noise = torch.randn((T, E, D * 4), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    env.set_state(step_counter=sc)
    out["final_obs"], out["final_values"] = _nan_filled((T, E, D, od)), _nan_filled((T, E))
    out = env.rollout(policy=pol, noise=noise, out=out, final_obs=True, final_values=True)
    done = out["terminated"] | out["truncated"]
    assert 0 < int(done.sum()) < done.numel()
    assert bool((_bits(out["final_obs"][~done]) == _NAN_BITS).all()) and bool((_bits(out["final_values"][~done]) == _NAN_BITS).all())
    assert bool(torch.isfinite(out["final_values"][done]).all())


def _values_ratio(ref, out):
    """Worst |final_values - float64 critic| / tolerance over the terminal rows, the reference evaluated on them as the kernel's
    saturating fp16 split sees them.  The criterion's fp32 yardstick (PolicyRef.tolerance) is taken over a tick's terminal rows
    together with that tick's observations: a batch of the size `values` is checked with, not of the few finished aviaries."""
    worst = 0.0
    for k in range(out["obs"].shape[0]):
        done = (out["terminated"][k] | out["truncated"][k]).cpu().numpy()
        if not done.any():
            continue
        x_fin = ref.flat(out["final_obs"][k].cpu().numpy()[done])
        x = PolicyRef.saturate(np.concatenate([x_fin, ref.flat(out["obs"][k])])).astype(np.float32)
        v, tol = ref.tolerance(ref.critic, ref.floor_critic, x)
        got = out["final_values"][k].cpu().numpy()[done].astype(np.float64)
        worst = max(worst, float((np.abs(got - v[:len(got), 0]) / tol[:len(got), 0]).max()))
    return worst


# (name, cls, act, D, E, physics, T, options): D = 3 leaves the CTAs partial (21 aviaries, 63 of 64 threads)
POLICY_CASES = [
    ("rpm-multi2", "MultiHoverAviary", "RPM", 2, 300, "DYN", 10, {}),
    ("pid-multi2", "MultiHoverAviary", "PID", 2, 300, "DYN", 10, {}),
    ("vel-hover", "HoverAviary", "VEL", 1, 300, "DYN", 10, {}),
    ("one_d_pid-multi4", "MultiHoverAviary", "ONE_D_PID", 4, 100, "DYN", 12, {}),
    ("pid-multi3", "MultiHoverAviary", "PID", 3, 200, "DYN", 10, {}),
    ("rpm-dw-stack4", "MultiHoverAviary", "RPM", 4, 100, "PYB_DW", 10, {"initial_xyzs": _STACK4}),
    ("pid-all-multi2", "MultiHoverAviary", "PID", 2, 300, "PYB_GND_DRAG_DW", 10, {}),
    ("pid-clears-phys-multi2", "MultiHoverAviary", "PID", 2, 300, "DYN", 10,
     {"autoreset_clears_controllers": True, "autoreset_clears_action_buffer": True, "table": 82}),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", POLICY_CASES, ids=[c[0] for c in POLICY_CASES])
def test_policy_rollout_final_obs_and_values(case):
    from gym_pybullet_drones_b200.policy import MlpPolicy
    name, cls, act, D, E, physics, T, opts = case
    sc = np.random.default_rng(6).integers(1880, 1960, E)
    env, twin, _ = _pair(cls, act, D, E, physics, opts, sc)
    A, od = env._A, env._obs_dim
    pol = MlpPolicy.random(D * od, D * A, seed=11 + D + A, critic=True, log_std=-1.0)
    noise = torch.randn((T, E, D * A), device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    out = env.rollout(policy=pol, noise=noise, final_obs=True, final_values=True)
    assert out["final_values"].shape == (T, E) and out["final_values"].dtype == torch.float32
    assert _replay(out, twin, out["actions"].clamp(-1, 1)) > 0
    ratio = _values_ratio(PolicyRef(pol), out)
    if os.environ.get("QS_POLICY_REPORT"):
        print("final-values-ratio %-28s %.3g" % (name, ratio))
    assert ratio <= 1.0, (name, ratio)


@pytest.mark.gpu
@pytest.mark.parametrize("policy", [False, True], ids=["actions", "policy"])
def test_final_outputs_have_no_side_effects(policy):
    from gym_pybullet_drones_b200.policy import MlpPolicy
    E, D, T = 300, 2, 12
    sc = np.random.default_rng(7).integers(1880, 1960, E)
    env, twin, _ = _pair("MultiHoverAviary", "PID", D, E, "DYN", {}, sc)
    if policy:
        pol = MlpPolicy.random(D * env._obs_dim, D * 3, seed=4, critic=True, log_std=-1.0)
        noise = torch.randn((T, E, D * 3), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
        out = env.rollout(policy=pol, noise=noise, final_obs=True, final_values=True)
        ref = twin.rollout(policy=pol, noise=noise)
        keys = ("obs", "actions", "log_probs", "values", "rewards", "terminated", "truncated")
    else:
        actions = _actions("PID", T, E, D, 3, seed=8)
        out, ref = env.rollout(actions=actions, final_obs=True), twin.rollout(actions=actions)
        keys = ("obs", "rewards", "terminated", "truncated")
    assert int((out["terminated"] | out["truncated"]).sum()) > 0
    for k in keys:
        assert out[k].shape == ref[k].shape and torch.equal(_bits(out[k].float()), _bits(ref[k].float())), k
    for a, b in ((env._planes, twin._planes), (env._last_rpm, twin._last_rpm), (env._pid, twin._pid), (env._step_counter, twin._step_counter),
                 (env._obs_buf[env._cur], twin._obs_buf[twin._cur])):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_env_rollout_refuses_final_outputs_it_cannot_produce():
    from gym_pybullet_drones_b200.policy import MlpPolicy
    env = _make("MultiHoverAviary", "RPM", 2, 8, autoreset="disabled")
    env.reset()
    with pytest.raises(ValueError, match="same_step"):
        env.rollout(num_steps=2, final_obs=True)
    env = _make("MultiHoverAviary", "RPM", 2, 8)
    env.reset()
    with pytest.raises(ValueError, match="critic"):
        env.rollout(num_steps=2, final_values=True)
    actor_only = MlpPolicy.random(2 * env._obs_dim, 2 * 4, seed=1, critic=False)
    with pytest.raises(ValueError, match="critic"):
        env.rollout(policy=actor_only, num_steps=2, final_values=True)


# ---------------------------------------------------------------------------------------------------------------
# refusals at the C ABI (no GPU): returned before any launch
# ---------------------------------------------------------------------------------------------------------------
def _rollout_call(flags, final_obs=False, final_values=False, critic=False, policy=True):
    from gym_pybullet_drones_b200 import _native as N
    lib = N.lib()
    buf = (C.c_char * 16384)()
    base = (C.addressof(buf) + 63) & ~63
    P, st, rio = N.QsParams(), N.QsState(), N.QsRolloutIO()
    st.planes, st.step_counter, st.target_pos, st.last_rpm = base, base + 2048, base + 1024, base + 4096
    st.init_pos, st.init_quat = base + 5120, base + 5376
    rio.obs_init, rio.obs, rio.reward, rio.terminated, rio.truncated = base + 512, base + 768, base + 1280, base + 1536, base + 1600
    rio.T, rio.act_buffer_size = 4, 15
    rio.final_obs = base + 6144 if final_obs else None
    rio.final_values = base + 12288 if final_values else None
    q = N.QsPolicy()
    for f in ("w1", "b1", "w2", "b2", "w3", "b3", "log_std") + (("vw1", "vb1", "vw2", "vb2", "vw3", "vb3") if critic else ()):
        setattr(q, f, base + 8192)
    q.in_dim, q.out_dim, q.nt3 = 2 * 72, 2 * 4, 1
    rio.policy = C.addressof(q) if policy else None
    rc = lib.qs_rollout(C.byref(P), C.byref(st), C.byref(rio), N.ACT_RPM, N.TASK_HOVER, 4, 2, 8, 0, flags, None)
    return rc, lib.qs_last_error().decode()


def test_final_outputs_refused_without_same_step_autoreset():
    for kw in (dict(final_obs=True), dict(final_values=True, critic=True), dict(final_obs=True, policy=False)):
        rc, msg = _rollout_call(0, **kw)
        assert rc == -5 and "SAME_STEP" in msg, (kw, rc, msg)


def test_final_values_refused_without_a_critic():
    from gym_pybullet_drones_b200 import _native as N
    same_step = N.FLAG_AUTORESET_SAME_STEP
    rc, msg = _rollout_call(same_step, final_values=True, critic=False)
    assert rc == -1 and "critic" in msg, (rc, msg)
    rc, msg = _rollout_call(same_step, final_obs=True, final_values=True, policy=False)
    assert rc == -1 and "critic" in msg, (rc, msg)
