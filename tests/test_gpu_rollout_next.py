"""rollout() under next-step autoreset (gymnasium >= 1.0's default): an aviary that finishes at tick k is reset by tick k+1, which
ignores its action and leaves its action history unshifted.

Episodes start near their time limit (set_state(step_counter=...)), so aviaries finish and are reset inside the rollout; every
case asserts that resets happened.
* Action rollouts: a twin env steps the same actions one tick at a time; obs, rewards and flags are its step() results bit for
  bit, out["autoreset"] is its pending latch before each step, and afterwards the planes, step counters, latch, PID state,
  last RPMs and current observation are the twin's.  The launch split carries the latch across launches, and a rollout
  starts from, and leaves, a latch that step() honours.
* Policy rollouts: the physics equals an action twin fed out["actions"].clamp(-1, 1); log_probs / values are teacher-forced
  against the float64 PolicyRef; on the reset ticks, values[k+1] is the critic on the terminal observation obs[k].
* The float64 oracle: next-step autoreset with drag, through step() and through rollout(), as the manual reset loop of
  test_gpu_parity.py's next-step test; the reset tick zeroes last_clipped_action like the reference's reset().
* Refusals at the C ABI without a GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

from qs_testlib import PolicyRef, relerr
from test_gpu_rollout_final import _STACK4, _actions, _bits, _pair

OBS_TOL = 2e-6          # test_gpu_parity.py: float32 cast of the observation + float32 atan2f/asinf


def _state(env):
    out = dict(planes=env._planes, last_rpm=env._last_rpm, step_counter=env._step_counter, pending=env._pending,
               obs_buf=env._obs_buf[env._cur])
    if env._pid is not None:
        out["pid"] = env._pid
    return out


def _assert_same_state(env, twin):
    sa, sb = _state(env), _state(twin)
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k


def _replay(out, twin, actions):
    """Steps the twin through `actions` ([T, E, D, A], CUDA), checking the rollout's outputs tick by tick.  Returns the number
    of reset ticks (aviaries x ticks)."""
    n_reset = 0
    for k in range(actions.shape[0]):
        pending = twin._pending.bool()
        obs, rew, term, trunc, _ = twin.step(actions[k].contiguous())
        assert torch.equal(out["autoreset"][k], pending), k
        assert torch.equal(_bits(obs), _bits(out["obs"][k])), k
        assert torch.equal(_bits(rew), _bits(out["rewards"][k])), k
        assert torch.equal(term, out["terminated"][k]) and torch.equal(trunc, out["truncated"][k]), k
        assert not bool((out["rewards"][k][pending] != 0).any() or (term | trunc)[pending].any()), k
        n_reset += int(pending.sum())
    return n_reset


# (name, cls, act, D, E, physics, T, options)
ACTION_CASES = [
    ("rpm-multi2", "MultiHoverAviary", "RPM", 2, 300, "DYN", 12, {}),
    ("one_d_rpm-hover", "HoverAviary", "ONE_D_RPM", 1, 300, "DYN", 12, {}),
    ("pid-clears-multi2", "MultiHoverAviary", "PID", 2, 300, "DYN", 12,
     {"autoreset_clears_controllers": True, "autoreset_clears_action_buffer": True}),
    ("vel-hover", "HoverAviary", "VEL", 1, 300, "DYN", 12, {}),
    ("one_d_pid-multi4", "MultiHoverAviary", "ONE_D_PID", 4, 100, "DYN", 12, {}),
    ("rpm-all-stack4", "MultiHoverAviary", "RPM", 4, 100, "PYB_GND_DRAG_DW", 12, {"initial_xyzs": _STACK4}),
    ("rpm-drag-multi2", "MultiHoverAviary", "RPM", 2, 300, "PYB_DRAG", 12, {}),
    ("rpm-phys-multi2", "MultiHoverAviary", "RPM", 2, 300, "DYN", 12, {"table": 91}),
    ("rpm-tables-multi2", "MultiHoverAviary", "RPM", 2, 300, "DYN", 12, {"initial_xyzs": "per-env"}),
]


def _options(opts, E, D):
    opts = dict(opts, autoreset="next_step")
    if isinstance(opts.get("initial_xyzs"), str):          # per-aviary pose tables (QsState.tables_per_env)
        rng = np.random.default_rng(12)
        xyz = np.stack([rng.uniform(-0.5, 0.5, (E, D)), rng.uniform(-0.5, 0.5, (E, D)), rng.uniform(0.05, 0.6, (E, D))], axis=-1)
        opts["initial_xyzs"] = xyz
    return opts


@pytest.mark.gpu
@pytest.mark.parametrize("case", ACTION_CASES, ids=[c[0] for c in ACTION_CASES])
def test_action_rollout_equals_step(case):
    name, cls, act, D, E, physics, T, opts = case
    sc = np.random.default_rng(3).integers(1880, 1960, E)              # 8 s at 240 Hz = 1920 physics steps
    env, twin, _ = _pair(cls, act, D, E, physics, _options(opts, E, D), sc)
    assert env._tables_per_env == isinstance(opts.get("initial_xyzs"), str)
    actions = _actions(act, T, E, D, env._A, seed=5)
    out = env.rollout(actions=actions)
    assert out["autoreset"].shape == (T, E) and out["autoreset"].dtype == torch.bool
    assert "final_obs" not in out and "final_values" not in out
    assert _replay(out, twin, actions) > 0
    _assert_same_state(env, twin)
    if opts.get("autoreset_clears_action_buffer"):
        assert bool((out["obs"][out["autoreset"]][..., 12:] == 0).all())


@pytest.mark.gpu
def test_latch_across_the_launch_split_and_step():
    """PID at 440/44 Hz allows 84 ticks per launch: T = 100 takes two launches.  One group of aviaries times out on tick 83, the
    last tick of the first launch, so its reset is the first tick of the second (8 s = 3520 physics steps, 10 per tick).  A step()
    before the rollout leaves another group pending, and a third group finishes on the last tick, which the step() after the
    rollout resets."""
    E, D, T = 90, 2, 100
    kw = dict(pyb_freq=440, ctrl_freq=44)
    sc = np.random.default_rng(4).integers(3300, 3520, E)
    sc[:12] = 2700 - 10                                    # after the first step(): 2700, truncated at tick 83
    sc[12:24] = 2540 - 10                                  # truncated at tick 99
    sc[24:36] = 3525                                       # truncated by the first step(): pending at tick 0
    env, twin, _ = _pair("MultiHoverAviary", "PID", D, E, "DYN", dict(kw, autoreset="next_step"), sc)
    tmax = env._lib.qs_rollout_max_ticks(env._act_type(), env._B, D)
    assert tmax == 84, tmax
    # PID targets at the drones' initial positions: they hover, so only the time-outs end episodes, at the ticks set up above
    home = torch.as_tensor(np.broadcast_to(env.INIT_XYZS, (E, D, 3)), dtype=torch.float32, device="cuda")
    actions = (home + 0.01 * (_actions("RPM", T + 2, E, D, 3, seed=6))).clamp(-1, 1).contiguous()
    for e in (env, twin):
        e.step(actions[0].contiguous())
    _assert_same_state(env, twin)
    assert bool(env._pending[24:36].bool().any())
    out = env.rollout(actions=actions[1:T + 1])
    assert bool(out["autoreset"][0, 24:36].any())
    assert bool(out["truncated"][tmax - 1, :12].any()) and bool(out["autoreset"][tmax, :12].any())
    assert bool(out["truncated"][T - 1, 12:24].any())
    assert _replay(out, twin, actions[1:T + 1]) > 0
    _assert_same_state(env, twin)
    pending = env._pending.bool().clone()
    assert bool(pending[12:24].any())
    r1, r2 = env.step(actions[T + 1].contiguous()), twin.step(actions[T + 1].contiguous())
    for a, b in zip(r1[:4], r2[:4]):
        assert torch.equal(_bits(a.float()), _bits(b.float()))
    assert bool((r1[1][pending] == 0).all())
    _assert_same_state(env, twin)


# (name, cls, act, D, E, physics, T, options)
POLICY_CASES = [
    ("rpm-multi2", "MultiHoverAviary", "RPM", 2, 300, "DYN", 10, {}),
    ("pid-clears-multi2", "MultiHoverAviary", "PID", 2, 300, "DYN", 10,
     {"autoreset_clears_controllers": True, "autoreset_clears_action_buffer": True}),
    ("rpm-all-stack4", "MultiHoverAviary", "RPM", 4, 100, "PYB_GND_DRAG_DW", 10, {"initial_xyzs": _STACK4}),
    # physics and latch only: the reference's 1/dz^2 downwash throws some drones to observations of 1e9-1e10 here, far past the
    # fp16 split's saturation, and the teacher-forced check then reached 1.2 x its tolerance (test_gpu_policy_actions.py checks the
    # network for this configuration)
    ("pid-all-multi2", "MultiHoverAviary", "PID", 2, 300, "PYB_GND_DRAG_DW", 10, {"teacher_forced": False}),
]


def _bootstrap_ratio(ref, out):
    """Worst |values[k+1] - float64 critic(obs[k])| / tolerance over the aviaries reset at k+1, with PolicyRef's criterion; the
    fp32 yardstick is taken over the whole tick's observations (the batch `values` is computed on).  Returns (ratio, count)."""
    worst, n = 0.0, 0
    for k in range(out["obs"].shape[0] - 1):
        m = out["autoreset"][k + 1].cpu().numpy()
        if not m.any():
            continue
        x = PolicyRef.saturate(ref.flat(out["obs"][k])).astype(np.float32)
        v, tol = ref.tolerance(ref.critic, ref.floor_critic, x)
        got = out["values"][k + 1].cpu().numpy().astype(np.float64)
        worst = max(worst, float((np.abs(got[m] - v[m, 0]) / tol[m, 0]).max()))
        n += int(m.sum())
    return worst, n


@pytest.mark.gpu
@pytest.mark.parametrize("case", POLICY_CASES, ids=[c[0] for c in POLICY_CASES])
def test_policy_rollout(case):
    from gym_pybullet_drones_b200.policy import MlpPolicy
    from test_gpu_policy_actions import _ratio, _teacher_forced
    name, cls, act, D, E, physics, T, opts = case
    opts = dict(opts)
    forced = opts.pop("teacher_forced", True)
    sc = np.random.default_rng(6).integers(1880, 1960, E)
    env, twin, obs0 = _pair(cls, act, D, E, physics, _options(opts, E, D), sc)
    A, od = env._A, env._obs_dim
    pol = MlpPolicy.random(D * od, D * A, seed=13 + D + A, critic=True, log_std=-1.0)
    ref = PolicyRef(pol)
    noise = torch.randn((T, E, D * A), device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    out = env.rollout(policy=pol, noise=noise)
    twin_out = twin.rollout(actions=out["actions"].clamp(-1, 1))
    for k in ("obs", "rewards", "terminated", "truncated", "autoreset"):
        assert torch.equal(out[k], twin_out[k]), k
    _assert_same_state(env, twin)
    assert bool(out["autoreset"].any())
    if not forced:
        return
    worst = _teacher_forced(ref, obs0, out, noise)
    assert _ratio(worst) <= 1.0, (name, worst)
    ratio, n = _bootstrap_ratio(ref, out)
    assert n > 0 and ratio <= 1.0, (name, ratio, n)


# ---------------------------------------------------------------------------------------------------------------
# the float64 oracle
# ---------------------------------------------------------------------------------------------------------------
def _oracle_next_step(ora, acts, pending):
    """One tick of the manual next-step loop of test_gpu_parity.py: aviaries that finished last tick are reset now (their action is
    ignored, their buffer untouched; the reset zeroes last_clipped_action).  Returns (obs, reward, term, trunc)."""
    buf_before = [b.copy() for b in ora.action_buffer]
    snap = {f: getattr(ora, f).copy() for f in ("pos", "quat", "vel", "rpy_rates", "ang_v", "rpy", "last_clipped_action")}
    sc = ora.step_counter.copy()
    o_obs, o_rew, o_term, o_trunc = ora.step(acts)
    if pending.any():
        for f, v in snap.items():
            getattr(ora, f)[pending] = v[pending]
        ora.step_counter[pending] = sc[pending]
        for b_new, b_old in zip(ora.action_buffer, buf_before):
            b_new[pending] = b_old[pending]
        o_obs[pending] = ora.reset(mask=pending)[pending]
        o_rew[pending] = 0; o_term[pending] = False; o_trunc[pending] = False
    return o_obs, o_rew, o_term, o_trunc


def _oracle_pair(E):
    from gym_pybullet_drones_b200.envs import HoverAviary
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    from oracle import dyn_oracle as O
    env = HoverAviary(physics=Physics.PYB_DRAG, act=ActionType.RPM, num_envs=E, autoreset="next_step")
    ora = O.OracleAviary("hover", E, 1, act="rpm", effects=O.EFFECT_DRAG)
    env.reset(); ora.reset()
    return env, ora


@pytest.mark.gpu
def test_oracle_step_next_step_with_drag():
    """step() with drag: the tick after a reset reads last_clipped_action = 0 in its drag term, as the reference does after
    reset(), and last_clipped_action reports the zeros."""
    E, T = 256, 200
    acts = np.random.default_rng(79).uniform(-1, 1, (T, E, 1, 4)).astype(np.float32)
    env, ora = _oracle_pair(E)
    pending = np.zeros(E, bool)
    saw = 0
    for t in range(T):
        obs, rew, term, trunc, _ = env.step(torch.from_numpy(acts[t]).cuda())
        o_obs, o_rew, o_term, o_trunc = _oracle_next_step(ora, acts[t], pending)
        if pending.any():
            saw += int(pending.sum())
            assert bool((env.last_clipped_action.cpu().numpy()[pending] == 0).all()), t
        assert relerr(env.last_clipped_action.cpu().numpy(), ora.last_clipped_action) < OBS_TOL, t
        assert relerr(obs.cpu().numpy(), o_obs) < OBS_TOL, t
        assert relerr(rew.cpu().numpy(), o_rew) < OBS_TOL, t
        assert np.array_equal((term | trunc).cpu().numpy(), o_term | o_trunc), t
        pending = o_term | o_trunc
    assert saw > E // 4


@pytest.mark.gpu
def test_oracle_rollout_next_step_with_drag():
    E, T = 256, 200
    acts = np.random.default_rng(80).uniform(-1, 1, (T, E, 1, 4)).astype(np.float32)
    env, ora = _oracle_pair(E)
    out = env.rollout(actions=torch.from_numpy(acts).cuda())
    obs, rew = out["obs"].cpu().numpy(), out["rewards"].cpu().numpy()
    done, autoreset = (out["terminated"] | out["truncated"]).cpu().numpy(), out["autoreset"].cpu().numpy()
    pending = np.zeros(E, bool)
    for t in range(T):
        o_obs, o_rew, o_term, o_trunc = _oracle_next_step(ora, acts[t], pending)
        assert np.array_equal(autoreset[t], pending), t
        assert relerr(obs[t], o_obs) < OBS_TOL, t
        assert relerr(rew[t], o_rew) < OBS_TOL, t
        assert np.array_equal(done[t], o_term | o_trunc), t
        pending = o_term | o_trunc
    assert int(autoreset.sum()) > E // 4
    assert relerr(env.last_clipped_action.cpu().numpy(), ora.last_clipped_action) < OBS_TOL
    assert np.array_equal(env._pending.bool().cpu().numpy(), pending)


# ---------------------------------------------------------------------------------------------------------------
# refusals at the C ABI (no GPU): returned before any launch
# ---------------------------------------------------------------------------------------------------------------
def _call(flags, pending=True, final_obs=False, final_values=False, policy=False):
    """qs_rollout on host buffers (as test_gpu_rollout_final._rollout_call, with the pending_reset latch): refused before any
    launch, so no GPU is needed."""
    from gym_pybullet_drones_b200 import _native as N
    lib = N.lib()
    buf = (C.c_char * 16384)()
    base = (C.addressof(buf) + 63) & ~63
    P, st, rio = N.QsParams(), N.QsState(), N.QsRolloutIO()
    st.planes, st.step_counter, st.target_pos, st.last_rpm = base, base + 2048, base + 1024, base + 4096
    st.init_pos, st.init_quat = base + 5120, base + 5376
    st.pending_reset = base + 5632 if pending else None
    rio.obs_init, rio.obs, rio.reward, rio.terminated, rio.truncated = base + 512, base + 768, base + 1280, base + 1536, base + 1600
    rio.T, rio.act_buffer_size = 4, 15
    rio.final_obs = base + 6144 if final_obs else None
    rio.final_values = base + 12288 if final_values else None
    q = N.QsPolicy()
    for f in ("w1", "b1", "w2", "b2", "w3", "b3", "log_std", "vw1", "vb1", "vw2", "vb2", "vw3", "vb3"):
        setattr(q, f, base + 8192)
    q.in_dim, q.out_dim, q.nt3 = 2 * 72, 2 * 4, 1
    rio.policy = C.addressof(q) if policy else None
    rc = lib.qs_rollout(C.byref(P), C.byref(st), C.byref(rio), N.ACT_RPM, N.TASK_HOVER, 4, 2, 8, 0, flags, None)
    return rc, lib.qs_last_error().decode()


def test_next_step_refusals():
    from gym_pybullet_drones_b200 import _native as N
    nxt, same = N.FLAG_AUTORESET_NEXT_STEP, N.FLAG_AUTORESET_SAME_STEP
    rc, msg = _call(nxt, pending=False)
    assert rc == -1 and "pending_reset" in msg, (rc, msg)
    rc, msg = _call(nxt | same)
    assert rc == -4 and "two autoreset modes" in msg, (rc, msg)
    for kw in (dict(final_obs=True), dict(final_values=True, policy=True), dict(final_obs=True, final_values=True, policy=True)):
        rc, msg = _call(nxt, **kw)
        assert rc == -5 and "SAME_STEP" in msg, (kw, rc, msg)
