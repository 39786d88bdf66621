"""The on-device policy of qs_rollout (rollout_kernel<0, false, true>: SB3-MlpPolicy-shaped actor and critic on the tensor cores
with a two-term fp16 split of both operands) against the float64 reference tests/qs_testlib.PolicyRef, at every shape the
kernel accepts.

Two independent checks per rollout:
* MLP, teacher-forced per tick: the reference evaluates the kernel's own observation before tick t (`out["obs"][t-1]`, or the
  env's observation at the start), so trajectory drift can neither hide nor cause an MLP error.  Actions, log-probabilities and
  values must meet PolicyRef's criterion (worst error / tolerance <= 1).
* Physics, bit for bit: a twin env replays the applied actions `out["actions"].clamp(-1, 1)` through the action path of the
  same kernel from the same reset; observations, rewards, flags, state planes, last RPMs and step counters are equal.

Set QS_POLICY_REPORT=1 to print every case's worst error / tolerance."""
import copy
import os

import numpy as np
import pytest
import torch

from qs_testlib import PolicyRef

pytestmark = pytest.mark.gpu


def _report(name, r):
    if os.environ.get("QS_POLICY_REPORT"):
        print("policy-ratio %-40s %s" % (name, " ".join("%s=%.3g" % kv for kv in sorted(r.items()))))


def _envs(cls, act, D, E, autoreset="same_step"):
    import gym_pybullet_drones_b200.envs as envs
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    kw = dict(physics=Physics.DYN, act=ActionType[act], num_envs=E, autoreset=autoreset, track_last_action=True)
    if cls == "MultiHoverAviary":
        kw["num_drones"] = D
    return getattr(envs, cls)(**kw), getattr(envs, cls)(**kw)


def _state(env):
    return [env._planes.clone(), env._last_rpm.clone(), env._step_counter.clone(), env._obs_buf[env._cur].clone()]


def _assert_same_physics(out, twin_out, env, twin):
    for k in ("obs", "rewards", "terminated", "truncated"):
        a, b = out[k], twin_out[k]
        assert a.shape == b.shape and torch.equal(a, b), k
    for name, a, b in zip(("planes", "last_rpm", "step_counter", "obs_buf"), _state(env), _state(twin)):
        assert torch.equal(a, b), name


def _teacher_forced(ref, obs0, out, noise, rows=None):
    """Worst error / tolerance over the ticks of `out`, the reference evaluated on the kernel's observation before each tick
    (restricted to aviaries `rows` if given)."""
    T = out["obs"].shape[0]
    sel = (lambda a: a) if rows is None else (lambda a: a[rows])
    worst = {}
    for t in range(T):
        x = obs0 if t == 0 else out["obs"][t - 1]
        r = ref.check(sel(x), None if noise is None else sel(noise[t]), sel(out["actions"][t]), sel(out["log_probs"][t]),
                      sel(out["values"][t]) if "values" in out else None)
        for k, v in r.items():
            worst[k] = max(worst.get(k, 0.0), v)
    return worst


# (cls, act, D, E, critic, noise, T): E leaves the last CTA partial (a policy CTA holds 64 // D aviaries); D = 3 and 5 leave idle
# threads (63 and 60 drones in a 64-thread CTA); nt3 = 4 for D * A in 17..32; ONE_D_RPM with D = 4, 8, 32 makes in_dim a
# multiple of 4, so layer 1 takes its 128-bit path on every fourth tick (the window slides by one float per tick)
CASES = [
    ("HoverAviary", "ONE_D_RPM", 1, 200, True, True, 10),        # in_dim 27: always the scalar path
    ("HoverAviary", "RPM", 1, 17, False, False, 10),             # 17 aviaries: the second m-tile has one real row
    ("MultiHoverAviary", "RPM", 2, 200, True, True, 10),
    ("MultiHoverAviary", "RPM", 2, 1, True, True, 10),           # a single aviary
    ("MultiHoverAviary", "RPM", 3, 100, True, True, 10),         # 21 aviaries per CTA, nt3 = 2
    ("MultiHoverAviary", "RPM", 4, 50, False, True, 10),         # nt3 = 2
    ("MultiHoverAviary", "RPM", 5, 30, True, True, 10),          # 12 aviaries per CTA, nt3 = 4
    ("MultiHoverAviary", "RPM", 8, 20, True, False, 10),         # out_dim 32, in_dim 576
    ("MultiHoverAviary", "ONE_D_RPM", 2, 70, True, True, 10),
    ("MultiHoverAviary", "ONE_D_RPM", 4, 37, True, True, 12),    # in_dim 108
    ("MultiHoverAviary", "ONE_D_RPM", 8, 19, False, True, 12),   # in_dim 216
    ("MultiHoverAviary", "ONE_D_RPM", 32, 5, True, True, 12),    # in_dim 864, out_dim 32, 2 aviaries per CTA
]


def _case_id(c):
    return "%s-%s-D%d-E%d-%s-%s" % (c[0][:-len("Aviary")], c[1], c[2], c[3], "critic" if c[4] else "actor", "noise" if c[5] else "mean")


@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_policy_rollout_matches_float64_reference(case):
    from gym_pybullet_drones_b200.policy import MlpPolicy
    cls, act, D, E, critic, with_noise, T = case
    env, twin = _envs(cls, act, D, E)
    A, od = env._A, env._obs_dim
    pol = MlpPolicy.random(D * od, D * A, seed=5 + D, critic=critic, log_std=-1.0)
    ref = PolicyRef(pol)
    g = torch.Generator(device="cuda").manual_seed(9)
    noise = torch.randn((T, E, D * A), device="cuda", generator=g) if with_noise else None
    obs0 = env.reset()[0].clone()
    twin.reset()
    # episodes near their time limit, ending at different ticks: the rollout autoresets aviaries on the way
    sc = np.random.default_rng(1).integers(1880, 1960, E)
    env.set_state(step_counter=sc); twin.set_state(step_counter=sc)
    out = env.rollout(policy=pol, noise=noise, num_steps=T)
    assert out["actions"].shape == (T, E, D, A) and out["log_probs"].shape == (T, E) and (("values" in out) == critic)
    twin_out = twin.rollout(actions=out["actions"].clamp(-1, 1))
    torch.cuda.synchronize()
    _assert_same_physics(out, twin_out, env, twin)
    resets = int((out["terminated"] | out["truncated"]).sum())
    assert resets > 0
    worst = _teacher_forced(ref, obs0, out, noise)
    _report(_case_id(case), worst)
    assert max(worst.values()) <= 1.0, worst


def _injected(kind, rng, E, n):
    """[E, n] observation rows of one kind, and the scale of each column's W1 row that keeps the pre-activations O(1)."""
    if kind == "ordinary":
        x = rng.uniform(-1, 1, (E, n))
    elif kind == "large":                                    # positions / velocities of hundreds of metres next to O(1) values
        x = rng.uniform(-1, 1, (E, n))
        x[:, : n // 3] *= rng.uniform(100, 1000, (E, n // 3))
    elif kind == "spanning":                                 # 1e-6 .. 3e4 in the same row, below the fp16 normal range included
        x = np.logspace(-6, np.log10(3e4), n)[None, :] * rng.choice([-1.0, 1.0], (E, n))
        x = x[:, rng.permutation(n)]
    elif kind == "fp16_exact":                               # x_lo' = 0 everywhere
        x = rng.uniform(-300, 300, (E, n)).astype(np.float16).astype(np.float64)
    elif kind == "saturating":                               # a few entries past fp16's range, the rest O(1)
        x = rng.uniform(-1, 1, (E, n))
        big = np.array([65504.0, 65510.0, 65535.0, 65535.984375, 65536.0, 7e4, 1e6, 3e38])
        for e in range(E):
            cols = rng.choice(n, 3, replace=False)
            x[e, cols] = rng.choice(big, 3) * rng.choice([-1.0, 1.0], 3)
    x = x.astype(np.float32)
    scale = 1.0 / np.clip(np.abs(PolicyRef.saturate(x)).max(axis=0), 1.0, 1e3)
    return x, scale


@pytest.mark.parametrize("kind", ["ordinary", "large", "spanning", "fp16_exact", "saturating"])
def test_policy_on_injected_observations(kind):
    """Chosen rows written into the env's current observation buffer after reset(): the policy reads them at tick 0 (the
    physics does not).  W1's rows are scaled so that pre-activations stay in tanh's active range and the inputs' low bits
    matter.  Past fp16's range the kernel sees +-65535.984375 (PolicyRef.OBS_SATURATION), not +-65504 and not the input."""
    from gym_pybullet_drones_b200.policy import MlpPolicy
    E, D = 96, 2
    env, _ = _envs("MultiHoverAviary", "RPM", D, E)
    n = D * env._obs_dim
    rng = np.random.default_rng(11)
    x, scale = _injected(kind, rng, E, n)
    base = MlpPolicy.random(n, D * 4, seed=3, critic=True, log_std=-1.0, device="cpu")
    actor = [(w, b) for w, b in base.actor]
    critic = [(w, b) for w, b in base.critic]
    s = torch.from_numpy(scale.astype(np.float32))[:, None]
    actor[0], critic[0] = (actor[0][0] * s, actor[0][1]), (critic[0][0] * s, critic[0][1])
    pol = MlpPolicy(actor, base.log_std, critic)
    ref = PolicyRef(pol)
    env.reset()
    env._obs_buf[env._cur].view(E, n).copy_(torch.from_numpy(x))
    noise = torch.randn((1, E, D * 4), device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    out = env.rollout(policy=pol, noise=noise)
    torch.cuda.synchronize()
    xs = PolicyRef.saturate(x).astype(np.float32)
    r = ref.check(x, noise[0], out["actions"][0], out["log_probs"][0], out["values"][0], ref_obs=xs)
    _report("injected-" + kind, r)
    assert max(r.values()) <= 1.0, r
    if kind == "saturating":
        # the two other readings of "saturate" are far off: clipping at 65504, and no clipping at all
        for other in (np.clip(x, -65504.0, 65504.0), x):
            o = ref.check(x, noise[0], out["actions"][0], out["log_probs"][0], out["values"][0], ref_obs=other)
            assert o["actions"] > 10 and o["values"] > 10, o


def test_policy_rollout_across_the_launch_split():
    """RPM D = 2 allows 255 ticks per launch (qs_rollout_max_ticks): T = 300 takes two launches, and BaseRLAviary.rollout slices
    noise, actions, log-probs and values at the split.  A second rollout() continues from the first one's last observation."""
    from gym_pybullet_drones_b200.policy import MlpPolicy
    E, D, T, T2 = 100, 2, 300, 20
    env, twin = _envs("MultiHoverAviary", "RPM", D, E)
    assert env._lib.qs_rollout_max_ticks(env._act_type(), env._B, D) == 255
    pol = MlpPolicy.random(D * env._obs_dim, D * 4, seed=8, critic=True, log_std=-1.0)
    ref = PolicyRef(pol)
    g = torch.Generator(device="cuda").manual_seed(4)
    noise = torch.randn((T, E, D * 4), device="cuda", generator=g)
    noise2 = torch.randn((T2, E, D * 4), device="cuda", generator=g)
    obs0 = env.reset()[0].clone()
    twin.reset()
    out = env.rollout(policy=pol, noise=noise)
    twin_out = twin.rollout(actions=out["actions"].clamp(-1, 1))
    torch.cuda.synchronize()
    _assert_same_physics(out, twin_out, env, twin)
    assert int(out["truncated"].sum()) > 0                  # 300 ticks outlast the 240-tick episode
    worst = _teacher_forced(ref, obs0, out, noise)
    last = out["obs"][-1].clone()
    out2 = env.rollout(policy=pol, noise=noise2)
    twin_out2 = twin.rollout(actions=out2["actions"].clamp(-1, 1))
    torch.cuda.synchronize()
    _assert_same_physics(out2, twin_out2, env, twin)
    w2 = _teacher_forced(ref, last, out2, noise2)
    worst = {k: max(v, w2[k]) for k, v in worst.items()}
    _report("split-T300+20", worst)
    assert max(worst.values()) <= 1.0, worst


def test_policy_without_weight_low_parts_fails_the_criterion():
    """Negative control of the weight operand: the packed actor with its lo' half-words zeroed (a valid input: the kernel then
    multiplies by fp16(W)) misses the criterion by more than 10x, while the intact weights meet it on the same observations."""
    from gym_pybullet_drones_b200.policy import MlpPolicy
    E, D, T = 128, 2, 3
    env, _ = _envs("MultiHoverAviary", "RPM", D, E)
    pol = MlpPolicy.random(D * env._obs_dim, D * 4, seed=5, critic=True, log_std=-1.0)
    bad = copy.copy(pol)
    bad._split = dict(pol._split)
    bad._split["actor"] = []
    for w, b in pol._split["actor"]:
        w = w.clone()
        w[..., 2:] = 0                                       # words 2, 3 of every lane: the {b0, b1} pairs of w_lo'
        bad._split["actor"].append((w, b))
    ref = PolicyRef(pol)
    worst = {}
    for name, p in (("intact", pol), ("no_w_lo", bad)):
        obs0 = env.reset()[0].clone()
        out = env.rollout(policy=p, num_steps=T)
        torch.cuda.synchronize()
        worst[name] = _teacher_forced(ref, obs0, out, None)
        _report("weights-" + name, worst[name])
    assert max(worst["intact"].values()) <= 1.0, worst
    assert worst["no_w_lo"]["actions"] > 10 and worst["no_w_lo"]["values"] <= 1.0, worst


def test_fp16_rounded_observation_fails_the_criterion():
    """Negative control of the observation operand, on the host: on observations of a real policy rollout, evaluating the
    reference on fp16(obs) moves it by more than 10x the criterion."""
    from gym_pybullet_drones_b200.policy import MlpPolicy
    E, D, T = 128, 2, 8
    env, _ = _envs("MultiHoverAviary", "RPM", D, E)
    pol = MlpPolicy.random(D * env._obs_dim, D * 4, seed=5, critic=True, log_std=-1.0)
    ref = PolicyRef(pol)
    env.reset()
    out = env.rollout(policy=pol, noise=torch.randn((T, E, D * 4), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1)))
    x = ref.flat(out["obs"][-1])
    mean, raw, lp, v = ref.forward(x.astype(np.float16).astype(np.float32))
    r = ref.check(x, None, raw, lp, v)
    _report("obs-fp16-host", r)
    assert r["actions"] > 10 and r["values"] > 10, r


def test_policy_rollout_full_size():
    """The bench shape: 32 768 aviaries of 2 drones, RPM, with a critic, T = 16.  Physics bit-identical to the twin, the
    reference on a random sample of 512 aviaries in every tick, and a second identical run gives identical bits."""
    from gym_pybullet_drones_b200.policy import MlpPolicy
    E, D, T = 32768, 2, 16
    env, twin = _envs("MultiHoverAviary", "RPM", D, E)
    pol = MlpPolicy.random(D * env._obs_dim, D * 4, seed=12, critic=True, log_std=-1.0)
    ref = PolicyRef(pol)
    noise = torch.randn((T, E, D * 4), device="cuda", generator=torch.Generator(device="cuda").manual_seed(6))
    obs0 = env.reset()[0].clone()
    twin.reset()
    out = env.rollout(policy=pol, noise=noise)
    twin_out = twin.rollout(actions=out["actions"].clamp(-1, 1))
    torch.cuda.synchronize()
    _assert_same_physics(out, twin_out, env, twin)
    rows = torch.from_numpy(np.sort(np.random.default_rng(3).choice(E, 512, replace=False))).cuda()
    worst = _teacher_forced(ref, obs0, out, noise, rows)
    _report("full-E32768-D2-T16", worst)
    assert max(worst.values()) <= 1.0, worst
    first = {k: v.clone() for k, v in out.items()}
    env.reset(options={"reset_action_buffer": True})         # the fresh env's history was zeros too
    again = env.rollout(policy=pol, noise=noise)
    torch.cuda.synchronize()
    for k, v in first.items():
        assert torch.equal(v, again[k]), k
