"""The on-device policy with any supported SB3 net_arch (qs_rollout_mlp: rollout_mlp_kernel<EFF, PIDACT, PHYS, MODE>).

Every case runs the two checks of test_gpu_policy_actions.py, with same-step autoresets inside the rollout:
* network, teacher-forced per tick against the float64 tests/mlp_ref.MlpRef (PolicyRef's criterion generalised to any depth and
  activation): worst error / tolerance <= 1;
* physics, bit for bit that of a twin env fed `out["actions"].clamp(-1, 1)` through the action rollout.
Then: a [64, 64] Tanh policy forced through the general path gives the bits of the classic one; terminal values under both
autoreset modes; the launch split; the bench shape at the widest accepted width; two negative controls.

Set QS_POLICY_REPORT=1 to print every case's worst error / tolerance."""
import copy

import numpy as np
import pytest
import torch

from mlp_ref import MlpRef
from qs_testlib import PolicyRef
from test_gpu_policy_actions import _STACK4, _assert_same_physics, _make, _physical_table, _ratio, _report, _teacher_forced

PI2 = dict(pi=[128, 64], vf=[256, 256])

# (name, act, D, E, physics, T, net_arch, activation, noise, options): E leaves the last 64-drone CTA partial
CASES = [
    ("relu64-rpm-d2", "RPM", 2, 150, "DYN", 10, [64, 64], "relu", True, {}),
    ("tanh128-rpm-d1", "RPM", 1, 200, "DYN", 10, [128, 128], "tanh", False, {}),
    ("relu256-rpm-d4", "RPM", 4, 50, "DYN", 10, [256, 256], "relu", True, {}),
    ("tanh100-one_d_rpm-d1", "ONE_D_RPM", 1, 200, "DYN", 12, [100], "tanh", True, {}),
    ("deep4-one_d_rpm-d3", "ONE_D_RPM", 3, 100, "DYN", 12, [256, 128, 64, 32], "tanh", False, {}),
    ("split-rpm-d2", "RPM", 2, 150, "DYN", 10, PI2, "relu", True, {}),
    ("deep4-pid-d2", "PID", 2, 150, "DYN", 10, [256, 128, 64, 32], "tanh", True, {}),
    ("relu128-vel-d2", "VEL", 2, 150, "DYN", 10, [128, 128], "relu", True, {}),
    ("split-one_d_pid-d4", "ONE_D_PID", 4, 37, "DYN", 12, PI2, "relu", True, {}),
    ("tanh128-gnd", "RPM", 2, 150, "PYB_GND", 10, [128, 128], "tanh", True, {}),
    ("tanh128-drag", "RPM", 2, 150, "PYB_DRAG", 10, [128, 128], "tanh", True, {}),
    ("relu256-dw-stack4", "RPM", 4, 50, "PYB_DW", 10, [256, 256], "relu", True, {"initial_xyzs": _STACK4}),
    ("split-all-stack4", "RPM", 4, 50, "PYB_GND_DRAG_DW", 10, PI2, "relu", True, {"initial_xyzs": _STACK4}),
    ("deep4-pid-phys", "PID", 2, 150, "DYN", 10, [256, 128, 64, 32], "tanh", True, {"table": 71}),
]


def _policy(env, D, arch, activation, seed):
    from gym_pybullet_drones_b200.policy import MlpPolicy
    return MlpPolicy.random(D * env._obs_dim, D * env._A, seed=seed, critic=True, log_std=-1.0, net_arch=arch, activation=activation)


def _pair(act, D, E, physics="DYN", autoreset="same_step", **opts):
    table = opts.pop("table", None)
    env, twin = _make("MultiHoverAviary", act, D, E, physics, autoreset, **opts), _make("MultiHoverAviary", act, D, E, physics, autoreset, **opts)
    if table is not None:
        twin.set_physical_params(**_physical_table(env, table))
    return env, twin


def _near_time_limit(env, twin, E, seed=1):
    sc = np.random.default_rng(seed).integers(1880, 1960, E)
    env.set_state(step_counter=sc); twin.set_state(step_counter=sc)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_general_policy_matches_reference_and_physics_twin(case):
    name, act, D, E, physics, T, arch, activation, with_noise, opts = case
    env, twin = _pair(act, D, E, physics, **dict(opts))
    pol = _policy(env, D, arch, activation, seed=5 + D)
    assert not pol.classic
    ref = MlpRef(pol)
    noise = torch.randn((T, E, D * env._A), device="cuda", generator=torch.Generator(device="cuda").manual_seed(9)) if with_noise else None
    obs0 = env.reset()[0].clone()
    twin.reset()
    _near_time_limit(env, twin, E)
    out = env.rollout(policy=pol, noise=noise, num_steps=T)
    twin_out = twin.rollout(actions=out["actions"].clamp(-1, 1))
    torch.cuda.synchronize()
    _assert_same_physics(out, twin_out, env, twin)
    assert int((out["terminated"] | out["truncated"]).sum()) > 0
    worst = _teacher_forced(ref, obs0, out, noise)
    _report("arch-" + name, worst)
    assert _ratio(worst) <= 1.0, worst


@pytest.mark.gpu
@pytest.mark.parametrize("act,physics,D,opts", [("RPM", "DYN", 2, {}), ("PID", "DYN", 2, {}), ("RPM", "PYB_DW", 4, {"initial_xyzs": _STACK4})],
                         ids=["rpm-d2", "pid-d2", "dw-stack4"])
def test_default_shape_through_the_general_path_gives_the_classic_bits(act, physics, D, opts):
    """[64, 64] Tanh forced through qs_rollout_mlp: obs, actions, log-probs, values and final_values equal qs_rollout's."""
    E, T = 150 if D == 2 else 50, 10
    env, twin = _pair(act, D, E, physics, **opts)
    pol = _policy(env, D, None, "tanh", seed=3)
    gen = copy.copy(pol)
    gen.classic = False
    noise = torch.randn((T, E, D * env._A), device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    env.reset(); twin.reset()
    _near_time_limit(env, twin, E)
    a = env.rollout(policy=pol, noise=noise, final_obs=True, final_values=True)
    b = twin.rollout(policy=gen, noise=noise, final_obs=True, final_values=True)
    torch.cuda.synchronize()
    done = (a["terminated"] | a["truncated"])
    assert int(done.sum()) > 0
    for k in ("obs", "actions", "log_probs", "values", "rewards", "terminated", "truncated"):
        assert torch.equal(a[k], b[k]), k
    assert torch.equal(a["final_values"][done], b["final_values"][done]) and torch.equal(a["final_obs"][done], b["final_obs"][done])


@pytest.mark.gpu
def test_same_step_final_values_with_a_wide_critic():
    E, D, T = 150, 2, 10
    env, twin = _pair("RPM", D, E)
    pol = _policy(env, D, dict(pi=[64], vf=[256, 256, 128]), "tanh", seed=11)
    ref = MlpRef(pol)
    env.reset(); twin.reset()
    _near_time_limit(env, twin, E)
    out = env.rollout(policy=pol, num_steps=T, final_obs=True, final_values=True)
    twin_out = twin.rollout(actions=out["actions"].clamp(-1, 1), final_obs=True)
    torch.cuda.synchronize()
    _assert_same_physics(out, twin_out, env, twin)
    done = (out["terminated"] | out["truncated"]).cpu().numpy()
    assert done.sum() > 0
    worst = 0.0
    for t in range(T):
        rows = np.nonzero(done[t])[0]
        if rows.size == 0:
            continue
        x = ref.flat(out["final_obs"][t].cpu().numpy()[rows])
        v, tol = ref.tolerance(ref.critic, ref.floor_critic, PolicyRef.saturate(x).astype(np.float32))
        got = out["final_values"][t].cpu().numpy()[rows].astype(np.float64)
        worst = max(worst, float((np.abs(got - v[:, 0]) / tol[:, 0]).max()))
    _report("arch-final-values", {"values": worst})
    assert worst <= 1.0, worst


@pytest.mark.gpu
@pytest.mark.parametrize("clears", [False, True])
def test_next_step_values_bootstrap_the_terminal_observation(clears):
    """Next-step autoreset: values[k+1] where autoreset[k+1] is the critic on obs[k], the terminal observation."""
    E, D, T = 150, 2, 12
    kw = {"autoreset_clears_controllers": True, "autoreset_clears_action_buffer": True} if clears else {}
    env, twin = _pair("PID", D, E, "DYN", "next_step", **kw)
    pol = _policy(env, D, dict(pi=[128, 64], vf=[256, 200]), "relu", seed=13)
    ref = MlpRef(pol)
    env.reset(); twin.reset()
    _near_time_limit(env, twin, E, seed=4)
    out = env.rollout(policy=pol, num_steps=T)
    twin_out = twin.rollout(actions=out["actions"].clamp(-1, 1))
    torch.cuda.synchronize()
    _assert_same_physics(out, twin_out, env, twin)
    ar = out["autoreset"].cpu().numpy()
    assert ar[1:].sum() > 0
    worst = 0.0
    for k in range(T - 1):
        rows = np.nonzero(ar[k + 1])[0]
        if rows.size == 0:
            continue
        x = ref.flat(out["obs"][k].cpu().numpy()[rows])
        v, tol = ref.tolerance(ref.critic, ref.floor_critic, PolicyRef.saturate(x).astype(np.float32))
        got = out["values"][k + 1].cpu().numpy()[rows].astype(np.float64)
        worst = max(worst, float((np.abs(got - v[:, 0]) / tol[:, 0]).max()))
    _report("arch-next-step-values-clears%d" % clears, {"values": worst})
    assert worst <= 1.0, worst


@pytest.mark.gpu
def test_wide_policy_across_the_launch_split():
    """PID at 440/44 Hz (obs 78 floats): T = 100 exceeds qs_rollout_mlp_max_ticks at width 256 and takes two launches; it gives the
    bits of two consecutive rollout() calls of tmax and T - tmax ticks."""
    E, D, T = 90, 2, 100
    kw = dict(pyb_freq=440, ctrl_freq=44)
    env, twin = _pair("PID", D, E, **kw)
    pol = _policy(env, D, [256, 256], "relu", seed=8)
    tmax = env._lib.qs_rollout_mlp_max_ticks(env._act_type(), env._B, D, pol.max_width)
    assert 0 < tmax < T, tmax
    noise = torch.randn((T, E, D * 3), device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    env.reset(); twin.reset()
    sc = np.random.default_rng(2).integers(3300, 3520, E)
    env.set_state(step_counter=sc); twin.set_state(step_counter=sc)
    out = env.rollout(policy=pol, noise=noise)
    o1 = twin.rollout(policy=pol, noise=noise[:tmax])
    o1 = {k: v.clone() for k, v in o1.items()}
    o2 = twin.rollout(policy=pol, noise=noise[tmax:])
    torch.cuda.synchronize()
    assert int((out["terminated"] | out["truncated"]).sum()) > 0
    for k in ("obs", "actions", "log_probs", "values", "rewards", "terminated", "truncated"):
        assert torch.equal(out[k], torch.cat([o1[k], o2[k]])), k


@pytest.mark.gpu
def test_widest_policy_at_the_bench_shape():
    """32 768 aviaries of 2 drones, RPM, T = 16, actor + critic at the widest accepted width: physics bit-identical to the twin,
    the reference on 512 sampled aviaries at sampled ticks."""
    from gym_pybullet_drones_b200.policy import MlpPolicy
    E, D, T = 32768, 2, 16
    w = MlpPolicy.MAX_WIDTH
    env, twin = _pair("RPM", D, E)
    pol = _policy(env, D, [w, w], "tanh", seed=12)
    ref = MlpRef(pol)
    noise = torch.randn((T, E, D * 4), device="cuda", generator=torch.Generator(device="cuda").manual_seed(6))
    obs0 = env.reset()[0].clone()
    twin.reset()
    out = env.rollout(policy=pol, noise=noise)
    twin_out = twin.rollout(actions=out["actions"].clamp(-1, 1))
    torch.cuda.synchronize()
    _assert_same_physics(out, twin_out, env, twin)
    rows = np.sort(np.random.default_rng(3).choice(E, 512, replace=False))
    worst = {}
    for t in (0, 5, 15):
        x = ref.flat((obs0 if t == 0 else out["obs"][t - 1]).cpu().numpy()[rows])
        r = ref.check(x, noise[t].cpu().numpy()[rows], out["actions"][t].cpu().numpy()[rows], out["log_probs"][t].cpu().numpy()[rows],
                      out["values"][t].cpu().numpy()[rows], ref_obs=PolicyRef.saturate(x).astype(np.float32))
        worst = {k: max(worst.get(k, 0.0), v) for k, v in r.items()}
    _report("arch-bench-shape-w%d" % w, worst)
    assert max(worst.values()) <= 1.0, worst


@pytest.mark.gpu
def test_negative_controls():
    """(a) The depth-4 net with the lo' half-words of its middle layer 2 zeroed misses the criterion: by more than 10x with ReLU,
    and with Tanh, whose activation floor grows with every layer, still clearly (measured 5.5x on H100); (b) the reference evaluated
    with the other activation misses it grossly.  The intact policies meet it on the same observations."""
    E, D, T = 128, 2, 3
    env, _ = _pair("RPM", D, E)
    worst = {}
    for activation in ("relu", "tanh"):
        pol = _policy(env, D, [256, 128, 64, 32], activation, seed=7)
        bad = copy.copy(pol)
        bad._split = dict(pol._split)
        bad._split["actor"] = list(pol._split["actor"])
        w, b = bad._split["actor"][2]
        w = w.clone()
        w[..., 2:] = 0                                       # words 2, 3 of every lane: the {b0, b1} pairs of w_lo'
        bad._split["actor"][2] = (w, b)
        other = "tanh" if activation == "relu" else "relu"
        for name, p, ref in (("intact", pol, MlpRef(pol)), ("no_w_lo_layer2", bad, MlpRef(pol)), (other + "_reference", pol, MlpRef(pol, other))):
            obs0 = env.reset()[0].clone()
            out = env.rollout(policy=p, num_steps=T)
            torch.cuda.synchronize()
            worst[activation + "-" + name] = _teacher_forced(ref, obs0, out, None)
            _report("arch-negative-%s-%s" % (activation, name), worst[activation + "-" + name])
    assert _ratio(worst["relu-intact"]) <= 1.0 and _ratio(worst["tanh-intact"]) <= 1.0, worst
    assert worst["relu-no_w_lo_layer2"]["actions"] > 10 and worst["relu-no_w_lo_layer2"]["values"] <= 1.0, worst
    assert worst["tanh-no_w_lo_layer2"]["actions"] > 2 and worst["tanh-no_w_lo_layer2"]["values"] <= 1.0, worst
    assert worst["relu-tanh_reference"]["actions"] > 100 and worst["tanh-relu_reference"]["actions"] > 100, worst
