"""-m gpu: BaseAviary.differentiable_rollout(policy=MlpPolicy) (qs_dyn_policy_traj / qs_dyn_policy_traj_vjp, DESIGN.md 4.5).

The forward and the gradients are held to the float64 torch reference tests/diff_policy_ref.py on the same device (per-drone
normwise relative error per input block) and to the per-tick composition differentiable_rollout(rpm[k:k+1]) + torch; the
observations to rollout(policy=) at float32 level; the gradients to torch.autograd.gradcheck and to themselves (determinism); a
Morton-reordered aviary to its twin in drone-id order; and a short Adam run improves a hover policy."""

import numpy as np
import pytest
import torch

import diff_policy_ref as PR
import diff_ref as R
from diff_testlib import per_drone_relerr

pytestmark = pytest.mark.gpu

FWD_TOL, GRAD_TOL = 1e-12, 1e-9
OBS_F32_TOL = 5e-5          # max |obs - rollout(policy=) obs| over 16 ticks at 30 Hz, 256 x 2 drones: 6.1e-6 measured (H100, 700 W)
STATE_KEYS = ("pos", "quat", "vel", "rpy_rates")


def _env(E, D=1, act="RPM", physics="DYN", ctrl=30, seed=0, cls="MultiHoverAviary", **kw):
    import gym_pybullet_drones_b200.envs as envs
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    rng = np.random.default_rng(seed)
    if cls == "MultiHoverAviary":
        xyz = np.stack([rng.uniform(-1, 1, D), rng.uniform(-1, 1, D), rng.uniform(0.1, 1.0, D)], 1)
        kw = dict(kw, num_drones=D, initial_xyzs=xyz, initial_rpys=rng.uniform(-0.1, 0.1, (D, 3)))
    env = getattr(envs, cls)(act=ActionType[act], physics=Physics[physics], pyb_freq=240, ctrl_freq=ctrl, num_envs=E, **kw)
    env.reset()
    return env


def _policy(env, arch=(64, 64), activation="tanh", seed=3):
    from gym_pybullet_drones_b200.policy import MlpPolicy
    return MlpPolicy.random(env._D * env._obs_dim, env._D * env._A, seed=seed, critic=False, log_std=-1.0, net_arch=list(arch),
                            activation=activation)


def _leaves(env, pol, rng, T, noise=True, table=True):
    """Every differentiable input of the policy loop, as fresh float64 leaves."""
    E, D, A, B, dev = env._E, env._D, env._A, env._B, env.device
    t = lambda a: torch.tensor(a, device=dev, dtype=torch.float64)
    L = {"pos": env.pos.clone() + t(rng.uniform(-0.2, 0.2, (E, D, 3))), "quat": env.quat.clone(),
         "vel": t(rng.uniform(-0.5, 0.5, (E, D, 3))), "rpy_rates": t(rng.uniform(-1, 1, (E, D, 3))),
         "last_rpm": t(env.HOVER_RPM * rng.uniform(0.9, 1.1, (E, D, 4))),
         "action_buffer": t(rng.uniform(-1, 1, (E, D, B, A)))}
    if noise:
        L["noise"] = t(rng.standard_normal((T, E, D * A)))
    if table:
        L.update({k: v * t(rng.uniform(0.8, 1.2, E)) for k, v in env.physical_params().items()})
    theta = pol.parameters64()
    for j, p in enumerate(theta):
        L["theta%d" % j] = p
    return {k: v.detach().clone().requires_grad_(True) for k, v in L.items()}, len(theta)


def _run(env, pol, L, nth, T):
    from gym_pybullet_drones_b200.params import PHYS_KEYS
    return env.differentiable_rollout(policy=pol, params=[L["theta%d" % j] for j in range(nth)], num_steps=T, noise=L.get("noise"),
                                      state={k: L[k] for k in STATE_KEYS}, last_rpm=L["last_rpm"],
                                      phys={k: L[k] for k in PHYS_KEYS if k in L}, action_buffer=L["action_buffer"])


def _reference(env, pol, L, nth, T, flip=()):
    from gym_pybullet_drones_b200.params import PHYS_KEYS, physical_rows
    E, D, n, dev = env._E, env._D, env._N, env.device
    props = env.physical_params()
    props.update({k: L[k] for k in PHYS_KEYS if k in L})
    rows = physical_rows(env.DRONE_MODEL, props, env.G).repeat_interleave(D, dim=0)
    x0 = torch.cat([L[k].reshape(n, -1) for k in STATE_KEYS], dim=1)
    K = R.model_constants(env._P, dev)
    xs, raw, obs = PR.policy_loop(K, rows, [L["theta%d" % j] for j in range(nth)], pol.activation, x0,
                                  L["action_buffer"].reshape(n, env._B, env._A), L["last_rpm"].reshape(n, 4), L.get("noise"), T, E, D,
                                  env.PYB_STEPS_PER_CTRL, env._effects, flip)
    out = {"pos": xs[..., 0:3], "quat": xs[..., 3:7], "vel": xs[..., 7:10], "rpy_rates": xs[..., 10:13]}
    out = {k: v.reshape(T, E, D, -1) for k, v in out.items()}
    out["actions"], out["obs"] = raw.reshape(T, E, D, -1), obs.reshape(T, E, D, -1)
    return out


def _loss(out, cot):
    return sum((out[k] * cot[k]).sum() for k in cot)


def _cotangents(out, rng, dev):
    return {k: torch.tensor(rng.standard_normal(tuple(out[k].shape)), device=dev) for k in STATE_KEYS + ("actions",)}


def _worst(L, got, want, E):
    """{input: worst per-drone (per-aviary, or whole-tensor for the parameters) relative error}."""
    res = {}
    for (k, leaf), g, w in zip(L.items(), got, want):
        g = torch.zeros_like(leaf) if g is None else g
        w = torch.zeros_like(leaf) if w is None else w
        if k == "noise":
            g, w = g.transpose(0, 1), w.transpose(0, 1)
        if k.startswith("theta"):
            g, w = g.reshape(1, -1), w.reshape(1, -1)
        else:
            g, w = g.reshape(E, -1), w.reshape(E, -1)
        res[k] = float(np.max(per_drone_relerr(g.cpu().numpy(), w.cpu().numpy())))
    return res


def _check(env, pol, T, seed, noise=True, table=True):
    rng = np.random.default_rng(seed)
    L, nth = _leaves(env, pol, rng, T, noise, table)
    out = _run(env, pol, L, nth, T)
    ref = _reference(env, pol, L, nth, T)
    for k in STATE_KEYS + ("actions", "obs"):
        err = R.relerr(out[k], ref[k])
        assert err <= FWD_TOL, (k, err)
    assert not out["obs"].requires_grad
    cot = _cotangents(out, rng, env.device)
    got = torch.autograd.grad(_loss(out, cot), list(L.values()), allow_unused=True)
    want = torch.autograd.grad(_loss(ref, cot), list(L.values()), allow_unused=True)
    worst = _worst(L, got, want, env._E)
    assert max(worst.values()) <= GRAD_TOL, worst
    return L, nth, out, cot, got


# (arch, activation, D, act, E, ctrl_freq, T, physics, noise, table)
CASES = [
    ((64, 64), "tanh", 1, "RPM", 37, 30, 20, "DYN", True, True),                    # partial CTAs, T > B
    ((128, 64), "relu", 2, "RPM", 37, 30, 6, "PYB_GND", True, True),
    ((100,), "tanh", 4, "ONE_D_RPM", 9, 48, 30, "PYB_DRAG", True, False),           # B = 24, T > B
    ((256, 256, 256, 256), "relu", 1, "ONE_D_RPM", 1, 30, 1, "DYN", False, False),  # E = 1, T = 1
    ((256, 256, 256, 256), "tanh", 2, "RPM", 5, 30, 4, "PYB_DRAG", True, True),
    ((64, 64), "relu", 4, "RPM", 6, 30, 5, "DYN", False, True),
]


@pytest.mark.parametrize("case", CASES, ids=["-".join(map(str, c[:8])).replace(" ", "") for c in CASES])
def test_forward_and_gradients_match_the_reference(case):
    arch, activation, D, act, E, ctrl, T, physics, noise, table = case
    env = _env(E, D, act, physics, ctrl)
    _check(env, _policy(env, arch, activation), T, 100 + CASES.index(case), noise, table)


def test_4096_aviaries_32_ticks_repeatable_and_env_untouched():
    env = _env(4096, 1, "RPM", "DYN", 30)
    pol = _policy(env)
    keep = [x.clone() for x in (env._planes, env._last_rpm, env._step_counter, env._obs_buf[0], env._obs_buf[1])] + \
        [t.clone() for wb in pol.actor for t in wb] + [w.clone() for w, _ in pol._split["actor"]]
    L, nth, out, cot, got = _check(env, pol, 32, 11)
    again = torch.autograd.grad(_loss(_run(env, pol, L, nth, 32), cot), list(L.values()), allow_unused=True)
    for a, b in zip(got, again):
        assert torch.equal(a, b)
    now = [env._planes, env._last_rpm, env._step_counter, env._obs_buf[0], env._obs_buf[1]] + \
        [t for wb in pol.actor for t in wb] + [w for w, _ in pol._split["actor"]]
    for a, b in zip(keep, now):
        assert torch.equal(a, b)
    with pytest.raises(ValueError, match="double backward"):
        torch.autograd.grad(_run(env, pol, L, nth, 32)["pos"].sum(), L["theta0"], create_graph=True)


def test_matches_the_per_tick_composition():
    """differentiable_rollout(rpm[k:k+1]) + the observation and the actor in torch, tick by tick: an independent check of the
    position / velocity / history path only (quat, rpy_rates and last_rpm stay out of the gradient comparison).  The composition cannot see R_last (the attitude inside the tick), so it runs where ang_v = 0 either
    way: ONE_D_RPM from zero body rates makes no torque."""
    E, T = 64, 8
    env = _env(E, 1, "ONE_D_RPM", "DYN", 30)             # one action on four motors: no torque, w stays 0, ang_v = 0 both ways
    pol = _policy(env, (64, 64), "tanh")
    rng = np.random.default_rng(5)
    L, nth = _leaves(env, pol, rng, T, noise=True, table=False)
    with torch.no_grad():
        L["rpy_rates"].zero_()
    out = _run(env, pol, L, nth, T)
    theta = [L["theta%d" % j] for j in range(nth)]
    from gym_pybullet_drones_b200.diff import actor64
    st, hist, last = {k: L[k] for k in STATE_KEYS}, L["action_buffer"], L["last_rpm"]
    poss = []
    for k in range(T):
        obs = torch.cat([st["pos"], PR.PR.quat_to_euler(st["quat"].reshape(E, 4)).reshape(E, 1, 3), st["vel"], torch.zeros_like(st["vel"]),
                         hist.reshape(E, 1, -1)], dim=-1)
        raw = actor64(theta, "tanh", obs.reshape(E, -1), L["noise"][k]).reshape(E, 1, 1)
        a = raw.clamp(-1, 1)
        hist = torch.cat([hist[:, :, 1:], a[:, :, None, :]], dim=2)
        rpm = (env.HOVER_RPM * (1 + 0.05 * a)).expand(E, 1, 4)
        o = env.differentiable_rollout(rpm[None], state=st, last_rpm=last)
        st = {key: o[key][0] for key in STATE_KEYS}
        last = rpm.clamp(0, env.MAX_RPM)
        poss.append(st["pos"])
    comp = torch.stack(poss)
    assert R.relerr(out["pos"], comp) <= FWD_TOL
    cot = torch.tensor(rng.standard_normal(tuple(comp.shape)), device=env.device)
    leaves = [L[k] for k in L if k not in ("rpy_rates", "quat", "last_rpm")]
    got = torch.autograd.grad((out["pos"] * cot).sum(), leaves, allow_unused=True)
    want = torch.autograd.grad((comp * cot).sum(), leaves, allow_unused=True)
    for k, g, w in zip([k for k in L if k not in ("rpy_rates", "quat", "last_rpm")], got, want):
        assert R.relerr(g, w) <= GRAD_TOL, k


def test_gradcheck_tiny():
    env = _env(2, 2, "RPM", "PYB_DRAG", 30)
    pol = _policy(env, (8,), "tanh")
    L, nth = _leaves(env, pol, np.random.default_rng(2), 3, noise=True, table=False)
    names = ["theta0", "theta%d" % (nth - 1), "pos", "vel", "action_buffer", "noise"]

    def f(*xs):
        M = dict(L, **dict(zip(names, xs)))
        o = _run(env, pol, M, nth, 3)
        return o["pos"], o["vel"], o["actions"]
    assert torch.autograd.gradcheck(f, [L[k] for k in names], eps=1e-6, atol=1e-6, rtol=1e-5, nondet_tol=0.0)


def test_negative_controls_fail_the_bound():
    env = _env(16, 1, "RPM", "DYN", 30)
    for activation, flip in (("tanh", "history"), ("tanh", "clip"), ("relu", "relu")):
        pol = _policy(env, (64, 64), activation, seed=9)
        rng = np.random.default_rng(4)
        L, nth = _leaves(env, pol, rng, 6, noise=True, table=False)
        with torch.no_grad():
            L["noise"].mul_(8.0)                        # exp(-1) * 8 sigma: a good share of the actions saturate
        out = _run(env, pol, L, nth, 6)
        assert float((out["actions"].abs() > 1).double().mean()) > 0.05
        cot = _cotangents(out, rng, env.device)
        got = torch.autograd.grad(_loss(out, cot), list(L.values()), allow_unused=True)
        want = torch.autograd.grad(_loss(_reference(env, pol, L, nth, 6), cot), list(L.values()), allow_unused=True)
        bad = torch.autograd.grad(_loss(_reference(env, pol, L, nth, 6, flip=(flip,)), cot), list(L.values()), allow_unused=True)
        assert max(_worst(L, got, want, 16).values()) <= GRAD_TOL
        assert max(_worst(L, got, bad, 16).values()) > 1e-4, flip


def test_observations_agree_with_rollout_policy_at_float32_level():
    E, T = 256, 16
    env = _env(E, 2, "RPM", "DYN", 30)
    pol = _policy(env, (64, 64), "tanh")
    noise = torch.randn((T, E, 2 * 4), generator=torch.Generator().manual_seed(1)).to(env.device)
    out = env.differentiable_rollout(policy=pol, noise=noise.double())
    buf = env.rollout(policy=pol, noise=noise)
    # out["obs"][k] is what the policy saw at tick k; rollout's obs[k] is the observation after tick k
    err = float((out["obs"][1:] - buf["obs"][:-1].double()).abs().max())
    print("max |obs64 - obs32| over %d ticks: %.3e" % (T, err))
    assert err <= OBS_F32_TOL
    assert float((out["actions"] - buf["actions"].double()).abs().max()) <= OBS_F32_TOL


def test_morton_reordered_aviary_equals_its_twin():
    """reorder_by_morton() needs an aviary whose downwash comes from the external stage, and the adjoint refuses downwash: so, as
    in the open- and closed-loop tests, the reordered env's effects are switched to plain DYN after the reorder.  The default
    state and the default action buffer are then gathered from a permuted storage order."""
    import gym_pybullet_drones_b200.envs as envs
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics

    class External(envs.MultiHoverAviary):
        _EXTERNAL_DOWNWASH = True
    D, T = 8, 6
    rng = np.random.default_rng(3)
    xyz = np.stack([rng.uniform(-2, 2, D), rng.uniform(-2, 2, D), rng.uniform(0.3, 1.0, D)], 1)
    kw = dict(num_drones=D, initial_xyzs=xyz, act=ActionType.RPM, pyb_freq=240, ctrl_freq=30, num_envs=1)
    a, b = External(physics=Physics.PYB_DW, **kw), envs.MultiHoverAviary(physics=Physics.DYN, **kw)
    a.reset(); b.reset()
    acts = torch.tensor(rng.uniform(-1, 1, (3, 1, D, 4)), dtype=torch.float32, device=b.device)
    b.rollout(actions=acts)                                # a non-trivial state and action buffer, per drone
    order = a.reorder_by_morton().cpu().numpy()
    assert np.count_nonzero(order != np.arange(D)) >= D // 2
    a._effects, a._EXTERNAL_DOWNWASH = 0, False
    a.set_state(pos=b.pos, quat=b.quat, vel=b.vel, rpy_rates=b.rpy_rates)
    a._obs_buf[a._cur][:, 12:] = b._obs_buf[b._cur][:, 12:][torch.as_tensor(order, device=b.device)]    # slot i holds drone order[i]
    pol = _policy(b, (64, 64), "relu")
    res = []
    for e in (a, b):
        theta = pol.parameters64()
        out = e.differentiable_rollout(policy=pol, params=theta, num_steps=T)
        res.append((out, torch.autograd.grad((out["pos"] ** 2).sum() + out["actions"].sum(), theta[:-1])))    # no noise: log_std is unused
    assert float(res[1][0]["obs"][0, 0, :, 12:].abs().max()) > 0
    for k in res[0][0]:
        assert torch.equal(res[0][0][k], res[1][0][k]), k
    for x, y in zip(*(r[1] for r in res)):
        assert torch.equal(x, y)


def test_refusals_and_parameter_round_trip():
    from gym_pybullet_drones_b200.policy import MlpPolicy
    env = _env(4, 1, "RPM", "DYN", 30)
    pol = _policy(env)
    theta = pol.parameters64()
    with pytest.raises(ValueError, match="exactly one"):
        env.differentiable_rollout(policy=pol, num_steps=2, rpm=torch.zeros((2, 4, 1, 4), dtype=torch.float64, device=env.device))
    with pytest.raises(ValueError, match="policy rollout only"):
        env.differentiable_rollout(torch.zeros((2, 4, 1, 4), dtype=torch.float64, device=env.device), noise=torch.zeros(1))
    with pytest.raises(ValueError, match="num_steps"):
        env.differentiable_rollout(policy=pol)
    with pytest.raises(ValueError, match="float64"):
        env.differentiable_rollout(policy=pol, noise=torch.zeros((2, 4, 4), device=env.device))
    with pytest.raises(ValueError, match="params"):
        env.differentiable_rollout(policy=pol, params=theta[:-1], num_steps=2)
    with pytest.raises(ValueError, match="shape"):
        env.differentiable_rollout(policy=pol, num_steps=2, action_buffer=torch.zeros((4, 1, 3, 4), dtype=torch.float64, device=env.device))
    with pytest.raises(ValueError, match="inputs"):
        env.differentiable_rollout(policy=MlpPolicy.random(10, 4), num_steps=2)
    with pytest.raises(ValueError, match="controller rollout only"):
        env.differentiable_rollout(policy=pol, num_steps=2, gains={})
    for act in ("PID", "VEL", "ONE_D_PID"):
        e2 = _env(2, 1, act, "DYN", 30)
        with pytest.raises(ValueError, match="embedded"):
            e2.differentiable_rollout(policy=_policy(e2), num_steps=2)
    e3 = _env(2, 2, "RPM", "PYB_DW", 30)
    with pytest.raises(ValueError, match="downwash"):
        e3.differentiable_rollout(policy=_policy(e3), num_steps=2)
    e4 = _env(2, 1, "RPM", "DYN", 1, cls="HoverAviary")
    with pytest.raises(ValueError, match="action buffer"):
        e4.differentiable_rollout(policy=MlpPolicy.random(12, 4), num_steps=2)
    # parameters64 / load_parameters: fp32 values, and the re-packed fragments equal a freshly built policy's
    with torch.no_grad():
        new = [p + 0.01 * torch.randn_like(p) for p in theta]
    pol.load_parameters(new)
    fresh = MlpPolicy([(new[2 * k].float(), new[2 * k + 1].float()) for k in range(len(pol.actor))], new[-1].float(), None, env.device)
    for (w, b), (fw, fb) in zip(pol._split["actor"], fresh._split["actor"]):
        assert torch.equal(w, fw) and torch.equal(b, fb)
    for p, q in zip(pol.parameters64(), new):
        assert torch.equal(p, q.float().double())
    with pytest.raises(ValueError, match="load_parameters"):
        pol.load_parameters(new[:-1])


def test_adam_improves_a_hover_policy():
    from gym_pybullet_drones_b200.policy import MlpPolicy
    E, T, iters = 1024, 32, 30
    env = _env(E, 1, "ONE_D_RPM", "DYN", 30, cls="HoverAviary")
    pol = MlpPolicy.random(env._obs_dim, 1, seed=0, critic=False, log_std=-1.0)
    g = torch.Generator().manual_seed(0)
    pos0 = torch.tensor([0.0, 0.0, 0.6], dtype=torch.float64) + (torch.rand((E, 1, 3), generator=g, dtype=torch.float64) - 0.5) * 0.4
    pos0 = pos0.to(env.device)
    target = torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64, device=env.device)

    def mean_reward():
        env.reset()
        env.set_state(pos=pos0.reshape(-1, 3))
        return float(env.rollout(policy=pol, num_steps=T)["rewards"].mean())
    r0 = mean_reward()
    theta = pol.parameters64()
    opt = torch.optim.Adam(theta, lr=3e-3)
    losses = []
    env.reset()
    for _ in range(iters):
        out = env.differentiable_rollout(policy=pol, params=theta, num_steps=T, state={"pos": pos0})
        loss = ((out["pos"] - target) ** 2).sum(-1).mean() + 1e-3 * (out["actions"] ** 2).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    pol.load_parameters(theta)
    r1 = mean_reward()
    print("loss %.4f -> %.4f, mean reward %.4f -> %.4f" % (losses[0], losses[-1], r0, r1))
    assert losses[-1] < 0.9 * losses[0]
    assert r1 > r0
