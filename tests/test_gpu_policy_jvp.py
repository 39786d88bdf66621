"""-m gpu: forward mode of the policy loop (qs_dyn_policy_traj_jvp / qs_dyn_policy_tick_jac, DESIGN.md 4.5) through
BaseAviary.differentiable_rollout(policy=) with torch.autograd.forward_ad and BaseAviary.linearise(policy=).

Covered: the dot-product identity <J v, w> = <v, J^T w> per aviary between forward AD and the existing backward over every input,
the actor's parameters and the noise included; forward AD's primals against the call without duals (bits) and its tangents
against central differences; linearise's columns against unit-tangent JVPs (bits) and its nominal trajectory against
differentiable_rollout(policy=) (bits); the A / B chain over 16 ticks against a 16-tick JVP; partial CTAs, a Morton-reordered
aviary against its twin, the refusals; and a use: an LQR gain designed at hover from linearise(rpm), realised exactly as a ReLU
MlpPolicy, gives rho(A) < 1 through linearise(policy=), and > 1 with its sign flipped."""
import numpy as np
import pytest
import torch
import torch.autograd.forward_ad as fwAD

from test_gpu_diff_policy import STATE_KEYS, _env, _leaves, _policy, _run

pytestmark = pytest.mark.gpu

OUT_KEYS = STATE_KEYS + ("actions",)


def _jvp(env, pol, L, nth, T, V):
    """(primal outputs, tangents) of differentiable_rollout(policy=) with the leaves L dual along V (keys of L)"""
    with fwAD.dual_level():
        D = {k: (fwAD.make_dual(v.detach(), V[k]) if k in V else v.detach()) for k, v in L.items()}
        out = _run(env, pol, D, nth, T)
        res = {k: fwAD.unpack_dual(out[k]) for k in OUT_KEYS}
        obs = out["obs"]
        return {k: r.primal.clone() for k, r in res.items()}, {k: r.tangent.clone() for k, r in res.items()}, obs


def _per_aviary(d, E, outputs=False):
    """sum over everything but the aviary axis of {k: [.., E, ..]} tensors laid out as the leaves (or, outputs=True, the
    [T, E, D, k] outputs) are; the parameters (shared by every aviary) are left out"""
    tot = torch.zeros(E, dtype=torch.float64, device=next(iter(d.values())).device)
    for k, v in d.items():
        if k.startswith("theta"):
            continue
        if k == "noise":                                        # [T, E, D A]
            tot = tot + v.sum(dim=(0, 2))
        elif v.dim() == 1:                                      # phys: [E]
            tot = tot + v
        else:                                                   # [E, ...] or the outputs' [T, E, D, k]
            tot = tot + (v.sum(dim=(0, 2, 3)) if outputs else v.reshape(E, -1).sum(1))
    return tot


DOT = [("RPM", 1, "DYN", "tanh"), ("ONE_D_RPM", 2, "PYB_GND", "relu"), ("RPM", 2, "PYB_DRAG", "tanh"), ("ONE_D_RPM", 1, "PYB_DRAG", "relu")]


@pytest.mark.parametrize("act,D,physics,activation", DOT)
def test_dot_product_identity_per_aviary(act, D, physics, activation):
    """<J v, w> = <v, J^T w> per aviary, v over every input (state, last_rpm, phys, action_buffer, noise and the actor's
    parameters): the parameters' share of aviary e is <v_theta, J^T w_e> with w restricted to aviary e"""
    E, T = 3, 8
    env = _env(E, D, act, physics, 30, seed=D)
    pol = _policy(env, (32, 32), activation)
    rng = np.random.default_rng(DOT.index((act, D, physics, activation)))
    L, nth = _leaves(env, pol, rng, T)
    # each physical constant moves relative to its size: KF reaches the thrust twice, directly and through HOVER_RPM = sqrt(m g /
    # (4 KF)) in the decode, and the two nearly cancel (HOVER_RPM^2 KF = m g / 4); a unit step in KF (3e-10) would leave that
    # cancellation's rounding, not the identity, at the scale of the other blocks
    from gym_pybullet_drones_b200.params import PHYS_KEYS
    V = {k: torch.tensor(rng.standard_normal(tuple(v.shape)), device=env.device) * (v.detach().abs() if k in PHYS_KEYS else 1.0)
         for k, v in L.items()}
    _, Jv, _ = _jvp(env, pol, L, nth, T, V)
    out = _run(env, pol, L, nth, T)
    Wt = {k: torch.tensor(rng.standard_normal(tuple(out[k].shape)), device=env.device) for k in OUT_KEYS}
    keys = list(L)
    lhs = _per_aviary({k: Jv[k] * Wt[k] for k in OUT_KEYS}, E, True)
    nj = torch.sqrt(_per_aviary({k: Jv[k] ** 2 for k in OUT_KEYS}, E, True)) * torch.sqrt(_per_aviary({k: Wt[k] ** 2 for k in OUT_KEYS}, E, True))
    worst = 0.0
    for e in range(E):
        g = torch.autograd.grad(sum((out[k][:, e] * Wt[k][:, e]).sum() for k in OUT_KEYS), [L[k] for k in keys], retain_graph=True,
                                allow_unused=True)
        JTw = {k: (torch.zeros_like(L[k]) if x is None else x) for k, x in zip(keys, g)}
        rhs = float(_per_aviary({k: V[k] * JTw[k] for k in keys}, E)[e])
        rhs += sum(float((V[k] * JTw[k]).sum()) for k in keys if k.startswith("theta"))
        worst = max(worst, abs(float(lhs[e]) - rhs) / float(nj[e]))
    print("policy dot identity %s D=%d %s %s: worst %.1e" % (act, D, physics, activation, worst))
    assert worst <= 1e-12


def test_forward_ad_primals_and_central_differences():
    E, D, T = 5, 2, 6
    env = _env(E, D, "RPM", "PYB_DRAG", 30, seed=4)       # no ground-effect height clip for a difference to step across
    pol = _policy(env, (64, 64), "tanh")
    rng = np.random.default_rng(5)
    L, nth = _leaves(env, pol, rng, T)
    plain = _run(env, pol, {k: v.detach() for k, v in L.items()}, nth, T)
    from gym_pybullet_drones_b200.params import PHYS_KEYS
    blocks = {"state": STATE_KEYS, "last_rpm": ("last_rpm",), "action_buffer": ("action_buffer",), "noise": ("noise",),
              "phys": tuple(k for k in PHYS_KEYS if k in L), "params": tuple("theta%d" % j for j in range(nth))}
    for name, keys in blocks.items():
        V = {k: torch.tensor(rng.standard_normal(tuple(L[k].shape)), device=env.device) *
             torch.where(L[k].detach() != 0, L[k].detach().abs(), torch.full_like(L[k].detach(), 1e-3)) for k in keys}
        prim, tan, obs = _jvp(env, pol, L, nth, T, V)
        for k in OUT_KEYS:
            assert torch.equal(prim[k], plain[k]), (name, k)
        assert torch.equal(obs, plain["obs"])
        h = 1e-3 if name == "last_rpm" else 1e-5     # last_rpm reaches the state through drag's first substep only: a larger step
        f = lambda s: _run(env, pol, {k: (v.detach() + s * V[k] if k in V else v.detach()) for k, v in L.items()}, nth, T)
        fp, fm = f(h), f(-h)
        for k in OUT_KEYS:
            fd = (fp[k] - fm[k]) / (2 * h)
            err = float((tan[k] - fd).norm() / fd.norm().clamp(min=1e-300))
            assert err <= 1e-6, (name, k, err)


def test_tangent_that_requires_grad_raises():
    env = _env(2, 1, "RPM", "DYN", 30)
    pol = _policy(env)
    L, nth = _leaves(env, pol, np.random.default_rng(1), 3)
    L = {k: v.detach() for k, v in L.items()}
    with fwAD.dual_level():
        L["vel"] = fwAD.make_dual(L["vel"], torch.ones_like(L["vel"]).requires_grad_(True))
        with pytest.raises(ValueError, match="requires grad"):
            _run(env, pol, L, nth, 3)


def _lin(env, pol, L, nth, T):
    from gym_pybullet_drones_b200.params import PHYS_KEYS
    return env.linearise(policy=pol, params=[L["theta%d" % j].detach() for j in range(nth)], num_steps=T,
                         noise=None if "noise" not in L else L["noise"].detach(), state={k: L[k].detach() for k in STATE_KEYS},
                         last_rpm=L["last_rpm"].detach(), phys={k: L[k].detach() for k in PHYS_KEYS if k in L},
                         action_buffer=L["action_buffer"].detach())


def _nzd(env):
    from gym_pybullet_drones_b200 import _native as N
    return 16 + env._B * env._A + (4 if env._effects & N.EFFECT_DRAG else 0)


@pytest.mark.parametrize("physics,act,D", [("DYN", "RPM", 2), ("PYB_DRAG", "ONE_D_RPM", 3)])
def test_linearise_columns_are_unit_jvps(physics, act, D):
    """The columns of tick k that a JVP can seed on its own equal that JVP, bit for bit, in the rows it returns (the state and
    the raw action): delta_k through the noise's tangent at tick k (log_std = 0, so exp(log_std) = 1), and at tick 0 the
    position, velocity, history and (drag) last_rpm columns through the inputs'.  The nominal trajectory is
    differentiable_rollout(policy=)'s."""
    E, T = 11, 3                                               # 11 aviaries: a full CTA and a partial one
    env = _env(E, D, act, physics, 30, seed=7)
    pol = _policy(env, (32, 16), "relu")
    rng = np.random.default_rng(8)
    L, nth = _leaves(env, pol, rng, T)
    L = {k: v.detach() for k, v in L.items()}
    L["theta%d" % (nth - 1)] = torch.zeros_like(L["theta%d" % (nth - 1)])
    lin = _lin(env, pol, L, nth, T)
    ro = _run(env, pol, L, nth, T)
    for k in OUT_KEYS + ("obs",):
        assert torch.equal(lin[k], ro[k]), k
    A_, nzd, B = env._A, _nzd(env), env._B
    nz = D * nzd
    assert lin["A"].shape == (T, E, nz, nz) and lin["B"].shape == (T, E, nz, D * A_) and lin["K"].shape == (T, E, D * A_, nz)
    assert lin["A"].data_ptr() == lin["B"].data_ptr() - nz * 8                         # views of one tensor
    rows = torch.tensor([d * nzd + j for d in range(D) for j in range(13)], device=env.device)

    def check(tan, k, col, M):
        x = torch.cat([tan[q][k] for q in STATE_KEYS], dim=-1).reshape(E, D * 13)
        assert torch.equal(x, M[k][:, rows, col]), (k, col)
    for k in range(T):
        for c in range(D * A_):
            v = torch.zeros_like(L["noise"])
            v[k, :, c] = 1.0
            _, tan, _ = _jvp(env, pol, L, nth, T, {"noise": v})
            check(tan, k, c, lin["B"])
            assert torch.equal(tan["actions"][k].reshape(E, D * A_)[:, c], torch.ones(E, dtype=torch.float64, device=env.device))
    cols = [(s, d, j, d * nzd + o + j) for d in range(D) for s, o, w in (("pos", 0, 3), ("vel", 7, 3)) for j in range(w)]
    cols += [("action_buffer", d, j, d * nzd + 16 + j) for d in range(D) for j in range(B * A_)][::7]
    if physics == "PYB_DRAG":
        cols += [("last_rpm", d, j, d * nzd + 16 + B * A_ + j) for d in range(D) for j in range(4)]
    for s, d, j, col in cols:
        v = torch.zeros_like(L[s])
        v.reshape(E, D, -1)[:, d, j] = 1.0
        _, tan, _ = _jvp(env, pol, L, nth, T, {s: v})
        check(tan, 0, col, lin["A"])
        assert torch.equal(tan["actions"][0].reshape(E, D * A_), lin["K"][0][:, :, col]), (s, j)


def _ang0_tangent(quat, w, tq, tw):
    """the tangent of the first observation's ang_v = R(q / |q|) w"""
    import diff_policy_ref as PR

    def f(q, w_):
        qn = q / torch.sqrt((q * q).sum(-1, keepdim=True))
        return (PR.matrix_unit(qn.reshape(-1, 4)) @ w_.reshape(-1, 3, 1))[:, :, 0].reshape(w_.shape)
    return torch.func.jvp(f, (quat, w), (tq, tw))[1]


@pytest.mark.parametrize("physics", ["DYN", "PYB_DRAG"])
def test_linearise_chain_reproduces_trajectory_jvp(physics):
    """z_{k+1} = A_k z_k + B_k delta_k and raw_k = K_k z_k + delta_k over 16 ticks give the trajectory JVP's state and action
    tangents; z_0's ang_v tangent is the initial ang_v's, delta_k = exp(log_std) t_noise[k]"""
    E, D, T = 5, 2, 16
    env = _env(E, D, "RPM", physics, 30, seed=9)
    pol = _policy(env, (64, 64), "tanh")
    rng = np.random.default_rng(10)
    L, nth = _leaves(env, pol, rng, T)
    L = {k: v.detach() for k, v in L.items()}
    lin = _lin(env, pol, L, nth, T)
    drag = physics == "PYB_DRAG"
    keys = STATE_KEYS + ("action_buffer", "noise") + (("last_rpm",) if drag else ())
    V = {k: torch.tensor(rng.standard_normal(tuple(L[k].shape)), device=env.device) for k in keys}
    _, tan, _ = _jvp(env, pol, L, nth, T, V)
    ang0 = _ang0_tangent(L["quat"], L["rpy_rates"], V["quat"], V["rpy_rates"])
    parts = [V[k] for k in STATE_KEYS] + [ang0, V["action_buffer"].reshape(E, D, -1)] + ([V["last_rpm"]] if drag else [])
    z = torch.cat(parts, dim=-1).reshape(E, -1)
    scale = torch.exp(L["theta%d" % (nth - 1)])
    for k in range(T):
        dk = scale * V["noise"][k]                                                  # [E, D A]
        raw = (lin["K"][k] @ z[..., None])[..., 0] + dk
        z = (lin["A"][k] @ z[..., None] + lin["B"][k] @ dk[..., None])[..., 0]
        x = torch.cat([tan[q][k] for q in STATE_KEYS], dim=-1)
        zx = z.reshape(E, D, -1)[..., :13]
        ex = float((zx - x).norm() / x.norm())
        ea = float((raw - tan["actions"][k].reshape(E, -1)).norm() / tan["actions"][k].norm())
        assert ex <= 1e-12 and ea <= 1e-12, (k, ex, ea)


def test_morton_twin_partial_ctas_and_refusals():
    import gym_pybullet_drones_b200.envs as envs
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics

    class External(envs.MultiHoverAviary):
        _EXTERNAL_DOWNWASH = True
    D, T = 8, 3
    rng = np.random.default_rng(3)
    xyz = np.stack([rng.uniform(-2, 2, D), rng.uniform(-2, 2, D), rng.uniform(0.3, 1.0, D)], 1)
    kw = dict(num_drones=D, initial_xyzs=xyz, act=ActionType.RPM, pyb_freq=240, ctrl_freq=30, num_envs=1)
    a, b = External(physics=Physics.PYB_DW, **kw), envs.MultiHoverAviary(physics=Physics.DYN, **kw)
    a.reset(); b.reset()
    b.rollout(actions=torch.tensor(rng.uniform(-1, 1, (3, 1, D, 4)), dtype=torch.float32, device=b.device))
    pol = _policy(b, (64, 64), "relu")
    with pytest.raises(ValueError, match="downwash"):
        a.linearise(policy=pol, num_steps=T)
    order = a.reorder_by_morton().cpu().numpy()
    assert np.count_nonzero(order != np.arange(D)) >= D // 2
    a._effects, a._EXTERNAL_DOWNWASH = 0, False
    a.set_state(pos=b.pos, quat=b.quat, vel=b.vel, rpy_rates=b.rpy_rates)
    a._obs_buf[a._cur][:, 12:] = b._obs_buf[b._cur][:, 12:][torch.as_tensor(order, device=b.device)]
    la, lb = a.linearise(policy=pol, num_steps=T), b.linearise(policy=pol, num_steps=T)
    for k in la:
        assert torch.equal(la[k], lb[k]), k
    # partial CTAs: an aviary's Jacobian does not depend on the other aviaries of its CTA
    env = _env(13, 2, "RPM", "DYN", 30, seed=11)
    p2 = _policy(env, (32, 32), "tanh")
    full = env.linearise(policy=p2, num_steps=2)
    state = {k: getattr(env, k)[5:6].clone() for k in STATE_KEYS}
    one = _env(1, 2, "RPM", "DYN", 30, seed=11)
    one._obs_buf[one._cur][:, 12:] = env._obs_buf[env._cur][10:12, 12:]
    last = env._by_id(env._last_rpm).reshape(13, 2, 4)[5:6].clone() if env._track_last_action else None
    sub = one.linearise(policy=p2, num_steps=2, state=state, last_rpm=last)
    for k in ("A", "B", "K", "actions", "pos"):
        assert torch.equal(full[k][:, 5:6] if full[k].dim() > 2 else full[k], sub[k]), k
    # refusals
    with pytest.raises(ValueError, match="exactly one"):
        env.linearise(torch.zeros((1, 13, 2, 4), dtype=torch.float64, device=env.device), policy=p2, num_steps=1)
    with pytest.raises(ValueError, match="exactly one"):
        env.linearise()
    with pytest.raises(ValueError, match="controller linearisation"):
        env.linearise(policy=p2, num_steps=1, waypoints=torch.zeros((1, 3), dtype=torch.float64, device=env.device))
    with pytest.raises(ValueError, match="policy linearisation"):
        env.linearise(torch.zeros((1, 13, 2, 4), dtype=torch.float64, device=env.device), noise=torch.zeros(1))
    with pytest.raises(ValueError, match="num_steps"):
        env.linearise(policy=p2)
    for act in ("PID", "VEL", "ONE_D_PID"):
        e2 = _env(2, 1, act, "DYN", 30)
        with pytest.raises(ValueError, match="linearise\\(policy=\\).*embedded"):
            e2.linearise(policy=_policy(e2), num_steps=1)


def _hover_lqr(env, Q, Rw):
    """The discrete LQR gain [A, 12] at hover in observation coordinates (pos, rpy, vel, ang_v) and action units, from
    linearise(rpm): o_{k+1} = F o_k + G a_k with F = C A E, G = C B d rpm / d a, C = d obs / d x, E its pseudo-inverse"""
    import scipy.linalg
    import diff_policy_ref as PR
    dev = env.device
    hover = dict(pos=torch.tensor([[[0.0, 0.0, 1.0]]], dtype=torch.float64, device=dev), quat=torch.tensor([[[0.0, 0.0, 0.0, 1.0]]],
                 dtype=torch.float64, device=dev), vel=torch.zeros((1, 1, 3), dtype=torch.float64, device=dev),
                 rpy_rates=torch.zeros((1, 1, 3), dtype=torch.float64, device=dev))
    rpm = torch.full((1, 1, 1, 4), float(env.HOVER_RPM), dtype=torch.float64, device=dev)
    lin = env.linearise(rpm, state=hover)
    A, B = lin["A"][0, 0, 0].cpu().numpy(), lin["B"][0, 0, 0].cpu().numpy()

    def obs(x):
        return torch.cat([x[0:3], PR.PR.quat_to_euler(x[None, 3:7])[0], x[7:10], x[10:13]])
    x0 = torch.tensor([0.0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0], dtype=torch.float64)
    Cm = torch.func.jacfwd(obs)(x0).numpy()
    Em = np.linalg.pinv(Cm)
    F, G = Cm @ A @ Em, Cm @ B * (0.05 * float(env.HOVER_RPM))
    S = scipy.linalg.solve_discrete_are(F, G, Q, Rw)
    K = np.linalg.solve(Rw + G.T @ S @ G, G.T @ S @ F)
    return K, hover                                            # a = -K (o - o*)


def test_lqr_policy_at_hover_is_stable_and_its_sign_flip_is_not():
    """An LQR at hover, realised exactly as a one-hidden-layer ReLU MlpPolicy raw = (relu(y + c) - relu(-y + c)) / 2 with y =
    -K (o - o*), c > 0 (no unit on its kink): linearise(policy=) gives rho(A) < 1 and K_lin = -K d obs / d z; with y's sign
    flipped, rho(A) > 1"""
    from gym_pybullet_drones_b200.policy import MlpPolicy
    import diff_policy_ref as PR
    env = _env(1, 1, "RPM", "DYN", 48, cls="HoverAviary")
    K, hover = _hover_lqr(env, np.diag([10.0] * 3 + [1.0] * 3 + [1.0] * 3 + [0.1] * 3), np.eye(4))
    dev = env.device
    od, A_, B = env._obs_dim, env._A, env._B
    o_star = np.zeros(12)
    o_star[2] = 1.0
    c = 0.5
    for sign, stable in ((1.0, True), (-1.0, False)):
        Kp = -sign * K                                          # y = Kp (o - o*)
        W1 = np.zeros((od, 2 * A_))
        W1[:12, :A_], W1[:12, A_:] = Kp.T, -Kp.T
        b1 = np.concatenate([-Kp @ o_star + c, Kp @ o_star + c])
        W2 = 0.5 * np.concatenate([np.eye(A_), -np.eye(A_)])
        theta = [torch.tensor(t, dtype=torch.float64, device=dev) for t in (W1, b1, W2, np.zeros(A_), np.zeros(A_))]
        pol = MlpPolicy([(theta[0].float(), theta[1].float()), (theta[2].float(), theta[3].float())], theta[4].float(), None, dev, "relu")
        lin = env.linearise(policy=pol, params=theta, num_steps=1, state=hover,
                            action_buffer=torch.zeros((1, 1, B, A_), dtype=torch.float64, device=dev))
        assert float(lin["actions"].abs().max()) <= 1e-12                # hover: raw = (relu(c) - relu(c)) / 2 up to K o's rounding
        Az = lin["A"][0, 0].cpu()
        rho = float(torch.linalg.eigvals(Az).abs().max())
        # d obs / d z at hover: pos, rpy (from the quaternion), vel, the observation's ang_v; the history has zero weights
        nz = Az.shape[0]
        Dz = torch.zeros((12, nz), dtype=torch.float64)
        Dz[0:3, 0:3] = torch.eye(3)
        Dz[3:6, 3:7] = torch.func.jacfwd(lambda q: PR.PR.quat_to_euler(q[None])[0])(torch.tensor([0.0, 0, 0, 1], dtype=torch.float64))
        Dz[6:9, 7:10] = torch.eye(3)
        Dz[9:12, 13:16] = torch.eye(3)
        want = torch.tensor(Kp) @ Dz
        err = float((lin["K"][0, 0].cpu() - want).abs().max() / want.abs().max())
        print("LQR policy x %+g: rho(A) = %.6f, |K - K_lqr d obs / d z| / |K| = %.1e" % (sign, rho, err))
        assert err <= 1e-12
        assert (rho < 1.0) if stable else (rho > 1.0), rho
