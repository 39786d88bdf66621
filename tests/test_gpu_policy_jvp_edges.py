"""-m gpu: the policy loop's forward mode (qs_dyn_policy_traj_jvp, qs_dyn_policy_tick_jac) on the device at every shape it accepts
and at its decisions, against the float64 references tests/diff_policy_ref.py and policy_jvp_testlib.ref_tick on the same device.

Forward AD through differentiable_rollout(policy=) is compared with torch.func.jvp of diff_policy_ref.policy_loop over a shape
matrix (test_gpu_diff_policy.CASES and the shapes only forward mode has: M = 8 aviaries per JVP CTA, D A = 32, widths 1 and 5, an
input width of 27, 256 JVP CTAs), per aviary and input block; linearise(policy=) at every tick with jacfwd of the reference tick
at the kernel's own tick-k inputs (teacher-forced), with the entries that are exact by construction held to exact zeros and
ones; an aviary's tangents do not depend on the other rows of its CTA; the decisions (actions at +-1, a ReLU unit at 0, the
gimbal guard, saturated actions, a binding MAX_RPM clip) are taken on the device; and negative controls miss the device."""
import numpy as np
import pytest
import torch

from diff_testlib import batched_jvp, per_drone_relerr
from policy_jvp_testlib import kernel_layout, ref_tick_jac
from test_gpu_diff_policy import CASES, STATE_KEYS, _leaves, _policy, _reference
from test_gpu_diff_policy import _env as _env_of
from test_gpu_policy_jvp import OUT_KEYS, _jvp, _lin

pytestmark = pytest.mark.gpu

JVP_TOL = 1e-10             # per-tick Jacobians (the host tests' bound)
GRAD_TOL = 1e-9             # trajectory tangents over T ticks

# (arch, activation, D, act, E, ctrl_freq, T, physics, noise, table): test_gpu_diff_policy's matrix, then the forward-mode shapes
MATRIX = CASES + [
    ((256, 256, 256, 256), "relu", 4, "RPM", 37, 30, 3, "PYB_DRAG", True, True),     # 2 080 doubles per aviary: M = 8, partial CTA
    ((64, 64), "tanh", 8, "RPM", 5, 30, 3, "DYN", True, True),                        # D A = 32
    ((32, 32), "relu", 32, "ONE_D_RPM", 3, 30, 2, "PYB_GND", True, True),             # D A = 32, M D = 256, R = 1 024
    ((1,), "tanh", 2, "RPM", 9, 30, 4, "DYN", True, True),                            # width 1: n-tile masking, K % 4 != 0
    ((5, 5), "relu", 1, "RPM", 13, 30, 4, "GND_DRAG", True, True),                    # width 5, GND | DRAG, two tick-Jacobian CTAs
    ((64,), "tanh", 1, "ONE_D_RPM", 9, 30, 3, "DYN", True, False),                    # in_dim 27
    ((64, 64), "tanh", 1, "RPM", 4090, 30, 3, "DYN", True, True),                     # 256 JVP CTAs, the last with 10 aviaries
]
IDS = ["-".join(map(str, c[:8])).replace(" ", "") for c in MATRIX]


def _env(E, D, act, physics, ctrl, seed=0):
    """test_gpu_diff_policy's env; "GND_DRAG": ground effect and drag, reachable through the C ABI's effects only"""
    from gym_pybullet_drones_b200 import _native as N
    env = _env_of(E, D, act, "PYB_DRAG" if physics == "GND_DRAG" else physics, ctrl, seed=seed)
    if physics == "GND_DRAG":
        env._effects = N.EFFECT_GND | N.EFFECT_DRAG
    return env


def _jvp_m(env, arch):
    """Aviaries per JVP CTA, policy_ctas' formula (policy_actor.cuh) with the JVP's shared memory per aviary (dyn_policy_jvp.cu)"""
    D, A, B = env._D, env._A, env._B
    ind, maxw = D * (12 + B * A), max(arch)
    per = ind + len(arch) * maxw + D * A + 2 * maxw + D * B * A
    M = min(227 * 1024 // (8 * per), 256 // D, 16)
    return M - M % 8


def _per_aviary_out(d, E):
    """{key: [T, E, D, k]} -> {key: [E, T D k]} for OUT_KEYS"""
    return {k: d[k].detach().transpose(0, 1).reshape(E, -1).cpu().numpy() for k in OUT_KEYS}


def _blocks(L, nth):
    from gym_pybullet_drones_b200.params import PHYS_KEYS
    b = {"state": STATE_KEYS, "last_rpm": ("last_rpm",), "action_buffer": ("action_buffer",)}
    if "noise" in L:
        b["noise"] = ("noise",)
    if "m" in L:
        b["phys"] = PHYS_KEYS
    b.update({"theta%d" % j: ("theta%d" % j,) for j in range(nth)})
    return b


@pytest.mark.parametrize("case", MATRIX, ids=IDS)
def test_forward_ad_matches_reference_jvp(case):
    """One direction per input block (state, last_rpm, action_buffer, noise, phys as d / d log c, each parameter tensor with
    log_std), per aviary on the four state entries and the actions.  Tangents the reference has exactly zero (last_rpm without
    drag, log_std without noise) are exactly zero."""
    arch, activation, D, act, E, ctrl, T, physics, noise, table = case
    env = _env(E, D, act, physics, ctrl)
    M = _jvp_m(env, arch)
    assert M == (8 if max(arch) == 256 and D == 4 or D == 32 else 16), M
    pol = _policy(env, arch, activation)
    rng = np.random.default_rng(200 + MATRIX.index(case))
    L, nth = _leaves(env, pol, rng, T, noise, table)
    Ld = {k: v.detach() for k, v in L.items()}
    blocks = _blocks(L, nth)
    Vs = [{k: torch.tensor(rng.standard_normal(tuple(L[k].shape)), device=env.device) * (Ld[k] if name == "phys" else 1.0) for k in keys}
          for name, keys in blocks.items()]
    ref = batched_jvp(lambda d: _reference(env, pol, d, nth, T), Ld, Vs)
    worst = {}
    for j, (name, V) in enumerate(zip(blocks, Vs)):
        _, tan, _ = _jvp(env, pol, L, nth, T, V)
        got, want = _per_aviary_out(tan, E), _per_aviary_out({k: ref[k][j] for k in OUT_KEYS}, E)
        worst[name] = max(float(per_drone_relerr(got[k], want[k]).max()) for k in OUT_KEYS)
    w = max(worst, key=worst.get)
    print("policy forward AD %s (M = %d): worst per-aviary error %.1e (%s)" % (IDS[MATRIX.index(case)], M, worst[w], w))
    assert worst[w] <= GRAD_TOL, worst


def _decode(rows, raw, n, A):
    """The applied RPMs [n, 4] of raw actions [n, A]: HOVER_RPM (1 + 0.05 clip(raw)) clipped to [0, MAX_RPM]"""
    rpm = (rows[:, 12:13] * (1.0 + 0.05 * torch.clamp(raw, -1.0, 1.0))).expand(n, 4)
    return torch.clamp(rpm, min=torch.zeros_like(rpm), max=rows[:, 13:14].expand(n, 4))


def _tick_x(env, L, lin, k, e):
    """Aviary e's inputs of tick k as ref_tick takes them, the kernel's own: the stored state after tick k - 1 (state0 at k = 0),
    ang_v and the history from obs[k], the previous applied RPMs rebuilt from actions[k - 1] (last_rpm at k = 0), its row"""
    from gym_pybullet_drones_b200.params import PHYS_KEYS, physical_rows
    D, A, B = env._D, env._A, env._B
    props = env.physical_params()
    props.update({key: L[key].detach() for key in PHYS_KEYS if key in L})
    rows = physical_rows(env.DRONE_MODEL, props, env.G)[e:e + 1].expand(D, 16)
    src = {s: L[s].detach() for s in STATE_KEYS} if k == 0 else {s: lin[s][k - 1] for s in STATE_KEYS}
    obs = lin["obs"][k, e]
    up = L["last_rpm"].detach()[e] if k == 0 else _decode(rows, lin["actions"][k - 1, e], D, A)
    return dict(state=torch.cat([src[s][e] for s in STATE_KEYS], dim=1), ang=obs[:, 9:12], hist=obs[:, 12:].reshape(D, B, A), up=up,
                row=rows[0])


def _compare_tick(env, pol, L, nth, lin, k, e, flip=(), theta=None):
    """({block: relative error}, exact) of aviary e's tick-k Jacobian against jacfwd of ref_tick at the kernel's inputs, per
    input block over all R rows; exact: the entries that are exact by construction (the shifted history rows, whose entries
    are 0 or 1, and raw_k x delta_k = I) equal the reference's bit for bit.  theta: the reference's parameters (default L's)."""
    from gym_pybullet_drones_b200 import _native as N
    D, A, B = env._D, env._A, env._B
    drag = bool(env._effects & N.EFFECT_DRAG)
    theta = [L["theta%d" % j].detach() for j in range(nth)] if theta is None else theta
    noise = L["noise"].detach()[k, e] if "noise" in L else None
    want = ref_tick_jac(env._P, env._effects, env.PYB_STEPS_PER_CTRL, pol.activation, theta, noise, _tick_x(env, L, lin, k, e), flip,
                        env.device)
    rows, cols, groups = kernel_layout(D, A, B, drag)
    ref = np.concatenate([want[b] for b in ("state", "ang", "hist", "up", "row", "raw_in")], axis=1)[rows][:, cols]
    J = lin["A"]._base                          # the [T, E, R, R] tensor linearise's A, B and K are views of
    assert J is not None and J.data_ptr() == lin["A"].data_ptr()
    J = J[k, e].cpu().numpy()
    errs = {b: float(per_drone_relerr(J[None, :, c], ref[None, :, c])[0]) for b, c in groups.items()}
    nzd, nz = len(rows) // D - A, len(rows) - D * A
    shift = np.array([d * nzd + 16 + j for d in range(D) for j in range((B - 1) * A)], dtype=np.int64)
    exact = (np.array_equal(J[shift], ref[shift]) and np.isin(J[shift], (0.0, 1.0)).all()
             and np.array_equal(J[nz:, nz:], np.eye(D * A)) and np.array_equal(ref[nz:, nz:], np.eye(D * A)))
    return errs, exact


def _sample(E, M):
    """aviaries to compare: the first and last of the first two CTAs of M and of the last (partial) one"""
    return sorted({e for e in (0, M - 1, M, 2 * M - 1, (E - 1) // M * M, E - 1) if e < E})


# the linearise subset: M = 8 (drag), D = 32 (R = 1 024, every thread a drone), width 5 with GND | DRAG and E = 13 (R = 84, not a
# multiple of 8: the last seed group is partial; two CTAs per tick, the second partial)
LIN = [MATRIX[-7], MATRIX[-5], MATRIX[-3]]


@pytest.mark.parametrize("case", LIN, ids=[IDS[MATRIX.index(c)] for c in LIN])
def test_linearise_matches_reference_at_every_tick(case):
    arch, activation, D, act, E, ctrl, _, physics, noise, table = case
    T = 3
    env = _env(E, D, act, physics, ctrl)
    pol = _policy(env, arch, activation)
    L, nth = _leaves(env, pol, np.random.default_rng(300 + LIN.index(case)), T, noise, table)
    lin = _lin(env, pol, L, nth, T)
    worst = {}
    for k in range(T):
        for e in _sample(E, 8):
            errs, exact = _compare_tick(env, pol, L, nth, lin, k, e)
            assert exact, (k, e)
            for b, v in errs.items():
                worst[b] = max(worst.get(b, 0.0), v)
    w = max(worst, key=worst.get)
    R = lin["A"].shape[-1] + D * env._A
    print("policy linearise %s (R = %d): worst per-aviary error %.1e (%s)" % (IDS[MATRIX.index(case)], R, worst[w], w))
    assert worst[w] <= JVP_TOL, worst


@pytest.mark.parametrize("case", [MATRIX[-7], ((64, 64), "tanh", 2, "RPM", 37, 30, 3, "DYN", True, True)], ids=["M8", "M16"])
def test_no_leakage_between_rows_of_a_cta(case):
    """Aviary e's JVP tangents at E = 37 equal, bit for bit, the same aviary run alone (E = 1): cta_gemm's rows are independent.
    The directions are the state, last_rpm, the history and the noise (whose tangent reaches the kernel unmixed)."""
    arch, activation, D, act, E, ctrl, T, physics, noise, table = case
    env = _env(E, D, act, physics, ctrl)
    M = _jvp_m(env, arch)
    assert M == (8 if max(arch) == 256 else 16)
    pol = _policy(env, arch, activation)
    rng = np.random.default_rng(17)
    L, nth = _leaves(env, pol, rng, T, noise, table)
    keys = STATE_KEYS + ("last_rpm", "action_buffer", "noise")
    V = {k: torch.tensor(rng.standard_normal(tuple(L[k].shape)), device=env.device) for k in keys}
    _, tan, _ = _jvp(env, pol, L, nth, T, V)
    one = _env(1, D, act, physics, ctrl)
    for e in _sample(E, M) + [M // 2, M + 3]:
        sl = lambda k, v: v[:, e:e + 1] if k == "noise" else v[e:e + 1] if not k.startswith("theta") else v
        _, t1, _ = _jvp(one, pol, {k: sl(k, v) for k, v in L.items()}, nth, T, {k: sl(k, v) for k, v in V.items()})
        for k in OUT_KEYS:
            assert torch.equal(t1[k], tan[k][:, e:e + 1]), (e, k)


# (scenario, activation, A, D): test_policy_jvp_host._case on the device (B = 5: 10 Hz control)
DECISIONS = [("edge", "relu", 4, 2), ("edge", "tanh", 1, 4), ("gimbal", "tanh", 4, 2), ("saturated", "relu", 4, 1),
             ("max_rpm", "tanh", 4, 2)]


def _decision_case(scenario, activation, A, D, seed, T=2):
    """(env, pol, L, nth, lin) of test_policy_jvp_host._case placed on the device: one aviary, its state, history, last_rpm,
    parameters and noise (the same at every tick); max_rpm: the saturated case with thrust2weight = 1.05"""
    from test_policy_jvp_host import _case
    P, theta, noise, x, _ = _case(activation, A, D, "saturated" if scenario == "max_rpm" else scenario, seed)
    env = _env(1, D, "RPM" if A == 4 else "ONE_D_RPM", "DYN", 10)
    assert env._B == x["hist"].shape[1]
    pol = _policy(env, (16, 8), activation)
    dev = env.device
    t = lambda a: torch.tensor(np.asarray(a, dtype=np.float64), device=dev)
    L = {k: t(x["state"][None, :, a:b]) for k, (a, b) in zip(STATE_KEYS, ((0, 3), (3, 7), (7, 10), (10, 13)))}
    L.update(last_rpm=t(x["up"][None]), action_buffer=t(x["hist"][None]), noise=t(np.repeat(noise[None, None], T, 0)))
    if scenario == "max_rpm":
        L.update({k: v for k, v in env.physical_params().items()}, thrust2weight=torch.full((1,), 1.05, dtype=torch.float64, device=dev))
    L.update({"theta%d" % j: t(th) for j, th in enumerate(theta)})
    return env, pol, L, len(theta), _lin(env, pol, L, len(theta), T)


@pytest.mark.parametrize("scenario,activation,A,D", DECISIONS)
def test_decisions_on_the_device(scenario, activation, A, D):
    """Each decision is taken on the device, read from its outputs (or the state it linearised at), and the tick Jacobians of
    T = 2 match the reference there"""
    env, pol, L, nth, lin = _decision_case(scenario, activation, A, D, DECISIONS.index((scenario, activation, A, D)))
    raw = lin["actions"].reshape(2, -1)
    if scenario == "edge":
        assert torch.all(raw[:, 0] == 1.0) and (D * A == 1 or torch.all(raw[:, -1] == -1.0)), raw
        if activation == "relu":                                # z = pos_x - pos_x of the first unit, exact at tick 0
            assert float(lin["obs"][0, 0, 0, 0]) == -float(L["theta1"][0])
    if scenario == "gimbal":
        q = L["quat"][0, 0]
        assert abs(float(-2.0 * (q[0] * q[2] - q[3] * q[1]))) >= 0.99999
    if scenario in ("saturated", "max_rpm"):
        assert bool((raw.abs() > 1).any()) and bool((raw.abs() < 1).any()), raw
    if scenario == "max_rpm":
        from gym_pybullet_drones_b200.params import PHYS_KEYS, physical_rows
        row = physical_rows(env.DRONE_MODEL, {k: L[k] for k in PHYS_KEYS}, env.G)[0]
        assert bool((row[12] * (1.0 + 0.05 * raw.clamp(-1, 1)) > row[13]).any()), (raw, row[12:14])
    worst = {}
    for k in range(2):
        errs, exact = _compare_tick(env, pol, L, nth, lin, k, 0)
        assert exact, k
        for b, v in errs.items():
            worst[b] = max(worst.get(b, 0.0), v)
    w = max(worst, key=worst.get)
    print("policy decision %s %s A=%d D=%d: worst per-aviary error %.1e (%s)" % (scenario, activation, A, D, worst[w], w))
    assert worst[w] <= JVP_TOL, worst


@pytest.mark.parametrize("flip,activation", [("clip", "tanh"), ("relu", "relu"), ("ang_start", "tanh")])
def test_negative_controls_miss_the_device(flip, activation):
    """ref_tick's flips miss the device's tick-0 Jacobian of the saturated case by more than 1e-4"""
    env, pol, L, nth, lin = _decision_case("saturated", activation, 4, 2, 5, T=1)
    good, _ = _compare_tick(env, pol, L, nth, lin, 0, 0)
    bad, _ = _compare_tick(env, pol, L, nth, lin, 0, 0, flip=(flip,))
    print("policy negative control %s: %.1e against the reference, %.1e against the flipped one" % (flip, max(good.values()),
                                                                                                    max(bad.values())))
    assert max(good.values()) <= JVP_TOL
    assert max(bad.values()) > 1e-4, (flip, bad)


def test_one_perturbed_weight_fails_the_bound():
    """The reference with its largest hidden-layer weight moved by 1e-8 relative misses the device's Jacobian by more than
    JVP_TOL per aviary: the bound sees a single-weight error"""
    env, pol, L, nth, lin = _decision_case("saturated", "tanh", 4, 2, 5, T=1)
    theta = [L["theta%d" % j].clone() for j in range(nth)]
    W = theta[2]
    i = int(torch.argmax(W.abs()))
    W.view(-1)[i] *= 1.0 + 1e-8
    good, _ = _compare_tick(env, pol, L, nth, lin, 0, 0)
    bad, _ = _compare_tick(env, pol, L, nth, lin, 0, 0, theta=theta)
    print("policy weight perturbation: %.1e against the reference, %.1e against the perturbed one" % (max(good.values()),
                                                                                                      max(bad.values())))
    assert max(good.values()) <= JVP_TOL
    assert max(bad.values()) > JVP_TOL, bad
