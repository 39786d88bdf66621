"""-m gpu: the closed-loop forward mode (qs_dyn_ctrl_tick_jac, qs_dyn_ctrl_traj_jvp) and the closed-loop VJP (qs_dyn_ctrl_traj_vjp)
on the device at the controller's decisions, against the float64 reference tests/diff_pid_ref.py on the same device.

The six ctrl_scenarios batches (flight, integral clips, PWM saturation, torque clip, thrust scalar <= 0, gimbal guard) are placed
through the public API (state=, pid_state=, per-drone waypoints of length 1, target_rpy / target_vel / target_rpy_rates per drone,
a gain table and per-aviary constants).  linearise(controller=) is compared at every tick with torch.func.jacfwd of the reference
tick evaluated at the kernel's own tick-k inputs (teacher-forced: the loop's chaos cannot hide or fake a difference); forward AD
and the gradients of differentiable_rollout(controller=) with the reference's forward AD and autograd, per drone and input block.
Each scenario shows that its decision is taken on the device; drones one ulp either side of the integral clips, scalar = 0 and
the gimbal guard match the reference on the side the kernel took; and each of diff_pid_ref's flips misses the device."""
import copy

import numpy as np
import pytest
import torch

import diff_pid_ref as PR
from ctrl_jvp_testlib import ref_ctrl_tick_jac
from diff_ctrl_testlib import ctrl_scenarios
from diff_testlib import batched_jvp, params_of, per_drone_relerr
from test_gpu_ctrl_jvp import _env, _jvp, _lin
from test_gpu_diff_ctrl import GAIN_KEYS, PID_KEYS, STATE_KEYS, _call, _grads, _ref

pytestmark = pytest.mark.gpu

JVP_TOL = 1e-10             # per-tick Jacobians (the host tests' bound)
GRAD_TOL = 1e-9             # trajectory tangents and gradients over T ticks
SCENARIOS = ("flight", "integral", "pwm", "torque", "scalar", "gimbal")
PER = 6                     # drones per scenario: one drone per aviary, E = 36
CONFIGS = [(m, p, c) for m in ("CF2X", "CF2P") for p in ("DYN", "PYB_GND", "PYB_DRAG", "GND_DRAG") for c in (240, 30)]


def _place(env, ctl, state, pid, tg, up, gains, rng=None):
    """Leaves of the closed loop that put drone i (aviary i, D = 1) at state [E, 13], pid [E, 9], targets tg [E, 10] (target_pos,
    target yaw, target_vel, target_rpy_rates), last_rpm up [E, 4] and gains [E, 18]; rng: per-aviary constants.  Only the
    inertias, KM and the arm are drawn below nominal: m, KF and thrust2weight only move MAX_RPM up, so the PWM clip's RPM is
    the applied one where the PWM saturates."""
    E, dev = env._E, env.device
    t = lambda a: torch.tensor(np.asarray(a, dtype=np.float64).reshape(E, 1, -1), device=dev)
    L = {"waypoints": t(tg[:, 0:3])[None], "offset": torch.zeros((E, 1, 3), dtype=torch.float64, device=dev),
         "target_rpy": t(np.concatenate([np.zeros((E, 2)), tg[:, 3:4]], 1)), "target_vel": t(tg[:, 4:7]),
         "target_rpy_rates": t(tg[:, 7:10]), "last_rpm": t(up)}
    L.update({k: t(state[:, a:b]) for k, (a, b) in zip(STATE_KEYS, ((0, 3), (3, 7), (7, 10), (10, 13)))})
    L.update({k: t(pid[:, 3 * j:3 * j + 3]) for j, k in enumerate(PID_KEYS)})
    L.update({k: torch.tensor(gains[:, 3 * j:3 * j + 3], device=dev) for j, k in enumerate(GAIN_KEYS)})
    for k, v in env.physical_params().items():
        lo, hi = (1.0, 1.2) if k in ("m", "thrust2weight") else (0.85, 1.0) if k == "kf" else (0.9, 1.1)
        L[k] = v if rng is None else v * torch.tensor(rng.uniform(lo, hi, E), device=dev)
    return {k: v.detach().clone().requires_grad_(True) for k, v in L.items()}


def _scenario_leaves(env, ctl, model, seed):
    """(leaves, scenario name per drone) of the six ctrl_scenarios batches, PER drones each"""
    rng = np.random.default_rng(seed)
    _, c = params_of(model.lower(), 240, env.CTRL_FREQ)
    sc = ctrl_scenarios(c, rng, PER)
    state, pid, tg = (np.concatenate([sc[s][j] for s in SCENARIOS]) for j in range(3))
    E = len(state)
    co = PR.gains_of(ctl._P).numpy()
    gains = co[None, :] * rng.uniform(0.8, 1.2, (E, 18))
    up = float(env.HOVER_RPM) * rng.uniform(0.8, 1.2, (E, 4))
    return _place(env, ctl, state, pid, tg, up, gains, rng), np.repeat(SCENARIOS, PER)


def _tick_inputs(env, L, lin, k):
    """The kernel's own inputs of tick k per drone, as ref_ctrl_tick_jac takes them: (rows, gains, x_k, s_k, targets, u_{k-1}).
    x_k is the stored state after tick k - 1, s_k = pid_state[k], u_{k-1} the applied RPMs of tick k - 1 (last_rpm at k = 0)."""
    from gym_pybullet_drones_b200.params import PHYS_KEYS, physical_rows
    n, D = env._N, env._D
    d = {key: v.detach() for key, v in L.items()}
    rows = physical_rows(env.DRONE_MODEL, {key: d[key] for key in PHYS_KEYS}, env.G).repeat_interleave(D, dim=0)
    gains = torch.cat([d[g] for g in GAIN_KEYS], dim=1).repeat_interleave(D, dim=0)
    src = d if k == 0 else {s: lin[s][k - 1] for s in STATE_KEYS}
    x = torch.cat([src[s].reshape(n, -1) for s in STATE_KEYS], dim=1)
    s = lin["pid_state"][k].reshape(n, 9)
    tg = torch.cat([(d["waypoints"][0] + d["offset"]).reshape(n, 3), d["target_rpy"].reshape(n, 3)[:, 2:3], d["target_vel"].reshape(n, 3),
                    d["target_rpy_rates"].reshape(n, 3)], dim=1)
    up = (d["last_rpm"] if k == 0 else lin["rpm"][k - 1]).reshape(n, 4)
    return rows, gains, x, s, tg, up


def _ref_jac(env, ctl, ins, flip=()):
    return ref_ctrl_tick_jac(env._P, ctl._P, env._effects, env.PYB_STEPS_PER_CTRL, env.CTRL_TIMESTEP, *ins, flip=flip, device=env.device)


def _kernel_blocks(lin, k, drag):
    """{block: [n, 26, width]} of linearise's tick k in ref_ctrl_tick_jac's layout (targets: target_pos only)"""
    top = torch.cat([lin["A"][k], lin["B"][k]], dim=-1)
    J = top if drag else torch.cat([top, torch.cat([lin["K"][k], lin["K_target"][k]], dim=-1)], dim=-2)
    J = J.reshape(-1, 26, J.shape[-1]).cpu().numpy()
    out = dict(state=J[..., 0:13], pid=J[..., 13:22], targets=J[..., -3:])
    if drag:
        out["last_rpm"] = J[..., 22:26]
    return out


def _per_drone(got, want):
    """{block: [n] per-drone relative errors}"""
    return {b: per_drone_relerr(got[b], want[b][..., :3] if b == "targets" else want[b]) for b in got}


def _probe(env, ctl, ins):
    """diff_pid_ref's decision inputs (scalar, sarg, torque and PWM before their clips) at the tick inputs `ins`"""
    rows, gains, x, s, tg, up = ins
    probe = {}
    PR.pid(PR.controller_constants(ctl._P, env.device), gains, s, env.CTRL_TIMESTEP, x, tg[:, 0:3], tg[:, 3], tg[:, 4:7], tg[:, 7:10],
           probe=probe)
    return {k: v.cpu().numpy() for k, v in probe.items()}


def _decisions_taken(env, ctl, L, lin, names):
    """Each scenario's decision on the device: the integral clips and the PWM clip from the kernel's outputs, the thrust scalar,
    the gimbal guard and the torque clip from the reference's predicates at the kernel's own tick inputs"""
    T = lin["rpm"].shape[0]
    pid = lin["pid_state"].reshape(T, -1, 9).cpu().numpy()
    at = lambda m: np.concatenate([np.abs(pid[1:, m, 0:2]) == 2.0, np.abs(pid[1:, m, 2:3]) == 0.15, np.abs(pid[1:, m, 6:8]) == 1.0], -1)
    clipped = at(names == "integral")                                   # after ticks 0 .. T - 2, per drone and clipped entry
    assert clipped.any() and not clipped.all(), clipped
    Cc = PR.controller_constants(ctl._P)
    hi, lo = Cc["scale"] * Cc["max_pwm"] + Cc["const"], Cc["scale"] * Cc["min_pwm"] + Cc["const"]
    rpm = lin["rpm"].reshape(T, -1, 4).cpu().numpy()[:, names == "pwm"]
    sat = (rpm == hi) | (rpm == lo)
    assert sat.any(), (rpm, hi, lo)
    seen = {"scalar": [], "gimbal": [], "torque": []}
    for k in range(T):
        p = _probe(env, ctl, _tick_inputs(env, L, lin, k))
        seen["scalar"].append(p["scalar"][names == "scalar"] <= 0)
        seen["gimbal"].append(np.abs(p["sarg"][names == "gimbal"]) >= 0.99999)
        seen["torque"].append((np.abs(p["torque"][names == "torque"]) > 3200).any(1))
    for k, v in seen.items():
        assert np.any(v[0]), k                                          # tick 0 at least
    return {"integral": int(clipped.any(axis=(0, 2)).sum()), "pwm": int(sat.any(axis=(0, 2)).sum())} | {k: int(np.sum(v[0])) for k, v in seen.items()}


@pytest.mark.parametrize("model,physics,ctrl", CONFIGS)
def test_linearise_matches_reference_at_the_scenarios(model, physics, ctrl):
    """A, B, K and K_target of every tick of T = 3 against jacfwd of the reference at the kernel's tick-k inputs, per drone and
    input block (x, s, u_{k-1}, target_pos); each scenario's decision is taken on the device"""
    from gym_pybullet_drones_b200 import _native as N
    E, T = PER * len(SCENARIOS), 3
    env, ctl = _env(E, 1, physics, model, 240, ctrl)
    L, names = _scenario_leaves(env, ctl, model, CONFIGS.index((model, physics, ctrl)))
    lin = _lin(env, ctl, L, T, None)
    assert torch.equal(lin["pid_state"][0], torch.cat([L[k].detach() for k in PID_KEYS], dim=-1))
    drag = bool(env._effects & N.EFFECT_DRAG)
    worst = {}
    for k in range(T):
        err = _per_drone(_kernel_blocks(lin, k, drag), _ref_jac(env, ctl, _tick_inputs(env, L, lin, k)))
        for b, e in err.items():
            for s in SCENARIOS:
                worst[(s, b)] = max(worst.get((s, b), 0.0), float(e[names == s].max()))
    taken = _decisions_taken(env, ctl, L, lin, names)
    w = max(worst, key=worst.get)
    print("ctrl linearise %s %s %d Hz: worst per-drone error %.1e (%s %s); decisions taken by %s drones" % (model, physics, ctrl, worst[w],
          *w, taken))
    assert worst[w] <= JVP_TOL, worst


def _blocks():
    from gym_pybullet_drones_b200.params import PHYS_KEYS
    b = {"state": STATE_KEYS, "pid_state": PID_KEYS, "waypoints": ("waypoints",), "offset": ("offset",), "target_rpy": ("target_rpy",),
         "target_vel": ("target_vel",), "target_rpy_rates": ("target_rpy_rates",)}
    b.update({g: (g,) for g in GAIN_KEYS})
    b.update({"phys": PHYS_KEYS, "last_rpm": ("last_rpm",)})
    return b


def _per_drone_out(d, E):
    """{key: [T, E, 1, k]} -> {key: [E, T k]}"""
    return {k: v.detach().transpose(0, 1).reshape(E, -1).cpu().numpy() for k, v in d.items()}


@pytest.mark.parametrize("model,physics,ctrl", CONFIGS)
def test_trajectory_tangents_and_gradients_at_the_scenarios(model, physics, ctrl):
    """Forward AD through differentiable_rollout(controller=) against torch.func.jvp of diff_pid_ref.closed_loop, one direction
    per input block (phys as d / d log c; the reference's directions batched with vmap), and torch.autograd.grad against the reference's autograd per input block, per drone
    and output: T = 4 at 30 Hz, T = 32 at 240 Hz.  Without drag last_rpm's tangents and gradients are exactly zero."""
    from gym_pybullet_drones_b200.params import PHYS_KEYS
    E, T = PER * len(SCENARIOS), 4 if ctrl == 30 else 32
    env, ctl = _env(E, 1, physics, model, 240, ctrl)
    L, names = _scenario_leaves(env, ctl, model, 100 + CONFIGS.index((model, physics, ctrl)))
    Ld = {k: v.detach() for k, v in L.items()}
    eff = env._effects
    rng = np.random.default_rng(7)
    blocks = _blocks()
    Vs = [{k: torch.tensor(rng.standard_normal(tuple(L[k].shape)), device=env.device) * (Ld[k] if name == "phys" else 1.0) for k in keys}
          for name, keys in blocks.items()]
    ref = batched_jvp(lambda d: _ref(env, ctl, d, T, None, eff), Ld, Vs)
    fwd = {}
    for j, (name, V) in enumerate(zip(blocks, Vs)):
        _, tan = _jvp(env, ctl, L, V, T, None)
        got, want = _per_drone_out(tan, E), _per_drone_out({k: v[j] for k, v in ref.items()}, E)
        fwd[name] = max(float(per_drone_relerr(got[k], want[k]).max()) for k in got)
    out = _call(env, ctl, L, T, None)
    g = {k: torch.tensor(rng.standard_normal(tuple(v.shape)), device=env.device) for k, v in out.items()}
    got, want = _grads(out, L, g), _grads(_ref(env, ctl, L, T, None, eff), L, g)
    bwd = {}
    for name, keys in _blocks().items():
        if name == "phys":                                              # d / d log c
            a = torch.stack([got[k] * Ld[k] for k in PHYS_KEYS], 1)
            b = torch.stack([want[k] * Ld[k] for k in PHYS_KEYS], 1)
        else:
            a = torch.cat([got[k].reshape(E, -1) for k in keys], 1)
            b = torch.cat([want[k].reshape(E, -1) for k in keys], 1)
        bwd[name] = float(per_drone_relerr(a.cpu().numpy(), b.cpu().numpy()).max())
    wf, wb = max(fwd, key=fwd.get), max(bwd, key=bwd.get)
    print("ctrl trajectory %s %s %d Hz T=%d: forward AD worst %.1e (%s), gradients worst %.1e (%s)" % (model, physics, ctrl, T, fwd[wf], wf,
                                                                                                        bwd[wb], wb))
    assert fwd[wf] <= GRAD_TOL, fwd
    assert bwd[wb] <= GRAD_TOL, bwd


@pytest.mark.parametrize("model", ["CF2X", "CF2P"])
def test_one_ulp_either_side_of_the_decisions(model):
    """test_ctrl_jvp_host's lattice on the device: drones one ulp below, at and above the integral clips, scalar = 0 and the
    gimbal guard (MIN_PWM low enough that the thrust is not saturated).  The device may round across a bound, so the side is
    read from the kernel: an integral stored inside its bound passes the tangent, one stored at the bound may go either way and
    matches the reference with that decision (plain, or flip "integral": the tangent passed); scalar and the guard match the
    reference whose predicate at the kernel's tick-0 state decides.  Both sides occur for every decision."""
    from test_ctrl_jvp_host import DT, _lattice
    P, CP, rows, gains, state, pid, tg, up, label = _lattice(model.lower(), np.random.default_rng(61 if model == "CF2X" else 62))
    env, ctl = _env(len(state), 1, "DYN", model, 240, 48)
    assert env.CTRL_TIMESTEP == DT
    ctl._P = CP
    L = _place(env, ctl, state, pid, tg, up, gains)
    lin = _lin(env, ctl, L, 2, None)
    ins = _tick_inputs(env, L, lin, 0)
    got = _kernel_blocks(lin, 0, False)
    p = _probe(env, ctl, ins)
    pid1 = lin["pid_state"][1].reshape(-1, 9).cpu().numpy()
    worst = 0.0
    for name in np.unique(label):
        i = np.flatnonzero(label == name)
        decision = "integral" if name[:2] in ("ip", "ir") else str(name)
        plain = _per_drone(got, _ref_jac(env, ctl, ins))
        flip = _per_drone(got, _ref_jac(env, ctl, ins, (decision,)))
        ep = np.max([plain[b][i] for b in plain], 0)
        ef = np.max([flip[b][i] for b in flip], 0)
        if decision == "integral":
            col, bound = (int(name[2]), float(name[3:])) if name[1] == "p" else (6, float(name[2:]))
            inside = np.abs(pid1[i, col]) < abs(bound)
            passed = ef <= JVP_TOL
            assert np.all(np.minimum(ep, ef) <= JVP_TOL), (name, ep, ef)
            assert np.all(passed[inside]), (name, ep, ef)
            sides = passed
        else:
            assert np.all(ep <= JVP_TOL), (name, ep)
            sides = p["scalar"][i] > 0 if decision == "scalar" else np.abs(p["sarg"][i]) >= 0.99999
        worst = max(worst, float(np.minimum(ep, ef).max()))
        assert sides.any() and not sides.all(), (name, sides, ep, ef)
    print("ctrl one-ulp lattice %s: worst per-drone error %.1e on the side the kernel took" % (model, worst))


@pytest.mark.parametrize("decision", ["integral", "pwm", "torque", "gimbal", "scalar"])
def test_negative_controls_miss_the_device(decision):
    """Each diff_pid_ref flip misses the device Jacobian of its own scenario by more than 1e-4, where the unflipped reference
    meets it (scalar: a MIN_PWM low enough that the thrust is not saturated, as the host test has it)"""
    env, ctl = _env(PER * len(SCENARIOS), 1, "DYN", "CF2X", 240, 48)
    if decision == "scalar":
        ctl._P = copy.copy(ctl._P)
        ctl._P.pid_min_pwm = -1e5
    L, names = _scenario_leaves(env, ctl, "CF2X", 21)
    lin = _lin(env, ctl, L, 1, None)
    ins = _tick_inputs(env, L, lin, 0)
    got = _kernel_blocks(lin, 0, False)
    m = names == decision
    good = max(float(e[m].max()) for e in _per_drone(got, _ref_jac(env, ctl, ins)).values())
    miss = max(float(e[m].max()) for e in _per_drone(got, _ref_jac(env, ctl, ins, (decision,))).values())
    print("ctrl negative control %s: %.1e against the reference, %.1e against the flipped one" % (decision, good, miss))
    assert good <= JVP_TOL
    assert miss > 1e-4, (decision, miss)
