"""-m gpu: the differentiable-trajectory kernels (dyn_traj_kernel<EFF>, dyn_traj_vjp_kernel<EFF>, DESIGN.md 4.5) at every decision
of the adjoint, per drone against the float64 torch reference tests/diff_ref.py on the same device.

Every comparison is the per-drone normwise relative error of each input block separately (rpm over all ticks, state0's pos /
quat / vel / rpy_rates, last_rpm, the 16-column row per aviary), and exactly zero where the reference's gradient is zero by
construction.  Covered: the scenario matrix of the host tests (diff_testlib.scenarios) through the device for every effect set,
GND|DRAG included, and S = 1, 5, 8, 24, with one tick also against the g++ build of the same adjoint; the forward of GND|DRAG
against the reference, the NumPy oracle and step(); the decision lattices (diff_testlib.lattices) on the device; partial CTAs
and aviaries of 1 to 7 drones; the C ABI's optional pointers; non-unit quaternions; long horizons; a negative control for each."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

import diff_ref as R
from diff_testlib import (MODELS, SIDE_PAIRS, aviary_rows, check_lattice, host_tick_vjp, lattices, params_of, per_drone_relerr,
                          quat_from_rpy, ref_tick_vjp, scenario_ticks, split_grads, worst_per_block)

pytestmark = pytest.mark.gpu

EFFECTS = {"dyn": 0, "gnd": R.EFFECT_GND, "drag": R.EFFECT_DRAG, "gnd_drag": R.EFFECT_GND | R.EFFECT_DRAG}
VJP_TOL = 1e-10          # per drone, T <= 8 (the host bound)
LONG_TOL = 1e-9          # per drone, long horizons
DEV = "cuda"


def _planes(x):
    """[..., n, 13] drones -> [..., 13 n] planes (diff.pack_state per leading index)."""
    from gym_pybullet_drones_b200.diff import pack_state
    x = torch.as_tensor(np.asarray(x, dtype=np.float64), device=DEV) if not isinstance(x, torch.Tensor) else x
    if x.dim() == 2:
        return pack_state(x[:, 0:3], x[:, 3:7], x[:, 7:10], x[:, 10:13]).contiguous()
    return torch.stack([_planes(t) for t in x])


def _drones(planes, n):
    """[..., 13 n] planes -> [..., n, 13] drones."""
    from gym_pybullet_drones_b200.diff import unpack_states
    u = unpack_states(planes, n)
    return torch.cat([u["pos"], u["quat"], u["vel"], u["rpy_rates"]], dim=-1)


def abi_vjp(P, E, D, S, eff, state, rpm, last, rows, g_states, null=()):
    """qs_dyn_traj, then qs_dyn_traj_vjp, through ctypes on torch buffers: state [n, 13], rpm [T, n, 4], last [n, 4], rows
    [E, 16], g_states [T, n, 13].  `null`: the optional pointers passed as NULL (phys, last_rpm, g_last_rpm, g_phys).  Returns
    numpy (states [T, n, 13], g_rpm [T, n, 4], g_state0 [n, 13], g_last [n, 4] or None, g_phys [n, 16] or None)."""
    from gym_pybullet_drones_b200 import _native as N
    t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64), device=DEV).contiguous()
    n = E * D
    rpm, last, rows = t(rpm), t(last), t(rows)
    T = rpm.shape[0]
    planes0, g_planes = _planes(t(state)), _planes(t(g_states))
    f64 = dict(dtype=torch.float64, device=DEV)
    states = torch.full((T, 13 * n), np.nan, **f64)
    g_rpm, g_state0 = torch.full((T, n, 4), np.nan, **f64), torch.full((13 * n,), np.nan, **f64)
    g_last, g_phys = torch.full((n, 4), np.nan, **f64), torch.full((n, 16), np.nan, **f64)
    scratch = torch.empty((S, 13, n), **f64)
    io = N.QsDynTrajIO()
    io.T = T
    io.state0, io.rpm, io.states = planes0.data_ptr(), rpm.data_ptr(), states.data_ptr()
    io.last_rpm = None if "last_rpm" in null else last.data_ptr()
    io.phys = None if "phys" in null else rows.data_ptr()
    stream = torch.cuda.current_stream().cuda_stream
    N.check(N.lib().qs_dyn_traj(C.byref(P), C.byref(io), E, D, S, eff, stream), "qs_dyn_traj")
    io.g_states, io.g_rpm, io.g_state0, io.scratch = g_planes.data_ptr(), g_rpm.data_ptr(), g_state0.data_ptr(), scratch.data_ptr()
    io.g_last_rpm = None if "g_last_rpm" in null else g_last.data_ptr()
    io.g_phys = None if "g_phys" in null else g_phys.data_ptr()
    N.check(N.lib().qs_dyn_traj_vjp(C.byref(P), C.byref(io), E, D, S, eff, stream), "qs_dyn_traj_vjp")
    torch.cuda.synchronize()
    c = lambda x: x.cpu().numpy()
    return (c(_drones(states, n)), c(g_rpm), c(_drones(g_state0, n)), None if "g_last_rpm" in null else c(g_last),
            None if "g_phys" in null else c(g_phys))


def ref_rollout(P, D, S, eff, state, rpm, last, rows, g_states, **kw):
    """diff_ref.rollout's autograd on the device: (states [T, n, 13], {block: gradient}), the row gradient per aviary [E, 16]."""
    t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64), device=DEV)
    x, r, u, rw = (t(a).requires_grad_(True) for a in (state, rpm, last, rows))
    out = R.rollout(R.model_constants(P, DEV), rw.repeat_interleave(D, dim=0), x, r, u, S, eff, **kw)
    gs = torch.autograd.grad(out, (x, r, u, rw), t(g_states), allow_unused=True)
    gs = [torch.zeros_like(v) if g is None else g for g, v in zip(gs, (x, r, u, rw))]
    return out.detach().cpu().numpy(), split_grads(gs[1].cpu().numpy(), gs[0].cpu().numpy(), gs[2].cpu().numpy(), gs[3].cpu().numpy())


def _fmt(d):
    return {k: "%.1e" % v for k, v in d.items()}


# ---- 1. the scenario matrix through the device kernels ----------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def _matrix_inputs(model, T, n_per=128, D=2):
    """Six scenarios x n_per drones, D drones per aviary with random rows; T ticks in each scenario's regime."""
    P, c = params_of(model)
    n = 6 * n_per
    rng = np.random.default_rng([MODELS.index(model), T])
    _, rows = aviary_rows(model, n // D, rng)
    names, state, raw, up = scenario_ticks(c, rows.numpy().repeat(D, axis=0), T, MODELS.index(model), n_per)
    return P, c, rows.numpy(), names, state, raw, up, rng.standard_normal((T, n, 13))


def _subset(inputs, keep, T):
    """The drones `keep` (whole aviaries) of _matrix_inputs over its first T ticks: (names, state, raw, up, rows, g)."""
    P, c, rows, names, state, raw, up, g = inputs
    D = len(names) // len(rows)
    return names[keep], state[keep], raw[:T, keep], up[keep], rows[keep.reshape(-1, D).all(1)], g[:T, keep]


def tumbling_ticks(S):
    """Ticks of the tumbling scenario in the matrix.  At 250-300 rad/s about body z the explicit Euler step of w x Jw grows the
    transverse rates every substep (CF2X: |w| reaches 2e3 after 4 ticks at S = 8 and 1e9 at S = 24), and the reference's own
    gradient becomes as ill-conditioned as the trajectory.  The tumbling drones run T S <= 24 substeps (the host tests' longest
    tick), where a 1-ulp change of the state moves the reference's gradient by < 1e-14."""
    return max(1, min(4, 24 // S))


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("eff", list(EFFECTS))
@pytest.mark.parametrize("S", [1, 5, 8, 24])
def test_scenario_matrix_matches_reference_per_drone(model, eff, S):
    """T = 4 ticks (tumbling: tumbling_ticks(S)) of the six scenarios, 128 drones each in aviaries of 2 with random rows,
    through DynTrajectory.apply, per drone against the reference's autograd on the device; one tick also against the g++ build."""
    from gym_pybullet_drones_b200.diff import DynTrajectory
    D = 2
    inputs = _matrix_inputs(model, 4)
    P, c = inputs[0], inputs[1]
    effects = EFFECTS[eff]
    tumbling = inputs[3] == "tumbling"
    for keep, T in ((~tumbling, 4), (tumbling, tumbling_ticks(S))):
        names, state, raw, up, rows, g = _subset(inputs, keep, T)
        n = state.shape[0]
        E = n // D
        t = lambda a: torch.tensor(a, device=DEV)
        # rpm as a strided view ([n, T, 4] storage): DynTrajectory once passed such a tensor's data_ptr to the kernels as if dense
        leaves = [t(np.ascontiguousarray(raw.transpose(1, 0, 2))).transpose(0, 1), _planes(state), t(up), t(rows)]
        assert T == 1 or not leaves[0].is_contiguous()
        leaves = [x.requires_grad_(True) for x in leaves]
        out = DynTrajectory.apply(leaves[0], leaves[1], leaves[2], leaves[3], (P, E, D, S, effects))
        gr = torch.autograd.grad(out, leaves, _planes(g))
        got = split_grads(gr[0].cpu().numpy(), _drones(gr[1], n).cpu().numpy(), gr[2].cpu().numpy(), gr[3].cpu().numpy())
        fwd, want = ref_rollout(P, D, S, effects, state, raw, up, rows, g)
        e_fwd = per_drone_relerr(np.moveaxis(_drones(out.detach(), n).cpu().numpy(), 0, 1), np.moveaxis(fwd, 0, 1))
        worst = worst_per_block(got, want)
        worst["forward"] = float(e_fwd.max())
        by = {s: max(float(np.max(per_drone_relerr(got[k][names == s], want[k][names == s]))) for k in got if k != "row")
              for s in dict.fromkeys(names)}
        print("matrix %s %s S=%d T=%d: worst per-drone error %s; by scenario %s" % (model, eff, S, T, _fmt(worst), _fmt(by)))
        # zero by construction: clipped RPM entries, last_rpm without drag; no radial part in the quaternion's gradient
        clipped = (raw < 0) | (raw > rows.repeat(D, axis=0)[None, :, 13:14])
        assert np.all(gr[0].cpu().numpy()[clipped] == 0)
        if not effects & R.EFFECT_DRAG:
            assert np.all(got["last_rpm"] == 0)
        radial = np.abs(np.sum(got["quat"] * state[:, 3:7], axis=1)) / np.linalg.norm(got["quat"], axis=1)
        assert radial.max() <= 1e-12, radial.max()
        assert worst["forward"] <= 1e-12
        for k, e in worst.items():
            assert e <= VJP_TOL, (k, e)

        # one tick against the g++ build of the same adjoint: tells "the device build differs" from "the adjoint is wrong"
        dev = abi_vjp(P, E, D, S, effects, state, raw[:1], up, rows, g[:1])
        host = host_tick_vjp(P, effects, S, state, raw[0], up, g[0], rows.repeat(D, axis=0))
        e_host = worst_per_block(split_grads(dev[1][0], dev[2], dev[3], dev[4]), split_grads(host[2], host[1], host[3], host[4]))
        e_host["forward"] = float(np.max(per_drone_relerr(dev[0][0], host[0])))
        print("   T=1 device against the host build: %s" % _fmt(e_host))
        for k, e in e_host.items():
            assert e <= 1e-12, (k, e)


@pytest.mark.parametrize("model", MODELS)
def test_forward_gnd_drag_matches_reference_oracle_and_step(model):
    """dyn_traj_kernel<GND|DRAG> against diff_ref and the NumPy oracle (effects = 3), and against step() of a one-drone
    PYB_GND_DRAG_DW aviary, which has no downwash pair: bit for bit at 240/240 Hz.  At S > 1 that env runs its substeps one
    dyn_tick_k call at a time (the in-CTA downwash loop), so it renormalises the quaternion on every substep, not once per tick:
    there the two agree to rounding only."""
    from oracle import dyn_oracle as O
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.params import nominal_properties, physical_rows
    from diff_testlib import drone_model
    from gym_pybullet_drones_b200.utils.enums import Physics
    T, S = 4, 5
    inputs = _matrix_inputs(model, T)
    P, c, names = inputs[0], inputs[1], inputs[3]
    keep = (names != "hover") & (names != "tumbling")   # the oracle's isclose identity; tumbling: tumbling_ticks
    _, state, raw, up, _, _ = _subset(inputs, keep, T)
    n = int(keep.sum())
    up = np.minimum(up, float(c.MAX_RPM))
    nom = nominal_properties(drone_model(model))
    rows = physical_rows(drone_model(model), {k: torch.full((n,), v, dtype=torch.float64) for k, v in nom.items()}).numpy()
    got = abi_vjp(P, n, 1, S, 3, state, raw, up, rows, np.zeros((T, n, 13)))[0]
    fwd, _ = ref_rollout(P, 1, S, 3, state, raw, up, rows, np.zeros((T, n, 13)))
    OP = O.OracleParams({"race": "racer"}.get(model, model))
    x, u_prev, ora = state.copy(), up.copy(), []
    for k in range(T):
        u = np.clip(raw[k], 0, OP.MAX_RPM)
        pos, quat, vel, w = x[:, 0:3], x[:, 3:7], x[:, 7:10], x[:, 10:13]
        for s in range(S):
            pos, quat, vel, w, _ = O.dynamics_substep(OP, u, pos, quat, vel, w, 3, rpm_prev=u_prev if s == 0 else u)
        x, u_prev = np.concatenate([pos, quat, vel, w], axis=1), u
        ora.append(x)
    ora = np.stack(ora)
    e_ref = float(np.max(np.abs(got - fwd) / np.maximum(np.abs(fwd), 1.0)))
    e_ora = float(np.max(np.abs(got - ora) / np.maximum(np.abs(ora), 1.0)))
    print("forward GND|DRAG %s: against the reference %.1e, the oracle %.1e" % (model, e_ref, e_ora))
    assert e_ref <= 1e-13 and e_ora <= 1e-13

    for ctrl, bits in ((240, True), (48, False)):
        env = CtrlAviary(drone_model=drone_model(model), num_drones=1, physics=Physics.PYB_GND_DRAG_DW, pyb_freq=240, ctrl_freq=ctrl,
                         num_envs=n)
        env.reset()
        t = lambda a: torch.tensor(a, device=DEV).reshape(n, 1, -1)
        env.set_state(t(state[:, 0:3]), t(state[:, 3:7]), t(state[:, 7:10]), t(state[:, 10:13]))
        env._last_rpm.copy_(t(up).reshape(env._last_rpm.shape))
        start = torch.cat([env.pos, env.quat, env.vel, env.rpy_rates], dim=-1).reshape(n, 13).cpu().numpy()
        Pe = env._P
        kern = abi_vjp(Pe, n, 1, env.PYB_STEPS_PER_CTRL, 3, start, raw, env._last_rpm.reshape(n, 4).cpu().numpy(), rows, np.zeros((T, n, 13)),
                       null=("phys",))[0]
        worst, same = 0.0, True
        for k in range(T):
            env.step(t(raw[k]).reshape(n, 1, 4))
            st = torch.cat([env.pos, env.quat, env.vel, env.rpy_rates], dim=-1).reshape(n, 13).cpu().numpy()
            same &= bool(np.array_equal(st, kern[k]))
            worst = max(worst, float(np.max(np.abs(st - kern[k]) / np.maximum(np.abs(st), 1.0))))
        print("   step() of PYB_GND_DRAG_DW, D = 1, 240/%d Hz: bit-identical %s, worst %.1e" % (ctrl, same, worst))
        assert same if bits else worst <= 1e-13


# ---- 2. decision lattices -----------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def _lattices(model):
    P, c = params_of(model)
    _, rows = aviary_rows(model, 64, np.random.default_rng(20))
    return P, lattices(P, c, rows.numpy(), np.random.default_rng(21))


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("name", ["rpm", "clip", "half_angle", "upright"])
def test_lattice_on_device(model, name):
    """Each lattice drone is its own aviary (MAX_RPM is the row's).  Against the reference on the device, against the g++
    build, and with the negative controls of the RPM clip (strict at MAX_RPM) and the height clip (hz <= clip)."""
    P, L = _lattices(model)
    lat = L[name]
    n = len(lat["state"])
    d = abi_vjp(P, n, 1, lat["S"], lat["effects"], lat["state"], lat["raw"][None], lat["up"], lat["rows"], lat["g_out"][None])
    got = [d[0][0], d[2], d[1][0], d[3], d[4]]
    args = (lat["effects"], lat["S"], lat["state"], lat["raw"], lat["up"], lat["g_out"])
    want = ref_tick_vjp(P, lat["rows"], *args, device=DEV)
    fwd = ref_tick_vjp(P, lat["rows"], *args, device=DEV, exact_branch=True)[0] if name == "half_angle" else want[0]
    worst = check_lattice(name, lat, got, want, fwd, VJP_TOL)
    host = host_tick_vjp(P, *args, lat["rows"])
    e_host = max(float(np.max(per_drone_relerr(a, b))) for a, b in zip(got, host))
    print("device lattice %s %s: worst per-drone error %s, against the host build %.1e" % (model, name, _fmt(worst), e_host))
    assert e_host <= 1e-12
    for a, b in SIDE_PAIRS.get(name, []):           # the two sides of the decision differ in the gradient
        assert float(per_drone_relerr(got[1][a:a + 1], got[1][b:b + 1])[0] + per_drone_relerr(got[2][a:a + 1], got[2][b:b + 1])[0]) >= 1e-3
    controls = {"rpm": (dict(strict_clamp=True), lat["label"] == 1, 2), "clip": (dict(gnd_clip_le=True), lat["label"] == 0, 1)}
    if name in controls:
        kw, at, blk = controls[name]
        e = per_drone_relerr(got[blk], ref_tick_vjp(P, lat["rows"], *args, device=DEV, **kw)[blk])
        print("   negative control %s: at the boundary >= %.1e, elsewhere <= %.1e" % (kw, e[at].min(), e[~at].max()))
        assert e[at].min() >= 1e-3 and e[~at].max() <= VJP_TOL


# ---- 3. shapes and optional pointers ------------------------------------------------------------------------------------

@pytest.mark.parametrize("E,D,physics,model", [(37, 3, "PYB_GND", "CF2X"), (129, 1, "PYB_DRAG", "CF2P"), (5, 7, "DYN", "RACE"),
                                               (1, 1, "PYB", "CF2X")])
def test_partial_cta_per_aviary_constants(E, D, physics, model):
    """N not a multiple of 128 (the last CTA partial) and 1..7 drones per aviary: the row gradients summed over each aviary's
    drones reach every PHYS_KEYS value, per aviary against the reference."""
    from test_gpu_diff import _env, _ref_grads, _rpm
    from gym_pybullet_drones_b200.params import PHYS_KEYS
    T = 8
    env = _env(E, D, physics, model, 240, 48)
    rng = np.random.default_rng(E * 10 + D)
    props = {k: v * torch.tensor(rng.uniform(0.8, 1.2, E), device=DEV) for k, v in env.physical_params().items()}
    state = {"pos": env.pos.clone(), "quat": env.quat.clone(), "vel": torch.tensor(rng.uniform(-1, 1, (E, D, 3)), device=DEV),
             "rpy_rates": torch.tensor(rng.uniform(-2, 2, (E, D, 3)), device=DEV)}
    last = torch.tensor(env.HOVER_RPM * rng.uniform(0.9, 1.1, (E, D, 4)), device=DEV)
    rpm = _rpm(env, T, rng)
    leaves = [rpm] + [state[k] for k in ("pos", "quat", "vel", "rpy_rates")] + [last] + [props[k] for k in PHYS_KEYS]
    leaves = [x.clone().requires_grad_(True) for x in leaves]
    out = env.differentiable_rollout(leaves[0], state=dict(zip(("pos", "quat", "vel", "rpy_rates"), leaves[1:5])), last_rpm=leaves[5],
                                     phys=dict(zip(PHYS_KEYS, leaves[6:])))
    g = {k: torch.tensor(rng.standard_normal(tuple(v.shape)), device=DEV) for k, v in out.items()}
    got = torch.autograd.grad(sum((out[k] * g[k]).sum() for k in out), leaves)
    want = _ref_grads(env, rpm, state, last, props, g, env._effects)
    names = ["rpm", "pos", "quat", "vel", "rpy_rates", "last_rpm"] + list(PHYS_KEYS)
    worst = {}
    for name, a, b in zip(names, got, want):
        a, b = a.cpu().numpy(), b.cpu().numpy()
        if name == "rpm":
            a, b = np.moveaxis(a, 0, 2), np.moveaxis(b, 0, 2)             # [E, D, T, 4]: per drone below
        worst[name] = float(np.max(per_drone_relerr(a.reshape(E * D, -1) if a.ndim > 1 else a, b.reshape(E * D, -1) if b.ndim > 1 else b)))
    print("partial CTA E=%d D=%d %s: worst per-drone / per-aviary error %s" % (E, D, physics, _fmt(worst)))
    for name, e in worst.items():
        assert e <= VJP_TOL, (name, e)


def test_abi_optional_pointers():
    """phys = NULL is the nominal row bit for bit; last_rpm = NULL is zeros; g_last_rpm = NULL and g_phys = NULL leave every
    other output as it was.  GND|DRAG, 333 drones in aviaries of 3."""
    from gym_pybullet_drones_b200.params import nominal_properties, physical_rows
    from diff_testlib import drone_model
    P, c = params_of("cf2x")
    E, D, T, S = 111, 3, 3, 5
    n = E * D
    rng = np.random.default_rng(30)
    nom = nominal_properties(drone_model("cf2x"))
    rows = physical_rows(drone_model("cf2x"), {k: torch.full((E,), v, dtype=torch.float64) for k, v in nom.items()}).numpy()
    names, state, raw, up = scenario_ticks(c, np.repeat(rows[:1], 6 * (n // 6 + 1), axis=0), T, 31, n // 6 + 1)
    state, raw, up = state[:n], raw[:, :n], up[:n]
    g = rng.standard_normal((T, n, 13))
    full = abi_vjp(P, E, D, S, 3, state, raw, up, rows, g)
    same = lambda a, b: all(np.array_equal(x, y) for x, y in zip(a, b) if x is not None and y is not None)
    assert same(full, abi_vjp(P, E, D, S, 3, state, raw, up, rows, g, null=("phys",)))
    assert same(abi_vjp(P, E, D, S, 3, state, raw, np.zeros_like(up), rows, g), abi_vjp(P, E, D, S, 3, state, raw, up, rows, g, null=("last_rpm",)))
    part = abi_vjp(P, E, D, S, 3, state, raw, up, rows, g, null=("g_last_rpm", "g_phys"))
    assert part[3] is None and part[4] is None and same(full[:3], part[:3])
    assert np.all(np.isfinite(full[3])) and np.any(full[3] != 0) and np.all(np.isfinite(full[4]))


def test_non_unit_quaternion():
    """state["quat"] x 1.3, and with one component negated: the forward equals the reference, the gradient matches it per drone
    and has no radial component (the entry renormalisation is part of the function)."""
    inputs = _matrix_inputs("cf2x", 4)
    P = inputs[0]
    names, state, raw, up, rows, g = _subset(inputs, inputs[3] != "tumbling", 4)
    D, S = 2, 8
    state[:, 3:7] *= 1.3
    state[1::2, 4] *= -1.0
    d = abi_vjp(P, len(state) // D, D, S, 3, state, raw, up, rows, g)
    fwd, want = ref_rollout(P, D, S, 3, state, raw, up, rows, g)
    got = split_grads(d[1], d[2], d[3], d[4].reshape(-1, D, 16).sum(1))
    worst = worst_per_block(got, want)
    worst["forward"] = float(np.max(per_drone_relerr(np.moveaxis(d[0], 0, 1), np.moveaxis(fwd, 0, 1))))
    radial = np.abs(np.sum(got["quat"] * state[:, 3:7], axis=1)) / np.linalg.norm(got["quat"], axis=1)
    print("non-unit quaternion: worst per-drone error %s, radial part <= %.1e" % (_fmt(worst), radial.max()))
    assert worst["forward"] <= 1e-12 and radial.max() <= 1e-12
    for k, e in worst.items():
        assert e <= VJP_TOL, (k, e)


@pytest.mark.parametrize("T,S", [(240, 1), (60, 8)])
def test_long_horizon_near_hover_gnd_drag(T, S):
    """Near hover, some drones inside ground effect, with RPMs clipped above MAX_RPM and below 0 at several ticks: drag's
    first substep of the next tick reads the clipped values."""
    P, c = params_of("cf2x")
    E, D = 128, 2
    n = E * D
    rng = np.random.default_rng([T, S])
    _, rows = aviary_rows("cf2x", E, rng)
    rows = rows.numpy()
    hv = rows.repeat(D, axis=0)[:, 12]
    state = np.zeros((n, 13))
    state[:, 0:2] = rng.uniform(-1, 1, (n, 2))
    state[:, 2] = rng.uniform(0.02, 0.3, n)
    state[:, 3:7] = quat_from_rpy(rng.uniform(-0.05, 0.05, (n, 3)))
    state[:, 7:10] = rng.uniform(-0.1, 0.1, (n, 3))
    raw = hv[None, :, None] * (1 + 0.02 * rng.uniform(-1, 1, (T, n, 4)))
    spikes = [T // 8, 3 * T // 8, 5 * T // 8, 7 * T // 8]
    mx = rows.repeat(D, axis=0)[:, 13]
    for k in spikes:
        raw[k, 0::2, 0] = 1.2 * mx[0::2]
        raw[k, 1::2, 3] = -50.0
    up = hv[:, None] * np.ones((n, 4))
    g = rng.standard_normal((T, n, 13))
    d = abi_vjp(P, E, D, S, 3, state, raw, up, rows, g)
    fwd, want = ref_rollout(P, D, S, 3, state, raw, up, rows, g)
    got = split_grads(d[1], d[2], d[3], d[4].reshape(E, D, 16).sum(1))
    worst = worst_per_block(got, want)
    worst["forward"] = float(np.max(per_drone_relerr(np.moveaxis(d[0], 0, 1), np.moveaxis(fwd, 0, 1))))
    print("long horizon T=%d S=%d GND|DRAG: worst per-drone error %s" % (T, S, _fmt(worst)))
    for k in spikes:                      # the clipped entries pass nothing; MAX_RPM of the spiking aviaries receives it
        assert np.all(d[1][k, 0::2, 0] == 0) and np.all(d[1][k, 1::2, 3] == 0)
    assert np.all(got["row"][:, 13] != 0)
    assert worst["forward"] <= 1e-12
    for k, e in worst.items():
        assert e <= LONG_TOL, (k, e)


# ---- 4. negative controls of the device comparisons ---------------------------------------------------------------------

def test_negative_control_isclose_branch_at_hover_on_device():
    """At exact hover, a reference that takes np.isclose's identity (zero attitude derivative) misses the kernel's RPM gradient
    by >= 1e-2 per drone; the exponential map's reference agrees."""
    inputs = _matrix_inputs("cf2x", 4)
    P = inputs[0]
    names, state, raw, up, rows, g = _subset(inputs, inputs[3] == "hover", 4)
    D, S = 2, 8
    g[..., [0, 1, 2, 7, 8, 9, 10, 11, 12]] = 0.0
    d = abi_vjp(P, len(rows), D, S, 0, state, raw, up, rows, g)
    _, good = ref_rollout(P, D, S, 0, state, raw, up, rows, g)
    _, bad = ref_rollout(P, D, S, 0, state, raw, up, rows, g, exact_branch=True)
    e_good = per_drone_relerr(np.moveaxis(d[1], 0, 1), good["rpm"])
    e_bad = per_drone_relerr(np.moveaxis(d[1], 0, 1), bad["rpm"])
    print("negative control isclose branch: exponential map <= %.1e, identity branch >= %.1e" % (e_good.max(), e_bad.min()))
    assert e_good.max() <= VJP_TOL and e_bad.min() >= 1e-2


def test_negative_control_gnd_drag_against_gnd_only_reference():
    """The GND|DRAG gradient against a GND-only reference misses, on every drone."""
    inputs = _matrix_inputs("cf2x", 4)
    P = inputs[0]
    names, state, raw, up, rows, g = _subset(inputs, inputs[3] != "tumbling", 4)
    D, S = 2, 8
    d = abi_vjp(P, len(state) // D, D, S, 3, state, raw, up, rows, g)
    got = split_grads(d[1], d[2], d[3], d[4].reshape(-1, D, 16).sum(1))
    _, good = ref_rollout(P, D, S, 3, state, raw, up, rows, g)
    _, gnd = ref_rollout(P, D, S, 1, state, raw, up, rows, g)
    e_good = worst_per_block(got, good)
    e_vel = per_drone_relerr(got["vel"], gnd["vel"])
    moving = names != "hover"             # at rest drag's force, and so last_rpm's gradient, is zero
    e_last = per_drone_relerr(got["last_rpm"], gnd["last_rpm"])
    print("negative control GND-only reference: GND|DRAG's <= %.1e; GND's vel block >= %.1e, last_rpm missed on %d of %d moving drones"
          % (max(e_good.values()), e_vel.min(), np.count_nonzero(np.isinf(e_last[moving])), moving.sum()))
    assert max(e_good.values()) <= VJP_TOL
    assert e_vel.min() >= 1e-6 and np.all(np.isinf(e_last[moving]))
