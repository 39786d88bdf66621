"""CPU tests of differentiable_rollout(downwash=True) (DESIGN.md 4.5, downwash adjoint): the torch reference tests/diff_dw_ref.py
against the NumPy oracle's downwash flight, against mppi_ref's downwash rollout and against central differences; the kernels'
aviary tick adjoint (dyn_adjoint.cuh and quad_core.cuh, built for the host phase by phase) against the reference's autograd at
every pair decision; negative controls that show the comparison sees each part of the derivative; the C ABI without a GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

import diff_dw_ref as DW
import diff_ref as R
import mppi_ref as MR
from diff_testlib import params_of, per_drone_relerr, quat_from_rpy
from qs_testlib import drone_model, harness

EFFECTS = {"dw": DW.EFFECT_DW, "gnd_drag_dw": DW.EFFECT_GND | DW.EFFECT_DRAG | DW.EFFECT_DW}
VJP_TOL = 1e-10
BLOCKS = ("state", "rpm", "last_rpm", "phys")


def _h():
    L = harness("diff_dw_host")
    L.ddh_tick_vjp.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_int, C.c_int] + [C.c_void_p] * 9
    L.ddh_pair_grad.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    return L


def host_tick_vjp(P, effects, S, state, raw, up, g_out, rows=None):
    """The host-built aviary tick and its VJP: (out, g_state, g_raw, g_up, g_row), per drone."""
    D = state.shape[0]
    a = lambda x: np.ascontiguousarray(x, dtype=np.float64)
    state, raw, up, g_out = a(state), a(raw), a(up), a(g_out)
    rows = None if rows is None else a(rows)
    outs = [np.zeros((D, 13)), np.zeros((D, 13)), np.zeros((D, 4)), np.zeros((D, 4)), np.zeros((D, 16))]
    p = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)
    _h().ddh_tick_vjp(C.addressof(P), p(rows), effects, S, D, p(state), p(raw), p(up), p(g_out), *[p(o) for o in outs])
    return outs


def ref_tick_vjp(P, rows, effects, S, state, raw, up, g_out, **kw):
    """diff_dw_ref's aviary tick and its autograd VJP: (out, g_state, g_raw, g_up, g_row)."""
    t = lambda x: torch.tensor(np.asarray(x, dtype=np.float64))
    x, r, u, rw = (t(v).requires_grad_(True) for v in (state, raw, up, rows))
    out, _ = DW.tick(R.model_constants(P), P, rw, x, r, u, S, effects, state.shape[0], **kw)
    gs = torch.autograd.grad(out, (x, r, u, rw), t(g_out), allow_unused=True)
    gs = [torch.zeros_like(v) if g is None else g for g, v in zip(gs, (x, r, u, rw))]
    return [out.detach().numpy()] + [g.numpy() for g in gs]


def _rows(model, D, rng=None):
    from gym_pybullet_drones_b200.params import nominal_properties, physical_rows
    nom = nominal_properties(drone_model(model))
    rows = physical_rows(drone_model(model), {k: torch.full((D,), v, dtype=torch.float64) for k, v in nom.items()}).numpy()
    if rng is not None:                                  # per-drone constants: the table path
        rows[:, 0] *= rng.uniform(0.8, 1.2, D)
        rows[:, 2] *= rng.uniform(0.8, 1.2, D)
    return rows


def _level_pair(c, D, lo, hi):
    """D level drones at rest with equal hover RPMs: drone 0 at lo, drone 1 at hi (positions [3]), the others 20 m apart in x
    beyond them (no pair with anyone).  Level, at rest and with equal RPMs their xy stay exact over the substeps."""
    st = np.zeros((D, 13))
    st[:, 6] = 1.0
    st[:, 0] = 30.0 + 20.0 * np.arange(D)
    st[:, 2] = 1.0
    st[0, 0:3] = lo
    if D > 1:
        st[1, 0:3] = hi
    st[:, 9] = 0.05
    hover = float(c.HOVER_RPM)
    return st, np.full((D, 4), 1.01 * hover), np.full((D, 4), hover)


def scenarios(P, c, rng, D):
    """{name: (state [D, 13], raw [D, 4], up [D, 4], uniform)} of one aviary at the decisions of the downwash adjoint; `uniform`:
    every drone has the model's nominal row (the pair must stay where it was put)."""
    hover, mx = float(c.HOVER_RPM), float(c.MAX_RPM)

    def state(pos, rpy, vel, w):
        return np.concatenate([pos, quat_from_rpy(rpy), vel, w], axis=1)

    def column(xy):                                      # a stack about 1 m apart in z, where the pair term is strong
        z = 0.5 + 1.0 * np.arange(D) + rng.uniform(-0.1, 0.1, D)
        return np.concatenate([rng.uniform(-xy, xy, (D, 2)), z[:, None]], 1)

    u = lambda lo, hi: hover * rng.uniform(lo, hi, (D, 4))
    out = {}
    out["flight"] = (state(column(0.03), rng.uniform(-0.3, 0.3, (D, 3)), rng.uniform(-1, 1, (D, 3)), rng.uniform(-3, 3, (D, 3))),
                     u(0.9, 1.1), u(0.9, 1.1), False)
    pos = column(0.0)
    pos[:, 0:2] = rng.uniform(-1, 1, 2)                  # exactly stacked: dxy2 = 0 for every pair at the tick's start
    out["stacked"] = (state(pos, rng.uniform(-0.3, 0.3, (D, 3)), rng.uniform(-1, 1, (D, 3)), rng.uniform(-3, 3, (D, 3))),
                      u(0.9, 1.1), u(0.9, 1.1), False)
    rpy = rng.uniform(-0.3, 0.3, (D, 3))
    rpy[0] = [2.2, -0.7, 1.0]                           # body z far off vertical: the pair force is not along world z
    out["tumbling"] = (state(column(0.03), rpy, rng.uniform(-1, 1, (D, 3)), rng.uniform(-3, 3, (D, 3))), u(0.5, 1.5), u(0.5, 1.5), False)
    raw = u(0.9, 1.1)
    raw[:, 0] = mx * rng.uniform(1.01, 1.5, D)
    raw[:, 2] = -hover * rng.uniform(0.01, 0.5, D)
    out["clipped"] = (state(column(0.03), rng.uniform(-0.3, 0.3, (D, 3)), rng.uniform(-1, 1, (D, 3)), rng.uniform(-3, 3, (D, 3))),
                      raw, np.clip(u(0.9, 1.1), 0, mx), False)
    if D >= 2:
        for name, dxy2 in (("dxy2_100-2ulp", _below(100.0, 2)), ("dxy2_100-1ulp", _below(100.0, 1)), ("dxy2_100", 100.0)):
            dx, dy = DW.pair_offset_for(dxy2)
            out[name] = _level_pair(c, D, [0.0, 0.0, 1.0], [dx, dy, 21.0]) + (True,)      # dz = 20: a live term at |dxy| = 10
        out["equal_height"] = _level_pair(c, D, [0.0, 0.0, 1.0], [0.3, -0.2, 1.0]) + (True,)
        out["underflow"] = _level_pair(c, D, [0.0, 0.0, 1.0], [0.5, 0.0, 1.75]) + (True,)   # beta = 0.01: exp(-1250) = 0
        dz = DW.beta_zero_dz(P)
        if dz is not None:
            out["beta_zero"] = _level_pair(c, D, [0.0, 0.0, 0.0], [0.1, 0.0, dz]) + (True,)
    return out


def _below(v, k):
    for _ in range(k):
        v = float(np.nextafter(v, 0.0))
    return v


def _check(P, c, model, eff, S, D, seed):
    rng = np.random.default_rng(seed)
    worst = {}
    for name, (state, raw, up, uniform) in scenarios(P, c, rng, D).items():
        rows = _rows(model, D, None if uniform else rng)
        g_out = rng.standard_normal((D, 13))
        got = host_tick_vjp(P, eff, S, state, raw, up, g_out, rows)
        want = ref_tick_vjp(P, rows, eff, S, state, raw, up, g_out)
        e = float(np.max(per_drone_relerr(got[0], want[0])))
        assert e <= 1e-12, (name, "forward", e)
        for blk, g, w in zip(BLOCKS, got[1:], want[1:]):
            assert np.all(np.isfinite(g)), (name, blk)
            e = float(np.max(per_drone_relerr(g, w)))
            worst[(name, blk)] = e
            assert e <= VJP_TOL, (name, blk, e)
    return worst


# ---- the reference itself ------------------------------------------------------------------------------------------------

def _oracle_tick(O, OP, effects, S, state, raw, up, D):
    """S substeps of the NumPy oracle for aviaries of D drones, the pair force of each substep from its start positions."""
    u = np.clip(raw, 0, OP.MAX_RPM)
    pos, quat, vel, w = state[:, 0:3], state[:, 3:7], state[:, 7:10], state[:, 10:13]
    for s in range(S):
        fz = O.downwash_body_z(OP, pos.reshape(-1, D, 3)).reshape(-1)
        pos, quat, vel, w, _ = O.dynamics_substep(OP, u, pos, quat, vel, w, effects, rpm_prev=up if s == 0 else u, dw_fz=fz)
    return np.concatenate([pos, quat, vel, w], axis=1)


@pytest.mark.parametrize("model", ["cf2x", "cf2p"])
@pytest.mark.parametrize("eff", list(EFFECTS))
def test_reference_forward_matches_oracle_and_mppi_ref(model, eff):
    from oracle import dyn_oracle as O
    P, c = params_of(model)
    OP = O.OracleParams(model)
    rng = np.random.default_rng(1)
    K = R.model_constants(P)
    for D in (2, 3, 5):
        for name, (state, raw, up, _) in scenarios(P, c, rng, D).items():
            if name in ("beta_zero",):
                continue                                  # the oracle's dxy / beta is 0.1 / 0 there: it warns and gives the same 0
            rows = torch.tensor(_rows(model, D))
            up = np.clip(up, 0, OP.MAX_RPM)
            want = _oracle_tick(O, OP, EFFECTS[eff], 5, state, raw, up, D)
            got, _ = DW.tick(K, P, rows, torch.tensor(state), torch.tensor(raw), torch.tensor(up), 5, EFFECTS[eff], D)
            err = np.max(np.abs(got.numpy() - want) / np.maximum(np.abs(want), 1.0))
            assert err <= 1e-12, (name, D, err)
            mr = MR.rollout_dw(K, P, rows, torch.tensor(state), torch.tensor(up), torch.tensor(raw)[None], 5, EFFECTS[eff], D)[0]
            err = float(torch.max(torch.abs(got - mr) / torch.clamp(torch.abs(mr), min=1.0)))
            assert err <= 1e-13, (name, D, err)


def test_reference_gradient_matches_oracle_central_differences():
    """A three-drone stack in flight (every pair acts, away from the predicate): the gradients of one tick, the cross-drone
    ones included, against central differences of the oracle."""
    from oracle import dyn_oracle as O
    P, c = params_of("cf2x")
    OP = O.OracleParams("cf2x")
    OP.MAX_RPM = np.inf
    rng = np.random.default_rng(2)
    D, S, eff = 3, 4, EFFECTS["gnd_drag_dw"]
    state, raw, up, _ = scenarios(P, c, rng, D)["flight"]
    state[:, 2] = [0.12, 0.5, 0.85]
    g_out = rng.standard_normal((D, 13))

    def loss(st, rw, u):
        return float(np.sum(g_out * _oracle_tick(O, OP, eff, S, st, rw, u, D)))

    def central(f, x, scale, rel=1e-6):
        g = np.zeros_like(x)
        for idx in np.ndindex(x.shape):
            h = rel * scale
            xp, xm = x.copy(), x.copy()
            xp[idx] += h; xm[idx] -= h
            g[idx] = (f(xp) - f(xm)) / (2 * h)
        return g

    fd_state = central(lambda s: loss(s, raw, up), state, 1.0)
    fd_raw = central(lambda r: loss(state, r, up), raw, float(c.HOVER_RPM))
    fd_up = central(lambda u: loss(state, raw, u), up, float(c.HOVER_RPM), 1e-2)
    want = ref_tick_vjp(P, _rows("cf2x", D), eff, S, state, raw, up, g_out)
    q = state[:, 3:7]
    fd_state[:, 3:7] -= q * np.sum(q * fd_state[:, 3:7], axis=1, keepdims=True)     # the oracle does not renormalise
    assert R.relerr(want[1], fd_state) < 1e-6
    assert R.relerr(want[2], fd_raw) < 1e-6
    assert R.relerr(want[3], fd_up) < 1e-6
    # the cross-drone part alone: the lower drones' loss w.r.t. the top drone's position
    g_low = g_out.copy()
    g_low[2] = 0.0
    cross = central(lambda s: float(np.sum(g_low * _oracle_tick(O, OP, eff, S, s, raw, up, D))), state, 1.0)[2, 0:3]
    got = ref_tick_vjp(P, _rows("cf2x", D), eff, S, state, raw, up, g_low)[1][2, 0:3]
    assert np.any(got != 0) and R.relerr(got, cross) < 1e-6


# ---- the host-built aviary adjoint against the reference ------------------------------------------------------------------

@pytest.mark.parametrize("model", ["cf2x", "cf2p"])
@pytest.mark.parametrize("eff", list(EFFECTS))
@pytest.mark.parametrize("S", [1, 5, 8])
@pytest.mark.parametrize("D", [1, 2, 3, 5, 8])
def test_aviary_tick_vjp_matches_reference(model, eff, S, D):
    P, c = params_of(model)
    worst = _check(P, c, model, EFFECTS[eff], S, D, hash((model, eff, S, D)) % 2 ** 32)
    print("worst per-drone relative error %s %s S=%d D=%d: %.2e" % (model, eff, S, D, max(worst.values())))


def test_pair_grad_decisions():
    """Stacked drones get finite derivatives with a zero xy part; beta = 0 and an exp underflow give exactly 0."""
    P, _ = params_of("cf2x")
    dz0 = DW.beta_zero_dz(P)
    dz = np.array([0.5, 0.75, dz0 if dz0 is not None else 0.75])
    d2 = np.array([0.0, 0.25, 0.01])
    out = np.zeros((3, 2))
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    _h().ddh_pair_grad(C.addressof(P), p(dz), p(d2), 3, p(out))
    assert np.all(np.isfinite(out[0])) and out[0, 0] != 0 and out[0, 1] != 0
    assert np.all(out[1:] == 0)


# ---- negative controls --------------------------------------------------------------------------------------------------

def _control(name, D=3, S=5, eff=EFFECTS["gnd_drag_dw"], **kw):
    """(host, good reference, controlled reference) on one scenario, g_out on the lowest drone only (drone 0 of the pair
    scenarios; in the stacks the one with the smallest z) so that every other drone's state gradient is a pair term"""
    P, c = params_of("cf2x")
    rng = np.random.default_rng(11)
    state, raw, up, uniform = scenarios(P, c, rng, D)[name]
    rows = _rows("cf2x", D, None if uniform else rng)
    g_out = np.zeros((D, 13))
    g_out[int(np.argmin(state[:, 2]))] = rng.standard_normal(13)
    got = host_tick_vjp(P, eff, S, state, raw, up, g_out, rows)
    good = ref_tick_vjp(P, rows, eff, S, state, raw, up, g_out)
    bad = ref_tick_vjp(P, rows, eff, S, state, raw, up, g_out, **kw)
    return got, good, bad


@pytest.mark.parametrize("kw", [dict(source=False), dict(receiver=False)], ids=["source_dropped", "receiver_dropped"])
def test_negative_control_one_side_of_the_pair(kw):
    got, good, bad = _control("flight", **kw)
    assert R.relerr(got[1], good[1]) <= VJP_TOL
    assert R.relerr(got[1], bad[1]) > 1e-6


def test_negative_control_sqrt_derivative_at_stacked_drones():
    got, good, bad = _control("stacked", sqrt_form=True)
    assert np.all(np.isfinite(got[1])) and R.relerr(got[1], good[1]) <= VJP_TOL
    assert not np.all(np.isfinite(bad[1]))


def test_negative_control_predicate_dxy2_lt_100():
    """At dxy2 = 100 - 1 ulp the reference's sqrt(dxy2) < 10 fails; dxy2 < 100 keeps the pair, so the top drone gains a gradient
    that the kernel's (exactly zero) does not have."""
    got, good, bad = _control("dxy2_100-1ulp", D=2, lt100=True)
    assert np.all(got[1][1] == 0) and R.relerr(got[1], good[1]) <= VJP_TOL
    assert np.any(bad[1][1] != 0)
    got, good, _ = _control("dxy2_100-2ulp", D=2)
    assert np.any(got[1][1, 0:3] != 0) and R.relerr(got[1], good[1]) <= VJP_TOL


def test_renormalisation_per_substep_is_held_by_the_forward_bits():
    """Each substep renormalises the quaternion on entry.  Its derivative cannot be told from one renormalisation per tick:
    _integrateQ keeps |q| = 1 to rounding, so the extra renormalisations act on unit quaternions and their VJPs only remove
    radial cotangents that the tick's first one removes anyway (the radial part passes the exponential map unchanged and
    reaches no other input).  The two agree to rounding here; what tells them apart is the forward's bits, which
    test_gpu_diff_dw.py holds to step() and rollout()."""
    got, good, per_tick = _control("tumbling", renorm_per_tick=True)
    assert R.relerr(got[1], good[1]) <= VJP_TOL
    for g, w in zip(got[1:], per_tick[1:]):
        assert R.relerr(g, w) < 1e-13


# ---- the C ABI without a GPU --------------------------------------------------------------------------------------------

def test_abi_exports_and_refusals():
    from gym_pybullet_drones_b200 import _native as N
    L = N.lib()
    P, _ = params_of("cf2x")
    buf = (C.c_double * 64)()
    io = N.QsDynTrajIO()
    io.T = 2
    io.state0 = io.rpm = io.states = C.addressof(buf)
    cio = N.QsDynCtrlTrajIO()
    cio.T, cio.control_timestep = 2, 1.0 / 48
    cio.state0 = cio.pid0 = cio.target_pos = cio.states = cio.rpm = cio.pid_states = C.addressof(buf)
    calls = {"qs_dyn_traj_dw": lambda f, *a: f(C.byref(P), C.byref(io), *a, None),
             "qs_dyn_traj_dw_vjp": lambda f, *a: f(C.byref(P), C.byref(io), *a, None),
             "qs_dyn_ctrl_traj_dw": lambda f, *a: f(C.byref(P), C.byref(P), C.byref(cio), *a, None),
             "qs_dyn_ctrl_traj_dw_vjp": lambda f, *a: f(C.byref(P), C.byref(P), C.byref(cio), *a, None)}
    dw, all3 = N.EFFECT_DW, N.EFFECT_GND | N.EFFECT_DRAG | N.EFFECT_DW
    for name, call in calls.items():
        assert name in N.EXPORTS
        f = getattr(L, name)
        if name.endswith("_vjp"):
            assert call(f, 1, 2, 1, dw) == -1                           # no cotangents, outputs or scratch
            assert L.qs_last_error().startswith(name.encode() + b": ")
            if "ctrl" in name:
                cio.g_states = cio.g_state0 = cio.scratch = C.addressof(buf)
            else:
                io.g_states = io.g_rpm = io.g_state0 = io.scratch = C.addressof(buf)
        assert call(f, 0, 2, 1, dw) == -3                               # sizes before effects, as the twins
        for eff in (0, N.EFFECT_GND, N.EFFECT_DRAG, N.EFFECT_GND | N.EFFECT_DRAG, N.EFFECT_GND | N.EFFECT_DW,
                    N.EFFECT_DRAG | N.EFFECT_DW, 8, 8 | dw):
            assert call(f, 1, 2, 1, eff) == -5, (name, eff)
        assert call(f, 1, 129, 1, dw) == -5
        assert L.qs_last_error() == name.encode() + b": downwash needs drones_per_env <= 128"
        assert call(f, 1, 129, 1, all3) == -5
    for name in ("qs_dyn_traj", "qs_dyn_traj_vjp"):                    # the per-drone entries still refuse downwash
        assert getattr(L, name)(C.byref(P), C.byref(io), 1, 2, 1, dw, None) == -5
        assert b"downwash" in L.qs_last_error()
    for name in ("qs_dyn_ctrl_traj", "qs_dyn_ctrl_traj_vjp"):
        assert getattr(L, name)(C.byref(P), C.byref(P), C.byref(cio), 1, 2, 1, all3, None) == -5
        assert b"downwash" in L.qs_last_error()
    assert L.qs_abi_version() == N.ABI_VERSION == 4
