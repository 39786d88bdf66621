"""CPU tests of the differentiable trajectories (DESIGN.md 4.5): the torch reference tests/diff_ref.py against the NumPy oracle,
the kernels' tick adjoint (dyn_adjoint.cuh, built for the host) against the reference's autograd, negative controls that show
the comparison sees each derivative decision, and the C ABI's refusals without a GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

import diff_ref as R
from diff_testlib import MODELS, drone_model, host_tick_vjp, params_of, scenarios

EFFECTS = {"dyn": 0, "gnd": R.EFFECT_GND, "drag": R.EFFECT_DRAG, "gnd_drag": R.EFFECT_GND | R.EFFECT_DRAG}
VJP_TOL = 1e-10


def _nominal_rows(model, n):
    from gym_pybullet_drones_b200.params import nominal_properties, physical_rows
    nom = nominal_properties(drone_model(model))
    return physical_rows(drone_model(model), {k: torch.full((n,), v, dtype=torch.float64) for k, v in nom.items()})


def _ref_vjp(P, rows, effects, S, state, raw, up, g_out, **kw):
    """diff_ref's tick and its autograd VJP: (out, g_state, g_raw, g_up, g_row)."""
    K = R.model_constants(P)
    x = torch.tensor(state, requires_grad=True)
    r = torch.tensor(raw, requires_grad=True)
    u = torch.tensor(up, requires_grad=True)
    rw = rows.clone().requires_grad_(True)
    out, _ = R.tick(K, rw, x, r, u, S, effects, **kw)
    gs = torch.autograd.grad(out, (x, r, u, rw), torch.tensor(g_out), allow_unused=True)
    gs = [torch.zeros_like(t) if g is None else g for g, t in zip(gs, (x, r, u, rw))]
    return [out.detach().numpy()] + [g.numpy() for g in gs]


# ---- the reference itself ------------------------------------------------------------------------------------------------

def _oracle_tick(O, OP, effects, S, state, raw, up):
    """S substeps of the NumPy oracle with the clipped rpm; drag's first substep reads `up`."""
    u = np.clip(raw, 0, OP.MAX_RPM)
    pos, quat, vel, w = state[:, 0:3], state[:, 3:7], state[:, 7:10], state[:, 10:13]
    for s in range(S):
        pos, quat, vel, w, _ = O.dynamics_substep(OP, u, pos, quat, vel, w, effects, rpm_prev=up if s == 0 else u)
    return np.concatenate([pos, quat, vel, w], axis=1)


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("eff", list(EFFECTS))
def test_reference_forward_matches_oracle(model, eff):
    from oracle import dyn_oracle as O
    P, c = params_of(model)
    OP = O.OracleParams({"race": "racer"}.get(model, model))
    rng = np.random.default_rng(1)
    worst = 0.0
    for name, (state, raw, up) in scenarios(c, rng).items():
        if name == "hover":
            continue                     # w = 0: the oracle keeps the quaternion, the reference's exponential map is the identity too
        n = state.shape[0]
        want = _oracle_tick(O, OP, EFFECTS[eff], 5, state, raw, np.clip(up, 0, OP.MAX_RPM))
        got, _ = R.tick(R.model_constants(P), _nominal_rows(model, n), torch.tensor(state), torch.tensor(raw),
                        torch.tensor(np.clip(up, 0, OP.MAX_RPM)), 5, EFFECTS[eff])
        err = np.max(np.abs(got.numpy() - want) / np.maximum(np.abs(want), 1.0))
        worst = max(worst, err)
    assert worst <= 1e-13, worst


@pytest.mark.parametrize("model", MODELS)
def test_reference_gradient_matches_oracle_central_differences(model):
    """Away from the clip and branch points (flight at 0.1 m, ground effect live and unclipped, |w| >> 1e-8)."""
    from oracle import dyn_oracle as O
    from gym_pybullet_drones_b200.params import nominal_properties, physical_rows
    P, c = params_of(model)
    name = {"race": "racer"}.get(model, model)
    rng = np.random.default_rng(2)
    n, S, eff = 3, 4, R.EFFECT_GND | R.EFFECT_DRAG
    state, raw, up = scenarios(c, rng, n)["flight"]
    state[:, 2] = 0.1
    g_out = rng.standard_normal((n, 13))
    nom = nominal_properties(drone_model(model))

    def loss(state, raw, up, m=nom["m"], kf=nom["kf"], ixx=nom["ixx"]):
        OP = O.OracleParams(name)
        OP.M, OP.GRAVITY, OP.KF = m, OP.G * m, kf
        OP.J = OP.J.copy(); OP.J[0] = ixx; OP.J_INV = 1.0 / OP.J
        OP.MAX_RPM = np.inf
        return float(np.sum(g_out * _oracle_tick(O, OP, eff, S, state, raw, up)))

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
    fd_up = central(lambda u: loss(state, raw, u), up, float(c.HOVER_RPM), 1e-2)      # drag's tiny term: a larger step
    fd_p = {k: central(lambda v: loss(state, raw, up, **{k: float(v[0])}), np.array([nom[k]]), nom[k])[0] for k in ("m", "kf", "ixx")}

    props = {k: torch.full((n,), v, dtype=torch.float64, requires_grad=k in fd_p) for k, v in nom.items()}
    rows = physical_rows(drone_model(model), props)
    x, r, u = (torch.tensor(a, requires_grad=True) for a in (state, raw, up))
    out, _ = R.tick(R.model_constants(P), rows, x, r, u, S, eff)
    gx, gr, gu, gm, gkf, gixx = torch.autograd.grad(out, (x, r, u, props["m"], props["kf"], props["ixx"]), torch.tensor(g_out))
    q = state[:, 3:7]
    tangent = lambda g: g - q * np.sum(q * g, axis=1, keepdims=True)     # the oracle does not renormalise: compare the tangent part
    fd_state[:, 3:7] = tangent(fd_state[:, 3:7])
    assert R.relerr(gx, fd_state) < 1e-6
    assert R.relerr(gr, fd_raw) < 1e-6
    assert R.relerr(gu, fd_up) < 1e-6
    for k, g in (("m", gm), ("kf", gkf), ("ixx", gixx)):
        assert R.relerr(g.sum(), fd_p[k]) < 1e-6, k


# ---- the host-built adjoint core against the reference --------------------------------------------------------------------

@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("eff", list(EFFECTS))
@pytest.mark.parametrize("S", [1, 5, 8, 24])
def test_tick_vjp_matches_reference(model, eff, S):
    P, c = params_of(model)
    rng = np.random.default_rng(hash((model, eff, S)) % 2 ** 32)
    worst = {}
    for name, (state, raw, up) in scenarios(c, rng).items():
        n = state.shape[0]
        rows = _nominal_rows(model, n)
        rows[:, 0] *= torch.from_numpy(rng.uniform(0.8, 1.2, n))      # per-drone constants: the table path
        rows[:, 2] *= torch.from_numpy(rng.uniform(0.8, 1.2, n))
        g_out = rng.standard_normal((n, 13))
        got = host_tick_vjp(P, EFFECTS[eff], S, state, raw, up, g_out, rows.numpy())
        want = _ref_vjp(P, rows, EFFECTS[eff], S, state, raw, up, g_out)
        assert R.relerr(got[0], want[0]) < 1e-12, (name, "forward")
        for blk, g, w in zip(("state", "rpm", "last_rpm", "phys"), got[1:], want[1:]):
            e = R.relerr(g, w)
            worst[(name, blk)] = e
            assert e <= VJP_TOL, (name, blk, e)
    print("worst normwise relative error %s %s S=%d: %.2e" % (model, eff, S, max(worst.values())))


def test_tick_vjp_qsparams_constants():
    """rows = NULL: the constants of QsParams, the same gradient as their nominal row."""
    P, c = params_of("cf2x")
    state, raw, up = scenarios(c, np.random.default_rng(3))["flight"]
    g_out = np.random.default_rng(4).standard_normal(state.shape[:1] + (13,))
    a = host_tick_vjp(P, 3, 8, state, raw, up, g_out)
    b = host_tick_vjp(P, 3, 8, state, raw, up, g_out, _nominal_rows("cf2x", state.shape[0]).numpy())
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_half_angle_grad_matches_reference():
    from diff_testlib import diff_harness
    dt = 1.0 / 240
    n2 = np.concatenate([[0.0, 1e-20, 1e-16], np.geomspace(1e-8, 1e7, 400), [(2 / dt) ** 2 * 0.25 * (1 - 1e-12), (2 / dt) ** 2 * 0.25]])
    out = np.zeros((n2.size, 4))
    diff_harness().dh_half_angle_grad(n2.ctypes.data_as(C.c_void_p), n2.size, dt, out.ctypes.data_as(C.c_void_p))
    t = torch.tensor(n2, requires_grad=True)
    cr, sr = R.half_angle(t, dt)
    dc, = torch.autograd.grad(cr.sum(), t, retain_graph=True)
    ds, = torch.autograd.grad(sr.sum(), t)
    for j, ref in enumerate((cr.detach(), sr.detach(), dc, ds)):
        assert R.relerr(out[:, j], ref) < 1e-14, j


# ---- negative controls --------------------------------------------------------------------------------------------------

def test_negative_control_isclose_branch_derivative():
    """At exact hover the reference's isclose branch has a zero attitude derivative: a reference that takes it misses the
    kernel's RPM gradient by >= 1e-2, while the exponential map's reference agrees."""
    P, c = params_of("cf2x")
    state, raw, up = scenarios(c, np.random.default_rng(5))["hover"]
    g_out = np.zeros((state.shape[0], 13))
    g_out[:, 3:7] = np.random.default_rng(6).standard_normal((state.shape[0], 4))
    rows = _nominal_rows("cf2x", state.shape[0])
    got = host_tick_vjp(P, 0, 1, state, raw, up, g_out, rows.numpy())
    good = _ref_vjp(P, rows, 0, 1, state, raw, up, g_out)
    branch = _ref_vjp(P, rows, 0, 1, state, raw, up, g_out, exact_branch=True)
    assert R.relerr(got[2], good[2]) <= VJP_TOL
    assert R.relerr(branch[2], got[2]) >= 1e-2


def test_negative_control_drag_last_rpm_path():
    """Drag's first substep reads the previous tick's RPMs: a reference that reads the current ones misses."""
    P, c = params_of("cf2x")
    state, raw, up = scenarios(c, np.random.default_rng(7))["flight"]
    g_out = np.random.default_rng(8).standard_normal((state.shape[0], 13))
    rows = _nominal_rows("cf2x", state.shape[0])
    got = host_tick_vjp(P, R.EFFECT_DRAG, 5, state, raw, up, g_out, rows.numpy())
    good = _ref_vjp(P, rows, R.EFFECT_DRAG, 5, state, raw, up, g_out)
    dropped = _ref_vjp(P, rows, R.EFFECT_DRAG, 5, state, raw, np.clip(raw, 0, float(c.MAX_RPM)), g_out)
    assert R.relerr(got[3], good[3]) <= VJP_TOL and R.relerr(got[2], good[2]) <= VJP_TOL
    assert np.any(got[3] != 0) and R.relerr(got[2], dropped[2]) > 1e-9 and R.relerr(dropped[0], got[0]) > 1e-12


def test_negative_control_entry_renormalisation():
    """Without the entry renormalisation the state-0 quaternion gradient gains a radial part."""
    P, c = params_of("cf2x")
    state, raw, up = scenarios(c, np.random.default_rng(9))["flight"]
    g_out = np.random.default_rng(10).standard_normal((state.shape[0], 13))
    rows = _nominal_rows("cf2x", state.shape[0])
    got = host_tick_vjp(P, 0, 8, state, raw, up, g_out, rows.numpy())
    good = _ref_vjp(P, rows, 0, 8, state, raw, up, g_out)
    raw_q = _ref_vjp(P, rows, 0, 8, state, raw, up, g_out, renormalise=False)
    assert R.relerr(got[1][:, 3:7], good[1][:, 3:7]) <= VJP_TOL
    assert R.relerr(got[1][:, 3:7], raw_q[1][:, 3:7]) > 1e-3
    q = state[:, 3:7]
    assert np.max(np.abs(np.sum(got[1][:, 3:7] * q, axis=1))) < 1e-12 * np.max(np.abs(got[1][:, 3:7]))   # no radial component


# ---- the C ABI without a GPU --------------------------------------------------------------------------------------------

def test_abi_exports_struct_and_refusals():
    from gym_pybullet_drones_b200 import _native as N
    L = N.lib()
    for name in ("qs_dyn_traj", "qs_dyn_traj_vjp", "qs_sizeof_dyn_traj_io"):
        assert name in N.EXPORTS
        getattr(L, name)
    assert L.qs_sizeof_dyn_traj_io() == C.sizeof(N.QsDynTrajIO) == 8 + 11 * 8
    P, _ = params_of("cf2x")
    io = N.QsDynTrajIO()
    io.T = 2
    buf = (C.c_double * 64)()
    io.state0 = io.rpm = io.states = C.addressof(buf)
    call = lambda f, io_, *a: f(C.byref(P), C.byref(io_) if io_ is not None else None, *a, None)
    assert call(L.qs_dyn_traj, None, 1, 1, 1, 0) == -1
    assert call(L.qs_dyn_traj, io, 1, 1, 1, N.EFFECT_DW) == -5
    assert call(L.qs_dyn_traj, io, 1, 1, 1, N.EFFECT_GND | N.EFFECT_DW) == -5
    assert call(L.qs_dyn_traj, io, 1, 1, 1, 8) == -4
    assert call(L.qs_dyn_traj, io, 0, 1, 1, 0) == -3
    assert call(L.qs_dyn_traj, io, 1, 1, 0, 0) == -3
    assert call(L.qs_dyn_traj_vjp, io, 1, 1, 1, 0) == -1          # no cotangents, outputs or scratch
    assert L.qs_last_error().startswith(b"qs_dyn_traj_vjp: ")      # a refusal names the entry point that was called
    io.g_states = io.g_rpm = io.g_state0 = io.scratch = C.addressof(buf)
    assert call(L.qs_dyn_traj_vjp, io, 1, 1, 1, N.EFFECT_DW) == -5
    io.T = 0
    assert call(L.qs_dyn_traj_vjp, io, 1, 1, 1, 0) == -3
    assert L.qs_last_error().startswith(b"qs_dyn_traj_vjp: ")
    io.T, io.phys = 1, C.addressof(buf) + 8
    assert call(L.qs_dyn_traj, io, 1, 1, 1, 0) == -2
    assert b"downwash" in (call(L.qs_dyn_traj, io, 1, 1, 1, N.EFFECT_DW) and L.qs_last_error())
