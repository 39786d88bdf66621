"""CPU tests of the closed-loop differentiable trajectories (DESIGN.md 4.5): the torch reference tests/diff_pid_ref.py against the
reference controller's known answers and the NumPy oracle, the kernels' closed-loop tick adjoint (pid_adjoint.cuh with
dyn_adjoint.cuh, built for the host) against the reference's autograd per input block, a negative control for each derivative
decision of the controller, and the C ABI's refusals without a GPU."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

import diff_pid_ref as PR
import diff_ref as R
from diff_ctrl_testlib import BLOCKS, ctrl_scenarios, host_ctrl_tick_vjp, ref_ctrl_tick_vjp
from diff_testlib import drone_model, params_of

EFFECTS = {"dyn": 0, "gnd": R.EFFECT_GND, "drag": R.EFFECT_DRAG, "gnd_drag": R.EFFECT_GND | R.EFFECT_DRAG}
VJP_TOL = 1e-10
MODELS = ("cf2x", "cf2p")


def _ctrl_params(model):
    from gym_pybullet_drones_b200.params import AviaryConstants, fill_params
    return fill_params(AviaryConstants(drone_model(model)), pid_model=drone_model(model))


def _rows(model, n):
    from gym_pybullet_drones_b200.params import nominal_properties, physical_rows
    nom = nominal_properties(drone_model(model))
    return physical_rows(drone_model(model), {k: torch.full((n,), v, dtype=torch.float64) for k, v in nom.items()})


# ---- the reference itself ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("model", MODELS)
def test_reference_pid_known_answers(golden, model):
    """The reference controller's answers on 256 random states, three stateful calls (tests/golden/pid_kat.npz)."""
    g = golden("pid_kat")
    k = model + "_"
    CP = _ctrl_params(model)
    Cc, gains = PR.controller_constants(CP), PR.gains_of(CP)
    n = g[k + "pos"].shape[0]
    st = torch.zeros((n, 9), dtype=torch.float64)
    t = lambda name: torch.tensor(g[k + name])
    for call in range(3):
        x = torch.cat([t("pos") + 0.01 * call, t("quat"), t("vel"), torch.zeros((n, 3), dtype=torch.float64)], dim=1)
        rpm, st, pe, ye = PR.pid(Cc, gains.expand(n, 18), st, 1 / 48, x, t("target_pos"), t("target_rpy")[:, 2], t("target_vel"),
                                 t("target_rpy_rates"))
        assert R.relerr(rpm, g[k + "rpm"][call]) < 1e-9
        assert R.relerr(pe, g[k + "pos_e"][call]) < 1e-12
        assert float(np.max(np.abs(ye.numpy() - g[k + "yaw_e"][call]))) < 1e-10
        assert R.relerr(st[:, 0:3], g[k + "integral_pos_e"][call]) < 1e-12
        assert R.relerr(st[:, 3:6], g[k + "last_rpy"][call]) < 1e-12
        assert R.relerr(st[:, 6:9], g[k + "integral_rpy_e"][call]) < 1e-10


def _oracle_closed_loop(model, x0, tpos, tyaw, dt, S, eff, T, gains=None):
    """OraclePID + the oracle's substeps (no renormalisation): states [T, n, 13]."""
    from oracle import dyn_oracle as O
    n = x0.shape[0]
    OP = O.OracleParams(model)
    ctrl = O.OraclePID(n, model)
    if gains is not None:
        ctrl.P_FOR, ctrl.I_FOR, ctrl.D_FOR, ctrl.P_TOR, ctrl.I_TOR, ctrl.D_TOR = (gains[3 * j:3 * j + 3] for j in range(6))
    pos, quat, vel, w = x0[:, 0:3], x0[:, 3:7], x0[:, 7:10], x0[:, 10:13]
    trpy = np.zeros((n, 3))
    trpy[:, 2] = tyaw
    up, out = np.zeros((n, 4)), []
    for k in range(T):
        rpm, _, _ = ctrl.compute(dt, pos, quat, vel, tpos[k], trpy)
        u = np.clip(np.clip(rpm, 0, OP.MAX_RPM), 0, OP.MAX_RPM)
        for s in range(S):
            pos, quat, vel, w, _ = O.dynamics_substep(OP, u, pos, quat, vel, w, eff, rpm_prev=up if s == 0 else u)
        up = u
        out.append(np.concatenate([pos, quat, vel, w], axis=1))
    return np.stack(out)


def _flight(n, T, rng):
    from diff_testlib import quat_from_rpy
    x0 = np.concatenate([rng.uniform(-0.5, 0.5, (n, 3)) + [0, 0, 1.0], quat_from_rpy(rng.uniform(-0.2, 0.2, (n, 3))),
                         rng.uniform(-0.3, 0.3, (n, 3)), rng.uniform(-0.5, 0.5, (n, 3))], axis=1)
    tpos = x0[None, :, 0:3] + 0.2 * np.sin(np.arange(T)[:, None, None] / 5.0 + rng.uniform(0, 6, (1, n, 3)))
    return x0, tpos, rng.uniform(-0.5, 0.5, n)


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("eff", list(EFFECTS))
def test_reference_closed_loop_matches_oracle(model, eff):
    P, c = params_of(model, 240, 48)
    CP = _ctrl_params(model)
    n, T, S, dt = 8, 12, 5, 1 / 48
    x0, tpos, tyaw = _flight(n, T, np.random.default_rng(11))
    want = _oracle_closed_loop(model, x0, tpos, tyaw, dt, S, EFFECTS[eff], T)
    z = torch.zeros((n, 3), dtype=torch.float64)
    got, _ = PR.closed_loop(R.model_constants(P), PR.controller_constants(CP), _rows(model, n), PR.gains_of(CP).expand(n, 18),
                            torch.tensor(x0), torch.zeros((n, 9), dtype=torch.float64), torch.tensor(tpos), torch.tensor(tyaw), z, z,
                            torch.zeros((n, 4), dtype=torch.float64), dt, S, EFFECTS[eff])
    err = np.max(np.abs(got.numpy() - want) / np.maximum(np.abs(want), 1.0))
    assert err <= 1e-10, err


@pytest.mark.parametrize("model", MODELS)
def test_reference_gradient_matches_oracle_central_differences(model):
    """Away from the clamp and branch points: gradients of a closed-loop loss w.r.t. the initial state, the gains and the
    targets against central differences of the oracle."""
    P, c = params_of(model, 240, 48)
    CP = _ctrl_params(model)
    n, T, S, dt, eff = 2, 4, 3, 1 / 48, R.EFFECT_GND | R.EFFECT_DRAG
    rng = np.random.default_rng(12)
    x0, tpos, tyaw = _flight(n, T, rng)
    x0[:, 2] = 0.1                        # ground effect live
    g_out = rng.standard_normal((T, n, 13))
    g0 = PR.gains_of(CP).numpy()

    def loss(x0=x0, tpos=tpos, tyaw=tyaw, gains=g0):
        return float(np.sum(g_out * _oracle_closed_loop(model, x0, tpos, tyaw, dt, S, eff, T, gains)))

    def central(f, x, scale, rel=1e-6):
        g = np.zeros_like(x)
        for idx in np.ndindex(x.shape):
            h = rel * (scale if np.isscalar(scale) else scale[idx])
            xp, xm = x.copy(), x.copy()
            xp[idx] += h
            xm[idx] -= h
            g[idx] = (f(xp) - f(xm)) / (2 * h)
        return g

    fd_x = central(lambda v: loss(x0=v), x0, 1.0)
    fd_tp = central(lambda v: loss(tpos=v), tpos, 1.0)
    fd_ty = central(lambda v: loss(tyaw=v), tyaw, 1.0)
    live = np.abs(g0) > 0
    fd_g = central(lambda v: loss(gains=v), g0, np.where(live, np.abs(g0), 1.0))
    x, tp, ty, gn = (torch.tensor(a, requires_grad=True) for a in (x0, tpos, tyaw, g0))
    z = torch.zeros((n, 3), dtype=torch.float64)
    out, _ = PR.closed_loop(R.model_constants(P), PR.controller_constants(CP), _rows(model, n), gn.expand(n, 18), x,
                            torch.zeros((n, 9), dtype=torch.float64), tp, ty, z, z, torch.zeros((n, 4), dtype=torch.float64), dt, S, eff)
    gx, gtp, gty, gg = torch.autograd.grad(out, (x, tp, ty, gn), torch.tensor(g_out))
    q = x0[:, 3:7]
    fd_x[:, 3:7] -= q * np.sum(q * fd_x[:, 3:7], axis=1, keepdims=True)      # the oracle does not renormalise: tangent part
    gx = gx.numpy().copy()
    gx[:, 3:7] -= q * np.sum(q * gx[:, 3:7], axis=1, keepdims=True)
    assert R.relerr(gx, fd_x) < 1e-6
    assert R.relerr(gtp, fd_tp) < 1e-6
    assert R.relerr(gty, fd_ty) < 1e-6
    assert R.relerr(gg, fd_g) < 1e-6


# ---- the host-built adjoint core against the reference --------------------------------------------------------------------

def _case(model, name, rng, S=5, eff=0, CP=None):
    P, c = params_of(model, 240, 48)
    CP = CP or _ctrl_params(model)
    state, pid, tg = ctrl_scenarios(c, rng)[name]
    n = state.shape[0]
    rows = _rows(model, n).numpy()
    rows[:, 0] *= rng.uniform(0.8, 1.2, n)                 # per-drone constants
    rows[:, 2] *= rng.uniform(0.8, 1.2, n)
    gains = PR.gains_of(CP).numpy()[None, :] * rng.uniform(0.7, 1.3, (n, 18))
    up = float(c.HOVER_RPM) * rng.uniform(0.8, 1.2, (n, 4))
    args = (P, CP, eff, S, 1 / 48, rows, gains, state, pid, tg, up,
            rng.standard_normal((n, 13)), rng.standard_normal((n, 4)), rng.standard_normal((n, 9)))
    return args


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("eff", list(EFFECTS))
@pytest.mark.parametrize("S", [1, 8])
def test_ctrl_tick_vjp_matches_reference(model, eff, S):
    rng = np.random.default_rng(hash((model, eff, S)) % 2 ** 32)
    worst = {}
    for name in ("flight", "integral", "pwm", "torque", "scalar", "gimbal"):
        args = _case(model, name, rng, S, EFFECTS[eff])
        got, want = host_ctrl_tick_vjp(*args), ref_ctrl_tick_vjp(*args)
        for k in ("out", "rpm", "pid_out"):
            assert R.relerr(got[k], want[k]) < 1e-12, (name, k)
        for blk in BLOCKS:
            e = R.relerr(got[blk], want[blk])
            worst[(name, blk)] = e
            assert e <= VJP_TOL, (name, blk, e)
    print("worst normwise relative error %s %s S=%d: %.2e" % (model, eff, S, max(worst.values())))


# ---- negative controls: each decision of the controller's adjoint is seen by the comparison -------------------------------

@pytest.mark.parametrize("decision,scenario", [("integral", "integral"), ("pwm", "pwm"), ("torque", "torque"), ("gimbal", "gimbal"),
                                               ("scalar", "scalar")])
def test_negative_control(decision, scenario):
    CP = None
    if decision == "scalar":
        # with the default constants a negative scalar always saturates the PWM at MIN_PWM, which hides the thrust; a
        # controller with a lower MIN_PWM shows the decision
        CP = copy.copy(_ctrl_params("cf2x"))
        CP.pid_min_pwm = -1e5
    args = _case("cf2x", scenario, np.random.default_rng(21), 3, 0, CP)
    got, good = host_ctrl_tick_vjp(*args), ref_ctrl_tick_vjp(*args)
    bad = ref_ctrl_tick_vjp(*args, flip=(decision,))
    assert max(R.relerr(got[b], good[b]) for b in BLOCKS) <= VJP_TOL
    assert not max(R.relerr(got[b], bad[b]) for b in BLOCKS) <= 1e-6, decision


# ---- the C ABI without a GPU --------------------------------------------------------------------------------------------

def test_abi_exports_struct_and_refusals():
    from gym_pybullet_drones_b200 import _native as N
    L = N.lib()
    for name in ("qs_dyn_ctrl_traj", "qs_dyn_ctrl_traj_vjp", "qs_sizeof_dyn_ctrl_traj_io"):
        assert name in N.EXPORTS
        getattr(L, name)
    assert L.qs_sizeof_dyn_ctrl_traj_io() == C.sizeof(N.QsDynCtrlTrajIO) == 16 + 24 * 8
    P, _ = params_of("cf2x")
    CP = _ctrl_params("cf2x")
    io = N.QsDynCtrlTrajIO()
    io.T, io.control_timestep = 2, 1 / 48
    buf = (C.c_double * 64)()
    io.state0 = io.pid0 = io.target_pos = io.states = io.rpm = io.pid_states = C.addressof(buf)
    call = lambda f, io_, *a, cp=CP: f(C.byref(P), C.byref(cp) if cp is not None else None, C.byref(io_) if io_ is not None else None, *a, None)
    assert call(L.qs_dyn_ctrl_traj, None, 1, 1, 1, 0) == -1
    assert call(L.qs_dyn_ctrl_traj, io, 1, 1, 1, 0, cp=None) == -1
    assert call(L.qs_dyn_ctrl_traj, io, 1, 1, 1, N.EFFECT_DW) == -5
    assert b"downwash" in L.qs_last_error()
    assert call(L.qs_dyn_ctrl_traj, io, 1, 1, 1, N.EFFECT_GND | N.EFFECT_DW) == -5
    assert call(L.qs_dyn_ctrl_traj, io, 1, 1, 1, 8) == -4
    assert call(L.qs_dyn_ctrl_traj, io, 0, 1, 1, 0) == -3
    assert call(L.qs_dyn_ctrl_traj, io, 1, 1, 0, 0) == -3
    io.control_timestep = 0.0
    assert call(L.qs_dyn_ctrl_traj, io, 1, 1, 1, 0) == -3
    io.control_timestep = 1 / 48
    assert call(L.qs_dyn_ctrl_traj_vjp, io, 1, 1, 1, 0) == -1          # no cotangents, gradient or scratch
    assert L.qs_last_error().startswith(b"qs_dyn_ctrl_traj_vjp: ")      # a refusal names the entry point that was called
    io.g_states = io.g_state0 = io.scratch = C.addressof(buf)
    assert call(L.qs_dyn_ctrl_traj_vjp, io, 1, 1, 1, N.EFFECT_DW) == -5
    io.T = 0
    assert call(L.qs_dyn_ctrl_traj_vjp, io, 1, 1, 1, 0) == -3
    assert L.qs_last_error().startswith(b"qs_dyn_ctrl_traj_vjp: ")
    io.T, io.phys = 1, C.addressof(buf) + 8
    assert call(L.qs_dyn_ctrl_traj, io, 1, 1, 1, 0) == -2
    io.phys, io.pid0 = None, None
    assert call(L.qs_dyn_ctrl_traj, io, 1, 1, 1, 0) == -1
