"""CPU tests of the forward mode of the closed-loop trajectories (DESIGN.md 4.5): the kernels' closed-loop tick tangent
(pid_tangent.cuh with dyn_tangent.cuh, built for the host) against torch.func.jacfwd of the reference controller and tick, and
against the transpose of the host-built closed-loop adjoint, also one ulp either side of the controller's decisions; negative
controls that show the comparison sees each decision; and the C ABI's refusals of qs_dyn_ctrl_traj_jvp / qs_dyn_ctrl_tick_jac
without a GPU."""
import copy
import ctypes as C

import numpy as np
import pytest

import diff_ref as R
from ctrl_jvp_testlib import BLOCKS, host_ctrl_tick_jac, ref_ctrl_tick_jac, vjp_ctrl_tick_jac
from diff_ctrl_testlib import ctrl_scenarios
from diff_testlib import params_of, per_drone_relerr, quat_from_rpy
from test_diff_ctrl_host import _ctrl_params, _rows

EFFECTS = {"dyn": 0, "gnd": R.EFFECT_GND, "drag": R.EFFECT_DRAG, "gnd_drag": R.EFFECT_GND | R.EFFECT_DRAG}
SCENARIOS = ("flight", "integral", "pwm", "torque", "scalar", "gimbal")
MODELS = ("cf2x", "cf2p")
JVP_TOL = 1e-10
DT = 1 / 48


def _case(model, name, rng, CP=None):
    """(P, CP, rows, gains, state, pid, targets, up) of one ctrl_scenarios batch with per-drone constants and gains"""
    P, c = params_of(model, 240, 48)
    CP = CP or _ctrl_params(model)
    state, pid, tg = ctrl_scenarios(c, rng)[name]
    n = state.shape[0]
    rows = _rows(model, n).numpy()
    rows[:, 0] *= rng.uniform(0.8, 1.2, n)
    rows[:, 2] *= rng.uniform(0.8, 1.2, n)
    gains = np.asarray([float(getattr(CP, f)[a]) for f in ("pid_p_for", "pid_i_for", "pid_d_for", "pid_p_tor", "pid_i_tor", "pid_d_tor")
                        for a in range(3)])[None, :] * rng.uniform(0.7, 1.3, (n, 18))
    up = float(c.HOVER_RPM) * rng.uniform(0.8, 1.2, (n, 4))
    return P, CP, rows, gains, state, pid, tg, up


def _worst(got, want):
    return {k: float(np.max(per_drone_relerr(got[k], want[k]))) for k in got}


# ---- the host-built tangent against jacfwd of the reference ---------------------------------------------------------------

@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("eff", list(EFFECTS))
@pytest.mark.parametrize("S", [1, 8])
def test_ctrl_tick_jvp_matches_reference_jacfwd(model, eff, S):
    rng = np.random.default_rng(MODELS.index(model) * 1000 + list(EFFECTS).index(eff) * 10 + S)
    worst = {}
    for name in SCENARIOS:
        P, CP, rows, gains, state, pid, tg, up = _case(model, name, rng)
        args = (P, CP, EFFECTS[eff], S, DT, rows, gains, state, pid, tg, up)
        got, want = host_ctrl_tick_jac(*args), ref_ctrl_tick_jac(*args)
        for k, e in _worst(got, want).items():
            worst[(name, k)] = e
            assert e <= JVP_TOL, (name, k, e)
        if not EFFECTS[eff] & R.EFFECT_DRAG:
            assert np.all(got["last_rpm"] == 0)
    print("ctrl tick jvp %s %s S=%d: worst per-drone error %.1e" % (model, eff, S, max(worst.values())))


# ---- the same build against the transpose of the host adjoint ---------------------------------------------------------------

def _ulps(x, k):
    """x moved by k ulps"""
    for _ in range(abs(k)):
        x = np.nextafter(x, np.inf if k > 0 else -np.inf)
    return x


def _edge(c, bound):
    """(inside, last inside, first outside) values s of a clip's input s + c at `bound` (the upper bound if > 0): one ulp apart,
    the clip passing the tangent at the first two (torch.clamp's lo <= x <= hi) and not at the third"""
    out = 1 if bound > 0 else -1                        # the direction out of the clip's range
    inside = (lambda v: v + c <= bound) if bound > 0 else (lambda v: v + c >= bound)
    s = bound - c
    while not inside(s):
        s = _ulps(s, -out)
    while inside(_ulps(s, out)):
        s = _ulps(s, out)
    return _ulps(s, -out), s, _ulps(s, out)


def _lattice(model, rng):
    """Drones one ulp below, at and above the controller's decisions: the integral clips (x at +-2, z at +-0.15, roll at +-1),
    the thrust scalar at 0 and the gimbal guard at +-0.99999.  (P, CP, rows, gains, state, pid, targets, up, label); CP has a
    MIN_PWM low enough that the thrust is not saturated at scalar = 0."""
    P, CP, rows, gains, state, pid, tg, up = _case(model, "flight", rng, copy.copy(_ctrl_params(model)))
    CP.pid_min_pwm = -1e5
    take = lambda idx: [np.repeat(a[:1], len(idx), 0).copy() for a in (rows, gains, state, pid, tg, up)]
    out, labels = [], []

    def add(batch, label):
        out.append(batch)
        labels.extend([label] * len(batch[0]))

    # integral_pos_e: ip0 = st + e dt across the bound (st moved)
    for axis, bound in ((0, 2.0), (0, -2.0), (2, 0.15), (2, -0.15)):
        b = take(range(3))
        c = (b[4][0, axis] - b[2][0, axis]) * DT
        b[3][:, axis] = _edge(c, bound)
        add(b, "ip%d%+g" % (axis, bound))
    # integral_rpy_e (roll): ir0 = ir_in + c with c = -(re dt), read from a call at ir_in = 0
    from ctrl_jvp_testlib import host_ctrl_tick_jvp
    zero = {k: np.zeros((1, w)) for k, w in BLOCKS}
    for bound in (1.0, -1.0):
        b = take(range(3))
        probe = [x[:1].copy() for x in b]
        probe[3][0, 6] = 0.0
        c = host_ctrl_tick_jvp(P, CP, 0, 1, DT, *probe, zero)["pid_out"][0, 6]
        b[3][:, 6] = _edge(c, bound)
        add(b, "ir%+g" % bound)
    # the thrust scalar: identity attitude (R = I, scalar = tt_z = fl(P_z e_z) + g with I_z = D_z = 0), e_z nudged across 0
    b = take(range(3))
    b[2][:, 3:7] = [0.0, 0.0, 0.0, 1.0]
    b[1][:, 5] = b[1][:, 8] = 0.0
    g = float(CP.pid_gravity)
    kp = b[1][0, 2]
    ez = -g / kp
    for _ in range(64):
        if kp * ez + g >= 0:
            break
        ez = _ulps(ez, 1)
    for _ in range(64):
        if kp * _ulps(ez, -1) + g < 0:
            break
        ez = _ulps(ez, -1)
    b[2][:, 2] = 0.0                        # e_z = target_z - 0 exactly
    for j, k in enumerate((-1, 0, 1)):
        b[4][j, 2] = _ulps(ez, k)
    add(b, "scalar")
    # the gimbal guard: sarg = -2 (x z - w y) at 0.99999, one ulp either side (w moved)
    b = take(range(3))
    q = quat_from_rpy(np.array([[0.1, np.arcsin(0.99999), 0.2]]))[0]
    x_, y_, z_, w_ = q
    sarg = lambda w: -2.0 * (x_ * z_ - w * y_)
    for _ in range(256):
        if sarg(w_) >= 0.99999 and sarg(_ulps(w_, -1)) < 0.99999:
            break
        w_ = _ulps(w_, -1 if sarg(w_) >= 0.99999 else 1)
    for j, k in enumerate((-1, 0, 1)):
        b[2][j, 3:7] = [x_, y_, z_, _ulps(w_, k)]
    add(b, "gimbal")
    cat = [np.concatenate([o[j] for o in out]) for j in range(6)]
    return (P, CP) + tuple(cat) + (np.array(labels),)


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("eff", ["dyn", "gnd_drag"])
def test_ctrl_tick_jvp_is_the_transpose_of_the_vjp(model, eff):
    """Both modes take every decision on the same side, on the scenarios and one ulp either side of the decisions: the
    Jacobians agree per drone and block to 1e-12, and the two sides of each decision differ."""
    rng = np.random.default_rng(40 + MODELS.index(model))
    cases = [_case(model, name, rng) for name in SCENARIOS]
    lat = _lattice(model, rng)
    cases.append(lat[:8])
    for P, CP, rows, gains, state, pid, tg, up in cases:
        args = (P, CP, EFFECTS[eff], 5, DT, rows, gains, state, pid, tg, up)
        got, want = host_ctrl_tick_jac(*args), vjp_ctrl_tick_jac(*args)
        for k, e in _worst(got, want).items():
            assert e <= 1e-12, (k, e)
    got = host_ctrl_tick_jac(P, CP, EFFECTS[eff], 5, DT, *lat[2:8])
    label = lat[8]
    for name in np.unique(label):
        i = np.flatnonzero(label == name)
        d = [float(per_drone_relerr(got["pid"][a:a + 1], got["pid"][b:b + 1])[0]) +
             float(per_drone_relerr(got["state"][a:a + 1], got["state"][b:b + 1])[0]) for a, b in ((i[0], i[2]),)]
        assert d[0] >= 1e-6, (name, d)


# ---- negative controls: each decision of the tangent is seen by the comparison ------------------------------------------

@pytest.mark.parametrize("decision,scenario", [("integral", "integral"), ("pwm", "pwm"), ("torque", "torque"), ("gimbal", "gimbal"),
                                               ("scalar", "scalar")])
def test_negative_control(decision, scenario):
    CP = None
    if decision == "scalar":                # as in test_diff_ctrl_host: a low MIN_PWM keeps the thrust visible
        CP = copy.copy(_ctrl_params("cf2x"))
        CP.pid_min_pwm = -1e5
    P, CP, rows, gains, state, pid, tg, up = _case("cf2x", scenario, np.random.default_rng(21), CP)
    args = (P, CP, 0, 3, DT, rows, gains, state, pid, tg, up)
    got, good = host_ctrl_tick_jac(*args), ref_ctrl_tick_jac(*args)
    bad = ref_ctrl_tick_jac(*args, flip=(decision,))
    assert max(_worst(got, good).values()) <= JVP_TOL
    miss = max(R.relerr(got[b], bad[b]) for b, _ in BLOCKS)
    assert miss >= 1e-6, (decision, miss)


# ---- the C ABI without a GPU --------------------------------------------------------------------------------------------

def test_abi_exports_struct_and_refusals():
    from gym_pybullet_drones_b200 import _native as N
    L = N.lib()
    for name in ("qs_dyn_ctrl_traj_jvp", "qs_dyn_ctrl_tick_jac", "qs_sizeof_dyn_ctrl_traj_jvp_io"):
        assert name in N.EXPORTS
        getattr(L, name)
    assert L.qs_sizeof_dyn_ctrl_traj_jvp_io() == C.sizeof(N.QsDynCtrlTrajJvpIO) == 16 + 24 * 8
    assert L.qs_sizeof_dyn_ctrl_traj_io() == C.sizeof(N.QsDynCtrlTrajIO) == 16 + 24 * 8
    P, _ = params_of("cf2x")
    CP = _ctrl_params("cf2x")
    buf = (C.c_double * 64)()
    for f, outs in ((L.qs_dyn_ctrl_traj_jvp, ("t_states", "t_rpm")), (L.qs_dyn_ctrl_tick_jac, ("jac",))):
        io = N.QsDynCtrlTrajJvpIO()
        io.T, io.control_timestep = 2, 1 / 48
        call = lambda io_, *a, cp=CP: f(C.byref(P), C.byref(cp) if cp is not None else None, C.byref(io_) if io_ is not None else None,
                                        *a, None)
        assert call(None, 1, 1, 1, 0) == -1
        assert call(io, 1, 1, 1, 0, cp=None) == -1
        assert call(io, 1, 1, 1, 0) == -1                               # no primal inputs
        assert L.qs_last_error().startswith(f.__name__.encode() + b": ")       # a refusal names the entry point that was called
        io.state0 = io.pid0 = io.target_pos = io.states = io.rpm = io.pid_states = C.addressof(buf)
        for k in range(len(outs)):                                      # each output missing in turn
            for j, o in enumerate(outs):
                setattr(io, o, None if j == k else C.addressof(buf))
            assert call(io, 1, 1, 1, 0) == -1
            assert L.qs_last_error().startswith(f.__name__.encode() + b": ")
        for o in outs:
            setattr(io, o, C.addressof(buf))
        assert call(io, 1, 1, 1, N.EFFECT_DW) == -5
        assert b"downwash" in L.qs_last_error()
        assert L.qs_last_error().startswith(f.__name__.encode() + b": ")
        assert call(io, 1, 1, 1, N.EFFECT_GND | N.EFFECT_DW) == -5
        assert call(io, 1, 1, 1, 8) == -4
        assert call(io, 0, 1, 1, 0) == -3
        assert call(io, 1, 0, 1, 0) == -3
        assert call(io, 1, 1, 0, 0) == -3
        assert call(io, 65536, 65536, 1, 0) == -3                       # N > 2^31 - 1
        io.control_timestep = 0.0
        assert call(io, 1, 1, 1, 0) == -3
        io.control_timestep = 1 / 48
        io.T = 0
        assert call(io, 1, 1, 1, 0) == -3
        io.T, io.phys = 1, C.addressof(buf) + 8
        assert call(io, 1, 1, 1, 0) == -2
        io.phys, io.t_phys = C.addressof(buf), C.addressof(buf) + 8
        assert call(io, 1, 1, 1, 0) == -2
        assert L.qs_last_error().startswith(f.__name__.encode() + b": ")
    io = N.QsDynCtrlTrajJvpIO()
    io.T, io.control_timestep = 1 << 30, 1 / 48
    io.state0 = io.pid0 = io.target_pos = io.states = io.rpm = io.pid_states = io.jac = C.addressof(buf)
    assert L.qs_dyn_ctrl_tick_jac(C.byref(P), C.byref(CP), C.byref(io), 1 << 9, 1, 1, 0, None) == -3   # T N C / 128 CTAs > 2^31 - 1
    assert b"CTAs" in L.qs_last_error()
