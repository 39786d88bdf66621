"""CPU tests of the forward mode of the differentiable trajectories (DESIGN.md 4.5): the kernels' tick tangent (dyn_tangent.cuh,
built for the host) against torch.func.jacfwd of the reference tests/diff_ref.py and against the transpose of the host-built
adjoint at every decision lattice, negative controls that show the comparison sees each decision, and the C ABI's refusals of
qs_dyn_traj_jvp / qs_dyn_tick_jac without a GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

import diff_ref as R
from diff_testlib import MODELS, SIDE_PAIRS, aviary_rows, lattices, params_of, per_drone_relerr, scenario_ticks
from jvp_testlib import host_tick_jac, ref_tick_jac, vjp_tick_jac, worst_per_block

EFFECTS = {"dyn": 0, "gnd": R.EFFECT_GND, "drag": R.EFFECT_DRAG, "gnd_drag": R.EFFECT_GND | R.EFFECT_DRAG}
JVP_TOL = 1e-10


def _scenario_batch(model, seed, n=4):
    """The six scenarios of diff_testlib, n drones each, every drone with its own random row: (state, raw, up, rows)."""
    P, c = params_of(model)
    _, rows = aviary_rows(model, 6 * n, np.random.default_rng(seed))
    _, state, raw, up = scenario_ticks(c, rows.numpy(), 1, seed, n)
    return P, state, raw[0], up, rows.numpy()


# ---- the host-built tangent against jacfwd of the reference ---------------------------------------------------------------

@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("eff", list(EFFECTS))
@pytest.mark.parametrize("S", [1, 5, 8, 24])
def test_tick_jvp_matches_reference_jacfwd(model, eff, S):
    P, state, raw, up, rows = _scenario_batch(model, MODELS.index(model) * 100 + S)
    got = host_tick_jac(P, EFFECTS[eff], S, state, raw, up, rows)
    want = ref_tick_jac(P, EFFECTS[eff], S, state, raw, up, rows)
    worst = worst_per_block(got, want)
    print("tick jvp %s %s S=%d: worst per-drone error %s" % (model, eff, S, {k: "%.1e" % v for k, v in worst.items()}))
    for k, e in worst.items():
        assert e <= JVP_TOL, (k, e)
    if not EFFECTS[eff] & R.EFFECT_DRAG:
        assert np.all(got["up"] == 0)


# ---- the same build against the transpose of the host adjoint on the decision lattices --------------------------------------

@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("name", ["rpm", "clip", "half_angle", "upright"])
def test_tick_jvp_is_the_transpose_of_the_vjp_on_lattices(model, name):
    """Both modes take every decision on the same side, also one ulp either side of it: the Jacobians agree per drone and
    block, the two sides of each decision differ, and the RPM clip passes or stops the derivative at the same lattice points."""
    P, c = params_of(model)
    _, rows = aviary_rows(model, 64, np.random.default_rng(20))
    lat = lattices(P, c, rows.numpy(), np.random.default_rng(21))[name]
    args = (P, lat["effects"], lat["S"], lat["state"], lat["raw"], lat["up"], lat["rows"])
    got, want = host_tick_jac(*args), vjp_tick_jac(*args)
    worst = worst_per_block(got, want)
    print("lattice %s %s: worst per-drone error against the VJP %s" % (model, name, {k: "%.1e" % v for k, v in worst.items()}))
    for k, e in worst.items():
        assert e <= 1e-12, (k, e)
    for a, b in SIDE_PAIRS.get(name, []):
        d = sum(float(per_drone_relerr(got[k][a:a + 1], got[k][b:b + 1])[0]) for k in ("state", "rpm"))
        assert d >= 1e-3, (a, b, d)
    if name == "rpm":                       # raw's tangent passes at max-, max, -0.0, 0.0, 0+; MAX_RPM's only strictly above
        lab = lat["label"]
        j = np.arange(len(lab)) // 7
        for jac in (got, want):
            col = jac["rpm"][np.arange(len(lab)), :, j]
            assert np.all(np.all(col == 0, axis=1) == np.isin(lab, (2, 3)))
            assert np.all(np.any(jac["row"][:, :, 13] != 0, axis=1) == (lab == 2))


# ---- negative controls: a perturbed tangent fails the check -------------------------------------------------------------

def test_negative_control_isclose_branch_zero_derivative():
    """At exact hover the reference's isclose identity has a zero attitude derivative: its tangent misses the kernel's."""
    P, c = params_of("cf2x")
    _, rows = aviary_rows("cf2x", 4, np.random.default_rng(30))
    rows = rows.numpy()
    state = np.tile([0, 0, 1.0, 0, 0, 0, 1.0, 0, 0, 0, 0, 0, 0], (4, 1))
    raw = up = np.tile(rows[:, 12:13], (1, 4))
    got = host_tick_jac(P, 0, 1, state, raw, up, rows)
    good = ref_tick_jac(P, 0, 1, state, raw, up, rows)
    bad = ref_tick_jac(P, 0, 1, state, raw, up, rows, exact_branch=True)
    assert worst_per_block(got, good)["rpm"] <= JVP_TOL
    quat = lambda j: j["rpm"][:, 3:7, :]                                # the attitude's rows: differential RPM reaches q
    assert np.any(quat(got) != 0)
    assert float(np.max(per_drone_relerr(quat(got), quat(bad)))) >= 1e-2


def test_negative_control_missing_entry_renormalisation():
    """Without the entry renormalisation's tangent the quaternion columns gain a radial part."""
    P, state, raw, up, rows = _scenario_batch("cf2x", 31)
    got = host_tick_jac(P, 0, 8, state, raw, up, rows)
    good = ref_tick_jac(P, 0, 8, state, raw, up, rows)
    bad = ref_tick_jac(P, 0, 8, state, raw, up, rows, renormalise=False)
    assert worst_per_block(got, good)["state"] <= JVP_TOL
    assert float(np.max(per_drone_relerr(got["state"][:, :, 3:7], bad["state"][:, :, 3:7]))) >= 1e-3
    q = state[:, 3:7]
    radial = np.einsum("nrc,nc->nr", got["state"][:, :, 3:7], q)           # A[:, 3:7] q = 0
    assert np.max(np.abs(radial)) <= 1e-12 * np.max(np.abs(got["state"]))


def test_negative_control_drag_without_up_path():
    """Drag's first substep reads the previous tick's RPMs: a reference that reads the current ones has no `up` tangent and a
    different rpm tangent."""
    P, state, raw, up, rows = _scenario_batch("cf2x", 32)
    got = host_tick_jac(P, R.EFFECT_DRAG, 5, state, raw, up, rows)
    good = ref_tick_jac(P, R.EFFECT_DRAG, 5, state, raw, up, rows)
    assert max(worst_per_block(got, good).values()) <= JVP_TOL
    cur = np.minimum(np.maximum(raw, 0.0), rows[:, 13:14])
    bad = ref_tick_jac(P, R.EFFECT_DRAG, 5, state, raw, cur, rows)
    assert np.any(got["up"] != 0)
    assert worst_per_block(got, bad)["rpm"] > 1e-9


def test_negative_control_strict_clamp():
    """A clip whose tangent passes only strictly below MAX_RPM misses the kernel's at raw == MAX_RPM (and only there)."""
    P, c = params_of("cf2x")
    _, rows = aviary_rows("cf2x", 64, np.random.default_rng(20))
    lat = lattices(P, c, rows.numpy(), np.random.default_rng(21))["rpm"]
    args = (P, lat["effects"], lat["S"], lat["state"], lat["raw"], lat["up"], lat["rows"])
    got = host_tick_jac(*args)
    good, bad = ref_tick_jac(*args), ref_tick_jac(*args, strict_clamp=True)
    assert max(worst_per_block(got, good).values()) <= JVP_TOL
    e = per_drone_relerr(got["rpm"], bad["rpm"])
    at = lat["label"] == 1
    assert e[at].min() >= 1e-3 and e[~at].max() <= JVP_TOL


# ---- the C ABI without a GPU --------------------------------------------------------------------------------------------

def test_abi_exports_struct_and_refusals():
    from gym_pybullet_drones_b200 import _native as N
    L = N.lib()
    for name in ("qs_dyn_traj_jvp", "qs_dyn_tick_jac", "qs_sizeof_dyn_traj_jvp_io"):
        assert name in N.EXPORTS
        getattr(L, name)
    assert L.qs_sizeof_dyn_traj_jvp_io() == C.sizeof(N.QsDynTrajJvpIO) == 8 + 11 * 8
    assert L.qs_sizeof_dyn_traj_io() == C.sizeof(N.QsDynTrajIO) == 8 + 11 * 8
    P, _ = params_of("cf2x")
    buf = (C.c_double * 64)()
    for f, out in ((L.qs_dyn_traj_jvp, "t_states"), (L.qs_dyn_tick_jac, "jac")):
        io = N.QsDynTrajJvpIO()
        io.T = 2
        call = lambda io_, *a: f(C.byref(P), C.byref(io_) if io_ is not None else None, *a, None)
        assert call(None, 1, 1, 1, 0) == -1
        assert f(None, C.byref(io), 1, 1, 1, 0, None) == -1
        assert call(io, 1, 1, 1, 0) == -1                               # no state0 / rpm / states
        io.state0 = io.rpm = io.states = C.addressof(buf)
        assert call(io, 1, 1, 1, 0) == -1                               # no output
        setattr(io, out, C.addressof(buf))
        assert call(io, 1, 1, 1, N.EFFECT_DW) == -5
        assert b"downwash" in L.qs_last_error() and b"pairwise" in L.qs_last_error()
        assert L.qs_last_error().startswith(f.__name__.encode() + b": ")       # a refusal names the entry point that was called
        assert call(io, 1, 1, 1, N.EFFECT_GND | N.EFFECT_DW) == -5
        assert call(io, 1, 1, 1, 8) == -4
        assert call(io, 0, 1, 1, 0) == -3
        assert call(io, 1, 0, 1, 0) == -3
        assert call(io, 1, 1, 0, 0) == -3
        assert call(io, 65536, 65536, 1, 0) == -3                       # N > 2^31 - 1
        io.T = 0
        assert call(io, 1, 1, 1, 0) == -3
        io.T, io.phys = 1, C.addressof(buf) + 8
        assert call(io, 1, 1, 1, 0) == -2
        io.phys, io.t_phys = C.addressof(buf), C.addressof(buf) + 8
        assert call(io, 1, 1, 1, 0) == -2
    io = N.QsDynTrajJvpIO()
    io.T, io.state0, io.rpm, io.states, io.jac = 1 << 30, C.addressof(buf), C.addressof(buf), C.addressof(buf), C.addressof(buf)
    assert L.qs_dyn_tick_jac(C.byref(P), C.byref(io), 1 << 10, 1, 1, 0, None) == -3     # T N C / 128 CTAs exceed 2^31 - 1
