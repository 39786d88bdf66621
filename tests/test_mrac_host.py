"""MRAC without a GPU: the tier-2 oracle and the g++ build of mrac_core.cuh against the reference's fixtures (tests/golden/mrac.npz,
made by make_golden_mrac.py from the unmodified reference MRAC), the package's gain synthesis, the derived free-running horizon,
and the C ABI's exports, struct sizes and refusals without a launch.

The controller is fed the reference's inputs (its calls chained, from the same initial gains): on its own it does not amplify
rounding.  The reference's closed loop does (see free_running_horizon), which a free-running comparison could not tell apart from
an error."""
import ctypes as C

import numpy as np
import pytest

from mrac_testlib import (DT, MODELS, TF_TOL, drone_model, err, free_running_horizon, gains_of, kat_worst, loop_inputs, loop_worst,
                          mrac_harness, pack_state, unpack_state)
from qs_testlib import ptr

ORACLE_TOL = 1e-12


class _Oracle:
    """Tier 2 behind the interface of kat_worst / loop_worst."""

    def __init__(self, G, m, n):
        from oracle.mrac_oracle import OracleMRAC
        self.c = OracleMRAC(n, m, gains_=G)

    def call(self, pos, quat, vel, angv, t):
        return self.c.compute(DT, pos, quat, vel, angv, t[:, 0:3], t[:, 3:6], t[:, 6:9], t[:, 9:12])

    def state(self):
        return self.c.Kx, self.c.Kr, self.c.Xm


class _Host:
    """The g++ build of mrac_core.cuh behind the interface of kat_worst / loop_worst."""

    def __init__(self, P, G, n):
        self.P, self.n, self.init = P, n, 1
        self.st = pack_state(np.broadcast_to(G["Kx"], (n, 12, 4)), np.broadcast_to(G["Kr"], (n, 4, 4)), np.zeros((n, 12)))

    def call(self, *inp):
        n = self.n
        a = [np.ascontiguousarray(x, dtype=np.float64) for x in inp]
        rpm, pe, re = np.zeros((n, 4)), np.zeros((n, 3)), np.zeros((n, 3))
        mrac_harness().hh_mrac(C.addressof(self.P), ptr(self.st), n, self.init, DT, ptr(a[0]), ptr(a[1]), ptr(a[2]), ptr(a[3]),
                               ptr(a[4]), ptr(rpm), ptr(pe), ptr(re))
        self.init = 0
        return rpm, pe, re

    def state(self):
        return unpack_state(self.st)


@pytest.mark.parametrize("m", MODELS)
def test_oracle_matches_the_reference(golden, m):
    """Tier 2 fed the reference's inputs, its calls chained, against the reference's outputs and states at 1e-12."""
    g = golden("mrac")
    G = gains_of(g, m)
    worst = kat_worst(_Oracle(G, m, 256), g, m)
    if m == "cf2x":
        for k, v in loop_worst(_Oracle(G, m, 1), g).items():
            worst[k] = max(worst.get(k, 0.0), v)
    print(m, {k: "%.1e" % v for k, v in worst.items()})
    assert max(worst.values()) <= ORACLE_TOL, worst


@pytest.mark.parametrize("m", MODELS)
def test_package_gains_match_the_reference(golden, m):
    from gym_pybullet_drones_b200.control.MRAC import mrac_gains
    g = golden("mrac")
    G = mrac_gains(drone_model(m))
    for key, gk in (("K", "K"), ("Am", "Am"), ("P", "P"), ("Kr_ref_gain", "Kr_ref_gain"), ("Kx", "Kx0"), ("Kr", "Kr0")):
        ref = g[m + "_" + gk]
        assert np.max(np.abs(G[key] - ref)) <= 1e-10 * np.max(np.abs(ref)), key


@pytest.mark.parametrize("m", MODELS)
def test_host_core_matches_the_reference_kat(golden, m):
    """The g++ build of mrac_core.cuh on the KAT (and, for CF2X, every call of mrac.py's loop), fed the reference's inputs, at
    TF_TOL."""
    from gym_pybullet_drones_b200.control.MRAC import mrac_params
    g = golden("mrac")
    P = mrac_params(drone_model(m))
    assert mrac_harness().hh_sizeof_mrac_params() == C.sizeof(P)
    G = gains_of(g, m)
    worst = kat_worst(_Host(P, G, 256), g, m)
    if m == "cf2x":
        for k, v in loop_worst(_Host(P, G, 1), g).items():
            worst[k] = max(worst.get(k, 0.0), v)
    print(m, {k: "%.1e" % v for k, v in worst.items()})
    assert max(worst.values()) <= TF_TOL, worst


def test_host_ang_v_matches_the_reference_state_vector(golden):
    """The state vector's ang_v rebuilt from quaternion and body rates, as the kernels do, against the reference's rows: the
    golden keeps no body rates, so they are recovered from ang_v first (R^T ang_v) and mapped back."""
    from oracle.dyn_oracle import quat_to_matrix
    g = golden("mrac")
    _, q, _, av = loop_inputs(np.concatenate([g["loop_state"], g["p_state"]]))
    q = np.ascontiguousarray(q)
    w = np.ascontiguousarray(np.einsum("nji,nj->ni", quat_to_matrix(q), av))
    out = np.zeros_like(w)
    mrac_harness().hh_mrac_ang_v(ptr(q), ptr(w), q.shape[0], ptr(out))
    assert err(out, av) <= 1e-14


def test_free_running_horizon():
    """Where a free-running comparison with the reference can hold at mrac_testlib.TOL: tier 2 against its own twin with a one-ulp
    perturbation of the controller's z input at every tick.  Measured: in mrac.py's CF2X loop the twins part by more than TOL
    at tick 186 (the RPMs leave saturation at about tick 140 and the loop amplifies from there), so the GPU test compares the
    first 93 ticks; in the CF2P offset case they never do, and all 1800 ticks are compared.  Tier 2 itself leaves the reference
    by more than TOL at tick 190 of the CF2X loop: the same amplification, from its own rounding."""
    first, horizon = free_running_horizon("cf2x")
    print("cf2x: twins part at tick", first, "horizon", horizon)
    assert 150 < first < 300 and horizon == first // 2
    assert free_running_horizon("cf2p") == (1800, 1800)


def test_abi_exports_sizes_and_refusals():
    from gym_pybullet_drones_b200 import _native as N
    lib = N.lib()
    for s in ("qs_mrac_control", "qs_mrac_control_state", "qs_ctrl_rollout_mrac", "qs_sizeof_mrac_params", "qs_sizeof_mrac_rollout_io"):
        assert s in N.EXPORTS and getattr(lib, s) is not None
    assert lib.qs_sizeof_mrac_params() == C.sizeof(N.QsMracParams) == 2112
    assert lib.qs_sizeof_mrac_rollout_io() == C.sizeof(N.QsMracRolloutIO) == 32
    P, MP, st = N.QsParams(), N.QsMracParams(), N.QsState()
    buf = (C.c_char * 8192)()
    base = (C.addressof(buf) + 63) & ~63
    d = [base + 256 * j for j in range(8)]
    assert lib.qs_mrac_control(None, d[0], 1, DT, d[1], d[2], d[3], d[4], d[5], None, None, None, 4, d[6], None, None, None) == -1
    assert lib.qs_mrac_control(C.byref(MP), d[0], 1, DT, d[1], d[2], d[3], None, d[5], None, None, None, 4, d[6], None, None, None) == -1
    assert lib.qs_mrac_control(C.byref(MP), d[0], 1, DT, d[1], d[2], d[3], d[4], d[5], None, None, None, 0, d[6], None, None, None) == -3
    assert lib.qs_mrac_control(C.byref(MP), d[0], 1, 0.0, d[1], d[2], d[3], d[4], d[5], None, None, None, 4, d[6], None, None, None) == -3
    assert lib.qs_mrac_control(C.byref(MP), d[0], 1, DT, d[1], d[2], d[3], d[4], d[5], None, None, None, 4, d[6] + 8, None, None, None) == -2
    assert lib.qs_mrac_control_state(C.byref(MP), d[0], 1, DT, C.byref(st), 4, d[5], None, None, None, d[6], None, None, None) == -1
    st.planes = d[7] + 8
    assert lib.qs_mrac_control_state(C.byref(MP), d[0], 1, DT, C.byref(st), 4, d[5], None, None, None, d[6], None, None, None) == -2
    io, mio = N.QsCtrlRolloutIO(), N.QsMracRolloutIO()
    st.planes, st.step_counter = d[7], d[6]
    io.T, io.control_timestep, io.W, io.M, io.waypoints, io.start = 2, DT, 1, 1, d[1], d[2]
    call = lambda m, eff=0: lib.qs_ctrl_rollout_mrac(C.byref(P), C.byref(st), C.byref(io), m, 1, 4, 2, eff, 0, None)   # noqa: E731
    assert call(None) == -1 and b"mio" in lib.qs_last_error()
    assert call(C.byref(mio)) == -1 and b"controller" in lib.qs_last_error()                   # no params / state
    mio.params, mio.state = C.addressof(MP), d[0]
    io.actions = d[3]
    assert call(C.byref(mio)) == -5 and b"not actions" in lib.qs_last_error()
    io.actions = None
    assert call(C.byref(mio), eff=N.EFFECT_GND | N.EFFECT_DRAG) == -5
    io.W = 0
    assert call(C.byref(mio)) == -3
    # the mode belongs to its own entry point
    io.W = 1
    assert lib.qs_ctrl_rollout(C.byref(P), C.byref(st), C.byref(io), N.CTRL_MRAC, 1, 4, 2, 0, 0, None) == -4
