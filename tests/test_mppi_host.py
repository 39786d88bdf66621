"""-m "not gpu": the rules of mppi() (DESIGN.md 4.5.2) on the host build of philox.cuh and mppi.cuh (tests/host_harness/mppi_host.cpp)
against the float64 restatement tests/mppi_ref.py: Philox4x32-10 known answers, Box-Muller against NumPy, the weights, the candidate
and the commit's choice on hand-worked cases, with a negative control; and the C ABI of qs_mppi_* (exports, struct, refusals)."""
import ctypes as C
import math

import numpy as np
import pytest

import mppi_ref as MR
from diff_testlib import params_of
from qs_testlib import harness


def _h():
    return harness("mppi_host")


def _philox(ctr, key):
    c, k, o = (C.c_uint32 * 4)(*ctr), (C.c_uint32 * 2)(*key), (C.c_uint32 * 4)()
    _h().mppi_philox(c, k, o)
    return tuple(o)


@pytest.mark.parametrize("ctr, key, want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    assert _philox(ctr, key) == want
    assert MR.philox(ctr, key) == want


def test_philox_host_matches_python_on_random_counters():
    rng = np.random.default_rng(0)
    for _ in range(200):
        ctr = tuple(int(x) for x in rng.integers(0, 2 ** 32, 4))
        key = tuple(int(x) for x in rng.integers(0, 2 ** 32, 2))
        assert _philox(ctr, key) == MR.philox(ctr, key)


def test_box_muller_against_numpy():
    rng = np.random.default_rng(1)
    worst = 0.0
    words = [tuple(int(x) for x in rng.integers(0, 2 ** 32, 4)) for _ in range(2000)]
    words += [(0, 0, 0, 0), (0xffffffff,) * 4, (0, 1, 0x80000000, 0)]          # the smallest and largest uniforms
    for w in words:
        z = (C.c_double * 2)()
        _h().mppi_box_muller((C.c_uint32 * 4)(*w), z)
        want = MR.box_muller(w)
        for g, r in zip(z, want):
            assert math.isfinite(g)
            worst = max(worst, abs(g - r) / max(abs(r), 1e-300) if abs(r) > 1e-12 else abs(g - r))
    assert worst < 8 * np.finfo(np.float64).eps, worst
    # the uniforms are in (0, 1]: never log(0)
    assert MR.uniform(0, 0) == 0.5 * 2.0 ** -53 and MR.uniform(0xffffffff, 0xffffffff) == 1.0


def test_eps_counter_layout():
    """eps of (k, s, id, it): the host build against the restatement; sample 0 is exactly zero; each counter word matters"""
    seed = (0x0123456789abcdef)
    got = {}
    for k, s, i, it in ((0, 1, 0, 0), (3, 5, 7, 2), (47, 63, 65535, 29), (0, 0, 3, 1), (1, 1, 0, 0), (0, 2, 0, 0), (0, 1, 1, 0),
                        (0, 1, 0, 1)):
        e = (C.c_double * 4)()
        _h().mppi_eps_host(C.c_ulonglong(seed), k, s, C.c_longlong(i), it, e)
        want = MR.eps(seed, k, s, i, it)
        np.testing.assert_allclose(np.array(e), want, rtol=1e-14, atol=1e-15)
        got[(k, s, i, it)] = tuple(e)
    assert got[(0, 0, 3, 1)] == (0.0, 0.0, 0.0, 0.0)
    base = got[(0, 1, 0, 0)]
    for other in ((1, 1, 0, 0), (0, 2, 0, 0), (0, 1, 1, 0), (0, 1, 0, 1)):
        assert got[other] != base
    # the key is (seed low, seed high): another high word gives other noise
    e = (C.c_double * 4)()
    _h().mppi_eps_host(C.c_ulonglong(seed ^ (1 << 40)), 0, 1, C.c_longlong(0), 0, e)
    assert tuple(e) != base


def _update(J, temperature, delta, u):
    J = np.ascontiguousarray(J, dtype=np.float64)
    delta = np.ascontiguousarray(delta, dtype=np.float64)
    u = np.ascontiguousarray(u, dtype=np.float64)
    K, n = delta.shape
    w, cand = np.zeros(K), np.zeros(n)
    p = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    best = _h().mppi_update_host(p(J), K, C.c_double(temperature), p(delta), p(u), n, p(w), p(cand))
    return w, cand, best


def _commit(jc, J):
    J = np.ascontiguousarray(J, dtype=np.float64)
    return _h().mppi_commit_host(C.c_double(jc), J.ctypes.data_as(C.POINTER(C.c_double)), len(J))


CASES = {
    # name: (J, temperature)
    "plain": ([3.0, 2.0, 5.0, 2.5], 0.1),
    "ties": ([3.0, 1.0, 1.0, 4.0, 1.0], 0.5),                 # best = the lowest s of the tie
    "lambda0": ([2.0, 2.0, 2.0], 0.1),                        # every J equal: lambda = 0, w = 1
    "nan_sample": ([3.0, float("nan"), 1.5, float("inf")], 0.2),
    "k2": ([1.0, 0.5], 1.0),
    "dominating": ([1e6, 1.0, 2e6, 3e6], 1e-4),              # one sample carries the weight
    "all_bad": ([float("nan"), float("inf")], 0.1),           # no finite sample: the nominal
    "huge_costs": ([1e5 + 1.0, 1e5, 1e5 + 2.0], 1e-3),        # large J: only the J_min shift keeps the weights finite
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_update_against_reference(name):
    J, temperature = CASES[name]
    K = len(J)
    rng = np.random.default_rng(len(name))
    n = 12
    delta = rng.normal(size=(K, n)) * 100.0
    delta[0] = 0.0                                            # sample 0 is the nominal
    u = 14000.0 + rng.normal(size=n)
    w, cand, best = _update(J, temperature, delta, u)
    w_ref, best_ref = MR.weights(J, temperature)
    np.testing.assert_allclose(w, w_ref, rtol=1e-15, atol=0)
    assert best == best_ref
    np.testing.assert_allclose(cand, MR.candidate(u, delta, w_ref), rtol=1e-14, atol=1e-12)
    if name == "ties":
        assert best == 1 and w[1] == w[2] == w[4] == 1.0
    if name == "lambda0":
        assert list(w) == [1.0, 1.0, 1.0]
    if name == "nan_sample":
        assert w[1] == 0.0 and w[3] == 0.0 and w[2] == 1.0
    if name == "dominating":
        assert w[1] == 1.0 and w[0] < 1e-300 and np.array_equal(cand, u + delta[1])
    if name == "all_bad":
        assert np.array_equal(cand, u) and best == 0


def test_weights_without_the_shift_underflow():
    """negative control: exp(-J / lambda) without J_min underflows to 0 / 0 where the shifted weights are finite"""
    J, temperature = CASES["huge_costs"]
    J = np.array(J)
    lam = temperature * (J.mean() - J.min())
    with np.errstate(invalid="ignore", divide="ignore"):
        raw = np.exp(-J / lam)
        assert raw.sum() == 0.0 and np.isnan((raw * 1.0).sum() / raw.sum())
    w, _ = MR.weights(J, temperature)
    assert w.sum() >= 1.0


@pytest.mark.parametrize("jc, J, want", [
    (1.0, [2.0, 1.5, 3.0], -1),                               # the candidate beats every sample
    (1.5, [2.0, 1.5, 3.0], -1),                               # a tie keeps the candidate
    (1.6, [2.0, 1.5, 3.0], 1),                                # the candidate loses to the best sample
    (float("nan"), [2.0, 1.5, 1.5], 1),                       # a NaN candidate: the lowest s of the best
    (5.0, [float("nan"), 4.0], 1),
    (5.0, [float("nan"), float("inf")], 0),                   # no finite sample: the nominal
])
def test_commit_choice(jc, J, want):
    assert _commit(jc, J) == want == MR.pick(jc, np.array(J))


def test_delta_with_and_without_box():
    d = _h().mppi_delta_host
    d.restype = C.c_double
    dd = lambda *a: d(*[C.c_double(x) for x in a[:5]], a[5])
    assert dd(100.0, 10.0, 0.5, 0.0, 1e9, 0) == 5.0
    assert dd(100.0, 10.0, 0.5, 0.0, 102.0, 1) == 2.0          # clamped: the perturbation stays in the box
    assert dd(100.0, 10.0, -20.0, 90.0, 102.0, 1) == -10.0
    assert dd(100.0, 10.0, -20.0, 90.0, 102.0, 0) == -200.0


def test_abi_exports_struct_and_refusals():
    from gym_pybullet_drones_b200 import _native as N
    L = N.lib()
    for name in ("qs_mppi_sample", "qs_mppi_update", "qs_mppi_commit", "qs_mppi_noise", "qs_sizeof_mppi_io"):
        assert name in N.EXPORTS
        getattr(L, name)
    assert L.qs_sizeof_mppi_io() == C.sizeof(N.QsMppiIO) == 16 + 8 + 8 + 16 * 8
    P, _ = params_of("cf2x")
    buf = (C.c_double * 64)()
    a = C.addressof(buf)
    common = ("state0", "rpm", "targets", "weights", "rpm_ref", "sigma")
    for f, outs in ((L.qs_mppi_sample, ("J",)), (L.qs_mppi_update, ("J", "cand")), (L.qs_mppi_commit, ("states", "cost_out"))):
        io = N.QsMppiIO(T=2, K=4, temperature=0.1)
        call = lambda *args: f(C.byref(P), C.byref(io), *args, None)
        assert f(None, C.byref(io), 1, 1, 1, 0, None) == -1
        assert f(C.byref(P), None, 1, 1, 1, 0, None) == -1
        for k in common + outs:
            assert call(1, 1, 1, 0) == -1, k                      # each missing pointer is refused
            assert L.qs_last_error().startswith(f.__name__.encode() + b": ")
            setattr(io, k, a)
        if f is L.qs_mppi_commit:
            io.cand = a                                           # J is needed with a candidate
            assert call(1, 1, 1, 0) == -1
            io.J = a
        assert call(1, 1, 1, 8) == -4
        assert call(1, 1, 1, 5) == -5 and call(1, 1, 1, 6) == -5   # GND|DW, DRAG|DW
        assert call(1, 129, 1, N.EFFECT_DW) == -5 and b"128" in L.qs_last_error()
        for bad in (1, 1025):
            io.K = bad
            assert call(1, 1, 1, 0) == -3 and b"K" in L.qs_last_error()
        io.K = 4
        io.iteration = -1
        assert call(1, 1, 1, 0) == -3
        io.iteration = 0
        io.per_tick = 2
        assert call(1, 1, 1, 0) == -3
        io.per_tick = 0
        io.rpm_lo = a
        assert call(1, 1, 1, 0) == -1
        io.rpm_lo = None
        if f is L.qs_mppi_update:
            for t in (0.0, -1.0, float("nan"), float("inf")):
                io.temperature = t
                assert call(1, 1, 1, 0) == -3 and b"temperature" in L.qs_last_error()
            io.temperature = 0.1
        io.phys = a + 8
        assert call(1, 1, 1, 0) == -2
        io.phys = None
        assert call(0, 1, 1, 0) == -3
        assert call(1, 0, 1, 0) == -3
        assert call(1, 1, 0, 0) == -3
        assert call(65536, 65536, 1, 0) == -3
        io.T = 0
        assert call(1, 1, 1, 0) == -3
    io = N.QsMppiIO(T=2, K=4)
    assert L.qs_mppi_noise(None, 1, 1, None) == -1
    assert L.qs_mppi_noise(C.byref(io), 1, 1, None) == -1
    io.noise = a
    io.K = 1
    assert L.qs_mppi_noise(C.byref(io), 1, 1, None) == -3


# ---- the float64 references of the GPU edge tests ------------------------------------------------------------------------------

def test_eps_counter_past_2_to_the_30():
    """the counter's fourth word is 2 it + h in unsigned arithmetic: every iteration in [0, 2^31) has its own noise, and the host
    build agrees with the restatement on both sides of 2^30 (where 2 it no longer fits an int)"""
    seed = 0x9e3779b97f4a7c15
    got = {}
    for it in (2 ** 30 - 1, 2 ** 30, 2 ** 31 - 1):
        e = (C.c_double * 4)()
        _h().mppi_eps_host(C.c_ulonglong(seed), 3, 7, C.c_longlong(11), it, e)
        np.testing.assert_allclose(np.array(e), MR.eps(seed, 3, 7, 11, it), rtol=1e-14, atol=1e-15)
        got[it] = tuple(e)
    assert len(set(got.values())) == 3


def test_vectorised_philox_matches_the_restatement():
    rng = np.random.default_rng(7)
    seed = 0x0123456789abcdef
    k, s, i, it = (rng.integers(0, 48, 64), rng.integers(0, 1024, 64), rng.integers(0, 2 ** 31, 64), rng.integers(0, 2 ** 31, 64))
    s[:4] = 0
    got = MR.eps_vec(seed, k, s, i, it)
    want = np.array([MR.eps(seed, *(int(x) for x in c)) for c in zip(k, s, i, it)])
    assert np.array_equal(got[:4], np.zeros((4, 4)))
    np.testing.assert_allclose(got, want, rtol=1e-14, atol=1e-15)


def test_weights_sum_in_s_order():
    """lambda's sum of the finite J runs in s order, as the kernel's scan: the restatement gives the host build's weights bit for
    bit at K = 1024, where np.mean's pairwise partial sums round otherwise (the negative control); a finite sum that overflows
    gives lambda = inf and every finite weight 1"""
    rng = np.random.default_rng(8)
    J = rng.uniform(0.0, 1.0, 1024) * 10.0 ** rng.integers(-3, 4, 1024)
    J[5], J[77] = float("nan"), float("inf")
    delta, u = np.zeros((1024, 1)), np.zeros(1)
    w, _, best = _update(J, 1e-3, delta, u)
    w_ref, best_ref = MR.weights(J, 1e-3)
    assert best == best_ref and np.array_equal(w, w_ref)
    assert not np.array_equal(w, MR.weights(J, 1e-3, order="numpy")[0])
    big = np.array([1e308, 0.5, 1e308, 2.0])
    w, _, best = _update(big, 0.1, np.zeros((4, 1)), u)
    assert best == 1 and np.array_equal(w, np.ones(4)) and np.array_equal(MR.weights(big, 0.1)[0], w)
    # the unit sum: drone order from 0.0, and the reverse order rounds otherwise
    Jd = np.array([[1.0, 1e16, -1e16]])
    assert MR.unit_sum(Jd, 3)[0, 0] == 0.0 and MR.unit_sum(Jd, 3, reverse=True)[0, 0] == 1.0


def _stacked_states(rng, E, D, model):
    from diff_testlib import quat_from_rpy
    n = E * D
    pos = np.zeros((E, D, 3))
    pos[:, :, 2] = 0.06 + 1.5 * np.arange(D)                          # the lowest drone in ground effect
    pos[:, :, :2] = rng.uniform(-0.05, 0.05, (E, D, 2))
    pos[:, -1, 0] += 12.0                                             # the top drone beyond 10 m in xy: no pair with it
    rpy = rng.uniform(-0.2, 0.2, (n, 3))
    q = np.stack([quat_from_rpy(r) for r in rpy])
    vel, w = rng.uniform(-0.5, 0.5, (n, 3)), rng.uniform(-2, 2, (n, 3))
    return np.concatenate([pos.reshape(n, 3), q, vel, w], axis=1)


@pytest.mark.parametrize("model", ["cf2x", "cf2p"])
def test_downwash_reference_matches_oracle(model):
    """mppi_ref.rollout_dw (GND|DRAG|DW, 240/48 Hz) against the NumPy oracle's downwash_body_z + dynamics_substep over four ticks
    of stacked drones, drag's substep 0 reading the previous tick's rpm; a reference without the downwash is far off"""
    import torch
    import diff_ref as DR
    from oracle import dyn_oracle as O
    from test_diff_host import _nominal_rows
    P, c = params_of(model, 240, 48)
    OP = O.OracleParams(model, 240, 48)
    rng = np.random.default_rng(3)
    E, D, T, S = 3, 4, 4, 5
    n = E * D
    x0 = _stacked_states(rng, E, D, model)
    v = float(c.HOVER_RPM) * (1 + 0.05 * rng.uniform(-1, 1, (T, n, 4)))
    up0 = float(c.HOVER_RPM) * (1 + 0.05 * rng.uniform(-1, 1, (n, 4)))
    got = MR.rollout_dw(DR.model_constants(P), P, _nominal_rows(model, n), torch.tensor(x0), torch.tensor(up0), torch.tensor(v), S, 7, D)
    pos, quat, vel, w = x0[:, 0:3], x0[:, 3:7], x0[:, 7:10], x0[:, 10:13]
    up, want, fz_seen = up0, [], 0.0
    for k in range(T):
        u = np.clip(v[k], 0, OP.MAX_RPM)
        for s in range(S):
            fz = O.downwash_body_z(OP, pos.reshape(E, D, 3)).reshape(n)
            fz_seen = max(fz_seen, np.abs(fz).max())
            pos, quat, vel, w, _ = O.dynamics_substep(OP, u, pos, quat, vel, w, 7, rpm_prev=up if s == 0 else u, dw_fz=fz)
        up = u
        want.append(np.concatenate([pos, quat, vel, w], axis=1))
    want = np.stack(want)
    err = np.max(np.abs(got.numpy() - want) / np.maximum(np.abs(want), 1.0))
    assert fz_seen > 1e-3 and err <= 1e-12, (fz_seen, err)
    none = DR.rollout(DR.model_constants(P), _nominal_rows(model, n), torch.tensor(x0), torch.tensor(v), torch.tensor(up0), S, 3)
    assert np.max(np.abs(none.numpy() - want)) > 1e-6
