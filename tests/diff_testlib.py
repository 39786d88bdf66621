"""Shared helpers of the differentiable-trajectory tests (test infrastructure): the g++ build of dyn_adjoint.cuh (the adjoint core
of the dyn_traj kernels) and the drone batches the tests differentiate at."""
import ctypes as C
import functools

import numpy as np

from qs_testlib import drone_model, harness

MODELS = ("cf2x", "cf2p", "race")


def diff_harness():
    """tests/host_harness/diff_host.cpp: the kernels' tick adjoint compiled for the host."""
    L = harness("diff_host")
    L.dh_tick_vjp.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_int, C.c_int] + [C.c_void_p] * 9
    L.dh_half_angle_grad.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_void_p]
    return L


def params_of(model, pyb_freq=240, ctrl_freq=240):
    """(QsParams, AviaryConstants) of a drone model."""
    from gym_pybullet_drones_b200.params import AviaryConstants, fill_params
    c = AviaryConstants(drone_model(model), pyb_freq, ctrl_freq)
    return fill_params(c), c


def quat_from_rpy(rpy):
    from gym_pybullet_drones_b200.params import quaternion_from_euler
    return quaternion_from_euler(np.asarray(rpy, dtype=np.float64))


def scenarios(c, rng, n=4):
    """{name: (state [n, 13], raw rpm [n, 4], previous clipped rpm [n, 4])} at the decision points of DESIGN.md 4.5.  c: the
    model's AviaryConstants."""
    hover, mx = float(c.HOVER_RPM), float(c.MAX_RPM)
    clip = float(c.GND_EFF_H_CLIP)

    def state(pos, rpy, vel, w):
        q = quat_from_rpy(rpy)
        return np.concatenate([pos, q, vel, w], axis=1)

    def rnd(lo, hi, shape):
        return rng.uniform(lo, hi, shape)

    z3 = np.zeros((n, 3))
    out = {}
    # exact hover: level, at rest, equal RPMs -- w = 0 in every substep (the isclose branch of the forward)
    out["hover"] = (state(np.tile([0.0, 0.0, 1.0], (n, 1)), z3, z3, z3), np.full((n, 4), hover), np.full((n, 4), hover))
    # generic flight
    out["flight"] = (state(rnd(-1, 1, (n, 3)) + [0, 0, 1.5], rnd(-0.4, 0.4, (n, 3)), rnd(-1, 1, (n, 3)), rnd(-3, 3, (n, 3))),
                     hover * rnd(0.8, 1.2, (n, 4)), hover * rnd(0.8, 1.2, (n, 4)))
    # tumbling: |w| dt / 2 beyond 1/2 (the sqrt / sincos range of half_angle_terms) at 240 Hz, mostly about the body z axis (about
    # a transverse axis the explicit Euler step of w x Jw amplifies the rates by ~1.7 per substep at these speeds)
    w = np.concatenate([rnd(-5, 5, (n, 2)), rnd(250, 300, (n, 1)) * np.sign(rnd(-1, 1, (n, 1)))], 1)
    out["tumbling"] = (state(rnd(-1, 1, (n, 3)) + [0, 0, 2], rnd(-3, 3, (n, 3)), rnd(-2, 2, (n, 3)), w),
                       hover * rnd(0.5, 1.5, (n, 4)), hover * rnd(0.5, 1.5, (n, 4)))
    # propellers below the ground-effect height clip (and some above it)
    out["ground"] = (state(np.concatenate([rnd(-1, 1, (n, 2)), rnd(0.1 * clip, 1.5 * clip, (n, 1))], 1), rnd(-0.2, 0.2, (n, 3)),
                           rnd(-0.5, 0.5, (n, 3)), rnd(-2, 2, (n, 3))), hover * rnd(0.8, 1.2, (n, 4)), hover * rnd(0.8, 1.2, (n, 4)))
    # RPM commands beyond the clip on both sides
    raw = hover * rnd(0.8, 1.2, (n, 4))
    raw[:, 0] = mx * rnd(1.01, 1.5, n)
    raw[:, 2] = -hover * rnd(0.01, 0.5, n)
    out["clipped"] = (state(rnd(-1, 1, (n, 3)) + [0, 0, 0.05], rnd(-0.3, 0.3, (n, 3)), rnd(-1, 1, (n, 3)), rnd(-3, 3, (n, 3))),
                      raw, np.clip(hover * rnd(0.8, 1.2, (n, 4)), 0, mx))
    # tilted past the upright switch (|roll| > pi/2), near the ground
    rpy = np.concatenate([rnd(1.7, 2.8, (n, 1)) * np.sign(rnd(-1, 1, (n, 1))), rnd(-0.3, 0.3, (n, 2))], 1)
    out["tilted"] = (state(np.concatenate([rnd(-1, 1, (n, 2)), rnd(0.02, 0.2, (n, 1))], 1), rpy, rnd(-1, 1, (n, 3)), rnd(-3, 3, (n, 3))),
                     hover * rnd(0.8, 1.2, (n, 4)), hover * rnd(0.8, 1.2, (n, 4)))
    return out


def host_tick_vjp(P, effects, S, state, raw, up, g_out, rows=None):
    """The host-built kernel core: one tick and its VJP.  Returns (out, g_state, g_raw, g_up, g_row)."""
    L = diff_harness()
    n = state.shape[0]
    a = lambda x: np.ascontiguousarray(x, dtype=np.float64)
    state, raw, up, g_out = a(state), a(raw), a(up), a(g_out)
    rows = None if rows is None else a(rows)
    outs = [np.zeros((n, 13)), np.zeros((n, 13)), np.zeros((n, 4)), np.zeros((n, 4)), np.zeros((n, 16))]
    p = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)
    L.dh_tick_vjp(C.addressof(P), p(rows), effects, S, n, p(state), p(raw), p(up), p(g_out), *[p(o) for o in outs])
    return outs


# ---- per-drone comparison ------------------------------------------------------------------------------------------------

def per_drone_relerr(got, want):
    """[n] normwise relative errors ||got_i - want_i|| / ||want_i|| of arrays whose first axis is the drone (or aviary).  Where
    want_i is zero the error is 0 only if got_i is exactly zero too (inf otherwise)."""
    got = np.asarray(got, dtype=np.float64).reshape(len(want), -1)
    want = np.asarray(want, dtype=np.float64).reshape(len(want), -1)
    n = np.linalg.norm(want, axis=1)
    d = np.linalg.norm(got - want, axis=1)
    return np.where(n > 0, d / np.where(n > 0, n, 1.0), np.where(np.any(got != 0, axis=1), np.inf, 0.0))


BLOCKS = ("rpm", "pos", "quat", "vel", "rpy_rates", "last_rpm", "row")


def split_grads(g_rpm, g_state, g_last, g_row):
    """{block: [n, ...]} of one VJP: g_rpm [T, n, 4] (drone first after this), g_state [n, 13], g_last [n, 4], g_row [n or E, 16]."""
    g_rpm = np.moveaxis(np.asarray(g_rpm), 0, 1) if np.ndim(g_rpm) == 3 else np.asarray(g_rpm)
    g_state = np.asarray(g_state)
    return {"rpm": g_rpm, "pos": g_state[:, 0:3], "quat": g_state[:, 3:7], "vel": g_state[:, 7:10], "rpy_rates": g_state[:, 10:13],
            "last_rpm": np.asarray(g_last), "row": np.asarray(g_row)}


def worst_per_block(got, want):
    """{block: worst per-drone relative error} of two split_grads dicts."""
    return {k: float(np.max(per_drone_relerr(got[k], want[k]))) for k in got}


def aviary_rows(model, E, rng, device=None):
    """(props, rows [E, 16]): the model's PHYS_KEYS values with m, J and kf scaled by U[0.8, 1.2] per aviary.  J is scaled as a
    whole: independent factors can make body z the intermediate axis of inertia, about which the tumbling scenario's spin is
    unstable (the rates grow by 1e20 within 24 substeps and the trajectory's own condition number passes 1e13)."""
    import torch
    from gym_pybullet_drones_b200.params import PHYS_KEYS, nominal_properties, physical_rows
    nom = nominal_properties(drone_model(model))
    f = {k: rng.uniform(0.8, 1.2, E) for k in ("m", "J", "kf")}
    props = {}
    for k in PHYS_KEYS:
        v = np.full(E, nom[k]) * f.get("J" if k in ("ixx", "iyy", "izz") else k, 1.0)
        props[k] = torch.tensor(v, dtype=torch.float64, device=device)
    return props, physical_rows(drone_model(model), props)


def scenario_ticks(c, rows, T, seed, n):
    """The six scenarios as one batch, each over T ticks in its own regime: (names [6 n], state [6 n, 13], raw rpm [T, 6 n, 4],
    previous clipped rpm [6 n, 4]).  rows: [6 n, 16] per-drone rows; every RPM is scaled by the row's HOVER_RPM over the model's
    (MAX_RPM / HOVER_RPM is the same in every row), so hover is the row's exact hover and clipped entries stay beyond its clip."""
    draws = [scenarios(c, np.random.default_rng([seed, k]), n) for k in range(T)]
    names = list(draws[0])
    scale = np.asarray(rows)[:, 12] / float(c.HOVER_RPM)
    state = np.concatenate([draws[0][s][0] for s in names])
    raw = np.stack([np.concatenate([d[s][1] for s in names]) for d in draws]) * scale[None, :, None]
    up = np.concatenate([draws[0][s][2] for s in names]) * scale[:, None]
    return np.repeat(names, n), state, raw, np.minimum(up, np.asarray(rows)[:, 13:14])


# ---- decision lattices: states and commands exactly on each boundary of DESIGN.md 4.5 and one ulp either side -------------
# Everything is decided in float64 with the kernels' operation order (the library builds with -fmad=false, the harness with
# -ffp-contract=off), so Python floats evaluate each predicate exactly as the kernels and the reference do.

_UPRIGHT_T = 1.722546424198833e-16


def _fma(a, b, c):
    from fractions import Fraction
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def _ulps(v, k):
    """v moved by k float64 ulps (toward +inf for k > 0)."""
    if v == 0 or abs(k) <= 1:
        return float(np.nextafter(v, np.inf if k > 0 else -np.inf)) if k else float(v)
    i = np.array(v, dtype=np.float64).view(np.int64)
    return float((i + (k if v > 0 else -k)).view(np.float64))


def unit_exact(q):
    """|q|^2 is 1.0 exactly however it is evaluated (quat_norm2's fma chain, any order of float64 sums): the entry renormalisation
    is then the identity on the device (rsqrt), on the host (1 / sqrt) and in the reference (q / sqrt), and the state the
    decision is taken on is the given one on every build."""
    import itertools
    x, y, z, w = q
    if _fma(w, w, _fma(z, z, _fma(y, y, x * x))) != 1.0:
        return False
    s = [x * x, y * y, z * z, w * w]
    if any(((s[a] + s[b]) + s[c]) + s[d] != 1.0 for a, b, c, d in itertools.permutations(range(4))):
        return False
    return (s[0] + s[1]) + (s[2] + s[3]) == 1.0 and (s[0] + s[2]) + (s[1] + s[3]) == 1.0


def upright_terms(q):
    """(sarg, ra, rb) of quad_core.cuh upright() for the quaternion (x, y, z, w), in its operation order."""
    x, y, z, w = q
    return -2.0 * (x * z - w * y), 2.0 * (y * z + w * x), w * w - x * x - y * y + z * z


def is_upright(q):
    sarg, ra, rb = upright_terms(q)
    return (sarg > -0.99999) and (sarg < 0.99999) and (rb > _UPRIGHT_T * abs(ra) or (rb == 0.0 and ra == 0.0))


def prop_heights(P, pz, q):
    """hz of the four propellers (quad_core.cuh dyn_tick_k's ground-effect height, its operation order)."""
    x, y, z, w = q
    xs, ys, zs = x + x, y + y, z + z
    r20, r21, r22 = x * zs - w * ys, y * zs + w * xs, 1.0 - (x * xs + y * ys)
    return [pz + r20 * P.prop_xyz[i][0] + r21 * P.prop_xyz[i][1] + r22 * P.prop_xyz[i][2] for i in range(4)]


@functools.lru_cache(maxsize=None)
def _upright_rb_lattice():
    """{-1, 0, +1: q}: roll near pi/2 with rb one ulp below, exactly at and one ulp above T |ra| (the upright switch's roll
    threshold).  rb = fl(w^2) - fl(x^2) - y^2 with x ~ w ~ 1/sqrt(2): y (~1e-8) sets rb to the ulp."""
    import math
    found = {}
    c = math.sqrt(0.5)
    for dx in range(-6, 7):
        x = _ulps(c, dx)
        for dw in range(-6, 7):
            w = _ulps(c, dw)
            a0 = w * w - x * x
            thr = _UPRIGHT_T * abs(2.0 * (0.0 + w * x))
            if not thr < a0 < 4e-16:
                continue
            y0 = math.sqrt(a0 - thr)
            for dy in range(-400, 400):
                q = (x, _ulps(y0, dy), 0.0, w)
                _, ra, rb = upright_terms(q)
                for off in (-1, 0, 1):
                    if off not in found and rb == _ulps(_UPRIGHT_T * abs(ra), off) and unit_exact(q):
                        found[off] = q
                if len(found) == 3:
                    return found
    raise AssertionError("no upright-threshold lattice found")


@functools.lru_cache(maxsize=None)
def _upright_sarg_lattice(sign):
    """{-1, 0, +1: q}: pitch near sign * pi/2 with sarg = sign * 0.99999 one ulp below, at and one ulp above (the gimbal guard)."""
    import math
    s0 = sign * 0.99999
    found = {}
    p = math.asin(0.99999)
    y0 = math.sin(p / 2)
    for dy in range(-4000, 4000):
        y = _ulps(y0, dy)
        for dw in range(-8, 9):
            q = (0.0, sign * y, 0.0, _ulps(math.sqrt(1 - y * y), dw))
            sarg = upright_terms(q)[0]
            for off in (-1, 0, 1):
                if off not in found and sarg == _ulps(s0, off) and unit_exact(q):
                    found[off] = q
            if len(found) == 3:
                return found
    raise AssertionError("no gimbal-guard lattice found")


def _exact_unit_near(q):
    """The unit_exact quaternion nearest q in a few ulps of its components."""
    for k in range(0, 40):
        for dw in (k, -k):
            for dx in range(-3, 4):
                c = (_ulps(q[0], dx), q[1], q[2], _ulps(q[3], dw))
                if unit_exact(c):
                    return c
    raise AssertionError("no exactly unit quaternion near %s" % (q,))


def lattices(P, c, rows, rng):
    """{name: dict(state [n, 13], raw [n, 4], up [n, 4], S, effects, label [n], rows [n, 16])} for one model: the decision
    lattices of DESIGN.md 4.5, one tick each.  rows: [>= n, 16] per-drone rows (each lattice drone gets its own).  Within a
    lattice every drone shares velocity, rates and RPMs unless the decision is about them, so neighbours differ by the decision.
      rpm        raw in {MAX_RPM of the row, 0.0, -0.0} and their float64 neighbours, one rotor at a time.  S = 2 with drag: at
                 u = 0 thrust's gradient 2 u kf vanishes, drag's sum over the current RPMs (substeps 1..) carries it.  label: the
                 lattice value's index (0..6 = max-, max, max+, -0-, -0, 0, 0+).
      clip       level, with the propellers' height pz + prop_z one ulp below, on and one ulp above GND_EFF_H_CLIP, and a roll of
                 0.5 rad whose propeller 0 lands on it.  label: +1 above the clip, 0 on it, -1 below (propeller 0).
      half_angle |w|^2 (dt/2)^2 (half_angle_terms' t) one ulp below, at and one ulp above 1/4 about each axis, w = 0, |w| = 1e-8
                 and |w|^2 one ulp either side of the isclose bound 1e-16; equal RPMs so the substep leaves w unchanged.  label:
                 -1 below, 0 at, +1 above t = 1/4; 2 w = 0; 3 isclose taken, 4 not.
      upright    rb one ulp below, at and above T |ra| (roll near pi/2), sarg one ulp below, at and above +-0.99999, with the
                 propellers live just above the clip.  label: 1 upright, 0 not."""
    import math
    rows = np.asarray(rows)
    hover = float(c.HOVER_RPM)
    clip = float(P.gnd_eff_h_clip)
    out = {}

    def flight(n, pz, q, w):
        st = np.zeros((n, 13))
        st[:, 0:2] = rng.uniform(-1, 1, 2)
        st[:, 2] = pz
        st[:, 3:7] = q
        st[:, 7:10] = rng.uniform(-1, 1, 3)
        st[:, 10:13] = w
        return st

    # RPM clip
    vals = lambda mx: [_ulps(mx, -1), mx, _ulps(mx, 1), _ulps(-0.0, -1), -0.0, 0.0, _ulps(0.0, 1)]
    n = 7 * 4
    r = rows[:n]
    raw = np.tile(hover * np.array([1.02, 0.98, 1.01, 0.99]), (n, 1)) * (r[:, 12:13] / hover)
    label = np.zeros(n, dtype=int)
    for i in range(n):
        label[i], j = i % 7, i // 7
        raw[i, j] = vals(float(r[i, 13]))[label[i]]
    st = flight(n, 1.0, quat_from_rpy(rng.uniform(-0.3, 0.3, 3)), rng.uniform(-2, 2, 3))
    out["rpm"] = dict(state=st, raw=raw, up=np.tile(hover * rng.uniform(0.9, 1.1, 4), (n, 1)), S=2, effects=2, label=label, rows=r)

    # ground-effect height clip (prop_z = 0 for every model: a level drone's propellers sit at pz)
    qs = [(0.0, 0.0, 0.0, 1.0)]
    qt = _exact_unit_near((math.sin(0.25), 0.0, 0.0, math.cos(0.25)))
    states, label = [], []
    w = rng.uniform(-2, 2, 3)
    for off in (-1, 0, 1):
        pz = _ulps(clip, off)
        assert all(h == pz for h in prop_heights(P, pz, qs[0])) and P.prop_xyz[0][2] == 0.0
        states.append(flight(1, pz, qs[0], w)); label.append(off)
    pz0 = clip - (prop_heights(P, 0.0, qt)[0])
    hit = None
    for k in range(-64, 65):
        if prop_heights(P, _ulps(pz0, k), qt)[0] == clip:
            hit = _ulps(pz0, k)
            break
    assert hit is not None
    for off in (-1, 0, 1):
        pz = _ulps(hit, off)
        h0 = prop_heights(P, pz, qt)[0]
        states.append(flight(1, pz, qt, w)); label.append((h0 > clip) - (h0 < clip))
    st = np.concatenate(states)
    n = len(st)
    r = rows[:n]
    out["clip"] = dict(state=st, raw=np.tile(hover * np.array([1.05, 0.97, 1.02, 0.96]), (n, 1)) * (r[:, 12:13] / hover),
                       up=np.zeros((n, 4)), S=1, effects=1, label=np.array(label), rows=r)

    # half_angle_grad's switch and the isclose region
    dt = float(P.dt)
    h = 0.5 * dt
    tt = lambda a: a * a * h * h
    a0 = 1.0 / dt
    while tt(a0) < 0.25:
        a0 = _ulps(a0, 1)
    while tt(_ulps(a0, -1)) >= 0.25:
        a0 = _ulps(a0, -1)
    assert tt(a0) == 0.25 and tt(_ulps(a0, -1)) < 0.25
    a1 = a0
    while tt(a1) == 0.25:
        a1 = _ulps(a1, 1)
    ai = 1e-8
    while ai * ai > 1e-16:
        ai = _ulps(ai, -1)
    while _ulps(ai, 1) ** 2 <= 1e-16:
        ai = _ulps(ai, 1)
    rates, label = [], []
    for axis in range(3):
        for a, lab in ((_ulps(a0, -1), -1), (a0, 0), (a1, 1)):
            v = np.zeros(3); v[axis] = a
            rates.append(v); label.append(lab)
    for a, lab in ((0.0, 2), (1e-8, 3 if 1e-8 * 1e-8 <= 1e-16 else 4), (ai, 3), (_ulps(ai, 1), 4)):
        rates.append(np.array([0.0, a, 0.0])); label.append(lab)
    n = len(rates)
    r = rows[:n]
    q = quat_from_rpy(rng.uniform(-0.4, 0.4, 3))
    st = np.concatenate([flight(1, 1.0, q, v) for v in rates])
    out["half_angle"] = dict(state=st, raw=np.full((n, 4), 1.05 * hover) * (r[:, 12:13] / hover), up=np.zeros((n, 4)), S=1,
                             effects=0, label=np.array(label), rows=r)

    # the upright switch
    quats = [lat[k] for lat in (_upright_rb_lattice(), _upright_sarg_lattice(1.0), _upright_sarg_lattice(-1.0)) for k in (-1, 0, 1)]
    reach = max(abs(P.prop_xyz[i][a]) for i in range(4) for a in range(2))
    w = rng.uniform(-2, 2, 3)
    st = np.concatenate([flight(1, clip + reach + 0.01, q, w) for q in quats])
    n = len(st)
    r = rows[:n]
    out["upright"] = dict(state=st, raw=np.tile(hover * np.array([1.05, 0.97, 1.02, 0.96]), (n, 1)) * (r[:, 12:13] / hover),
                          up=np.zeros((n, 4)), S=1, effects=1, label=np.array([int(is_upright(q)) for q in quats]), rows=r)
    for lat in out.values():
        lat["g_out"] = np.tile(rng.standard_normal(13), (len(lat["state"]), 1))
    return out


# pairs of lattice drones one ulp apart on the two sides of each decision (indices into the lattice's drones)
SIDE_PAIRS = {"clip": [(0, 1), (3, 4)], "upright": [(1, 2), (3, 4), (7, 8)], "rpm": [(1, 2), (3, 4)]}


def ref_tick_vjp(P, rows, effects, S, state, raw, up, g_out, device=None, **kw):
    """diff_ref's tick and its autograd VJP on `device` (numpy in and out): (out, g_state, g_raw, g_up, g_row)."""
    import torch
    import diff_ref as R
    t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64), device=device)
    x, r, u, rw = (t(a).requires_grad_(True) for a in (state, raw, up, rows))
    out, _ = R.tick(R.model_constants(P, device), rw, x, r, u, S, effects, **kw)
    gs = torch.autograd.grad(out, (x, r, u, rw), t(g_out), allow_unused=True)
    gs = [torch.zeros_like(v) if g is None else g for g, v in zip(gs, (x, r, u, rw))]
    return [out.detach().cpu().numpy()] + [g.cpu().numpy() for g in gs]


def check_lattice(name, lat, got, want, fwd_ref, tol):
    """Asserts one tick's outputs `got` (out, g_state, g_raw, g_up, g_row; per drone) on a lattice against the reference `want`
    per drone: forward <= 1e-12 against `fwd_ref` (the forward takes np.isclose's identity where |w|^2 <= 1e-16, the reference's
    exact_branch=True), every block <= tol; the RPM clip's gradient exactly 0 outside [0, MAX_RPM] and MAX_RPM's only strictly
    above; last_rpm's exactly 0 without drag.  Returns {block: worst}."""
    e_fwd = float(np.max(per_drone_relerr(got[0], fwd_ref)))
    assert e_fwd <= 1e-12, (name, "forward", e_fwd)
    g, w = split_grads(got[2], got[1], got[3], got[4]), split_grads(want[2], want[1], want[3], want[4])
    worst = worst_per_block(g, w)
    worst["forward"] = e_fwd
    for k, e in worst.items():
        assert e <= tol, (name, k, e)
    if name == "rpm":
        lab = lat["label"]
        j = np.arange(len(lab)) // 7                                  # the lattice rotor
        g_lat = got[2][np.arange(len(lab)), j]
        assert np.all((g_lat == 0) == np.isin(lab, (2, 3))), (lab, g_lat)      # passes at max-, max, -0.0, 0.0, 0+ only
        assert np.all((got[4][:, 13] != 0) == (lab == 2))                     # MAX_RPM receives it only strictly above
    if not lat["effects"] & 2:
        assert np.all(got[3] == 0)
    return worst
