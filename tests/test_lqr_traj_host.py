"""CPU tests of the differentiable tracker loop (qs_dyn_lqr_traj_vjp, DESIGN.md 4.5): one tracker tick's VJP -- the law and its
adjoint (lqr_law.cuh), the box, the env's clip and the tick adjoint (dyn_adjoint.cuh), built for the host -- against torch autograd
of tests/ilqr_tracker_ref.py's law and tests/diff_ref.py's tick, per input block; every clamp decision at its boundary with
torch.clamp's convention, a strict-inequality reference as the negative control; and the C ABI's refusals without a GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

import diff_ref as R
import ilqr_tracker_ref as TR
from diff_testlib import params_of, quat_from_rpy
from qs_testlib import harness

EFFECTS = {"dyn": 0, "gnd": R.EFFECT_GND, "drag": R.EFFECT_DRAG, "gnd_drag": R.EFFECT_GND | R.EFFECT_DRAG}
BLOCKS = ("state", "last_rpm", "phys", "rpm_nom", "K", "z_nom")
VJP_TOL = 1e-10                                   # normwise relative, the test_diff_host standard


def lqr_harness():
    """tests/host_harness/lqr_traj_host.cpp"""
    L = harness("lqr_traj_host")
    L.lh_tick_vjp.argtypes = [C.c_void_p, C.c_uint, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 17
    return L


def host_tick_vjp(P, eff, S, rows, state, up, rpm_nom, K, z_nom, lo, hi, g_out, g_rpm):
    """The host-built kernel core: one tracker tick and its VJP.  Returns {out, rpm} and the gradients of BLOCKS."""
    n, nz = state.shape[0], z_nom.shape[1]
    a = lambda x: None if x is None else np.ascontiguousarray(x, dtype=np.float64)
    ins = [a(x) for x in (rows, state, up, rpm_nom, K, z_nom, lo, hi, g_out, g_rpm)]
    outs = [np.zeros((n, w)) for w in (13, 4, 13, 4, 16, 4)] + [np.zeros((n, 4, nz)), np.zeros((n, nz))]
    p = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)
    lqr_harness().lh_tick_vjp(C.addressof(P), eff, S, nz, n, *[p(x) for x in ins], *[p(o) for o in outs])
    res = dict(out=outs[0], rpm=outs[1])
    res.update(zip(BLOCKS, outs[2:]))
    return res


def strict_clampd(v, lo, hi):
    """clampd whose gradient passes only strictly inside (lo, hi): a negative control"""
    return torch.where(v <= lo, lo.detach() if isinstance(lo, torch.Tensor) else lo, torch.where(v >= hi, hi, v))


def ref_tick_vjp(P, eff, S, rows, state, up, rpm_nom, K, z_nom, lo, hi, g_out, g_rpm, strict=False):
    """ilqr_tracker_ref.control (box only) then diff_ref.tick (the env's clip as torch.clamp) and their autograd VJP, in the
    layout of host_tick_vjp.  strict=True: both clamps pass the gradient only strictly inside their bounds."""
    t = {k: torch.tensor(np.asarray(v, dtype=np.float64), requires_grad=True) for k, v in
         dict(state=state, last_rpm=up, phys=rows, rpm_nom=rpm_nom, K=K, z_nom=z_nom).items()}
    b = TR.control(t["state"], t["last_rpm"], t["z_nom"], t["K"], t["rpm_nom"])
    if lo is not None:
        lo_t, hi_t = torch.tensor(lo), torch.tensor(hi)
        b = strict_clampd(b, lo_t, hi_t) if strict else TR.clampd(b, lo_t, hi_t)
    if strict:
        mx = t["phys"][:, 13:14].expand_as(b)
        b = strict_clampd(b, torch.zeros_like(b), mx)
    out, u = R.tick(R.model_constants(P), t["phys"], t["state"], b, t["last_rpm"], S, eff)
    loss = (out * torch.tensor(g_out)).sum() + (u * torch.tensor(g_rpm)).sum()
    gs = torch.autograd.grad(loss, [t[k] for k in BLOCKS], allow_unused=True)
    res = {k: (torch.zeros_like(t[k]) if g is None else g).numpy() for k, g in zip(BLOCKS, gs)}
    res.update(out=out.detach().numpy(), rpm=u.detach().numpy())
    return res


def _rows(model, n, rng):
    from gym_pybullet_drones_b200.params import nominal_properties, physical_rows
    from diff_testlib import drone_model
    nom = nominal_properties(drone_model(model))
    rows = physical_rows(drone_model(model), {k: torch.full((n,), v, dtype=torch.float64) for k, v in nom.items()}).numpy()
    rows[:, 0] *= rng.uniform(0.85, 1.15, n)                  # per-drone constants
    rows[:, 2] *= rng.uniform(0.85, 1.15, n)
    return rows


def _case(model, eff, nz, box, rng, n=16, S=5):
    """n drones around hover, some near the ground (ground effect live), quaternions off unit length (the radial part of the
    state's cotangent), plans whose feedback moves u by a few percent, rotors on both sides of the box and of MAX_RPM."""
    P, c = params_of(model, 240, 48)
    h, mx = float(c.HOVER_RPM), float(c.MAX_RPM)
    rows = _rows(model, n, rng)
    pos = rng.uniform(-1, 1, (n, 3)) + [0, 0, 1.0]
    pos[: n // 4, 2] = rng.uniform(0.02, 0.1, n // 4)
    quat = quat_from_rpy(rng.uniform(-0.3, 0.3, (n, 3))) * rng.uniform(0.98, 1.02, (n, 1))
    state = np.concatenate([pos, quat, rng.uniform(-0.5, 0.5, (n, 3)), rng.uniform(-1, 1, (n, 3))], axis=1)
    up = h * rng.uniform(0.9, 1.1, (n, 4))
    z_nom = np.concatenate([state + rng.normal(0, 0.05, (n, 13)), up + rng.normal(0, 300.0, (n, 4))], axis=1)[:, :nz]
    K = rng.normal(0, 1.0, (n, 4, nz)) * np.concatenate([np.full(13, 0.02 * h), np.full(4, 0.1)])[:nz]
    rpm_nom = h * rng.uniform(0.9, 1.1, (n, 4))
    rpm_nom[-2:] = mx * rng.uniform(0.97, 1.03, (2, 4))       # the env's clip binds on some rotors
    lo = hi = None
    if box == "fixed":
        lo, hi = np.full((n, 4), 0.95 * h), np.full((n, 4), 1.05 * h)
    elif box == "per_tick":
        lo, hi = h * rng.uniform(0.9, 0.97, (n, 4)), h * rng.uniform(1.03, 1.1, (n, 4))
    return (P, eff, S, rows, state, up, rpm_nom, K, z_nom, lo, hi, rng.standard_normal((n, 13)), rng.standard_normal((n, 4)))


@pytest.mark.parametrize("box", [None, "fixed", "per_tick"], ids=["nobox", "fixed", "per_tick"])
@pytest.mark.parametrize("eff", list(EFFECTS))
@pytest.mark.parametrize("nz", [13, 17])
def test_tick_vjp_matches_reference(nz, eff, box):
    rng = np.random.default_rng(hash((nz, eff, box)) % 2 ** 32)
    worst = {}
    for model in ("cf2x", "cf2p"):
        args = _case(model, EFFECTS[eff], nz, box, rng)
        got, want = host_tick_vjp(*args), ref_tick_vjp(*args)
        assert np.array_equal(got["rpm"], want["rpm"]), model                   # the applied RPMs bit for bit
        assert R.relerr(got["out"], want["out"]) < 1e-12, model
        for blk in BLOCKS:
            e = R.relerr(got[blk], want[blk])
            worst[(model, blk)] = e
            assert e <= VJP_TOL, (model, blk, e)
        if box is not None:                                                      # the box binds somewhere
            b = TR.control(torch.tensor(args[4]), torch.tensor(args[5]), torch.tensor(args[8]), torch.tensor(args[7]), torch.tensor(args[6]))
            assert bool(((b < torch.tensor(args[9])) | (b > torch.tensor(args[10]))).any())
    print("n_z %d %s %s: worst normwise relative error %.2e" % (nz, eff, box, max(worst.values())))


def test_second_path_of_nz17_and_the_radial_part_are_seen():
    """Negative controls: dropping K^T lambda's last four entries (the n_z = 17 path into the previous RPMs) or its quaternion
    part (the radial component z reads) moves the gradients far beyond the tolerance."""
    args = _case("cf2x", R.EFFECT_DRAG, 17, None, np.random.default_rng(3))
    got, want = host_tick_vjp(*args), ref_tick_vjp(*args)
    Ktl = -want["z_nom"]
    assert R.relerr(got["last_rpm"], want["last_rpm"]) <= VJP_TOL
    assert R.relerr(got["last_rpm"], want["last_rpm"] - Ktl[:, 13:17]) > 1e-3
    assert R.relerr(got["state"], want["state"]) <= VJP_TOL
    no_radial = want["state"].copy()
    q = args[4][:, 3:7] / np.linalg.norm(args[4][:, 3:7], axis=1, keepdims=True)
    no_radial[:, 3:7] -= q * np.sum(q * Ktl[:, 3:7], axis=1, keepdims=True)
    assert R.relerr(got["state"], no_radial) > 1e-6


def _ulp_lattice(v):
    return [np.nextafter(v, -np.inf), v, np.nextafter(v, np.inf)]


@pytest.mark.parametrize("eff", [0, R.EFFECT_DRAG])
@pytest.mark.parametrize("nz", [13, 17])
def test_every_clamp_decision_at_its_boundary(nz, eff):
    """dz = 0 gives u = rpm_nom exactly, so rpm_nom puts u on lo, hi, 0 and MAX_RPM and one ulp either side.  The host build
    passes the gradient at equality (torch.clamp); a strict-inequality reference misses at exactly those rotors."""
    P, c = params_of("cf2x", 240, 48)
    h = float(c.HOVER_RPM)
    rng = np.random.default_rng(7 + nz + eff)
    cases = []                                          # (u, lo, hi) per rotor; lo = hi = None: no box (the env's clip alone)
    for v in _ulp_lattice(0.9 * h):
        cases.append((v, 0.9 * h, 1.1 * h))
    for v in _ulp_lattice(1.1 * h):
        cases.append((v, 0.9 * h, 1.1 * h))
    for v in [-5e-324, 0.0, 5e-324]:
        cases.append((v, None, None))
    cases += [(v, None, None) for v in _ulp_lattice(float(c.MAX_RPM))]
    rows = _rows("cf2x", 1, rng)
    rows[:, 13] = c.MAX_RPM                             # MAX_RPM of the row: the lattice above is about it
    for boxed in (True, False):
        sel = [k for k in cases if (k[1] is not None) == boxed]
        n = len(sel)                                    # one rotor per drone on the lattice, the others at hover
        rpm_nom = np.full((n, 4), h)
        for i, (v, _, _) in enumerate(sel):
            rpm_nom[i, i % 4] = v
        state = np.concatenate([np.tile([0.1, -0.2, 1.0], (n, 1)), quat_from_rpy(rng.uniform(-0.1, 0.1, (n, 3))),
                                rng.uniform(-0.2, 0.2, (n, 6))], axis=1)
        up = h * rng.uniform(0.95, 1.05, (n, 4))
        z_nom = np.concatenate([state, up], axis=1)[:, :nz]
        K = rng.normal(0, 1.0, (n, 4, nz)) * 50.0
        lo = np.full((n, 4), 0.9 * h) if boxed else None
        hi = np.full((n, 4), 1.1 * h) if boxed else None
        args = (P, eff, 3, np.repeat(rows, n, 0), state, up, rpm_nom, K, z_nom, lo, hi, rng.standard_normal((n, 13)),
                rng.standard_normal((n, 4)))
        got, want, bad = host_tick_vjp(*args), ref_tick_vjp(*args), ref_tick_vjp(*args, strict=True)
        assert np.array_equal(got["rpm"], want["rpm"])
        for blk in BLOCKS:
            assert R.relerr(got[blk], want[blk]) <= VJP_TOL, (boxed, blk)
        lam = got["rpm_nom"][np.arange(n), np.arange(n) % 4]
        for i, (v, lo_, hi_) in enumerate(sel):
            lo_, hi_ = (lo_, hi_) if boxed else (0.0, float(c.MAX_RPM))
            inside = lo_ <= v <= hi_
            assert (lam[i] != 0.0) == inside, (boxed, v, lam[i])
        on = [i for i, (v, lo_, hi_) in enumerate(sel) if v in ((lo_, hi_) if boxed else (0.0, float(c.MAX_RPM)))]
        bad_lam = bad["rpm_nom"][np.arange(n), np.arange(n) % 4]
        assert all(bad_lam[i] == 0.0 and lam[i] != 0.0 for i in on), (boxed, on)     # the strict reference misses each
        assert R.relerr(got["rpm_nom"], bad["rpm_nom"]) > 1e-3


def test_abi_exports_struct_and_refusals():
    from gym_pybullet_drones_b200 import _native as N
    L = N.lib()
    for name in ("qs_dyn_lqr_traj", "qs_dyn_lqr_traj_vjp", "qs_sizeof_dyn_lqr_traj_io"):
        assert name in N.EXPORTS
        getattr(L, name)
    assert L.qs_sizeof_dyn_lqr_traj_io() == C.sizeof(N.QsDynLqrTrajIO) == 24 + 19 * 8
    P, _ = params_of("cf2x")
    buf = (C.c_double * 256)()
    base = (C.addressof(buf) + 31) // 32 * 32
    io = N.QsDynLqrTrajIO()
    io.T, io.n_z, io.T_plan, io.tick0 = 2, 13, 4, 0
    io.state0 = io.K = io.z_nom = io.rpm_nom = io.states = io.rpm = base
    for f in (L.qs_dyn_lqr_traj, L.qs_dyn_lqr_traj_vjp):
        name = f.__name__.encode()
        call = lambda io_, *a: f(C.byref(P), C.byref(io_) if io_ is not None else None, *a, None)
        def refused(rc, *a):
            assert call(io, *a) == rc, (name, rc)
            assert L.qs_last_error().startswith(name + b": "), L.qs_last_error()
        assert call(None, 1, 1, 1, 0) == -1
        if f is L.qs_dyn_lqr_traj_vjp:
            refused(-1, 1, 1, 1, 0)                                            # no cotangents, gradient or scratch
            io.g_states = io.g_state0 = io.scratch = base
        io.K = None
        refused(-1, 1, 1, 1, 0)
        io.K = base
        refused(-3, 0, 1, 1, 0)
        refused(-3, 1, 1, 0, 0)
        refused(-4, 1, 1, 1, 8)
        refused(-5, 1, 1, 1, N.EFFECT_DW)
        assert b"downwash" in L.qs_last_error()
        refused(-5, 1, 1, 1, N.EFFECT_GND | N.EFFECT_DRAG | N.EFFECT_DW)
        io.n_z = 12
        refused(-3, 1, 1, 1, 0)
        io.n_z, io.tick0 = 17, -1
        refused(-3, 1, 1, 1, 0)
        io.tick0 = 3                                                           # ticks [3, 5) past T_plan = 4
        refused(-3, 1, 1, 1, 0)
        assert b"tick0" in L.qs_last_error()
        io.tick0, io.lo = 2, base
        refused(-1, 1, 1, 1, 0)
        io.hi, io.per_tick = base, 2
        refused(-3, 1, 1, 1, 0)
        io.per_tick, io.rpm_nom = 1, base + 8
        refused(-2, 1, 1, 1, 0)
        io.rpm_nom, io.lo, io.hi = base, base + 16, base + 16
        refused(-2, 1, 1, 1, 0)
        io.lo = io.hi = None
        io.per_tick, io.phys = 0, base + 8
        refused(-2, 1, 1, 1, 0)
        io.phys, io.n_z, io.tick0 = None, 13, 0
