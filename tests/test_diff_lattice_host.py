"""CPU tests of the differentiable trajectories' decisions at their boundaries (DESIGN.md 4.5): the g++ build of the tick adjoint
(dyn_adjoint.cuh) on states and commands exactly on each decision of the derivative and one ulp either side (diff_testlib.lattices),
per drone against the torch reference; torch.clamp's gradient convention, which the reference inherits; a negative control
for each decision and for the per-drone metric."""
import functools

import numpy as np
import pytest
import torch

import diff_ref as R
from diff_testlib import (MODELS, SIDE_PAIRS, aviary_rows, check_lattice, host_tick_vjp, lattices, params_of, per_drone_relerr,
                          ref_tick_vjp)

VJP_TOL = 1e-10
LATTICES = ("rpm", "clip", "half_angle", "upright")


@functools.lru_cache(maxsize=None)
def model_lattices(model):
    P, c = params_of(model)
    _, rows = aviary_rows(model, 64, np.random.default_rng(20))
    return P, lattices(P, c, rows.numpy(), np.random.default_rng(21))


def _run(P, lat, device=None, **kw):
    args = (lat["effects"], lat["S"], lat["state"], lat["raw"], lat["up"], lat["g_out"])
    return ref_tick_vjp(P, lat["rows"], *args, device=device, **kw)


def test_torch_clamp_gradient_convention():
    """diff_ref's RPM clip is torch.clamp with tensor bounds: the gradient passes at 0, -0.0 and MAX_RPM, and MAX_RPM receives
    it only strictly above.  The kernels implement this convention (rpm_clip_vjp); a torch that moved it would move the
    reference under them."""
    mx = 21702.64377525105
    x = torch.tensor([np.nextafter(mx, 0), mx, np.nextafter(mx, np.inf), np.nextafter(-0.0, -1), -0.0, 0.0, np.nextafter(0.0, 1),
                      -1.0, 0.5 * mx], dtype=torch.float64, requires_grad=True)
    m = torch.full_like(x, mx).requires_grad_(True)
    lo = torch.zeros_like(x).requires_grad_(True)
    gx, gm, gl = torch.autograd.grad(torch.clamp(x, min=lo, max=m).sum(), (x, m, lo))
    assert gx.tolist() == [1, 1, 0, 0, 1, 1, 1, 0, 1]
    assert gm.tolist() == [0, 0, 1, 0, 0, 0, 0, 0, 0]
    assert gl.tolist() == [0, 0, 0, 1, 0, 0, 0, 1, 0]


@pytest.mark.parametrize("model", MODELS)
def test_lattices_sit_on_their_boundaries(model):
    """The lattice states take each decision exactly at its boundary, in the reference's own float64 evaluation too."""
    from diff_testlib import prop_heights, upright_terms
    P, L = model_lattices(model)
    K = R.model_constants(P)
    st = L["clip"]["state"]
    hz = np.array([prop_heights(P, s[2], tuple(s[3:7]))[0] for s in st])
    assert np.array_equal(np.sign(hz - K["h_clip"]), L["clip"]["label"])
    x = torch.tensor(L["clip"]["state"])
    q = x[:, 3:7]
    r20, r21, r22 = 2 * (q[:, 0] * q[:, 2] - q[:, 3] * q[:, 1]), 2 * (q[:, 1] * q[:, 2] + q[:, 3] * q[:, 0]), 1 - 2 * (q[:, 0] ** 2 + q[:, 1] ** 2)
    Pp = K["props"]
    assert torch.equal(x[:, 2] + r20 * Pp[0, 0] + r21 * Pp[0, 1] + r22 * Pp[0, 2], torch.tensor(hz))
    w = L["half_angle"]["state"][:, 10:13]
    h = 0.5 * float(P.dt)
    t = np.array([(a * a + b * b + c * c) * h * h for a, b, c in w])
    lab = L["half_angle"]["label"]
    assert np.all(t[lab == 0] == 0.25) and np.all(t[lab == -1] < 0.25) and np.all(t[lab == 1] > 0.25)
    n2 = np.array([a * a + b * b + c * c for a, b, c in w])
    assert np.all(n2[lab == 3] <= 1e-16) and np.all(n2[lab == 4] > 1e-16) and np.any(lab == 3) and np.any(lab == 4)
    qs = L["upright"]["state"][:, 3:7]
    up = R.upright(*[torch.tensor(v) for v in zip(*[upright_terms(tuple(qq)) for qq in qs])])
    assert up.tolist() == [bool(v) for v in L["upright"]["label"]]
    sarg, ra, rb = zip(*[upright_terms(tuple(qq)) for qq in qs])
    assert rb[1] == 1.722546424198833e-16 * abs(ra[1]) and sarg[4] == 0.99999 and sarg[7] == -0.99999


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("name", LATTICES)
def test_lattice_host_build_matches_reference(model, name):
    P, L = model_lattices(model)
    lat = L[name]
    got = host_tick_vjp(P, lat["effects"], lat["S"], lat["state"], lat["raw"], lat["up"], lat["g_out"], lat["rows"])
    want = _run(P, lat)
    fwd = _run(P, lat, exact_branch=True)[0] if name == "half_angle" else want[0]
    worst = check_lattice(name, lat, got, want, fwd, VJP_TOL)
    print("host lattice %s %s: worst per-drone error %s" % (model, name, {k: "%.1e" % v for k, v in worst.items()}))


@pytest.mark.parametrize("model", MODELS)
def test_negative_controls_lattices(model):
    """A reference that clips strictly at MAX_RPM, or clips the ground-effect height at hz == clip, misses the lattice drones
    on the boundary; the two sides of the clip and of the upright switch differ in the gradient by >= 1e-3."""
    P, L = model_lattices(model)
    for name, kw, at in (("rpm", dict(strict_clamp=True), L["rpm"]["label"] == 1), ("clip", dict(gnd_clip_le=True), L["clip"]["label"] == 0)):
        lat = L[name]
        got = host_tick_vjp(P, lat["effects"], lat["S"], lat["state"], lat["raw"], lat["up"], lat["g_out"], lat["rows"])
        bad = _run(P, lat, **kw)
        blk = 2 if name == "rpm" else 1
        e = per_drone_relerr(got[blk], bad[blk])
        print("negative control %s %s: per-drone error at the boundary >= %.1e, elsewhere <= %.1e" % (model, name, e[at].min(), e[~at].max()))
        assert e[at].min() >= 1e-3 and e[~at].max() <= VJP_TOL
    for name, pairs in SIDE_PAIRS.items():
        want = _run(P, L[name])
        for a, b in pairs:
            e = float(per_drone_relerr(want[1][a:a + 1], want[1][b:b + 1])[0]) + float(per_drone_relerr(want[2][a:a + 1], want[2][b:b + 1])[0])
            assert e >= 1e-3, (name, a, b, e)


def test_per_drone_metric_sees_one_drone_of_4096():
    """A 1e-8 relative error in one drone of 4 096 passes the normwise metric over the batch (<= 1e-9) and fails the per-drone
    one (<= 1e-10)."""
    rng = np.random.default_rng(22)
    want = rng.standard_normal((4096, 13))
    got = want.copy()
    d = rng.standard_normal(13)
    got[1234] += 1e-8 * np.linalg.norm(want[1234]) * d / np.linalg.norm(d)
    assert R.relerr(got, want) <= 1e-9
    e = per_drone_relerr(got, want)
    assert e[1234] > 50 * VJP_TOL and np.count_nonzero(e) == 1
