"""-m gpu: differentiable tracker loops, differentiable_rollout(controller=ilqr.Tracker(sol), plan=) (qs_dyn_lqr_traj /
qs_dyn_lqr_traj_vjp, DESIGN.md 4.5).

Covered: the forward equals CtrlAviary.rollout(controller=Tracker(sol)) bit for bit (states and applied RPMs) across Physics modes,
models, control rates, phys tables, n_z 13 and 17, boxes and mid-plan starts, and GND|DRAG (which the rollout refuses) against the
host build; gradients of every input block against autograd of a float64 torch loop (tests/ilqr_tracker_ref.py + diff_ref.py),
with three negative controls that miss; central differences; every clamp decision on the device; the invariants (unflown plan
ticks, mid-plan slices, determinism, strides, partial CTAs, drone independence); the refusals; and a plan refined by gradient
descent over randomised plants, flown by the production rollout on held-out plants."""
import numpy as np
import pytest
import torch

import diff_ref as R
import ilqr_tracker_ref as TR

pytestmark = pytest.mark.gpu

DEV = "cuda"
KEYS = ("pos", "quat", "vel", "rpy_rates")
F64 = torch.float64
BLOCKS = ("rpm", "K", "z", "state", "last_rpm", "phys")
# normwise relative error of each gradient block against the float64 torch loop: about 2x the measured worst, 2.7e-14 on an H100
# (DESIGN.md 10)
GRAD_TOL = 5e-14


def _imports():
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.ilqr import Tracker
    from gym_pybullet_drones_b200.utils.enums import DroneModel, Physics
    return CtrlAviary, Tracker, DroneModel, Physics


def _env(E, D, physics="DYN", model="CF2X", pyb=240, ctrl=48, seed=0, xyz=None, rpy=0.3):
    """physics "gnd_drag": GND|DRAG without the downwash of PYB_GND_DRAG_DW"""
    CtrlAviary, _, DroneModel, Physics = _imports()
    rng = np.random.default_rng(seed)
    if xyz is None:
        xyz = np.stack([rng.uniform(-1, 1, D), rng.uniform(-1, 1, D), rng.uniform(0.3, 1.5, D)], 1)
    name = "PYB_GND_DRAG_DW" if physics == "gnd_drag" else physics
    env = CtrlAviary(drone_model=getattr(DroneModel, model), num_drones=D, physics=getattr(Physics, name), pyb_freq=pyb, ctrl_freq=ctrl,
                     initial_xyzs=xyz, initial_rpys=rng.uniform(-rpy, rpy, (D, 3)), num_envs=E)
    env.reset()
    if physics == "gnd_drag":
        env._effects = 3
    return env


def _phys(envs, seed, lo=0.85, hi=1.15):
    rng = np.random.default_rng(seed)
    e = envs[0]
    m, kf = e.M * rng.uniform(lo, hi, e._E), e.KF * rng.uniform(lo, hi, e._E)
    for env in envs:
        env.set_physical_params(m=m, kf=kf)


def _targets(env, seed, spread=0.4):
    rng = np.random.default_rng(seed)
    return {"pos": torch.tensor(rng.uniform(-spread, spread, (env._E, env._D, 3)) + np.array([0.0, 0.0, 1.0]), device=DEV)}


def _state(env):
    return torch.cat([getattr(env, k) for k in KEYS], dim=-1)


def _perturb(envs, seed, dp=0.03, dv=0.1, dw=0.2):
    rng = np.random.default_rng(seed)
    e = envs[0]
    shp = (e._E, e._D, 3)
    pos = e.pos.cpu().numpy() + rng.uniform(-dp, dp, shp)
    vel, w = rng.uniform(-dv, dv, shp), rng.uniform(-dw, dw, shp)
    for env in envs:
        env.set_state(pos=pos, vel=vel, rpy_rates=w)


def _bounds(kind, sol, env):
    T, E, D = sol["rpm"].shape[:3]
    h = env.HOVER_RPM
    if kind is None or kind == "motor":
        return kind
    if kind == "const":
        return (torch.full((4,), 0.92 * h, dtype=F64, device=DEV), torch.full((E, D, 4), 1.08 * h, dtype=F64, device=DEV))
    g = np.random.default_rng(5)
    return (torch.tensor(h * g.uniform(0.95, 0.99, (T, E, D, 4)), device=DEV), torch.tensor(h * g.uniform(1.01, 1.05, (T, E, D, 4)), device=DEV))


def _plan(case):
    """(plant env, a twin, Tracker, sol) of a case (plant, planner, model, rates, E, D, phys, box, T)"""
    _, Tracker, _, _ = _imports()
    plant, planner, model, (pyb, ctrl), E, D, phys, box, T = case
    a, b = _env(E, D, plant, model, pyb, ctrl, seed=7), _env(E, D, plant, model, pyb, ctrl, seed=7)
    p = _env(E, D, planner, model, pyb, ctrl, seed=7)
    if phys:
        _phys([a, b], 8)
    sol = p.ilqr(_targets(p, 9), num_steps=T, iters=3)
    _perturb([a, b], 10)
    return a, b, Tracker(sol, rpm_bounds=_bounds(box, sol, p)), sol


# ---- 1: the forward is the tracker rollout's bits ------------------------------------------------------------------------------

FWD = [
    # id, plant, planner, model, (pyb, ctrl), E, D, phys table, box, T, tick0
    ("dyn-cf2x", "DYN", "DYN", "CF2X", (240, 48), 37, 3, False, None, 12, 0),
    ("pyb-cf2p-240hz-box", "PYB", "DYN", "CF2P", (240, 240), 5, 7, False, "const", 12, 4),
    ("gnd-cf2x-phys-pertick", "PYB_GND", "PYB_GND", "CF2X", (240, 48), 10, 3, True, "per_tick", 12, 0),
    ("drag-nz17-240hz-mid", "PYB_DRAG", "PYB_DRAG", "CF2X", (240, 240), 13, 5, False, "per_tick", 12, 5),
    ("drag-nz17-cf2p-phys", "PYB_DRAG", "PYB_DRAG", "CF2P", (240, 48), 9, 4, True, "motor", 10, 0),
    ("plan-nz17-fly-dyn", "DYN", "PYB_DRAG", "CF2X", (240, 48), 9, 4, True, "const", 10, 3),
    ("plan-dyn-fly-drag-cf2p", "PYB_DRAG", "DYN", "CF2P", (240, 240), 7, 9, True, None, 10, 0),
]


@pytest.mark.parametrize("case", FWD, ids=[c[0] for c in FWD])
def test_forward_is_the_tracker_rollout_bit_for_bit(case):
    a, b, trk, sol = _plan(case[1:10])
    tick0 = case[10]
    T = trk.T - tick0
    trk.tick = tick0
    planes0, tick_before = a._planes.clone(), trk.tick
    out = a.differentiable_rollout(controller=trk)
    assert trk.tick == tick_before and torch.equal(a._planes, planes0)             # neither the tracker nor the env changed
    assert out["rpm"].shape == (T, a._E, a._D, 4) and all(out[k].grad_fn is None for k in KEYS)
    states, rpm = [], []
    for k in range(T):                                                             # split calls equal one call (Tracker's docstring)
        rpm.append(b.rollout(controller=trk, num_steps=1, record=False)["rpm"][0])
        states.append(_state(b))
    assert trk.tick == trk.T
    assert torch.equal(out["rpm"], torch.stack(rpm))
    assert torch.equal(torch.cat([out[k] for k in KEYS], dim=-1), torch.stack(states))


def _ref_loop(env, plan, tick0, T, x0, last, rows_e, box, variant=None):
    """The float64 torch loop of T tracker ticks: ilqr_tracker_ref.control, the box (torch.clamp's gradient), diff_ref.tick.
    plan = (rpm [T_plan, n, 4], K [T_plan, n, 4, n_z], z [T_plan, n, n_z]).  variant (negative controls): "no_radial" (dz reads
    the quaternion through its tangent part only), "box_everywhere" (the box passes the gradient everywhere), "no_second_path"
    (dz's previous RPMs carry no gradient).  Returns (states [T, n, 13], applied rpm [T, n, 4])."""
    rpm_nom, K, z = plan
    D = env._D
    Kc = R.model_constants(env._P, DEV)
    rows = rows_e.repeat_interleave(D, 0)
    x, up = x0, last
    xs, us = [], []
    for k in range(T):
        p = tick0 + k
        xz, upz = x, up
        if variant == "no_radial":
            q = x[:, 3:7]
            qh = q / torch.sqrt((q * q).sum(1, keepdim=True))
            xz = torch.cat([x[:, :3], qh + (q - qh).detach(), x[:, 7:]], dim=1)
        if variant == "no_second_path":
            upz = up.detach()
        bcmd = TR.control(xz, upz, z[p], K[p], rpm_nom[p])
        if box is not None:
            lo, hi, per_tick = box
            lo, hi = (lo[p], hi[p]) if per_tick else (lo, hi)
            cl = TR.clampd(bcmd, lo, hi)
            bcmd = bcmd + (cl - bcmd).detach() if variant == "box_everywhere" else cl
        x, u = R.tick(Kc, rows, x, bcmd, up, env.PYB_STEPS_PER_CTRL, env._effects)
        xs.append(x)
        us.append(u)
        up = u
    return torch.stack(xs), torch.stack(us)


def _leaves(env, trk, seed, phys_grad=True):
    """Inputs that require grad: plan (rpm, K, z: copies of the tracker's, K perturbed), state (pos, quat, vel, rpy_rates), last_rpm and
    phys (m, kf)"""
    E, D, T, nz = env._E, env._D, trk.T, trk.nz
    rng = np.random.default_rng(seed)
    # K scaled entry by entry by 1 + 0.1 N(0, 1): ilqr's K annihilates the quaternion's radial direction (the open loop's
    # Jacobians do), which would hide the radial part of the state's cotangent; with n_z = 17 a feedback of about 1 % from the
    # previous RPMs is added, where a drag plan's own is too weak to show the second path
    K = trk.K.view(T, E, D, 4, nz) * (1.0 + 0.1 * torch.tensor(rng.standard_normal((T, E, D, 4, nz)), device=DEV))
    if nz == 17:
        K[..., 13:] += 0.01 * torch.tensor(rng.standard_normal((T, E, D, 4, 4)), device=DEV)
    plan = {"rpm": trk.rpm_nom.view(T, E, D, 4).clone().requires_grad_(), "K": K.requires_grad_(),
            "z": trk.z_nom.view(T, E, D, nz).clone().requires_grad_()}
    state = {k: getattr(env, k).clone().requires_grad_() for k in KEYS}
    last = (env._last_rpm.view(E, D, 4) * torch.tensor(rng.uniform(0.97, 1.03, (E, D, 4)), device=DEV)).requires_grad_()
    props = env.physical_params()
    phys = {k: props[k].clone().requires_grad_(phys_grad) for k in ("m", "kf")}
    return plan, state, last, phys


def _flat_grads(loss, plan, state, last, phys):
    leaves = [plan["rpm"], plan["K"], plan["z"], *[state[k] for k in KEYS], last, phys["m"], phys["kf"]]
    g = torch.autograd.grad(loss, leaves, allow_unused=True)
    g = [torch.zeros_like(l) if x is None else x for x, l in zip(g, leaves)]
    return dict(rpm=g[0], K=g[1], z=g[2], state=torch.cat([x.flatten() for x in g[3:7]]), last_rpm=g[7], phys=torch.cat([g[8], g[9]]))


def _kernel_and_ref(env, trk, seed, variants=()):
    """The kernel's gradients and the reference loop's (and each variant's) of one random linear functional of the outputs"""
    from gym_pybullet_drones_b200.diff import _start_state
    E, D, n = env._E, env._D, env._N
    T = trk.T - trk.tick
    plan, state, last, phys = _leaves(env, trk, seed)
    out = env.differentiable_rollout(controller=trk, plan=plan, state=state, last_rpm=last, phys=phys)
    g = torch.Generator(device=DEV).manual_seed(seed)
    w = {k: torch.randn(out[k].shape, generator=g, dtype=F64, device=DEV) for k in (*KEYS, "rpm")}
    loss = sum((out[k] * w[k]).sum() for k in w)
    got = _flat_grads(loss, plan, state, last, phys)
    res = {}
    for v in (None, *variants):
        planes0, last_n, rows = _start_state(env, state, last, phys)
        x0 = TR.drone_vec(planes0, n)
        rp = (plan["rpm"].reshape(trk.T, n, 4), plan["K"].reshape(trk.T, n, 4, trk.nz), plan["z"].reshape(trk.T, n, trk.nz))
        xs, us = _ref_loop(env, rp, trk.tick, T, x0, last_n, rows, trk.box, v)
        o = {k: xs[..., s].reshape(T, E, D, -1) for k, s in zip(KEYS, (slice(0, 3), slice(3, 7), slice(7, 10), slice(10, 13)))}
        o["rpm"] = us.reshape(T, E, D, 4)
        res[v] = _flat_grads(sum((o[k] * w[k]).sum() for k in w), plan, state, last, phys)
        if v is None:
            fwd = max(R.relerr(out[k], o[k].detach()) for k in w)
    return got, res, fwd


GRAD = [
    # id, plant, planner, model, rates, E, D, phys, box, T, tick0
    ("dyn-cf2x", "DYN", "DYN", "CF2X", (240, 48), 19, 7, True, None, 16, 0),
    ("gnd-cf2p-box", "PYB_GND", "PYB_GND", "CF2P", (240, 48), 11, 3, True, "const", 16, 4),
    ("drag-nz17-pertick", "PYB_DRAG", "PYB_DRAG", "CF2X", (240, 48), 13, 5, True, "per_tick", 16, 0),
    ("gnd-drag-nz17-240hz", "gnd_drag", "gnd_drag", "CF2X", (240, 240), 6, 4, True, "const", 16, 2),
    ("dyn-plan-nz17", "DYN", "PYB_DRAG", "CF2P", (240, 48), 9, 3, True, "per_tick", 12, 0),
]


@pytest.mark.parametrize("case", GRAD, ids=[c[0] for c in GRAD])
def test_gradients_match_the_float64_loop(case):
    a, _, trk, sol = _plan(case[1:10])
    trk.tick = case[10]
    nz = trk.nz
    variants = ["no_radial"] + (["box_everywhere"] if trk.box is not None else []) + (["no_second_path"] if nz == 17 else [])
    got, res, fwd = _kernel_and_ref(a, trk, 40, variants)
    errs = {b: R.relerr(got[b], res[None][b]) for b in BLOCKS}
    print("%s: forward %.2e, gradients %s" % (case[0], fwd, " ".join("%s %.2e" % kv for kv in errs.items())))
    assert fwd <= 1e-12
    for b, e in errs.items():
        assert e <= GRAD_TOL, (b, e)
    for v in variants:
        miss = max(R.relerr(got[b], res[v][b]) for b in BLOCKS)
        print("  negative control %s misses by %.2e" % (v, miss))
        assert miss > 100 * GRAD_TOL, v
    assert float(got["K"][:trk.tick].abs().max() if trk.tick else 0.0) == 0.0       # unflown plan ticks


def test_gnd_drag_forward_against_host_build_and_reference():
    """GND|DRAG, which the tracker rollout refuses: the forward's applied RPMs equal the host build's tick by tick (teacher-forced
    on the device's states), its states within 1e-13, and the torch loop within 1e-12."""
    from test_lqr_traj_host import host_tick_vjp
    a, _, trk, sol = _plan(("gnd_drag", "gnd_drag", "CF2X", (240, 48), 5, 4, True, "const", 10))
    E, D, n, T, nz = a._E, a._D, a._N, trk.T, trk.nz
    out = a.differentiable_rollout(controller=trk)
    xs = torch.cat([out[k] for k in KEYS], dim=-1).reshape(T, n, 13)
    x_prev, up = _state(a).reshape(n, 13), a._last_rpm.reshape(n, 4).clone()
    from gym_pybullet_drones_b200.diff import _start_state
    rows = _start_state(a, None, None, None)[2].repeat_interleave(D, 0)
    lo, hi, _ = trk.box
    z = np.zeros((n, 13))
    for k in range(T):
        h = host_tick_vjp(a._P, 3, a.PYB_STEPS_PER_CTRL, rows.cpu().numpy(), x_prev.cpu().numpy(), up.cpu().numpy(),
                          trk.rpm_nom[k].cpu().numpy(), trk.K[k].cpu().numpy(), trk.z_nom[k].cpu().numpy(),
                          lo.expand(n, 4).cpu().numpy(), hi.expand(n, 4).cpu().numpy(), z, np.zeros((n, 4)))
        assert np.array_equal(h["rpm"], out["rpm"][k].reshape(n, 4).cpu().numpy()), k
        assert R.relerr(h["out"], xs[k].cpu().numpy()) < 1e-13, k
        x_prev, up = xs[k], out["rpm"][k].reshape(n, 4)
    _, res, fwd = _kernel_and_ref(a, trk, 41)
    assert fwd <= 1e-12


# ---- 2: central differences ------------------------------------------------------------------------------------------------------

def test_central_differences_along_random_directions():
    a, _, trk, sol = _plan(("PYB_DRAG", "PYB_DRAG", "CF2X", (240, 48), 6, 4, True, None, 12))
    plan, state, last, phys = _leaves(a, trk, 50)
    g = torch.Generator(device=DEV).manual_seed(51)

    def loss(pl, st, la, ph):
        out = a.differentiable_rollout(controller=trk, plan=pl, state=st, last_rpm=la, phys=ph)
        return (out["pos"][-1] ** 2).sum() + 1e-8 * (out["rpm"] ** 2).sum() + (out["vel"] * 0.3).sum()

    l0 = loss(plan, state, last, phys)
    got = _flat_grads(l0, plan, state, last, phys)
    blocks = {"rpm": [plan["rpm"]], "K": [plan["K"]], "z": [plan["z"]], "state": [state[k] for k in KEYS], "last_rpm": [last],
              "phys": [phys["m"], phys["kf"]]}
    worst = {}
    with torch.no_grad():
        for name, ts in blocks.items():
            for rep in range(2):
                # each component scaled by its own magnitude (z holds positions next to RPMs)
                scale = [(t.abs().flatten(0, -2).mean(0) if t.dim() > 1 else t.abs().mean()) + 1e-30 for t in ts]
                dirs = [torch.randn(t.shape, generator=g, dtype=F64, device=DEV) * c for t, c in zip(ts, scale)]
                gs = {"state": got["state"], "phys": got["phys"]}.get(name, got[name])
                an = float((gs.flatten() * torch.cat([d.flatten() for d in dirs])).sum())
                h = min(1e-4, 1e-5 * abs(float(l0)) / max(abs(an), 1e-300))     # moves the loss by at most 1e-5 of itself
                shift = lambda s: [t + s * d for t, d in zip(ts, dirs)]

                def f(s):
                    new = shift(s)
                    pl, st, la, ph = dict(plan), dict(state), last, dict(phys)
                    if name in ("rpm", "K", "z"):
                        pl[name] = new[0]
                    elif name == "state":
                        st = dict(zip(KEYS, new))
                    elif name == "last_rpm":
                        la = new[0]
                    else:
                        ph = dict(zip(("m", "kf"), new))
                    return float(loss(pl, st, la, ph))
                fd = (f(h) - f(-h)) / (2 * h)
                worst[(name, rep)] = abs(fd - an) / max(abs(an), 1e-12)
    print("central differences: " + " ".join("%s %.1e" % (k[0], v) for k, v in worst.items()))
    assert max(worst.values()) < 1e-3


# ---- 3: every decision on the device --------------------------------------------------------------------------------------------

def test_every_clamp_decision_on_the_device():
    """Plan tick 0 with dz = 0 (z[0] the start state and last_rpm) puts u = rpm[0] on lo, hi, 0 and MAX_RPM and one ulp either
    side; later ticks of a plan with rotors commanded above MAX_RPM, below 0 and outside the box make every decision occur in
    flight.  The device's lambda at tick 0 follows torch.clamp's convention rotor by rotor, and every gradient block matches the
    float64 loop."""
    _, Tracker, _, _ = _imports()
    E, D, T = 12, 1, 8
    a = _env(E, D, "PYB_DRAG", seed=60)
    h, mx = float(a.HOVER_RPM), float(a.MAX_RPM)
    rng = np.random.default_rng(61)
    n = E * D
    x0 = _state(a).reshape(n, 13)
    last = a._last_rpm.reshape(n, 4)
    z = torch.cat([x0, last], dim=1)[None].expand(T, n, 17).clone()
    z[1:] += torch.tensor(rng.normal(0, 0.02, (T - 1, n, 17)), device=DEV) * torch.tensor([1.0] * 13 + [500.0] * 4, device=DEV)
    K = torch.tensor(rng.normal(0, 1, (T, n, 4, 17)), device=DEV) * torch.tensor([0.05 * h] * 13 + [0.3] * 4, device=DEV)
    rpm = torch.tensor(h * rng.uniform(0.9, 1.1, (T, n, 4)), device=DEV)
    lo, hi = torch.full((n, 4), 0.92 * h, dtype=F64, device=DEV), torch.full((n, 4), 1.08 * h, dtype=F64, device=DEV)
    up = lambda v: float(np.nextafter(v, np.inf))
    dn = lambda v: float(np.nextafter(v, -np.inf))
    lattice = [(dn(0.92 * h), "box"), (0.92 * h, "box"), (up(0.92 * h), "box"), (dn(1.08 * h), "box"), (1.08 * h, "box"),
               (up(1.08 * h), "box"), (-5e-324, "clip"), (0.0, "clip"), (5e-324, "clip"), (dn(mx), "clip"), (mx, "clip"), (up(mx), "clip")]
    for i, (v, kind) in enumerate(lattice):
        rpm[0, i, i % 4] = v
        if kind == "clip":                               # the clip's rotors outside the box: no box on those drones
            lo[i], hi[i] = -1e30, 1e30
    rpm[2:5, ::3] = 1.3 * mx                              # the env's clip holds at MAX_RPM,
    rpm[2:5, 1::3] = -100.0                               # at 0,
    rpm[5:, 2::3, :2] = 1.2 * h                           # and the box at hi in flight
    sol = {"rpm": rpm.view(T, E, D, 4), "K": K.view(T, E, D, 4, 17), "z": z.view(T, E, D, 17)}
    trk = Tracker(sol, rpm_bounds=(lo.view(E, D, 4), hi.view(E, D, 4)))
    got, res, fwd = _kernel_and_ref(a, trk, 62, ["box_everywhere"])
    out = a.differentiable_rollout(controller=trk)["rpm"].reshape(T, n, 4)
    counts = dict(max_rpm=int((out[1:] == mx).sum()), zero=int((out[1:] == 0.0).sum()),
                  box=int(((out[1:] == lo) | (out[1:] == hi)).sum()))
    print("decisions in flight (ticks 1..%d): %s" % (T - 1, counts))
    assert all(v > 0 for v in counts.values()), counts
    for b in BLOCKS:
        assert R.relerr(got[b], res[None][b]) <= GRAD_TOL, b
    assert max(R.relerr(got[b], res["box_everywhere"][b]) for b in BLOCKS) > 100 * GRAD_TOL
    lam = got["rpm"].reshape(T, n, 4)[0]
    for i, (v, kind) in enumerate(lattice):
        l, u_ = (0.92 * h, 1.08 * h) if kind == "box" else (0.0, mx)
        assert (float(lam[i, i % 4]) != 0.0) == (l <= v <= u_), (i, v, kind, float(lam[i, i % 4]))
        assert float(lam[i, i % 4]) == float(res[None]["rpm"].reshape(T, n, 4)[0, i, i % 4]) or l <= v <= u_


# ---- 4: invariants ---------------------------------------------------------------------------------------------------------------

def test_invariants():
    _, Tracker, _, _ = _imports()
    a, _, trk, sol = _plan(("PYB_DRAG", "PYB_DRAG", "CF2X", (240, 48), 43, 3, True, "per_tick", 12))      # N = 129: partial CTA
    E, D, n, T = a._E, a._D, a._N, trk.T
    # unflown plan ticks get exactly zero gradient, and the slice from mid-plan equals the whole call
    plan, state, last, phys = _leaves(a, trk, 70)
    trk.tick = 3
    out = a.differentiable_rollout(controller=trk, num_steps=5, plan=plan, state=state, last_rpm=last, phys=phys)
    g = _flat_grads(sum(out[k].sum() for k in (*KEYS, "rpm")), plan, state, last, phys)
    for b in ("rpm", "K", "z"):
        assert float(g[b][:3].abs().max()) == 0.0 and float(g[b][8:].abs().max()) == 0.0, b
        assert float(g[b][3:8].abs().max()) > 0.0, b
    trk.tick = 0
    whole = a.differentiable_rollout(controller=trk)
    trk.tick = 5
    part = a.differentiable_rollout(controller=trk, state={k: whole[k][4] for k in KEYS}, last_rpm=whole["rpm"][4])
    for k in (*KEYS, "rpm"):
        assert torch.equal(part[k], whole[k][5:]), k
    trk.tick = 0
    # two backward passes are bitwise equal, and strided plan tensors give the dense gradients
    plan, state, last, phys = _leaves(a, trk, 71)
    out = a.differentiable_rollout(controller=trk, plan=plan, state=state, last_rpm=last, phys=phys)
    loss = sum((out[k] ** 2).sum() for k in (*KEYS, "rpm"))
    g1 = _flat_grads(loss, plan, state, last, phys)
    out = a.differentiable_rollout(controller=trk, plan=plan, state=state, last_rpm=last, phys=phys)
    g2 = _flat_grads(sum((out[k] ** 2).sum() for k in (*KEYS, "rpm")), plan, state, last, phys)
    for b in BLOCKS:
        assert torch.equal(g1[b], g2[b]), b
    strided = {k: v.detach().permute(1, 2, 0, *range(3, v.dim())).contiguous().permute(2, 0, 1, *range(3, v.dim())).requires_grad_()
               for k, v in plan.items()}
    assert not any(v.is_contiguous() for v in strided.values())
    out = a.differentiable_rollout(controller=trk, plan=strided, state=state, last_rpm=last, phys=phys)
    g3 = _flat_grads(sum((out[k] ** 2).sum() for k in (*KEYS, "rpm")), strided, state, last, phys)
    for b in BLOCKS:
        assert torch.equal(g1[b], g3[b]), b


def test_one_drones_gradients_ignore_its_neighbours():
    """One drone per aviary (its phys row is its own): moving every other drone's plan, state, last_rpm and constants leaves drone
    0's gradients bit for bit."""
    a, _, trk, sol = _plan(("PYB_GND", "PYB_GND", "CF2P", (240, 48), 130, 1, True, "const", 10))
    n = a._N
    mine = []
    for seed in (80, 81):
        plan, state, last, phys = _leaves(a, trk, 82)
        with torch.no_grad():
            g = torch.Generator(device=DEV).manual_seed(seed)
            for t in plan.values():                                    # [T, E, 1, ...]
                t[:, 1:] *= 1.0 + 1e-3 * torch.rand(t[:, 1:].shape, generator=g, dtype=F64, device=DEV)
            for t in (*state.values(), last, *phys.values()):          # [E, 1, k] and [E]
                t[1:] *= 1.0 + 1e-3 * torch.rand(t[1:].shape, generator=g, dtype=F64, device=DEV)
        out = a.differentiable_rollout(controller=trk, plan=plan, state=state, last_rpm=last, phys=phys)
        gr = _flat_grads(sum((out[k] ** 2).sum() for k in (*KEYS, "rpm")), plan, state, last, phys)
        st = torch.split(gr["state"], [3 * n, 4 * n, 3 * n, 3 * n])
        mine.append(dict(rpm=gr["rpm"][:, 0], K=gr["K"][:, 0], z=gr["z"][:, 0], last_rpm=gr["last_rpm"][0],
                         phys=gr["phys"].view(2, n)[:, 0], state=torch.cat([s.view(n, -1)[0] for s in st])))
    for b in BLOCKS:
        assert torch.equal(mine[0][b], mine[1][b]), b


# ---- 5: refusals -----------------------------------------------------------------------------------------------------------------

def test_refusals():
    CtrlAviary, Tracker, _, Physics = _imports()
    from gym_pybullet_drones_b200.control.DSLPIDControl import DSLPIDControl
    from gym_pybullet_drones_b200.utils.enums import DroneModel
    E, D, T = 2, 3, 6
    env = _env(E, D, "DYN", seed=30)
    sol = env.ilqr(_targets(env, 31), num_steps=T, iters=1)
    trk = Tracker(sol)
    pid = DSLPIDControl(drone_model=DroneModel.CF2X, num_drones=E * D)
    with pytest.raises(ValueError, match="plan= is the plan of a tracker loop"):
        env.differentiable_rollout(controller=pid, plan={"rpm": sol["rpm"]}, waypoints=torch.zeros((4, 3), dtype=F64, device=DEV))
    with pytest.raises(ValueError, match="plan= is the plan of a tracker loop"):
        env.differentiable_rollout(sol["rpm"], plan={"rpm": sol["rpm"]})
    with pytest.raises(ValueError, match="unknown plan keys"):
        env.differentiable_rollout(controller=trk, plan={"k": sol["k"]})
    with pytest.raises(ValueError, match="plan\\['K'\\] must have shape"):
        env.differentiable_rollout(controller=trk, plan={"K": sol["K"][..., :12]})
    with pytest.raises(ValueError, match="plan\\['rpm'\\] must be float64"):
        env.differentiable_rollout(controller=trk, plan={"rpm": sol["rpm"].float()})
    with pytest.raises(ValueError, match="plan\\['z'\\] must be on"):
        env.differentiable_rollout(controller=trk, plan={"z": sol["z"].cpu()})
    for kw in (dict(waypoints=torch.zeros((4, 3), dtype=F64, device=DEV)), dict(start=0), dict(offset=torch.zeros(3, dtype=F64, device=DEV)),
               dict(target_rpy=torch.zeros(3, dtype=F64, device=DEV)), dict(target_vel=torch.zeros(3, dtype=F64, device=DEV)),
               dict(target_rpy_rates=torch.zeros(3, dtype=F64, device=DEV)), dict(gains={}), dict(pid_state={}),
               dict(control_timestep=0.02)):
        with pytest.raises(ValueError, match="a Tracker flies its plan: %s" % list(kw)[0]):
            env.differentiable_rollout(controller=trk, **kw)
    with pytest.raises(ValueError, match="apply to a policy rollout only"):
        env.differentiable_rollout(controller=trk, noise=torch.zeros((T, E, D * 4), dtype=F64, device=DEV))
    with pytest.raises(ValueError, match="plan is for"):
        _env(E, D + 1, "DYN", seed=30).differentiable_rollout(controller=trk)
    other = Tracker(sol)
    other.device = torch.device("cpu")
    with pytest.raises(ValueError, match="plan is on"):
        env.differentiable_rollout(controller=other)
    for steps in (0, -2):
        with pytest.raises(ValueError, match="num_steps must be > 0"):
            env.differentiable_rollout(controller=trk, num_steps=steps)
    with pytest.raises(ValueError, match="do not fit"):
        env.differentiable_rollout(controller=trk, num_steps=T + 1)
    trk.tick = 4
    with pytest.raises(ValueError, match="do not fit"):
        env.differentiable_rollout(controller=trk, num_steps=3)
    trk.tick = -1
    with pytest.raises(ValueError, match="tick must be an integer >= 0"):
        env.differentiable_rollout(controller=trk)
    trk.tick = 0
    drag = _env(E, D, "PYB_DRAG", seed=30)
    sol17 = drag.ilqr(_targets(drag, 31), num_steps=T, iters=1)
    nolast = CtrlAviary(num_drones=D, physics=Physics.DYN, num_envs=E, track_last_action=False)
    nolast.reset()
    with pytest.raises(ValueError, match="last_clipped_action"):
        nolast.differentiable_rollout(controller=Tracker(sol17))
    assert nolast.differentiable_rollout(controller=Tracker(sol17), last_rpm=sol17["z"][0, ..., 13:])["rpm"].shape == (T, E, D, 4)
    dw = _env(E, D, "PYB_DW", seed=30)
    with pytest.raises(ValueError, match="differentiable_rollout\\(\\) does not support downwash"):
        dw.differentiable_rollout(controller=trk)
    from test_gpu_formation import stacks
    xyz = stacks(10, 9)[:333]
    a = CtrlAviary(num_drones=len(xyz), initial_xyzs=xyz, physics=Physics.PYB_DW, num_envs=1)
    p = CtrlAviary(num_drones=len(xyz), initial_xyzs=xyz, physics=Physics.DYN, num_envs=1)
    a.reset(); p.reset()
    a.reorder_by_morton()
    a._effects = 0                                         # the formation without its downwash, which is refused first
    with pytest.raises(ValueError, match="reorder_by_morton"):
        a.differentiable_rollout(controller=Tracker(p.ilqr({"pos": torch.tensor(xyz, device=DEV)[None]}, num_steps=4, iters=1)))
    with pytest.raises(ValueError, match="controller must be a DSLPIDControl, got Tracker"):
        env.linearise(controller=trk)
    plan = {"rpm": sol["rpm"].clone().requires_grad_()}
    out = env.differentiable_rollout(controller=trk, plan=plan)
    with pytest.raises(ValueError, match="double backward"):
        torch.autograd.grad(out["pos"].sum(), plan["rpm"], create_graph=True)
    import torch.autograd.forward_ad as fwAD
    with fwAD.dual_level():
        dual = fwAD.make_dual(sol["rpm"].clone(), torch.ones_like(sol["rpm"]))
        with pytest.raises(ValueError, match="reverse mode only"):
            env.differentiable_rollout(controller=trk, plan={"rpm": dual})
    assert trk.tick == 0 and int(env._step_counter[0]) == 0


# ---- 6: a plan refined over randomised plants -------------------------------------------------------------------------------------

# the refined plan's mean error on held-out plants must be below the unrefined's divided by this.  Measured on an H100 80GB HBM3 at
# 700 W: 17.2 mm unrefined, 1.23 mm refined (a factor of 14.0)
REFINE_FACTOR = 5.0


def test_robust_refinement_end_to_end():
    """Solve one plan on the nominal plant; refine its rpm and K by Adam (a fixed budget of steps) on the mean tracked error over
    a training batch of aviaries with mass and KF randomised by up to +-15 % and perturbed starts; then fly the refined plan with
    the production CtrlAviary.rollout(controller=Tracker(refined)) on held-out randomised plants."""
    _, Tracker, _, _ = _imports()
    T, E_train, E_test, steps = 48, 256, 1024, 100
    start = np.array([[0.0, 0.0, 1.0]])
    goal = torch.tensor([[[0.3, -0.2, 1.2]]], dtype=F64, device=DEV)
    from gym_pybullet_drones_b200.ilqr import Problem, solve
    nom = _env(1, 1, "DYN", seed=90, xyz=start, rpy=0.0)
    p = Problem(nom, {"pos": goal}, num_steps=T)
    sol = solve(p, 30)
    p.mu.zero_()
    p.backward()                                                               # the gains at mu = 0 (Tracker's docstring)
    sol = p.result(sol["cost"])
    pos_nom = sol["pos"]                                                        # [T, 1, 1, 3]

    def batch(E, seed):
        env = _env(E, 1, "DYN", seed=seed, xyz=start, rpy=0.0)
        _phys([env], seed + 1)
        rng = np.random.default_rng(seed + 2)
        env.set_state(pos=start[None] + rng.uniform(-0.02, 0.02, (E, 1, 3)), vel=rng.uniform(-0.05, 0.05, (E, 1, 3)))
        return env

    def expand(p, E):
        return {k: v.expand(v.shape[0], E, *v.shape[2:]) for k, v in p.items()}

    train = batch(E_train, 91)
    rpm0, K0 = sol["rpm"].detach(), sol["K"].detach()
    kscale = K0.abs().mean(dim=0, keepdim=True) + 1e-12
    a_rpm = torch.zeros_like(rpm0, requires_grad=True)
    a_K = torch.zeros_like(K0, requires_grad=True)
    opt = torch.optim.Adam([a_rpm, a_K], lr=0.02)
    trk = Tracker(expand({"rpm": rpm0, "K": K0, "z": sol["z"]}, E_train))
    losses = []
    for it in range(steps):
        plan = expand({"rpm": rpm0 + 100.0 * a_rpm, "K": K0 + kscale * a_K}, E_train)
        out = train.differentiable_rollout(controller=trk, plan=plan)
        loss = ((out["pos"] - pos_nom) ** 2).sum(-1).mean() + ((out["pos"][-1] - goal) ** 2).sum(-1).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    refined = {"rpm": (rpm0 + 100.0 * a_rpm).detach(), "K": (K0 + kscale * a_K).detach(), "z": sol["z"]}
    errs = []
    for p in (sol, refined):
        test = batch(E_test, 93)
        test.rollout(controller=Tracker(expand({k: p[k] for k in ("rpm", "K", "z")}, E_test)), record=False)
        errs.append(float((test.pos - goal).norm(dim=-1).mean()))
    print("robust refinement: training loss %.3e -> %.3e in %d steps; held-out mean final error %.3e m unrefined, %.3e m refined"
          % (losses[0], losses[-1], steps, errs[0], errs[1]))
    assert errs[1] * REFINE_FACTOR < errs[0]
