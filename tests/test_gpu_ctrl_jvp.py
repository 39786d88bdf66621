"""-m gpu: forward mode of the closed-loop trajectories (qs_dyn_ctrl_traj_jvp / qs_dyn_ctrl_tick_jac, DESIGN.md 4.5) through
BaseAviary.differentiable_rollout(controller=) with torch.autograd.forward_ad and BaseAviary.linearise(controller=).

Covered: the dot-product identity <J v, w> = <v, J^T w> per drone between the JVP and the VJP kernels along every input block
(both models, the four effect sets, 240/240 and 240/48 Hz, T = 4 and 240, per-drone waypoints, a gain table); forward AD's
primals against the call without duals (bits) and its tangents against central differences of the forward; linearise's columns
against T = 1 JVP launches with unit tangents (bits), K against the JVP's applied-RPM tangent, the A / B chain against a 16-tick
JVP; partial CTAs, a Morton-reordered formation against its twin, the refusals; and a use: the closed-loop spectral radius at
hover under the default gains and under a gain change that keeps hover an equilibrium but destabilises the attitude loop,
against the growth of a perturbation in rollout(controller=)."""
import numpy as np
import pytest
import torch
import torch.autograd.forward_ad as fwAD

from test_gpu_diff_ctrl import GAIN_KEYS, PID_KEYS, STATE_KEYS, _call, _imports, _leaves
from test_gpu_diff_ctrl import _env as _env_of

pytestmark = pytest.mark.gpu

OUT_KEYS = STATE_KEYS + ("rpm",)


def _env(E, D, physics, model, pyb, ctrl, **kw):
    """test_gpu_diff_ctrl's env; "GND_DRAG": ground effect and drag, reachable through the C ABI's effects only"""
    from gym_pybullet_drones_b200 import _native as N
    env, ctl = _env_of(E, D, "PYB_DRAG" if physics == "GND_DRAG" else physics, model, pyb, ctrl, **kw)
    if physics == "GND_DRAG":
        env._effects = N.EFFECT_GND | N.EFFECT_DRAG
    return env, ctl


def _jvp(env, ctl, L, V, T, start, **kw):
    """(primal outputs, tangents) of differentiable_rollout(controller=) with the leaves L dual along V (keys of L; the rest
    carry no tangent)"""
    with fwAD.dual_level():
        D = {k: (fwAD.make_dual(v.detach(), V[k]) if k in V else v.detach()) for k, v in L.items()}
        out = _call(env, ctl, D, T, start, **kw)
        res = {k: fwAD.unpack_dual(v) for k, v in out.items()}
        return {k: r.primal.clone() for k, r in res.items()}, {k: r.tangent.clone() for k, r in res.items()}


def _per_aviary(d, E, outputs=False):
    """sum over everything but the aviary axis of {k: [.., E, ..]} tensors laid out as the leaves (or, outputs=True, the
    [T, E, D, k] outputs) are"""
    tot = torch.zeros(E, dtype=torch.float64, device=next(iter(d.values())).device)
    for k, v in d.items():
        if outputs or k == "waypoints":                         # [T or W, E, D, k] (shared waypoints [W, 3] carry none here)
            tot = tot + v.sum(dim=(0, 2, 3))
        elif v.dim() == 1:                                      # phys: [E]
            tot = tot + v
        else:                                                   # [E, ...]
            tot = tot + v.reshape(E, -1).sum(1)
    return tot


DOT = [(m, p, c) for m in ("CF2X", "CF2P") for p in ("DYN", "PYB_GND", "PYB_DRAG", "GND_DRAG") for c in (240, 48)]


@pytest.mark.parametrize("model,physics,ctrl", DOT)
@pytest.mark.parametrize("T", [4, 240])
def test_dot_product_identity_per_drone(model, physics, ctrl, T):
    """<J v, w> = <v, J^T w> per drone (D = 1: the gain and phys rows are the drone's own) with v over every input block"""
    E, W = 37, 6                                            # not a multiple of the CTA's 128 drones
    env, ctl = _env(E, 1, physics, model, 240, ctrl, seed=T)
    rng = np.random.default_rng(hash((model, physics, ctrl, T)) % 2 ** 32)
    L = _leaves(env, ctl, rng, W, True)
    start = torch.tensor(rng.integers(0, W, (E, 1)), device=env.device)
    V = {k: torch.tensor(rng.standard_normal(tuple(v.shape)), device=env.device) for k, v in L.items()}
    prim, Jv = _jvp(env, ctl, L, V, T, start)
    out = _call(env, ctl, L, T, start)
    Wt = {k: torch.tensor(rng.standard_normal(tuple(v.shape)), device=env.device) for k, v in out.items()}
    g = torch.autograd.grad(sum((out[k] * Wt[k]).sum() for k in out), list(L.values()), allow_unused=True)
    JTw = {k: (torch.zeros_like(L[k]) if x is None else x) for k, x in zip(L, g)}
    lhs = _per_aviary({k: Jv[k] * Wt[k] for k in out}, E, True)
    rhs = _per_aviary({k: V[k] * JTw[k] for k in L}, E)
    nj = torch.sqrt(_per_aviary({k: Jv[k] ** 2 for k in out}, E, True)) * torch.sqrt(_per_aviary({k: Wt[k] ** 2 for k in out}, E, True))
    ok = torch.isfinite(lhs) & torch.isfinite(rhs) & torch.isfinite(nj)
    assert int(ok.sum()) >= E // 2, int(ok.sum())           # at 48 Hz the linearised loop may overflow over 240 ticks
    err = ((lhs - rhs).abs() / nj)[ok]
    print("dot identity %s %s %d Hz T=%d: worst %.1e over %d drones" % (model, physics, ctrl, T, float(err.max()), int(ok.sum())))
    assert float(err.max()) <= 1e-12


def test_forward_ad_primals_and_central_differences():
    E, D, T, W = 3, 11, 12, 5
    env, ctl = _env(E, D, "PYB_DRAG", "CF2X", 240, 240)     # no ground-effect height clip for a difference to step across
    rng = np.random.default_rng(3)
    L = _leaves(env, ctl, rng, W, True)
    start = torch.tensor(rng.integers(0, W, (E, D)), device=env.device)
    plain = _call(env, ctl, {k: v.detach() for k, v in L.items()}, T, start)
    from gym_pybullet_drones_b200.params import PHYS_KEYS
    blocks = {"state": STATE_KEYS, "pid": PID_KEYS, "waypoints": ("waypoints",), "offset": ("offset",),
              "targets": ("target_vel", "target_rpy", "target_rpy_rates"), "gains": GAIN_KEYS, "last_rpm": ("last_rpm",),
              "phys": PHYS_KEYS}
    for name, keys in blocks.items():
        # each leaf moved relative to its own size (KF is 3e-10, KM 7e-12); a zero entry by 1e-3
        V = {k: torch.tensor(rng.standard_normal(tuple(L[k].shape)), device=env.device) *
             torch.where(L[k].detach() != 0, L[k].detach().abs(), torch.full_like(L[k].detach(), 1e-3)) for k in keys}
        prim, tan = _jvp(env, ctl, L, V, T, start)
        for k in OUT_KEYS:
            assert torch.equal(prim[k], plain[k]), (name, k)
        h = 1e-5                # V is scaled to each leaf: a smaller step leaves rounding noise in the small tangents
        f = lambda s: _call(env, ctl, {k: (v.detach() + s * V[k] if k in V else v.detach()) for k, v in L.items()}, T, start)
        fp, fm = f(h), f(-h)
        for k in OUT_KEYS:
            fd = (fp[k] - fm[k]) / (2 * h)
            err = float((tan[k] - fd).norm() / fd.norm().clamp(min=1e-300))
            assert err <= 1e-6, (name, k, err)


def test_tangent_that_requires_grad_raises():
    env, ctl = _env(2, 2, "DYN", "CF2X", 240, 48)
    rng = np.random.default_rng(4)
    L = {k: v.detach() for k, v in _leaves(env, ctl, rng, 4, False).items()}
    t = torch.ones_like(L["offset"]).requires_grad_(True)
    with fwAD.dual_level():
        L["offset"] = fwAD.make_dual(L["offset"], t)
        with pytest.raises(ValueError, match="requires grad"):
            _call(env, ctl, L, 3, None)


def _lin(env, ctl, L, T, start):
    from gym_pybullet_drones_b200.params import PHYS_KEYS
    kw = dict(controller=ctl, num_steps=T, start=start, waypoints=L["waypoints"].detach(), offset=L["offset"].detach(),
              target_vel=L["target_vel"].detach(), target_rpy=L["target_rpy"].detach(),
              target_rpy_rates=L["target_rpy_rates"].detach(), state={k: L[k].detach() for k in STATE_KEYS},
              pid_state={k: L[k].detach() for k in PID_KEYS}, last_rpm=L["last_rpm"].detach(),
              gains={k: L[k].detach() for k in GAIN_KEYS}, phys={k: L[k].detach() for k in PHYS_KEYS})
    return env.linearise(**kw)


@pytest.mark.parametrize("physics", ["DYN", "GND_DRAG"])
def test_linearise_columns_are_unit_jvps(physics):
    """Each column of A / B and each row block of K at tick k equals a T = 1 JVP launch from the forward's stored state k - 1,
    controller state pid_state[k] and (drag) rpm[k - 1] with a unit tangent: bit for bit"""
    E, D, T, W = 3, 11, 3, 4
    env, ctl = _env(E, D, physics, "CF2P", 240, 48)
    rng = np.random.default_rng(6)
    L = {k: v.detach() for k, v in _leaves(env, ctl, rng, W, True).items()}
    start = torch.tensor(rng.integers(0, W, (E, D)), device=env.device)
    lin = _lin(env, ctl, L, T, start)
    drag = physics.endswith("DRAG")
    nz = 26 if drag else 22
    assert lin["A"].shape == (T, E, D, nz, nz) and lin["B"].shape == (T, E, D, nz, 3)
    assert lin["K"].shape == (T, E, D, 4, nz) and lin["K_target"].shape == (T, E, D, 4, 3)
    ro = _call(env, ctl, L, T, start)
    for k in STATE_KEYS + ("rpm",):
        assert torch.equal(lin[k], ro[k]), k
    for k in range(T):
        Lk = dict(L)
        if k > 0:
            Lk.update({s: lin[s][k - 1] for s in STATE_KEYS})
            Lk["last_rpm"] = lin["rpm"][k - 1]
        Lk.update({s: lin["pid_state"][k][..., 3 * j:3 * j + 3] for j, s in enumerate(PID_KEYS)})
        cols = [(s, j) for s in STATE_KEYS for j in range(L[s].shape[-1])] + [(s, j) for s in PID_KEYS for j in range(3)]
        cols += [("last_rpm", j) for j in range(4)] if drag else []
        cols += [("offset", j) for j in range(3)]
        for c, (s, j) in enumerate(cols):
            v = torch.zeros_like(L[s])
            v[..., j] = 1.0
            _, tan = _jvp(env, ctl, Lk, {s: v}, 1, start + k)
            x = torch.cat([tan[q][0] for q in STATE_KEYS], dim=-1)
            jac = torch.cat([lin["A"][k], lin["B"][k]], dim=-1)[..., :13, c]
            assert torch.equal(x, jac), (k, s, j)
            assert torch.equal(tan["rpm"][0], torch.cat([lin["K"][k], lin["K_target"][k]], dim=-1)[..., c]), (k, s, j)


@pytest.mark.parametrize("physics", ["DYN", "PYB_DRAG"])
def test_linearise_chain_reproduces_trajectory_jvp(physics):
    """z_{k+1} = A_k z_k + B_k dtp_k and u_k = K_k z_k + K_target_k dtp_k over 16 ticks give the trajectory JVP's state and RPM
    tangents: z is the whole closed-loop state (u_{k-1} included with drag)"""
    E, D, T = 4, 3, 16
    env, ctl = _env(E, D, physics, "CF2X", 240, 48)
    rng = np.random.default_rng(7)
    L = {k: v.detach() for k, v in _leaves(env, ctl, rng, T, True).items()}
    start = torch.zeros((E, D), dtype=torch.int64, device=env.device)
    lin = _lin(env, ctl, L, T, start)
    drag = physics.endswith("DRAG")
    keys = STATE_KEYS + PID_KEYS + (("last_rpm",) if drag else ()) + ("waypoints",)
    V = {k: torch.tensor(rng.standard_normal(tuple(L[k].shape)), device=env.device) for k in keys}
    _, tan = _jvp(env, ctl, L, V, T, start)
    z = torch.cat([V[k] for k in STATE_KEYS + PID_KEYS + (("last_rpm",) if drag else ())], dim=-1)
    for k in range(T):
        dtp = V["waypoints"][k]
        u = lin["K"][k] @ z[..., None] + lin["K_target"][k] @ dtp[..., None]
        z = (lin["A"][k] @ z[..., None] + lin["B"][k] @ dtp[..., None])[..., 0]
        x = torch.cat([tan[q][k] for q in STATE_KEYS], dim=-1)
        ex = float((z[..., :13] - x).norm() / x.norm())
        eu = float((u[..., 0] - tan["rpm"][k]).norm() / tan["rpm"][k].norm())
        assert ex <= 1e-12 and eu <= 1e-12, (k, ex, eu)
        if drag:
            assert torch.equal(z[..., 22:26], u[..., 0])


def test_morton_twin_and_refusals():
    DSLPIDControl, CtrlAviary, DroneModel, Physics = _imports()
    from test_gpu_formation import stacks
    from gym_pybullet_drones_b200.control import MRAC
    xyz = stacks(10, 9)[:150]
    xyz = xyz[np.random.default_rng(5).permutation(len(xyz))]
    a = CtrlAviary(num_drones=len(xyz), initial_xyzs=xyz, physics=Physics.PYB_DW, ctrl_freq=48, num_envs=1)
    b = CtrlAviary(num_drones=len(xyz), initial_xyzs=xyz, physics=Physics.DYN, ctrl_freq=48, num_envs=1)
    a.reset(); b.reset()
    wp = torch.tensor([[0.0, 0.0, 1.0], [0.1, 0.0, 1.0]], dtype=torch.float64, device=a.device)
    ca, cb = (DSLPIDControl(DroneModel.CF2X, num_drones=len(xyz), device=e.device) for e in (a, b))
    with pytest.raises(ValueError, match="downwash"):
        a.linearise(controller=ca, waypoints=wp)
    order = a.reorder_by_morton().cpu().numpy()
    assert np.count_nonzero(order == np.arange(len(order))) < len(order) // 10
    a._effects = 0
    la, lb = a.linearise(controller=ca, waypoints=wp, num_steps=3), b.linearise(controller=cb, waypoints=wp, num_steps=3)
    for k in la:
        assert torch.equal(la[k], lb[k]), k
    # refusals
    with pytest.raises(ValueError, match="exactly one"):
        b.linearise()
    with pytest.raises(ValueError, match="exactly one"):
        b.linearise(torch.zeros((1, 1, len(xyz), 4), dtype=torch.float64, device=b.device), controller=cb, waypoints=wp)
    with pytest.raises(ValueError, match="controller linearisation"):
        b.linearise(torch.zeros((1, 1, len(xyz), 4), dtype=torch.float64, device=b.device), waypoints=wp)
    with pytest.raises(ValueError, match="MRAC"):
        b.linearise(controller=MRAC(DroneModel.CF2X, num_drones=len(xyz), device=b.device), waypoints=wp)
    with pytest.raises(ValueError, match="waypoints"):
        b.linearise(controller=cb, waypoints=wp[:, :2])
    with pytest.raises(ValueError, match="num_drones"):
        b.linearise(controller=DSLPIDControl(DroneModel.CF2X, num_drones=3, device=b.device), waypoints=wp)
    with pytest.raises(ValueError, match="pid_state"):
        b.linearise(controller=cb, waypoints=wp, pid_state={"integral_pos_e": torch.zeros((1, 3), dtype=torch.float64, device=b.device)})


# z without integral_rpy_e x and y: with DSLPIDControl's I_COEFF_TOR = (0, 0, 500) nothing reads them, so they are integrators
# that add two eigenvalues of exactly 1 (A is block triangular there) and say nothing about the loop's stability
LIVE = [j for j in range(22) if j not in (19, 20)]


def _spectral_radius(A):
    return float(torch.linalg.eigvals(A.cpu()[LIVE][:, LIVE]).abs().max())


def test_closed_loop_stability_at_hover():
    """CF2X drones at 240 Hz settled at hover under the default gains: rho(A) < 1 (on LIVE) and a body-rate kick decays by 10x in
    rollout(controller=).  With D_COEFF_TOR's sign flipped hover stays an equilibrium (the rate error it multiplies is ~0
    there), rho(A) > 1 and the same kick grows by 10x."""
    DSLPIDControl, CtrlAviary, DroneModel, Physics = _imports()
    E, D = 4, 1
    env = CtrlAviary(drone_model=DroneModel.CF2X, num_drones=D, physics=Physics.DYN, pyb_freq=240, ctrl_freq=240,
                     initial_xyzs=np.array([[0.0, 0.0, 1.0]]), num_envs=E)
    env.reset()
    ctl = DSLPIDControl(DroneModel.CF2X, num_drones=E * D, device=env.device)
    hover = torch.tensor([[0.0, 0.0, 1.0]], dtype=torch.float64, device=env.device)
    for _ in range(20):                                                                  # settle: 20 s
        env.rollout(controller=ctl, waypoints=hover, num_steps=240, record=False)
    base = ctl._P
    dtor = torch.tensor(list(base.pid_d_tor), dtype=torch.float64, device=env.device)
    state0 = {k: getattr(env, k).clone() for k in STATE_KEYS}
    pid0 = {k: ctl._state[3 * j:3 * j + 3].t().reshape(E, D, 3).clone() for j, k in enumerate(PID_KEYS)}
    kick = torch.zeros_like(state0["rpy_rates"])
    kick[..., 0] = 1e-3
    steps = 240 * 5
    for sign, stable in ((1.0, True), (-1.0, False)):
        gains = {"D_COEFF_TOR": sign * dtor}
        lin = env.linearise(controller=ctl, waypoints=hover, num_steps=1, gains=gains, state=state0, pid_state=pid0)
        rho = max(_spectral_radius(lin["A"][0, e, 0]) for e in range(E))
        kw = dict(controller=ctl, waypoints=hover, num_steps=steps, gains=gains, pid_state=pid0)
        nom = env.differentiable_rollout(state=state0, **kw)
        per = env.differentiable_rollout(state=dict(state0, rpy_rates=state0["rpy_rates"] + kick), **kw)
        dev = torch.cat([per[k] - nom[k] for k in STATE_KEYS], dim=-1).detach()
        ratio = float(dev[-1].norm() / kick.norm())
        print("D_COEFF_TOR x %+g: rho(A) = %.6f, |perturbation| after %d ticks / at start = %.3e" % (sign, rho, steps, ratio))
        if stable:
            assert rho < 1.0 and ratio <= 0.1, (rho, ratio)
        else:
            assert rho > 1.0 and ratio >= 10.0, (rho, ratio)
