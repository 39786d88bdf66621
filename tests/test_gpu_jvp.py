"""-m gpu: the forward mode of the differentiable trajectories (dyn_traj_jvp_kernel<EFF>, dyn_tick_jac_kernel<EFF>, DESIGN.md 4.5).

Covered: the dot-product identity <J v, w> = <v, J^T w> per drone between qs_dyn_traj_jvp and qs_dyn_traj_vjp (three models,
the four effect sets, S = 1, 5, 8, 24, T = 4 and 240, the decision lattices); BaseAviary.linearise against the JVP kernel with
unit tangents and its chain of A / B / B_last against the JVP of a whole trajectory; forward AD through differentiable_rollout
against central differences of the forward kernel, with primal outputs bit for bit; the radial null space of A's quaternion
columns; partial CTAs, a strided rpm and the refusals; and a discrete LQR designed on linearise's Jacobians that stabilises
CtrlAviary drones of different masses (with K = 0 as the negative control)."""
import ctypes as C

import numpy as np
import pytest
import torch

import diff_ref as R
from diff_testlib import MODELS, aviary_rows, lattices, params_of, quat_from_rpy, scenario_ticks

pytestmark = pytest.mark.gpu

EFFECTS = {"dyn": 0, "gnd": R.EFFECT_GND, "drag": R.EFFECT_DRAG, "gnd_drag": R.EFFECT_GND | R.EFFECT_DRAG}
DEV = "cuda"
KEYS = ("pos", "quat", "vel", "rpy_rates")


def _t(a):
    return torch.as_tensor(np.asarray(a, dtype=np.float64), device=DEV).contiguous()


def _planes(x):
    from gym_pybullet_drones_b200.diff import pack_state
    return pack_state(x[..., 0:3], x[..., 3:7], x[..., 7:10], x[..., 10:13]).contiguous()


def _drones(planes, n):
    from gym_pybullet_drones_b200.diff import unpack_states
    u = unpack_states(planes, n)
    return torch.cat([u[k] for k in KEYS], dim=-1)


def abi_dot(P, E, D, S, eff, state, rpm, last, rows, v, w):
    """qs_dyn_traj, qs_dyn_traj_jvp along v = (t_state [n, 13], t_rpm [T, n, 4], t_last [n, 4], t_rows [E, 16]) and
    qs_dyn_traj_vjp with w [T, n, 13]: per drone (<J v, w>, <v, J^T w>, |J v|, |w|)."""
    from gym_pybullet_drones_b200 import _native as N
    n, T = E * D, rpm.shape[0]
    f64 = dict(dtype=torch.float64, device=DEV)
    planes0, rpm, last, rows = _planes(_t(state)), _t(rpm), _t(last), _t(rows)
    t_state, t_rpm, t_last, t_rows = (_t(x) for x in v)
    states, t_states = torch.empty((T, 13 * n), **f64), torch.empty((T, 13 * n), **f64)
    stream = torch.cuda.current_stream().cuda_stream
    io = N.QsDynTrajIO()
    io.T, io.state0, io.rpm, io.last_rpm, io.phys, io.states = T, planes0.data_ptr(), rpm.data_ptr(), last.data_ptr(), rows.data_ptr(), states.data_ptr()
    N.check(N.lib().qs_dyn_traj(C.byref(P), C.byref(io), E, D, S, eff, stream), "qs_dyn_traj")
    jo = N.QsDynTrajJvpIO()
    jo.T, jo.state0, jo.rpm, jo.last_rpm, jo.phys, jo.states = T, io.state0, io.rpm, io.last_rpm, io.phys, io.states
    t_planes = _planes(t_state)
    jo.t_state0, jo.t_rpm, jo.t_last_rpm, jo.t_phys = t_planes.data_ptr(), t_rpm.data_ptr(), t_last.data_ptr(), t_rows.data_ptr()
    jo.t_states = t_states.data_ptr()
    N.check(N.lib().qs_dyn_traj_jvp(C.byref(P), C.byref(jo), E, D, S, eff, stream), "qs_dyn_traj_jvp")
    g_planes = torch.stack([_planes(x) for x in _t(w)])
    g_rpm, g_state0 = torch.empty((T, n, 4), **f64), torch.empty((13 * n,), **f64)
    g_last, g_phys, scratch = torch.empty((n, 4), **f64), torch.empty((n, 16), **f64), torch.empty((S, 13, n), **f64)
    io.g_states, io.g_rpm, io.g_state0, io.g_last_rpm, io.g_phys, io.scratch = (x.data_ptr() for x in (g_planes, g_rpm, g_state0, g_last,
                                                                                                          g_phys, scratch))
    N.check(N.lib().qs_dyn_traj_vjp(C.byref(P), C.byref(io), E, D, S, eff, stream), "qs_dyn_traj_vjp")
    jv = _drones(t_states, n)                                                       # [T, n, 13]
    lhs = (jv * _t(w)).sum(dim=(0, 2))
    rhs = ((g_rpm * t_rpm).sum(dim=(0, 2)) + (_drones(g_state0, n) * t_state).sum(1) + (g_last * t_last).sum(1)
           + (g_phys * t_rows.repeat_interleave(D, dim=0)).sum(1))
    return [x.cpu().numpy() for x in (lhs, rhs, jv.norm(dim=(0, 2)), _t(w).norm(dim=(0, 2)))]


def _random_v(rng, T, n, E, rows, hover):
    """Tangents of all four input blocks, each on the scale of its input."""
    return (rng.standard_normal((n, 13)), hover * 1e-2 * rng.standard_normal((T, n, 4)), hover * 1e-2 * rng.standard_normal((n, 4)),
            np.asarray(rows) * 1e-2 * rng.standard_normal((E, 16)))


def _check_dot(out, tol=1e-12, finite_share=1.0):
    """Asserts the identity per drone; `finite_share`: the share of drones whose trajectory must stay finite (open-loop flights of
    tens of seconds overflow: the identity is checked on the drones whose tangents are finite)."""
    lhs, rhs, jv, w = out
    ratio = np.abs(lhs - rhs) / (jv * w)
    fin = np.isfinite(ratio)
    assert fin.mean() >= finite_share, fin.mean()
    assert np.all(jv[fin] > 0), "zero tangent"
    assert ratio[fin].max() <= tol, ratio[fin].max()
    return float(ratio[fin].max())


# ---- 1. <J v, w> = <v, J^T w> per drone ---------------------------------------------------------------------------------

@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("eff", list(EFFECTS))
@pytest.mark.parametrize("S", [1, 5, 8, 24])
@pytest.mark.parametrize("T", [4, 240])
def test_dot_product_jvp_against_vjp(model, eff, S, T):
    """The scenario matrix of the host tests, each drone its own aviary with a random row.  T = 240: the tumbling drones are
    left out (their rates overflow within a few hundred substeps of explicit Euler on w x Jw); at S = 24 (24 s of open-loop
    flight under random RPMs) some of the others overflow too, and the identity is checked on the drones that stay finite."""
    P, c = params_of(model)
    n_per = 16
    rng = np.random.default_rng([MODELS.index(model), S, T])
    _, rows = aviary_rows(model, 6 * n_per, rng)
    rows = rows.numpy()
    names, state, raw, up = scenario_ticks(c, rows, T, MODELS.index(model) + S, n_per)
    keep = names != "tumbling" if T > 4 else np.ones(len(names), bool)
    state, raw, up, rows = state[keep], raw[:, keep], up[keep], rows[keep]
    n = len(state)
    v = _random_v(rng, T, n, n, rows, float(c.HOVER_RPM))
    w = rng.standard_normal((T, n, 13))
    out = abi_dot(P, n, 1, S, EFFECTS[eff], state, raw, up, rows, v, w)
    worst = _check_dot(out, finite_share=1.0 if T * S <= 240 * 8 else 0.5)
    print("dot product %s %s S=%d T=%d: worst |<Jv,w> - <v,J^T w>| / (|Jv||w|) = %.1e over %d of %d drones (the rest overflow)"
          % (model, eff, S, T, worst, int(np.isfinite(out[0] - out[1]).sum()), n))


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("name", ["rpm", "clip", "half_angle", "upright"])
def test_dot_product_on_lattices(model, name):
    P, c = params_of(model)
    _, rows = aviary_rows(model, 64, np.random.default_rng(20))
    lat = lattices(P, c, rows.numpy(), np.random.default_rng(21))[name]
    n = len(lat["state"])
    rng = np.random.default_rng(22)
    v = _random_v(rng, 1, n, n, lat["rows"], float(c.HOVER_RPM))
    out = abi_dot(P, n, 1, lat["S"], lat["effects"], lat["state"], lat["raw"][None], lat["up"], lat["rows"], v, lat["g_out"][None])
    print("dot product lattice %s %s: %.1e" % (model, name, _check_dot(out)))


def test_dot_product_negative_control():
    """A JVP whose rpm tangent misses one drone's ticks breaks the identity for that drone only."""
    P, c = params_of("cf2x")
    rng = np.random.default_rng(23)
    _, rows = aviary_rows("cf2x", 12, rng)
    _, state, raw, up = scenario_ticks(c, rows.numpy(), 4, 3, 2)
    v = _random_v(rng, 4, 12, 12, rows.numpy(), float(c.HOVER_RPM))
    w = rng.standard_normal((4, 12, 13))
    lhs, rhs, jv, wn = abi_dot(P, 12, 1, 5, 3, state, raw, up, rows.numpy(), v, w)
    v2 = (v[0], v[1].copy(), v[2], v[3])
    v2[1][:, 3] = 0.0
    lhs2 = abi_dot(P, 12, 1, 5, 3, state, raw, up, rows.numpy(), v2, w)[0]
    ratio = np.abs(lhs2 - rhs) / (jv * wn)
    assert ratio[3] >= 1e-6 and np.delete(ratio, 3).max() <= 1e-12


# ---- 2. linearise against the JVP kernel ----------------------------------------------------------------------------------

def _env(E, D, physics, model="CF2X", pyb=240, ctrl=48):
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils.enums import DroneModel, Physics
    rng = np.random.default_rng(E * 100 + D)
    xyz = np.stack([rng.uniform(-1, 1, D), rng.uniform(-1, 1, D), rng.uniform(0.02, 1.0, D)], 1)
    env = CtrlAviary(drone_model=getattr(DroneModel, model), num_drones=D, physics=getattr(Physics, physics), pyb_freq=pyb, ctrl_freq=ctrl,
                     initial_xyzs=xyz, initial_rpys=rng.uniform(-0.3, 0.3, (D, 3)), num_envs=E)
    env.reset()
    env.set_physical_params(m=env.M * rng.uniform(0.8, 1.2, E), kf=env.KF * rng.uniform(0.8, 1.2, E))
    return env


def _max_rpm(env):
    """[E, 1, 1] MAX_RPM of each aviary's row."""
    from gym_pybullet_drones_b200.params import physical_rows
    return physical_rows(env.DRONE_MODEL, env.physical_params(), env.G)[:, 13].to(env.device)[:, None, None]


def _inputs(env, T, seed):
    rng = np.random.default_rng(seed)
    E, D = env._E, env._D
    rpm = torch.tensor(env.HOVER_RPM * (1 + 0.05 * rng.uniform(-1, 1, (T, E, D, 4))), device=env.device)
    rpm[0, 0, 0, 0] = _max_rpm(env)[0, 0, 0] * 1.1        # one clipped rotor: its B column is zero
    state = {"pos": env.pos.clone(), "quat": torch.tensor(np.stack([quat_from_rpy(r) for r in rng.uniform(-0.5, 0.5, (E * D, 3))]),
                                                          device=env.device).reshape(E, D, 4) * 1.0000001,
             "vel": torch.tensor(rng.uniform(-1, 1, (E, D, 3)), device=env.device),
             "rpy_rates": torch.tensor(rng.uniform(-3, 3, (E, D, 3)), device=env.device)}
    last = torch.tensor(env.HOVER_RPM * (1 + 0.05 * rng.uniform(-1, 1, (E, D, 4))), device=env.device)
    return rpm, state, last


def _jvp(env, rpm, state, last, t_rpm=None, t_state=None, t_last=None):
    """Forward AD through differentiable_rollout: (outputs, tangents) as dicts of [T, E, D, k]."""
    import torch.autograd.forward_ad as fwAD
    with fwAD.dual_level():
        r = rpm if t_rpm is None else fwAD.make_dual(rpm, t_rpm)
        st = {k: (x if t_state is None else fwAD.make_dual(x, t_state[k])) for k, x in state.items()}
        lr = last if t_last is None else fwAD.make_dual(last, t_last)
        out = env.differentiable_rollout(r, state=st, last_rpm=lr)
        prim = {k: fwAD.unpack_dual(v).primal.clone() for k, v in out.items()}
        tan = {k: fwAD.unpack_dual(v).tangent for k, v in out.items()}
        tan = {k: torch.zeros_like(prim[k]) if t is None else t.clone() for k, t in tan.items()}
    return prim, tan


def _cat(d):
    return torch.cat([d[k] for k in KEYS], dim=-1)


@pytest.mark.parametrize("E,D,physics,model", [(37, 3, "PYB_GND", "CF2X"), (129, 1, "PYB_DRAG", "CF2P"), (5, 7, "DYN", "RACE"),
                                               (1, 1, "PYB_DRAG", "CF2X")])
def test_linearise_columns_match_unit_jvps(E, D, physics, model):
    """T = 1, partial CTAs and 1..7 drones per aviary: every column of A, B and B_last is the JVP kernel's tangent along the unit
    input, and the nominal trajectory is differentiable_rollout's bits."""
    env = _env(E, D, physics, model)
    rpm, state, last = _inputs(env, 1, E)
    lin = env.linearise(rpm, state=state, last_rpm=last)
    ref = env.differentiable_rollout(rpm, state=state, last_rpm=last)
    for k in KEYS:
        assert torch.equal(lin[k], ref[k]), k
    drag = physics == "PYB_DRAG"
    assert ("B_last" in lin) == drag
    z = lambda w: torch.zeros((1, E, D, w) if w == 4 else (E, D, w), dtype=torch.float64, device=env.device)
    worst = 0.0
    for col in range(21 if drag else 17):
        t_state = {k: torch.zeros_like(x) for k, x in state.items()}
        t_rpm, t_last = z(4), torch.zeros_like(last)
        if col < 13:
            key, j = [(k, j) for k, w in zip(KEYS, (3, 4, 3, 3)) for j in range(w)][col]
            t_state[key][..., j] = 1.0
            want = lin["A"][..., col]
        elif col < 17:
            t_rpm[..., col - 13] = 1.0
            want = lin["B"][..., col - 13]
        else:
            t_last[..., col - 17] = 1.0
            want = lin["B_last"][..., col - 17]
        _, tan = _jvp(env, rpm, state, last, t_rpm, t_state, t_last)
        got = _cat(tan)
        err = ((got - want).norm(dim=-1) / want.norm(dim=-1).clamp_min(1e-300)).max().item()
        worst = max(worst, err)
        assert err <= 1e-13, (col, err)
    assert torch.all(lin["B"][0, 0, 0, :, 0] == 0)                     # the clipped rotor
    print("linearise %s E=%d D=%d: worst column error against the JVP kernel %.1e" % (physics, E, D, worst))


@pytest.mark.parametrize("physics", ["DYN", "PYB_GND", "PYB_DRAG"])
def test_linearise_chain_matches_trajectory_jvp(physics):
    """dx_{k+1} = A_k dx_k + B_k drpm_k + B_last_k dup_k (dup_0 = dlast_rpm, dup_k = the clip's tangent of drpm_{k-1}) equals the
    JVP of the whole trajectory at every tick, per drone."""
    env = _env(64, 2, physics)
    T = 16
    rpm, state, last = _inputs(env, T, 7)
    rng = np.random.default_rng(8)
    t_state = {k: torch.tensor(rng.standard_normal(tuple(x.shape)), device=env.device) for k, x in state.items()}
    t_rpm = torch.tensor(rng.standard_normal(tuple(rpm.shape)), device=env.device) * 10
    t_last = torch.tensor(rng.standard_normal(tuple(last.shape)), device=env.device) * 10
    _, tan = _jvp(env, rpm, state, last, t_rpm, t_state, t_last)
    lin = env.linearise(rpm, state=state, last_rpm=last)
    mv = lambda M, x: (M @ x[..., None])[..., 0]
    dx, dup = _cat(t_state), t_last
    live = (rpm >= 0) & (rpm <= _max_rpm(env)[None])
    worst = 0.0
    for k in range(T):
        du = torch.where(live[k], t_rpm[k], torch.zeros_like(t_rpm[k]))
        dx = mv(lin["A"][k], dx) + mv(lin["B"][k], t_rpm[k])
        if "B_last" in lin:
            dx = dx + mv(lin["B_last"][k], dup)
        dup = du
        want = _cat(tan)[k]
        err = ((dx - want).norm(dim=-1) / want.norm(dim=-1)).max().item()
        worst = max(worst, err)
    print("chain %s T=%d: worst per-drone error %.1e" % (physics, T, worst))
    assert worst <= 1e-10


def test_quaternion_columns_null_on_stored_quaternion():
    env = _env(256, 2, "PYB_GND")
    rpm, state, last = _inputs(env, 4, 9)
    lin = env.linearise(rpm, state=state, last_rpm=last)
    q0 = state["quat"][None]
    q = torch.cat([q0, lin["quat"][:-1]], dim=0)
    qh = q / q.norm(dim=-1, keepdim=True)
    radial = (lin["A"][..., 3:7] @ qh[..., None])[..., 0].norm(dim=-1)
    scale = lin["A"].flatten(-2).norm(dim=-1)
    print("|A[..., 3:7] q_hat| / |A|: %.1e" % (radial / scale).max().item())
    assert (radial / scale).max().item() <= 1e-12


# ---- 3. forward AD through differentiable_rollout ------------------------------------------------------------------------

@pytest.mark.parametrize("block", ["state", "rpm", "last_rpm", "m"])
def test_forward_ad_matches_central_differences(block):
    env = _env(8, 2, "PYB_DRAG")
    T = 8
    rpm, state, last = _inputs(env, T, 10)
    rpm[0, 0, 0, 0] = env.HOVER_RPM                                # away from the clip: central differences straddle no kink
    rng = np.random.default_rng(11)
    m = env.physical_params()["m"]
    if block == "state":
        v = {k: torch.tensor(rng.standard_normal(tuple(x.shape)), device=env.device) * (0.1 if k == "quat" else 1.0) for k, x in state.items()}
    elif block == "m":
        v = torch.tensor(rng.uniform(0.5, 1.0, 8), device=env.device) * m
    else:
        x = rpm if block == "rpm" else last
        v = torch.tensor(rng.standard_normal(tuple(x.shape)), device=env.device) * env.HOVER_RPM

    def run(h, dual=None):
        import torch.autograd.forward_ad as fwAD
        st = {k: x + h * v[k] if block == "state" else x for k, x in state.items()}
        r = rpm + h * v if block == "rpm" else rpm
        lr = last + h * v if block == "last_rpm" else last
        phys = {"m": m + h * v} if block == "m" else None
        if dual is None:
            return _cat(env.differentiable_rollout(r, state=st, last_rpm=lr, phys=phys))
        with fwAD.dual_level():
            if block == "state":
                st = {k: fwAD.make_dual(x, v[k]) for k, x in st.items()}
            elif block == "rpm":
                r = fwAD.make_dual(r, v)
            elif block == "last_rpm":
                lr = fwAD.make_dual(lr, v)
            else:
                phys = {"m": fwAD.make_dual(phys["m"], v)}
            out = env.differentiable_rollout(r, state=st, last_rpm=lr, phys=phys)
            return _cat({k: fwAD.unpack_dual(x).primal for k, x in out.items()}), _cat({k: fwAD.unpack_dual(x).tangent for k, x in out.items()})

    plain = run(0.0)
    prim, tan = run(0.0, dual=True)
    assert torch.equal(prim, plain)                                 # the primal outputs, bit for bit
    h = 1e-6
    fd = (run(h) - run(-h)) / (2 * h)
    err = R.relerr(tan.cpu(), fd.cpu())
    print("forward AD %s against central differences: %.1e" % (block, err))
    assert err <= 1e-6


# ---- 4. shapes and refusals ---------------------------------------------------------------------------------------------

def test_strided_rpm_and_refusals():
    import torch.autograd.forward_ad as fwAD
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils.enums import Physics
    env = _env(4, 2, "DYN")
    rpm, state, last = _inputs(env, 3, 12)
    wide = torch.zeros((3, 4, 2, 8), dtype=torch.float64, device=env.device)
    wide[..., ::2] = rpm
    a, b = env.linearise(wide[..., ::2], state=state, last_rpm=last), env.linearise(rpm, state=state, last_rpm=last)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    with pytest.raises(ValueError):
        env.linearise(rpm.float(), state=state)
    with pytest.raises(ValueError):
        env.linearise(rpm[:, :, :1])
    with pytest.raises(ValueError):
        env.linearise(rpm[:0])
    with pytest.raises(ValueError):
        env.linearise(rpm.cpu())
    with pytest.raises(ValueError):
        env.linearise(rpm, state={"position": env.pos})
    dw = CtrlAviary(num_drones=2, physics=Physics.PYB_DW, num_envs=2)
    with pytest.raises(ValueError, match="downwash"):
        dw.linearise(torch.full((1, 2, 2, 4), dw.HOVER_RPM, dtype=torch.float64, device=dw.device))
    with fwAD.dual_level():                                          # a tangent that itself requires grad
        t = torch.ones_like(rpm).requires_grad_(True)
        with pytest.raises(ValueError, match="tangent"):
            env.differentiable_rollout(fwAD.make_dual(rpm, t), state=state)


# ---- 5. use: a discrete LQR on linearise's Jacobians stabilises the drones ---------------------------------------------------

def _lqr_gains(A, B):
    import scipy.linalg as sl
    Q = np.diag([100.0] * 3 + [10.0] * 4 + [10.0] * 3 + [1.0] * 3)       # pos, quat, vel, rpy_rates
    Rm = np.eye(4) * 1e-7                                                  # per RPM^2: about 1e3 RPM per metre of error
    K = []
    for a, b in zip(A, B):
        Pm = sl.solve_discrete_are(a, b, Q, Rm)
        K.append(np.linalg.solve(Rm + b.T @ Pm @ b, b.T @ Pm @ a))
    return np.stack(K)


@pytest.mark.parametrize("zero_gain", [False, True])
def test_lqr_on_linearised_hover_stabilises_ctrl_aviary(zero_gain):
    """CtrlAviary cf2x, DYN at 240 / 48 Hz, four aviaries with masses 0.8 .. 1.2 x nominal: linearise each at its own hover
    (T = 1), solve the discrete LQR per drone (Q, R in _lqr_gains), fly u = hover - K (x - x_eq) through step() with float64
    RPMs from 0.2 m and 0.3 rad away.  After 5 s the position error is below 1e-3 m; with K = 0 it is not."""
    from gym_pybullet_drones_b200.params import physical_rows
    env = _env(4, 1, "DYN")
    E = 4
    env.set_physical_params(m=env.M * np.array([0.8, 0.9, 1.1, 1.2]))
    dev = env.device
    hover = physical_rows(env.DRONE_MODEL, env.physical_params(), env.G)[:, 12].to(dev)
    u_eq = hover[:, None, None].expand(E, 1, 4).contiguous()
    f64 = dict(dtype=torch.float64, device=dev)
    x_eq = {"pos": torch.tensor([0, 0, 1.0], **f64).expand(E, 1, 3).clone(), "quat": torch.tensor([0, 0, 0, 1.0], **f64).expand(E, 1, 4).clone(),
            "vel": torch.zeros((E, 1, 3), dtype=torch.float64, device=dev), "rpy_rates": torch.zeros((E, 1, 3), dtype=torch.float64, device=dev)}
    lin = env.linearise(u_eq[None], state=x_eq, last_rpm=u_eq)
    drift = (_cat({k: lin[k][0] for k in KEYS}) - _cat(x_eq)).abs().max().item()
    assert drift <= 1e-12                                                   # each drone's hover is an equilibrium
    K = torch.tensor(_lqr_gains(lin["A"][0, :, 0].cpu().numpy(), lin["B"][0, :, 0].cpu().numpy()), device=dev)
    if zero_gain:
        K = torch.zeros_like(K)
    d = torch.tensor([1.0, -1.0, 1.0], dtype=torch.float64, device=dev) / 3 ** 0.5
    env.set_state(pos=x_eq["pos"] + 0.2 * d, quat=torch.tensor(quat_from_rpy(0.3 * np.array([1.0, 1.0, -1.0]) / 3 ** 0.5), device=dev).expand(E, 1, 4),
                  vel=x_eq["vel"], rpy_rates=x_eq["rpy_rates"])
    xe = _cat(x_eq)[:, 0]
    for _ in range(5 * env.CTRL_FREQ):
        x = torch.cat([env.pos, env.quat, env.vel, env.rpy_rates], dim=-1).reshape(E, 13)
        u = hover[:, None] - torch.einsum("eij,ej->ei", K, x - xe)
        env.step(u.reshape(E, 1, 4))
    err = (env.pos.reshape(E, 3) - x_eq["pos"][:, 0]).norm(dim=1)
    print("LQR%s: position error after 5 s %s" % (" (K = 0)" if zero_gain else "", err.cpu().numpy()))
    if zero_gain:
        assert torch.all(~(err < 1e-2))
    else:
        assert err.max().item() < 1e-3
