"""No GPU: the g++ build of mlp_adjoint.cuh (tests/host_harness/diff_policy_host.cpp: one aviary tick of the policy loop and its
VJP, the code of dyn_policy_traj.cu's kernels) against the torch reference tests/diff_policy_ref.py per input block, with negative
controls; the reference against its own central differences; the C ABI of qs_dyn_policy_traj (exports, struct size, every
argument refusal, which returns before any launch) and MlpPolicy.parameters64 / load_parameters on the CPU."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import diff_policy_ref as PR
import diff_ref as R
from diff_testlib import params_of
from qs_testlib import harness


def _case(activation, A, D, effects, seed):
    from gym_pybullet_drones_b200.params import PHYS_KEYS, nominal_properties, physical_rows
    from gym_pybullet_drones_b200.utils.enums import DroneModel
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64) * 2 - 1
    P, c = params_of("cf2x", 240, 30)
    E, B, T, H = 2, 15, 4, 6
    n, od = E * D, 12 + B * A
    nom = nominal_properties(DroneModel.CF2X)
    props = {k: torch.full((E,), float(nom[k]), dtype=torch.float64) * (1 + 0.1 * rnd(E)) for k in PHYS_KEYS}
    theta = [rnd(D * od, H) / (D * od) ** 0.5, 0.1 * rnd(H), rnd(H, D * A) / H ** 0.5, 0.1 * rnd(D * A), torch.full((D * A,), -1.0, dtype=torch.float64)]
    x0 = torch.cat([rnd(n, 3) + torch.tensor([0.0, 0.0, 1.0]), torch.nn.functional.normalize(rnd(n, 4) * 0.1 + torch.tensor([0, 0, 0, 1.0]), dim=1),
                    0.5 * rnd(n, 3), rnd(n, 3)], dim=1)
    leaves = dict(x0=x0, abuf=0.5 * rnd(n, B, A), last=float(c.HOVER_RPM) * (1 + 0.1 * rnd(n, 4)), noise=rnd(T, E, D * A),
                  **{"theta%d" % j: t for j, t in enumerate(theta)}, **props)
    leaves = {k: v.clone().requires_grad_(True) for k, v in leaves.items()}
    cot = rnd(T, n, 13)

    def f(L):
        rows = physical_rows(DroneModel.CF2X, {k: L[k] for k in PHYS_KEYS}, 9.8).repeat_interleave(D, dim=0)
        xs, raw, _ = PR.policy_loop(R.model_constants(P), rows, [L["theta%d" % j] for j in range(5)], activation, L["x0"], L["abuf"], L["last"],
                                    L["noise"], T, E, D, 8, effects)
        return (xs * cot).sum() + raw.sum()
    return leaves, f


@pytest.mark.parametrize("activation,A,D,effects", [("tanh", 4, 1, 0), ("relu", 1, 2, R.EFFECT_DRAG), ("tanh", 4, 2, R.EFFECT_GND)])
def test_reference_gradient_matches_central_differences(activation, A, D, effects):
    L, f = _case(activation, A, D, effects, 7)
    grads = dict(zip(L, torch.autograd.grad(f(L), list(L.values()), allow_unused=True)))
    rng = np.random.default_rng(0)
    for k in ("theta0", "theta2", "theta4", "x0", "abuf", "noise", "m", "kf"):
        v = torch.tensor(rng.standard_normal(tuple(L[k].shape)))
        h = 1e-6 * float(L[k].detach().abs().max())
        with torch.no_grad():
            up, dn = f(dict(L, **{k: L[k] + h * v})), f(dict(L, **{k: L[k] - h * v}))
        fd, an = float(up - dn) / (2 * h), float((grads[k] * v).sum())
        tol = 1e-6 if activation == "tanh" else 2e-5         # a ReLU unit or an action clip can change side inside the step
        assert abs(fd - an) <= tol * max(1.0, abs(an)), (k, fd, an)


def test_abi_lists_the_policy_trajectory():
    from gym_pybullet_drones_b200 import _native as N
    assert {"qs_dyn_policy_traj", "qs_dyn_policy_traj_vjp", "qs_sizeof_dyn_policy_traj_io"} <= set(N.EXPORTS)
    assert any(os.path.basename(s) == "dyn_policy_traj.cu" for s in N.SOURCES)
    assert any(os.path.basename(h) == "mlp_adjoint.cuh" for h in N.HEADERS)
    lib = C.CDLL(N.LIB_PATH)
    lib.qs_sizeof_dyn_policy_traj_io.restype = C.c_int
    assert lib.qs_sizeof_dyn_policy_traj_io() == C.sizeof(N.QsDynPolicyTrajIO)


def test_parameters64_round_trip_on_the_cpu():
    from gym_pybullet_drones_b200.policy import MlpPolicy
    pol = MlpPolicy.random(72, 4, seed=1, critic=True, net_arch=[100, 32], activation="relu", device="cpu")
    critic = [(w.clone(), b.clone()) for w, b in pol.critic]
    theta = pol.parameters64()
    assert [tuple(t.shape) for t in theta] == [(72, 100), (100,), (100, 32), (32,), (32, 4), (4,), (4,)]
    assert all(t.dtype == torch.float64 and t.requires_grad and t.is_leaf for t in theta)
    new = [t.detach() + 0.01 for t in theta]
    pol.load_parameters(new)
    fresh = MlpPolicy([(new[2 * k].float(), new[2 * k + 1].float()) for k in range(3)], new[-1].float(), None, "cpu", "relu")
    for (w, b), (fw, fb) in zip(pol._split["actor"], fresh._split["actor"]):
        assert torch.equal(w, fw) and torch.equal(b, fb)
    for p, q in zip(pol.parameters64(), new):
        assert torch.equal(p, q.float().double())
    for (w, b), (cw, cb) in zip(pol.critic, critic):
        assert torch.equal(w, cw) and torch.equal(b, cb)
    with pytest.raises(ValueError, match="load_parameters"):
        pol.load_parameters(new[:-1])
    with pytest.raises(ValueError, match="layer 0"):
        pol.load_parameters([new[0].t()] + new[1:])


# ---- the g++ build of the aviary tick adjoint ------------------------------------------------------------------------------

def _quat(rpy):
    from diff_testlib import quat_from_rpy
    return torch.tensor(quat_from_rpy(np.asarray(rpy, dtype=np.float64)))


def _tick_case(activation, A, D, effects, scenario, seed):
    """Inputs of one aviary tick (leaves), the constants around them and the cotangents of its four outputs."""
    from gym_pybullet_drones_b200.params import PHYS_KEYS, nominal_properties, physical_rows
    from gym_pybullet_drones_b200.utils.enums import DroneModel
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64) * 2 - 1
    P, c = params_of("cf2x", 240, 30)
    B, H = 15, (16, 8)
    od = 12 + B * A
    nom = nominal_properties(DroneModel.CF2X)
    row = physical_rows(DroneModel.CF2X, {k: torch.full((1,), float(nom[k]), dtype=torch.float64) * (1 + 0.1 * rnd(1)) for k in PHYS_KEYS}, 9.8)[0]
    widths = [D * od] + list(H) + [D * A]
    theta = []
    for i, o in zip(widths[:-1], widths[1:]):
        theta += [rnd(i, o) / i ** 0.5, 0.1 * rnd(o)]
    theta.append(torch.full((D * A,), -1.0, dtype=torch.float64))
    rpy = 0.3 * rnd(D, 3)
    pos = rnd(D, 3) + torch.tensor([0.0, 0.0, 1.0])
    noise = rnd(D * A)
    if scenario == "gimbal":
        rpy[0, 1] = 1.5705                                  # sarg = sin(pitch) beyond 0.99999: the guard's branch of rpy
    if scenario == "ground":
        pos[:, 2] = 0.02 + 0.02 * rnd(D).abs()
    if scenario == "saturated":
        noise = 8.0 * noise                                 # exp(-1) * 8: most actions leave [-1, 1]
    if scenario == "max_rpm":
        row = row.clone(); row[13] = row[12] * 1.01         # MAX_RPM just above HOVER_RPM: the env's clip cuts the positive actions
    x = torch.cat([pos, _quat(rpy.numpy()), 0.5 * rnd(D, 3), 2.0 * rnd(D, 3)], dim=1)
    ql = torch.nn.functional.normalize(_quat((rpy + 0.01 * rnd(D, 3)).numpy()), dim=1)
    L = dict(x=x, ql=ql, hist=0.5 * rnd(D, B, A), up=float(c.HOVER_RPM) * (1 + 0.1 * rnd(D, 4)), row=row, noise=noise,
             **{"theta%d" % j: t for j, t in enumerate(theta)})
    L = {k: v.clone().requires_grad_(True) for k, v in L.items()}
    cot = dict(x=rnd(D, 13), raw=rnd(D, A), ang=rnd(D, 3), hist=rnd(D, B, A))
    return P, L, cot, len(theta)


def _ref_tick(P, L, cot, nth, activation, D, effects, flip=()):
    theta = [L["theta%d" % j] for j in range(nth)]
    x1, _, ql1, raw, _, hist1 = PR.one_tick(R.model_constants(P), L["row"][None].expand(D, 16), theta, activation, L["x"], L["ql"], L["hist"],
                                            L["up"], L["noise"][None], 1, D, 8, effects, flip)
    ang1 = (PR.matrix_unit(ql1) @ x1[:, 10:13, None])[:, :, 0]
    loss = (x1 * cot["x"]).sum() + (raw * cot["raw"]).sum() + (ang1 * cot["ang"]).sum() + (hist1 * cot["hist"]).sum()
    return (x1, raw, hist1, ql1), dict(zip(L, torch.autograd.grad(loss, list(L.values()), allow_unused=True)))


def _host_tick(P, L, cot, nth, activation, D, A, effects):
    lib = harness("diff_policy_host")
    B = L["hist"].shape[1]
    depth = nth // 2 - 1
    arr = lambda t: np.ascontiguousarray(t.detach().numpy(), dtype=np.float64)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)
    th = [arr(L["theta%d" % j]) for j in range(nth)]
    Ws = (C.c_void_p * (depth + 1))(*[ptr(th[2 * l]).value for l in range(depth + 1)])
    bs = (C.c_void_p * (depth + 1))(*[ptr(th[2 * l + 1]).value for l in range(depth + 1)])
    width = (C.c_int * 4)(*([th[2 * l].shape[1] for l in range(depth)] + [0] * (4 - depth)))
    ins = [arr(L[k]) for k in ("row", "x", "ql", "hist", "up")] + [arr(cot["x"]), arr(cot["raw"]), arr(cot["ang"]), arr(cot["hist"])]
    noise = arr(L["noise"])
    shapes = [(D, 13), (D, A), (D, B, A), (D, 4), (D, 13), (D, 4), (D, B, A), (D, 4), (16,), (D, A)]
    outs = [np.zeros(s) for s in shapes]
    lib.dph_tick_vjp(C.addressof(P), C.c_uint(effects), 8, D, A, B, 0 if activation == "tanh" else 1, depth, width, Ws, bs, ptr(th[-1]), ptr(noise),
                     *[ptr(a) for a in ins], *[ptr(o) for o in outs])
    fwd = outs[:4]
    grads = dict(zip(("x", "ql", "hist", "up", "row", "g_raw"), outs[4:]))
    # the parameters' and the noise's gradients from g_raw, as diff.py's backward forms them
    from gym_pybullet_drones_b200.diff import actor64
    leaves = [L["theta%d" % j].detach().requires_grad_(True) for j in range(nth)]
    eps = L["noise"].detach().requires_grad_(True)
    obs = torch.tensor(_obs_of(L, D))
    got = torch.autograd.grad(actor64(leaves, activation, obs[None], eps[None]), leaves + [eps], torch.tensor(grads.pop("g_raw")).reshape(1, -1))
    grads.update({"theta%d" % j: g for j, g in enumerate(got[:-1])}, noise=got[-1])
    return fwd, grads


def _obs_of(L, D):
    x, ql, hist = L["x"].detach(), L["ql"].detach(), L["hist"].detach()
    ang = (PR.matrix_unit(ql) @ x[:, 10:13, None])[:, :, 0]
    return torch.cat([x[:, 0:3], PR.PR.quat_to_euler(x[:, 3:7]), x[:, 7:10], ang, hist.reshape(D, -1)], dim=1).reshape(-1).numpy()


def _worst(got, want):
    return {k: R.relerr(torch.as_tensor(got[k]).reshape(-1), (torch.zeros_like(torch.as_tensor(got[k])) if want[k] is None else want[k]).reshape(-1))
            for k in got}


TICKS = [("tanh", 4, 1, 0, "flight"), ("relu", 4, 2, R.EFFECT_GND, "ground"), ("tanh", 1, 4, R.EFFECT_DRAG, "flight"),
         ("relu", 1, 2, R.EFFECT_GND | R.EFFECT_DRAG, "flight"), ("tanh", 4, 2, 0, "saturated"), ("relu", 4, 1, R.EFFECT_DRAG, "saturated"),
         ("tanh", 4, 2, R.EFFECT_GND | R.EFFECT_DRAG, "gimbal"), ("tanh", 4, 1, 0, "max_rpm")]


@pytest.mark.parametrize("activation,A,D,effects,scenario", TICKS)
def test_host_tick_adjoint_matches_the_reference(activation, A, D, effects, scenario):
    P, L, cot, nth = _tick_case(activation, A, D, effects, scenario, 3)
    fwd, grads = _host_tick(P, L, cot, nth, activation, D, A, effects)
    ref_fwd, want = _ref_tick(P, L, cot, nth, activation, D, effects)
    for got, ref in zip(fwd, ref_fwd):
        assert R.relerr(torch.tensor(got).reshape(-1), ref.detach().reshape(-1)) <= 1e-12
    if scenario == "gimbal":
        x = L["x"].detach()
        assert abs(float(-2.0 * (x[0, 3] * x[0, 5] - x[0, 6] * x[0, 4]))) >= 0.99999
    if scenario == "saturated":
        assert (np.abs(fwd[1]) > 1).mean() > 0.3
    worst = _worst(grads, want)
    assert max(worst.values()) <= 1e-10, worst


@pytest.mark.parametrize("activation,flip", [("tanh", "history"), ("tanh", "clip"), ("relu", "relu")])
def test_host_tick_negative_controls_fail_the_bound(activation, flip):
    P, L, cot, nth = _tick_case(activation, 4, 2, 0, "saturated", 5)
    _, grads = _host_tick(P, L, cot, nth, activation, 2, 4, 0)
    _, bad = _ref_tick(P, L, cot, nth, activation, 2, 0, flip=(flip,))
    assert max(_worst(grads, bad).values()) > 1e-4


def test_c_abi_refusals_return_before_any_launch():
    """Every argument check of qs_dyn_policy_traj: a negative return code, no device needed (the pointers are never read)."""
    from gym_pybullet_drones_b200 import _native as N
    lib = N.lib()
    P, _ = params_of("cf2x", 240, 30)

    def io(**kw):
        q = N.QsDynPolicyTrajIO()
        q.T, q.act_buffer_size, q.activation, q.depth = 4, 15, N.MLP_TANH, 2
        q.width[0] = q.width[1] = 64
        q.in_dim, q.out_dim = 72, 4
        for l in range(3):
            q.w[l], q.b[l] = 256, 256
        for k in ("log_std", "state0", "action_buffer", "states", "actions", "obs"):
            setattr(q, k, 256)
        for k, v in kw.items():
            if k == "width0":
                q.width[0] = v
            elif k == "w2":
                q.w[2] = v
            else:
                setattr(q, k, v)
        return q

    def rc(q, act=N.ACT_RPM, E=8, D=1, S=8, eff=0, vjp=False):
        f = lib.qs_dyn_policy_traj_vjp if vjp else lib.qs_dyn_policy_traj
        return f(C.byref(P), C.byref(q), act, E, D, S, eff, None)
    assert rc(io(state0=None)) == -1 and rc(io(w2=None)) == -1 and rc(io(), vjp=True) == -1          # QS_ERR_NULL
    assert lib.qs_last_error().startswith(b"qs_dyn_policy_traj_vjp: ")      # a refusal names the entry point that was called
    assert rc(io(T=0)) == -3 and rc(io(act_buffer_size=0)) == -3 and rc(io(depth=0)) == -3 and rc(io(depth=5)) == -3
    assert rc(io(width0=257)) == -3 and rc(io(width0=0)) == -3 and rc(io(in_dim=73)) == -3 and rc(io(out_dim=8)) == -3
    assert rc(io(activation=2)) == -4 and rc(io(), eff=8) == -4                                      # QS_ERR_ENUM
    assert rc(io(), act=N.ACT_PID) == -5 and rc(io(), act=N.ACT_VEL) == -5 and rc(io(), eff=N.EFFECT_DW) == -5
    assert rc(io(in_dim=33 * 27, out_dim=33), act=N.ACT_ONE_D_RPM, D=33) == -5                       # D * A > 32
    big = io(act_buffer_size=120, in_dim=8 * 492, out_dim=32)                                        # 240 Hz control, 8 drones
    assert rc(big, D=8) == -5 and b"shared memory" in lib.qs_last_error()
    assert rc(io(phys=264)) == -2                                                                    # QS_ERR_ALIGN
