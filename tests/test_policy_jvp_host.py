"""CPU tests of the forward mode of the policy loop (DESIGN.md 4.5): the kernels' aviary tick tangent (mlp_tangent.cuh, built for
the host) against torch.func.jacfwd of the reference tick with the observation's ang_v as state, and against the transpose of the
host-built adjoint; at an action exactly at +-1, a ReLU unit exactly at 0 and a drone on the gimbal guard; negative controls that
show the comparison sees each decision; and the C ABI's refusals of qs_dyn_policy_traj_jvp / qs_dyn_policy_tick_jac without a
GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

import diff_ref as R
from diff_testlib import params_of, quat_from_rpy
from policy_jvp_testlib import (BLOCKS, compose_for_vjp, drop_u_rows, host_tick_jac, host_tick_jvp, ref_tick_jac, vjp_tick_jac,
                                widths)

JVP_TOL = 1e-10
VJP_TOL = 1e-12


def _relerr(got, want):
    scale = max(float(np.abs(want).max()), 1e-300)
    return float(np.abs(got - want).max()) / scale if want.size else 0.0


def _case(activation, A, D, scenario, seed):
    """(P, theta, noise, x, ql) of one aviary tick: x = {state, ang, hist, up, row} with ang = R(ql) w"""
    from gym_pybullet_drones_b200.params import PHYS_KEYS, nominal_properties, physical_rows
    from gym_pybullet_drones_b200.utils.enums import DroneModel
    import diff_policy_ref as PR
    rng = np.random.default_rng(seed)
    rnd = lambda *s: rng.uniform(-1.0, 1.0, s)
    P, c = params_of("cf2x", 240, 30)
    B, H = 5, (16, 8)
    od = 12 + B * A
    nom = nominal_properties(DroneModel.CF2X)
    row = physical_rows(DroneModel.CF2X, {k: torch.full((1,), float(nom[k]) * (1 + 0.1 * rnd(1)[0]), dtype=torch.float64) for k in PHYS_KEYS},
                        9.8)[0].numpy()
    sizes = [D * od] + list(H) + [D * A]
    theta = []
    for i, o in zip(sizes[:-1], sizes[1:]):
        theta += [rnd(i, o) / i ** 0.5, 0.1 * rnd(o)]
    theta.append(np.full(D * A, -1.0))
    rpy = 0.3 * rnd(D, 3)
    pos = rnd(D, 3) + np.array([0.0, 0.0, 1.0])
    noise = rnd(D * A)
    if scenario == "gimbal":
        rpy[0, 1] = 1.5705                                  # sarg = sin(pitch) beyond 0.99999: the guard's branch of rpy
    if scenario == "saturated":
        noise = 8.0 * noise                                 # exp(-1) * 8: most actions leave [-1, 1]
    state = np.concatenate([pos, quat_from_rpy(rpy), 0.5 * rnd(D, 3), 2.0 * rnd(D, 3)], axis=1)
    ql = quat_from_rpy(rpy + 0.01 * rnd(D, 3))
    ql = ql / np.linalg.norm(ql, axis=1, keepdims=True)
    if scenario == "edge":
        # raw actions exactly at +1 and -1 (a zero output column, bias +-1, no noise): torch.clamp passes the tangent there
        for j, v in ((0, 1.0), (D * A - 1, -1.0))[:min(2, D * A)]:
            theta[-3][:, j] = 0.0
            theta[-2][j] = v
            noise[j] = 0.0
        # first hidden unit exactly at 0 with a live input: z = pos_x * 1 - pos_x (ReLU passes nothing there)
        theta[0][:, 0] = 0.0
        theta[0][0, 0] = 1.0
        theta[1][0] = -state[0, 0]
    ang = (PR.matrix_unit(torch.tensor(ql)) @ torch.tensor(state[:, 10:13, None]))[:, :, 0].numpy()
    x = dict(state=state, ang=ang, hist=0.5 * rnd(D, B, A), up=float(c.HOVER_RPM) * (1 + 0.1 * rnd(D, 4)), row=row)
    return P, theta, noise, x, ql


EFF = {"dyn": 0, "gnd": R.EFFECT_GND, "drag": R.EFFECT_DRAG, "gnd_drag": R.EFFECT_GND | R.EFFECT_DRAG}
# (activation, A, D, effects, S, scenario): D = 1, 2, 4; RPM and ONE_D_RPM; tanh and relu; the four effect sets; S = 1 and 8;
# edge: actions at +-1 and a ReLU unit at 0; gimbal: a drone on the guard
TICKS = [("tanh", 4, 1, "dyn", 8, "flight"), ("relu", 4, 2, "gnd", 1, "edge"), ("tanh", 1, 4, "drag", 8, "edge"),
         ("relu", 1, 2, "gnd_drag", 8, "flight"), ("tanh", 4, 2, "gnd_drag", 1, "gimbal"), ("relu", 4, 1, "drag", 8, "gimbal"),
         ("relu", 1, 1, "dyn", 1, "edge"), ("tanh", 4, 4, "gnd", 8, "saturated"), ("relu", 4, 4, "dyn", 8, "edge")]


def _edge_checks(scenario, x, raw):
    if scenario == "edge":
        assert raw[0] == 1.0 and (len(raw) == 1 or raw[-1] == -1.0)
    if scenario == "gimbal":
        q = x["state"][0, 3:7]
        assert abs(-2.0 * (q[0] * q[2] - q[3] * q[1])) >= 0.99999


@pytest.mark.parametrize("activation,A,D,eff,S,scenario", TICKS)
def test_host_tick_jvp_matches_reference_jacfwd(activation, A, D, eff, S, scenario):
    P, theta, noise, x, _ = _case(activation, A, D, scenario, TICKS.index((activation, A, D, eff, S, scenario)))
    got = host_tick_jac(P, EFF[eff], S, activation, theta, noise, x)
    want = ref_tick_jac(P, EFF[eff], S, activation, theta, noise, x)
    zero = {k: np.zeros(s) for k, s in (("state", (D, 13)), ("ang", (D, 3)), ("hist", x["hist"].shape), ("up", (D, 4)),
                                        ("row", (16,)), ("raw_in", (D * A,)))}
    val, _ = host_tick_jvp(P, EFF[eff], S, activation, theta, noise, x, zero)
    _edge_checks(scenario, x, val["raw"])
    worst = {k: _relerr(got[k], want[k]) for k in BLOCKS}
    print("policy tick jvp %s A=%d D=%d %s S=%d %s: worst %.1e" % (activation, A, D, eff, S, scenario, max(worst.values())))
    assert max(worst.values()) <= JVP_TOL, worst
    if not EFF[eff] & R.EFFECT_DRAG:
        assert np.all(got["up"] == 0)


@pytest.mark.parametrize("activation,A,D,eff,S,scenario", TICKS[::2])
def test_host_tick_jvp_is_the_transpose_of_the_host_vjp(activation, A, D, eff, S, scenario):
    P, theta, noise, x, ql = _case(activation, A, D, scenario, 11 + TICKS.index((activation, A, D, eff, S, scenario)))
    jac = drop_u_rows(host_tick_jac(P, EFF[eff], S, activation, theta, noise, x), D, A, x["hist"].shape[1])
    J, dw, dq = vjp_tick_jac(P, EFF[eff], S, activation, theta, noise, x, ql)
    mine = compose_for_vjp(jac, D, dw, dq)
    worst = {k: _relerr(mine[k], J[k]) for k in J}
    print("policy tick jvp vs transposed vjp %s A=%d D=%d %s S=%d %s: worst %.1e" % (activation, A, D, eff, S, scenario, max(worst.values())))
    assert max(worst.values()) <= VJP_TOL, worst


@pytest.mark.parametrize("flip,activation", [("clip", "tanh"), ("relu", "relu"), ("ang_start", "tanh")])
def test_negative_controls_fail_the_bound(flip, activation):
    """A straight-through clip, ReLU always alive and ang_v through another attitude than the last substep's start each leave
    the bound far behind.  That attitude is the tick's start: the end of the tick gives the same function (policy_jvp_testlib)."""
    P, theta, noise, x, _ = _case(activation, 4, 2, "saturated", 5)
    got = host_tick_jac(P, 0, 8, activation, theta, noise, x)
    bad = ref_tick_jac(P, 0, 8, activation, theta, noise, x, flip=(flip,))
    worst = max(_relerr(got[k], bad[k]) for k in BLOCKS)
    assert worst > 1e-4, (flip, worst)


def test_abi_lists_the_policy_forward_mode():
    import os
    from gym_pybullet_drones_b200 import _native as N
    assert {"qs_dyn_policy_traj_jvp", "qs_dyn_policy_tick_jac", "qs_sizeof_dyn_policy_traj_jvp_io"} <= set(N.EXPORTS)
    assert any(os.path.basename(s) == "dyn_policy_jvp.cu" for s in N.SOURCES)
    assert {"mlp_tangent.cuh", "policy_actor.cuh"} <= {os.path.basename(h) for h in N.HEADERS}
    L = N.lib()
    assert L.qs_sizeof_dyn_policy_traj_jvp_io() == C.sizeof(N.QsDynPolicyTrajJvpIO)
    assert L.qs_sizeof_dyn_policy_traj_io() == C.sizeof(N.QsDynPolicyTrajIO)


def test_c_abi_refusals_return_before_any_launch():
    """Every argument check of both entry points: a negative return code naming the entry point, no device needed (the
    pointers are never read)"""
    from gym_pybullet_drones_b200 import _native as N
    L = N.lib()
    P, _ = params_of("cf2x", 240, 30)

    def io(**kw):
        q = N.QsDynPolicyTrajJvpIO()
        q.T, q.act_buffer_size, q.activation, q.depth = 4, 15, N.MLP_TANH, 2
        q.width[0] = q.width[1] = 64
        q.in_dim, q.out_dim = 72, 4
        for l in range(3):
            q.w[l], q.b[l] = 256, 256
        for k in ("log_std", "state0", "action_buffer", "states", "actions", "obs", "t_states", "t_actions", "jac"):
            setattr(q, k, 256)
        for k, v in kw.items():
            if k == "width0":
                q.width[0] = v
            elif k == "w2":
                q.w[2] = v
            else:
                setattr(q, k, v)
        return q

    for name in ("qs_dyn_policy_traj_jvp", "qs_dyn_policy_tick_jac"):
        f = getattr(L, name)

        def rc(q, act=N.ACT_RPM, E=8, D=1, S=8, eff=0):
            return f(C.byref(P), C.byref(q), act, E, D, S, eff, None)
        assert rc(io(state0=None)) == -1 and rc(io(obs=None)) == -1 and rc(io(w2=None)) == -1          # QS_ERR_NULL
        assert L.qs_last_error().startswith(name.encode() + b": ")
        if name.endswith("jvp"):
            assert rc(io(t_states=None)) == -1 and rc(io(t_actions=None)) == -1
        else:
            assert rc(io(jac=None)) == -1
        assert b"NULL" in L.qs_last_error()
        assert rc(io(T=0)) == -3 and rc(io(act_buffer_size=0)) == -3 and rc(io(depth=0)) == -3 and rc(io(depth=5)) == -3
        assert rc(io(width0=257)) == -3 and rc(io(width0=0)) == -3 and rc(io(in_dim=73)) == -3 and rc(io(out_dim=8)) == -3
        assert rc(io(activation=2)) == -4 and rc(io(), eff=8) == -4                                  # QS_ERR_ENUM
        assert rc(io(), act=N.ACT_PID) == -5 and rc(io(), act=N.ACT_VEL) == -5 and rc(io(), act=N.ACT_ONE_D_PID) == -5
        assert rc(io(), eff=N.EFFECT_DW) == -5 and b"downwash" in L.qs_last_error()
        assert rc(io(in_dim=33 * 27, out_dim=33), act=N.ACT_ONE_D_RPM, D=33) == -5                   # D * A > 32
        big = io(act_buffer_size=120, in_dim=8 * 492, out_dim=32)                                    # 240 Hz control, 8 drones
        assert rc(big, D=8) == -5 and b"shared memory" in L.qs_last_error()
        assert rc(io(phys=264)) == -2 and rc(io(t_phys=264)) == -2                                   # QS_ERR_ALIGN
        assert L.qs_last_error().startswith(name.encode() + b": ")
    # the Jacobian's grid: T ceil(E / 8) CTAs above 2^31 - 1
    assert L.qs_dyn_policy_tick_jac(C.byref(P), C.byref(io(T=1 << 30)), N.ACT_RPM, 24, 1, 8, 0, None) == -3
    assert b"2^31-1" in L.qs_last_error()


def test_nothing_the_vjp_accepts_is_refused():
    """The shared-memory bound of forward mode is the VJP's: at the widest accepted shapes, where the VJP's 8 aviaries only just
    fit, the forward-mode entry points pass every check (they fail only at the launch, for want of a device)"""
    from gym_pybullet_drones_b200 import _native as N
    L = N.lib()
    P, _ = params_of("cf2x", 240, 30)
    for B, D, width in ((120, 2, 256), (60, 4, 64), (30, 8, 256)):
        A = 4
        q = N.QsDynPolicyTrajJvpIO()
        q.T, q.act_buffer_size, q.activation, q.depth = 2, B, N.MLP_RELU, 4
        for l in range(4):
            q.width[l] = width
        q.in_dim, q.out_dim = D * (12 + B * A), D * A
        for l in range(5):
            q.w[l], q.b[l] = 256, 256
        for k in ("log_std", "state0", "action_buffer", "states", "actions", "obs", "t_states", "t_actions", "jac"):
            setattr(q, k, 256)
        v = N.QsDynPolicyTrajIO()
        C.memmove(C.addressof(v), C.addressof(q), N.QsDynPolicyTrajIO.g_states.offset)        # the layouts agree up to obs
        v.g_states = v.g_raw = v.g_state0 = v.scratch = 256
        vjp = L.qs_dyn_policy_traj_vjp(C.byref(P), C.byref(v), N.ACT_RPM, 16, D, 8, 0, None)
        msg_vjp = L.qs_last_error()
        for name in ("qs_dyn_policy_traj_jvp", "qs_dyn_policy_tick_jac"):
            r = getattr(L, name)(C.byref(P), C.byref(q), N.ACT_RPM, 16, D, 8, 0, None)
            msg = L.qs_last_error()
            if vjp == -5 and b"shared memory" in msg_vjp:
                assert r == -5 and b"shared memory" in msg, (B, D, width, name)
            else:
                assert b"shared memory" not in msg and b"NULL" not in msg, (B, D, width, name, msg)
