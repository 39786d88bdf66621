"""Shared helpers of the closed-loop differentiable-trajectory tests (test infrastructure): the g++ build of pid_adjoint.cuh with
the closed-loop tick of dyn_ctrl_traj.cu, its torch counterpart, and the drone / controller batches the tests differentiate at."""
import ctypes as C

import numpy as np
import torch

import diff_pid_ref as PR
import diff_ref as R
from diff_testlib import quat_from_rpy
from qs_testlib import harness

BLOCKS = ("state", "pid", "targets", "last_rpm", "phys", "gains")


def ctrl_harness():
    """tests/host_harness/diff_ctrl_host.cpp: the kernels' closed-loop tick adjoint compiled for the host."""
    L = harness("diff_ctrl_host")
    L.dh_ctrl_tick_vjp.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_int, C.c_double, C.c_int] + [C.c_void_p] * 18
    return L


def host_ctrl_tick_vjp(P, CP, effects, S, dt, rows, gains, state, pid, tg, up, g_out, g_rpm, g_pid):
    """The host-built kernel core: one closed-loop tick and its VJP.  Returns {out, rpm, pid_out} and the gradients of BLOCKS."""
    L = ctrl_harness()
    n = state.shape[0]
    a = lambda x: np.ascontiguousarray(x, dtype=np.float64)
    ins = [a(x) for x in (rows, gains, state, pid, tg, up, g_out, g_rpm, g_pid)]
    outs = [np.zeros((n, w)) for w in (13, 4, 9, 13, 9, 10, 4, 16, 18)]
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    L.dh_ctrl_tick_vjp(C.addressof(P), C.addressof(CP), effects, S, dt, n, *[p(x) for x in ins], *[p(o) for o in outs])
    res = dict(zip(("out", "rpm", "pid_out"), outs[:3]))
    res.update(zip(("state", "pid", "targets", "last_rpm", "phys", "gains"), outs[3:]))
    return res


def ref_ctrl_tick_vjp(P, CP, effects, S, dt, rows, gains, state, pid, tg, up, g_out, g_rpm, g_pid, flip=()):
    """diff_pid_ref's closed-loop tick and its autograd VJP, in the layout of host_ctrl_tick_vjp."""
    K, Cc = R.model_constants(P), PR.controller_constants(CP)
    t = {k: torch.tensor(np.asarray(v, dtype=np.float64), requires_grad=True) for k, v in
         dict(state=state, pid=pid, targets=tg, last_rpm=up, phys=rows, gains=gains).items()}
    tgt = t["targets"]
    raw, st, _, _ = PR.pid(Cc, t["gains"], t["pid"], dt, t["state"], tgt[:, 0:3], tgt[:, 3], tgt[:, 4:7], tgt[:, 7:10], flip)
    u1 = torch.clamp(raw, 0.0, Cc["max_rpm"])
    out, u = R.tick(K, t["phys"], t["state"], u1, t["last_rpm"], S, effects)
    loss = (out * torch.tensor(g_out)).sum() + (u * torch.tensor(g_rpm)).sum() + (st * torch.tensor(g_pid)).sum()
    gs = torch.autograd.grad(loss, [t[k] for k in BLOCKS], allow_unused=True)
    res = {k: (torch.zeros_like(t[k]) if g is None else g).numpy() for k, g in zip(BLOCKS, gs)}
    res.update(out=out.detach().numpy(), rpm=u.detach().numpy(), pid_out=st.detach().numpy())
    return res


def ctrl_scenarios(c, rng, n=6):
    """{name: (state [n, 13], pid [n, 9], targets [n, 10])} at the controller's decision points (DESIGN.md 4.5); c: the env
    model's AviaryConstants.  Targets are target_pos, target yaw, target_vel, target_rpy_rates."""
    def state(pos, rpy, vel, w):
        return np.concatenate([pos, quat_from_rpy(rpy), vel, w], axis=1)

    def rnd(lo, hi, shape):
        return rng.uniform(lo, hi, shape)

    def targets(pos, spread):
        return np.concatenate([pos + rnd(-spread, spread, (n, 3)), rnd(-1, 1, (n, 1)), rnd(-0.3, 0.3, (n, 3)), rnd(-0.1, 0.1, (n, 3))], 1)

    def pid(scale_i=0.05, scale_r=0.05):
        return np.concatenate([rnd(-scale_i, scale_i, (n, 3)), rnd(-0.2, 0.2, (n, 3)), rnd(-scale_r, scale_r, (n, 3))], 1)

    out = {}
    pos = rnd(-1, 1, (n, 3)) + [0, 0, 1.5]
    out["flight"] = (state(pos, rnd(-0.2, 0.2, (n, 3)), rnd(-0.5, 0.5, (n, 3)), rnd(-1, 1, (n, 3))), pid(), targets(pos, 0.05))
    # integral clips: integral_pos_e near +-2 (x, y) and +-0.15 (z), integral_rpy_e near +-1, half of them pushed over
    p = pid()
    sgn = np.sign(rnd(-1, 1, (n, 3)))
    p[:, 0:2] = sgn[:, 0:2] * rnd(1.9, 2.1, (n, 2)).clip(max=2.0)
    p[:, 2] = sgn[:, 2] * rnd(0.1, 0.2, n).clip(max=0.15)
    p[:, 6:8] = sgn[:, 0:2] * rnd(0.9, 1.1, (n, 2)).clip(max=1.0)
    pos = rnd(-1, 1, (n, 3)) + [0, 0, 1.5]
    out["integral"] = (state(pos, rnd(-0.3, 0.3, (n, 3)), rnd(-0.5, 0.5, (n, 3)), rnd(-2, 2, (n, 3))), p, targets(pos, 3.0))
    # PWM saturation: far targets
    pos = rnd(-1, 1, (n, 3)) + [0, 0, 1.5]
    out["pwm"] = (state(pos, rnd(-0.1, 0.1, (n, 3)), rnd(-0.5, 0.5, (n, 3)), rnd(-1, 1, (n, 3))), pid(), targets(pos + [0, 0, 4], 2.0))
    # torque clip: large attitude errors and rates
    pos = rnd(-1, 1, (n, 3)) + [0, 0, 1.5]
    out["torque"] = (state(pos, rnd(-0.8, 0.8, (n, 3)), rnd(-0.5, 0.5, (n, 3)), rnd(-8, 8, (n, 3))), pid(), targets(pos, 0.5))
    # upside down under a target above: the thrust scalar is negative
    pos = rnd(-1, 1, (n, 3)) + [0, 0, 1.5]
    rpy = np.concatenate([np.pi - rnd(0, 0.3, (n, 1)), rnd(-0.2, 0.2, (n, 2))], 1)
    out["scalar"] = (state(pos, rpy, rnd(-0.5, 0.5, (n, 3)), rnd(-1, 1, (n, 3))), pid(), targets(pos + [0, 0, 0.5], 0.1))
    # pitch within the gimbal guard (|sarg| >= 0.99999), both signs
    pos = rnd(-1, 1, (n, 3)) + [0, 0, 1.5]
    rpy = np.concatenate([rnd(-0.3, 0.3, (n, 1)), np.sign(rnd(-1, 1, (n, 1))) * (np.pi / 2 - rnd(1e-4, 3e-3, (n, 1))), rnd(-1, 1, (n, 1))], 1)
    out["gimbal"] = (state(pos, rpy, rnd(-0.5, 0.5, (n, 3)), rnd(-1, 1, (n, 3))), pid(), targets(pos, 0.3))
    return out
