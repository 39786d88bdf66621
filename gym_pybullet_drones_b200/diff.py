"""Differentiable raw-RPM trajectories of Physics.DYN: a torch.autograd.Function over qs_dyn_traj / qs_dyn_traj_vjp
(include/quadsim.h, DESIGN.md 4.5).  BaseAviary.differentiable_rollout is the public entry point; this module packs the state
into the kernels' planes layout, runs the forward and backward kernels and unpacks the result."""
import ctypes as C

import torch

from . import _native as N

STATE_KEYS = (("pos", 3), ("quat", 4), ("vel", 3), ("rpy_rates", 3))


def pack_state(pos, quat, vel, w):
    """[N, 3], [N, 4], [N, 3], [N, 3] -> the [13 N] planes of QsState ([pos|w.x] [quat] [vel|w.y] as [N][4], then w.z)."""
    return torch.cat([torch.cat([pos, w[:, 0:1]], 1).reshape(-1), quat.reshape(-1), torch.cat([vel, w[:, 1:2]], 1).reshape(-1), w[:, 2]])


def unpack_states(planes, n):
    """[..., 13 N] planes -> {pos, quat, vel, rpy_rates} as [..., N, k] views."""
    head = planes[..., :12 * n].unflatten(-1, (3, n, 4))
    p0, q, p2 = head[..., 0, :, :], head[..., 1, :, :], head[..., 2, :, :]
    w = torch.stack([p0[..., 3], p2[..., 3], planes[..., 12 * n:]], dim=-1)
    return {"pos": p0[..., 0:3], "quat": q, "vel": p2[..., 0:3], "rpy_rates": w}


class DynTrajectory(torch.autograd.Function):
    """states [T, 13 N] = the T ticks of qs_dyn_traj from planes0 [13 N] with rpm [T, N, 4], last_rpm [N, 4] and the per-aviary
    rows [E, 16]; backward = qs_dyn_traj_vjp, its per-drone row gradients summed over each aviary's drones (torch, deterministic).
    `cfg` = (QsParams, E, D, substeps, effects).  The inputs may have any strides (the kernels read dense buffers: they get
    contiguous copies).  Double backward raises ValueError."""

    @staticmethod
    def forward(ctx, rpm, planes0, last_rpm, rows, cfg):
        rpm, planes0, last_rpm, rows = (x.contiguous() for x in (rpm, planes0, last_rpm, rows))
        P, E, D, S, eff = cfg
        T, n = rpm.shape[0], E * D
        states = torch.empty((T, 13 * n), dtype=torch.float64, device=rpm.device)
        io = N.QsDynTrajIO()
        io.T = T
        io.state0, io.rpm, io.last_rpm, io.phys = planes0.data_ptr(), rpm.data_ptr(), last_rpm.data_ptr(), rows.data_ptr()
        io.states = states.data_ptr()
        with torch.cuda.device(rpm.device):
            N.check(N.lib().qs_dyn_traj(C.byref(P), C.byref(io), E, D, S, eff, torch.cuda.current_stream().cuda_stream), "qs_dyn_traj")
        ctx.save_for_backward(rpm, planes0, last_rpm, rows, states)
        ctx.cfg = cfg
        return states

    @staticmethod
    def backward(ctx, g_states):
        if torch.is_grad_enabled():
            raise ValueError("differentiable_rollout: double backward (create_graph=True) is not supported: the VJP kernel has no "
                             "derivative of its own")
        rpm, planes0, last_rpm, rows, states = ctx.saved_tensors
        P, E, D, S, eff = ctx.cfg
        T, n = rpm.shape[0], E * D
        f64 = dict(dtype=torch.float64, device=rpm.device)
        g_states = g_states.to(torch.float64).contiguous()
        g_rpm, g_state0 = torch.empty((T, n, 4), **f64), torch.empty((13 * n,), **f64)
        g_last, g_phys = torch.empty((n, 4), **f64), torch.empty((n, 16), **f64)
        scratch = torch.empty((S, 13, n), **f64)
        io = N.QsDynTrajIO()
        io.T = T
        io.state0, io.rpm, io.last_rpm, io.phys = planes0.data_ptr(), rpm.data_ptr(), last_rpm.data_ptr(), rows.data_ptr()
        io.states, io.g_states = states.data_ptr(), g_states.data_ptr()
        io.g_rpm, io.g_state0, io.g_last_rpm, io.g_phys = g_rpm.data_ptr(), g_state0.data_ptr(), g_last.data_ptr(), g_phys.data_ptr()
        io.scratch = scratch.data_ptr()
        with torch.cuda.device(rpm.device):
            N.check(N.lib().qs_dyn_traj_vjp(C.byref(P), C.byref(io), E, D, S, eff, torch.cuda.current_stream().cuda_stream),
                    "qs_dyn_traj_vjp")
        return g_rpm, g_state0, g_last, g_phys.view(E, D, 16).sum(dim=1), None


def _tensor(x, name, shape, device):
    if not isinstance(x, torch.Tensor):
        raise ValueError("%s must be a torch tensor, got %s" % (name, type(x).__name__))
    if x.device != device:
        raise ValueError("%s must be on %s, got %s" % (name, device, x.device))
    if x.dtype != torch.float64:
        raise ValueError("%s must be float64, got %s" % (name, x.dtype))
    if tuple(x.shape) != tuple(shape):
        raise ValueError("%s must have shape %s, got %s" % (name, tuple(shape), tuple(x.shape)))
    return x


def differentiable_rollout(env, rpm, state=None, last_rpm=None, phys=None):
    """BaseAviary.differentiable_rollout (see there)."""
    from .params import PHYS_KEYS, physical_rows
    if env._effects & N.EFFECT_DW or env._EXTERNAL_DOWNWASH:
        raise ValueError("differentiable_rollout() does not support downwash: the pairwise term has no adjoint (use Physics.DYN, PYB, "
                         "PYB_GND or PYB_DRAG)")
    E, D, n, dev = env._E, env._D, env._N, env.device
    if not isinstance(rpm, torch.Tensor) or rpm.dim() != 4:
        raise ValueError("rpm must be a [T, %d, %d, 4] float64 CUDA tensor" % (E, D))
    T = rpm.shape[0]
    if T <= 0:
        raise ValueError("rpm must hold at least one tick")
    _tensor(rpm, "rpm", (T, E, D, 4), dev)
    # the env's state in drone-id order (every drone is independent without downwash: the kernels need no storage order)
    cur = {"pos": env._plane[0, :, 0:3], "quat": env._plane[1], "vel": env._plane[2, :, 0:3],
           "rpy_rates": torch.stack([env._plane[0, :, 3], env._plane[2, :, 3], env._wz], dim=1)}
    state = dict(state or {})
    bad = set(state) - {k for k, _ in STATE_KEYS}
    if bad:
        raise ValueError("unknown state keys %s (expected pos, quat, vel, rpy_rates)" % sorted(bad))
    parts = []
    for k, w in STATE_KEYS:
        if k in state:
            parts.append(_tensor(state[k], "state[%r]" % k, (E, D, w), dev).reshape(n, w))
        else:
            parts.append(env._by_id(cur[k]).detach().clone())
    planes0 = pack_state(*parts).contiguous()
    if last_rpm is None:
        last_rpm = env._by_id(env._last_rpm).detach().clone() if env._track_last_action else torch.zeros((n, 4), dtype=torch.float64, device=dev)
    else:
        last_rpm = _tensor(last_rpm, "last_rpm", (E, D, 4), dev).reshape(n, 4)
    phys = dict(phys or {})
    bad = set(phys) - set(PHYS_KEYS)
    if bad:
        raise ValueError("unknown physical parameters %s (expected some of %s)" % (sorted(bad), ", ".join(PHYS_KEYS)))
    props = env.physical_params()
    for k, v in phys.items():
        props[k] = _tensor(v, "phys[%r]" % k, (E,), dev)
    with torch.cuda.device(dev):
        rows = physical_rows(env.DRONE_MODEL, props, env.G)
        cfg = (env._P, E, D, env.PYB_STEPS_PER_CTRL, env._effects)
        states = DynTrajectory.apply(rpm.reshape(T, n, 4).contiguous(), planes0, last_rpm.contiguous(), rows.contiguous(), cfg)
    return {k: v.reshape(T, E, D, v.shape[-1]) for k, v in unpack_states(states, n).items()}
