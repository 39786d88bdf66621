"""Differentiable trajectories of Physics.DYN: torch.autograd.Functions over qs_dyn_traj / qs_dyn_traj_vjp (raw RPMs),
qs_dyn_ctrl_traj / qs_dyn_ctrl_traj_vjp (a DSLPIDControl in the loop), with downwash their aviary-unit twins qs_dyn_traj_dw /
qs_dyn_traj_dw_vjp and qs_dyn_ctrl_traj_dw / qs_dyn_ctrl_traj_dw_vjp, qs_dyn_lqr_traj / qs_dyn_lqr_traj_vjp (an iLQR plan's
LQR tracker in the loop) and qs_dyn_policy_traj / qs_dyn_policy_traj_vjp (an MlpPolicy in the loop) (include/quadsim.h, DESIGN.md 4.5), and their forward mode: the jvp of each Function (qs_dyn_traj_jvp,
qs_dyn_ctrl_traj_jvp, qs_dyn_policy_traj_jvp) and the per-tick Jacobians of linearise (qs_dyn_tick_jac, qs_dyn_ctrl_tick_jac,
qs_dyn_policy_tick_jac).
BaseAviary.differentiable_rollout is the public entry point; this module packs the state into the kernels' planes layout, runs
the forward and backward kernels and unpacks the result."""
import ctypes as C

import torch

from . import _native as N

STATE_KEYS = (("pos", 3), ("quat", 4), ("vel", 3), ("rpy_rates", 3))
GAIN_KEYS = ("P_COEFF_FOR", "I_COEFF_FOR", "D_COEFF_FOR", "P_COEFF_TOR", "I_COEFF_TOR", "D_COEFF_TOR")    # QsDynCtrlTrajIO.gains
PID_KEYS = ("integral_pos_e", "last_rpy", "integral_rpy_e")                                              # rows of the [9, N] state


def pack_state(pos, quat, vel, w):
    """[N, 3], [N, 4], [N, 3], [N, 3] -> the [13 N] planes of QsState ([pos|w.x] [quat] [vel|w.y] as [N][4], then w.z)."""
    return torch.cat([torch.cat([pos, w[:, 0:1]], 1).reshape(-1), quat.reshape(-1), torch.cat([vel, w[:, 1:2]], 1).reshape(-1), w[:, 2]])


def unpack_states(planes, n):
    """[..., 13 N] planes -> {pos, quat, vel, rpy_rates} as [..., N, k] views."""
    head = planes[..., :12 * n].unflatten(-1, (3, n, 4))
    p0, q, p2 = head[..., 0, :, :], head[..., 1, :, :], head[..., 2, :, :]
    w = torch.stack([p0[..., 3], p2[..., 3], planes[..., 12 * n:]], dim=-1)
    return {"pos": p0[..., 0:3], "quat": q, "vel": p2[..., 0:3], "rpy_rates": w}


def unpack_traj(states, T, E, D):
    """[T, 13 N] planes -> {pos, quat, vel, rpy_rates} as [T, E, D, k]."""
    return {k: v.reshape(T, E, D, v.shape[-1]) for k, v in unpack_states(states, E * D).items()}


def dyn_cfg(env):
    """The launch configuration of the DYN kernels for `env`: (QsParams, E, D, substeps per control tick, effects)."""
    return env._P, env._E, env._D, env.PYB_STEPS_PER_CTRL, env._effects


def _call(name, *args, device):
    """N.lib().<name>(*args, stream) on `device` and its current stream; a refusal or launch error raises (N.check)."""
    with torch.cuda.device(device):
        N.check(getattr(N.lib(), name)(*args, torch.cuda.current_stream().cuda_stream), name)


def _io(cls, T, ptrs, **scalars):
    """A `cls` IO struct with T, the given scalar fields and a pointer field per entry of `ptrs` (a tensor, or None: NULL)."""
    io = cls()
    io.T = T
    for k, v in scalars.items():
        setattr(io, k, v)
    for k, x in ptrs.items():
        setattr(io, k, None if x is None else x.data_ptr())
    return io


def _entry(name, eff):
    """The entry point `name` of the per-drone kernels, or its downwash twin (name + "_dw" before any "_vjp") for effects with
    EFFECT_DW."""
    if not eff & N.EFFECT_DW:
        return name
    return name[:-4] + "_dw_vjp" if name.endswith("_vjp") else name + "_dw"


def _no_downwash_jvp(eff):
    if eff & N.EFFECT_DW:
        raise ValueError("differentiable_rollout(downwash=True) has reverse mode only: forward-mode (dual tensor) derivatives "
                         "with downwash are not implemented (their Jacobians are per aviary)")


def _no_double_backward():
    if torch.is_grad_enabled():
        raise ValueError("differentiable_rollout: double backward (create_graph=True) is not supported: the VJP kernel has no "
                         "derivative of its own")


def _traj_ptrs(rpm, planes0, last_rpm, rows, states):
    """The primal pointers of QsDynTrajIO and QsDynTrajJvpIO: dense rpm [T, N, 4], planes0 [13 N], last_rpm [N, 4], rows [E, 16]
    and the forward's states [T, 13 N]."""
    return dict(rpm=rpm, state0=planes0, last_rpm=last_rpm, phys=rows, states=states)


def _dyn_traj(cfg, rpm, planes0, last_rpm, rows):
    """states [T, 13 N] of qs_dyn_traj from dense rpm [T, N, 4], planes0 [13 N], last_rpm [N, 4] and rows [E, 16]."""
    P, E, D, S, eff = cfg
    T, n = rpm.shape[0], E * D
    states = torch.empty((T, 13 * n), dtype=torch.float64, device=rpm.device)
    io = _io(N.QsDynTrajIO, T, _traj_ptrs(rpm, planes0, last_rpm, rows, states))
    _call(_entry("qs_dyn_traj", eff), C.byref(P), C.byref(io), E, D, S, eff, device=rpm.device)
    return states


class DynTrajectory(torch.autograd.Function):
    """states [T, 13 N] = the T ticks of qs_dyn_traj from planes0 [13 N] with rpm [T, N, 4], last_rpm [N, 4] and the per-aviary
    rows [E, 16]; backward = qs_dyn_traj_vjp, its per-drone row gradients summed over each aviary's drones (torch, deterministic);
    jvp (torch.autograd.forward_ad) = qs_dyn_traj_jvp.  `cfg` = (QsParams, E, D, substeps, effects); effects with EFFECT_DW run
    qs_dyn_traj_dw and qs_dyn_traj_dw_vjp, and their jvp raises ValueError.  The inputs may have any
    strides (the kernels read dense buffers: they get contiguous copies).  Double backward and tangents that require grad raise
    ValueError."""

    @staticmethod
    def forward(ctx, rpm, planes0, last_rpm, rows, cfg):
        rpm, planes0, last_rpm, rows = (x.contiguous() for x in (rpm, planes0, last_rpm, rows))
        states = _dyn_traj(cfg, rpm, planes0, last_rpm, rows)
        ctx.save_for_backward(rpm, planes0, last_rpm, rows, states)
        ctx.save_for_forward(rpm, planes0, last_rpm, rows, states)
        ctx.cfg = cfg
        return states

    @staticmethod
    def jvp(ctx, t_rpm, t_planes0, t_last_rpm, t_rows, _t_cfg):
        """Forward mode: the tangent [T, 13 N] of the states along the inputs' tangents (qs_dyn_traj_jvp, which linearises
        each tick at the forward's stored states).  A tangent that requires grad raises ValueError."""
        tangents = (t_rpm, t_planes0, t_last_rpm, t_rows)
        if any(t is not None and t.requires_grad for t in tangents):
            raise ValueError("differentiable_rollout: a tangent that requires grad (reverse mode over forward mode) is not supported: "
                             "the JVP kernel has no derivative of its own")
        P, E, D, S, eff = ctx.cfg
        _no_downwash_jvp(eff)
        states = ctx.saved_tensors[4]
        t_states = torch.empty_like(states)
        dense = [None if t is None else t.to(torch.float64).contiguous() for t in tangents]
        if dense[3] is not None and dense[3].data_ptr() % 16:          # the kernel reads t_phys rows as 16-byte pairs
            dense[3] = dense[3].clone()
        ptrs = dict(_traj_ptrs(*ctx.saved_tensors), t_states=t_states, **dict(zip(("t_rpm", "t_state0", "t_last_rpm", "t_phys"), dense)))
        io = _io(N.QsDynTrajJvpIO, states.shape[0], ptrs)
        _call("qs_dyn_traj_jvp", C.byref(P), C.byref(io), E, D, S, eff, device=states.device)
        return t_states

    @staticmethod
    def backward(ctx, g_states):
        _no_double_backward()
        return (*_dyn_traj_vjp(ctx.cfg, *ctx.saved_tensors, g_states), None)


def _dyn_traj_vjp(cfg, rpm, planes0, last_rpm, rows, states, g_states):
    """qs_dyn_traj_vjp of the trajectory `states` (qs_dyn_traj's output for the other inputs) for the cotangent g_states
    [T, 13 N]: (g_rpm [T, N, 4], g_planes0 [13 N], g_last_rpm [N, 4], g_rows [E, 16]), the per-drone row gradients summed over
    each aviary's drones (torch, deterministic)."""
    P, E, D, S, eff = cfg
    T, n = rpm.shape[0], E * D
    f64 = dict(dtype=torch.float64, device=rpm.device)
    g = dict(g_rpm=torch.empty((T, n, 4), **f64), g_state0=torch.empty((13 * n,), **f64), g_last_rpm=torch.empty((n, 4), **f64),
             g_phys=torch.empty((n, 16), **f64))
    ptrs = dict(_traj_ptrs(rpm, planes0, last_rpm, rows, states), g_states=g_states.to(torch.float64).contiguous(),
                scratch=torch.empty((S, 13, n), **f64), **g)
    io = _io(N.QsDynTrajIO, T, ptrs)
    _call(_entry("qs_dyn_traj_vjp", eff), C.byref(P), C.byref(io), E, D, S, eff, device=rpm.device)
    return g["g_rpm"], g["g_state0"], g["g_last_rpm"], g["g_phys"].view(E, D, 16).sum(dim=1)


CTRL_INS = ("state0", "pid0", "target_pos", "target_vel", "target_rpy", "target_rpy_rates", "last_rpm", "phys", "gains")


def _dyn_ctrl_traj(cfg, ins):
    """{states [T, 13 N], rpm [T, N, 4], pid_states [T, 9, N]} of qs_dyn_ctrl_traj from the dense inputs `ins` (CTRL_INS)."""
    P, CP, dt, E, D, S, eff = cfg
    tpos = ins["target_pos"]
    T, n = tpos.shape[0], E * D
    f64 = dict(dtype=torch.float64, device=tpos.device)
    outs = dict(states=torch.empty((T, 13 * n), **f64), rpm=torch.empty((T, n, 4), **f64), pid_states=torch.empty((T, 9, n), **f64))
    io = _io(N.QsDynCtrlTrajIO, T, dict(ins, **outs), control_timestep=dt)
    _call(_entry("qs_dyn_ctrl_traj", eff), C.byref(P), C.byref(CP), C.byref(io), E, D, S, eff, device=tpos.device)
    return outs


class DynCtrlTrajectory(torch.autograd.Function):
    """(states [T, 13 N], rpm [T, N, 4]) = the T ticks of qs_dyn_ctrl_traj from planes0 [13 N] and the controller state pid0
    [9, N], with target_pos [T, N, 3], target_vel / target_rpy / target_rpy_rates [N, 3], last_rpm [N, 4], the per-aviary rows
    [E, 16] and gain sets [E, 18]; backward = qs_dyn_ctrl_traj_vjp, its per-drone row and gain gradients summed over each
    aviary's drones (torch, deterministic); jvp (torch.autograd.forward_ad) = qs_dyn_ctrl_traj_jvp.  `cfg` = (env QsParams,
    controller QsParams, control_timestep, E, D, substeps, effects); effects with EFFECT_DW run qs_dyn_ctrl_traj_dw and
    qs_dyn_ctrl_traj_dw_vjp, and their jvp raises ValueError.  The inputs may have any strides (the kernels get contiguous copies).  Double backward and tangents that require grad raise ValueError."""

    @staticmethod
    def forward(ctx, planes0, pid0, tpos, tvel, trpy, trr, last_rpm, rows, gains, cfg):
        ins = dict(zip(CTRL_INS, (x.contiguous() for x in (planes0, pid0, tpos, tvel, trpy, trr, last_rpm, rows, gains))))
        outs = _dyn_ctrl_traj(cfg, ins)
        ctx.save_for_backward(*ins.values(), *outs.values())
        ctx.save_for_forward(*ins.values(), *outs.values())
        ctx.cfg = cfg
        return outs["states"], outs["rpm"]

    @staticmethod
    def jvp(ctx, *tangents):
        """Forward mode: the tangents (t_states [T, 13 N], t_rpm [T, N, 4]) along the inputs' tangents (qs_dyn_ctrl_traj_jvp,
        which linearises each tick at the forward's stored states).  A tangent that requires grad raises ValueError."""
        tangents = tangents[:9]
        if any(t is not None and t.requires_grad for t in tangents):
            raise ValueError("differentiable_rollout: a tangent that requires grad (reverse mode over forward mode) is not supported: "
                             "the JVP kernel has no derivative of its own")
        saved = ctx.saved_tensors
        P, CP, dt, E, D, S, eff = ctx.cfg
        _no_downwash_jvp(eff)
        states = saved[9]
        dense = [None if t is None else t.to(torch.float64).contiguous() for t in tangents]
        if dense[7] is not None and dense[7].data_ptr() % 16:          # the kernel reads t_phys rows as 16-byte pairs
            dense[7] = dense[7].clone()
        t_states, t_rpm = torch.empty_like(states), torch.empty_like(saved[10])
        ptrs = dict(zip(CTRL_INS, saved[:9]), **dict(zip(("states", "rpm", "pid_states"), saved[9:])),
                    **dict(zip(("t_" + k for k in CTRL_INS), dense)), t_states=t_states, t_rpm=t_rpm)
        io = _io(N.QsDynCtrlTrajJvpIO, states.shape[0], ptrs, control_timestep=dt)
        _call("qs_dyn_ctrl_traj_jvp", C.byref(P), C.byref(CP), C.byref(io), E, D, S, eff, device=states.device)
        return t_states, t_rpm

    @staticmethod
    def backward(ctx, g_states, g_rpm):
        _no_double_backward()
        saved = ctx.saved_tensors
        ins = dict(zip(CTRL_INS, saved[:9]))
        outs = dict(zip(("states", "rpm", "pid_states"), saved[9:]))
        P, CP, dt, E, D, S, eff = ctx.cfg
        T, n = ins["target_pos"].shape[0], E * D
        f64 = dict(dtype=torch.float64, device=ins["target_pos"].device)
        grads = dict(g_state0=torch.empty((13 * n,), **f64), g_pid0=torch.empty((9, n), **f64), g_target_pos=torch.empty((T, n, 3), **f64),
                     g_target_vel=torch.empty((n, 3), **f64), g_target_rpy=torch.empty((n, 3), **f64),
                     g_target_rpy_rates=torch.empty((n, 3), **f64), g_last_rpm=torch.empty((n, 4), **f64),
                     g_phys=torch.empty((n, 16), **f64), g_gains=torch.empty((n, 18), **f64))
        outs.update(g_states=g_states.to(torch.float64).contiguous(), g_rpm_out=g_rpm.to(torch.float64).contiguous(),
                    scratch=torch.empty((S, 13, n), **f64))
        io = _io(N.QsDynCtrlTrajIO, T, dict(ins, **outs, **grads), control_timestep=dt)
        _call(_entry("qs_dyn_ctrl_traj_vjp", eff), C.byref(P), C.byref(CP), C.byref(io), E, D, S, eff, device=ins["target_pos"].device)
        g = grads
        return (g["g_state0"], g["g_pid0"], g["g_target_pos"], g["g_target_vel"], g["g_target_rpy"], g["g_target_rpy_rates"],
                g["g_last_rpm"], g["g_phys"].view(E, D, 16).sum(dim=1), g["g_gains"].view(E, D, 18).sum(dim=1), None)


LQR_INS = ("state0", "last_rpm", "phys", "rpm_nom", "K", "z_nom")
PLAN_KEYS = ("rpm", "K", "z")                                                          # plan= keys, in sol's names


class DynLqrTrajectory(torch.autograd.Function):
    """(states [T, 13 N], rpm [T, N, 4]) = the T ticks of qs_dyn_lqr_traj from planes0 [13 N], with last_rpm [N, 4], the
    per-aviary rows [E, 16] and the plan rpm_nom [T_plan, N, 4], K [T_plan, N, 4, n_z], z_nom [T_plan, N, n_z], flown from plan
    tick tick0; backward = qs_dyn_lqr_traj_vjp, its per-drone row gradients summed over each aviary's drones (torch,
    deterministic), the plan's gradients zero on the ticks not flown.  `cfg` = (QsParams, E, D, substeps, effects, tick0, box),
    box = (lo, hi, per_tick) of the tracker (constants) or None.  The inputs may have any strides (the kernels get contiguous
    copies).  Double backward and forward mode (dual tensors) raise ValueError: the tracker loop has reverse mode only."""

    @staticmethod
    def _lqr_io(cfg, T, ptrs):
        """The QsDynLqrTrajIO of T ticks with the tensors of `ptrs` and the tracker's box"""
        P, E, D, S, eff, tick0, box = cfg
        lo, hi, per_tick = box if box is not None else (None, None, False)
        K = ptrs["K"]
        return _io(N.QsDynLqrTrajIO, T, dict(ptrs, lo=lo, hi=hi), n_z=K.shape[-1], T_plan=K.shape[0], tick0=tick0,
                   per_tick=int(per_tick))

    @staticmethod
    def forward(ctx, planes0, last_rpm, rows, rpm_nom, K, z_nom, cfg, T):
        ins = dict(zip(LQR_INS, (x.contiguous() for x in (planes0, last_rpm, rows, rpm_nom, K, z_nom))))
        if ins["rpm_nom"].data_ptr() % 32:                  # the kernel reads a drone's 4 nominal RPMs as one 32-byte access
            ins["rpm_nom"] = ins["rpm_nom"].clone()
        P, E, D, S, eff, tick0, box = cfg
        n = E * D
        f64 = dict(dtype=torch.float64, device=planes0.device)
        outs = dict(states=torch.empty((T, 13 * n), **f64), rpm=torch.empty((T, n, 4), **f64))
        _call("qs_dyn_lqr_traj", C.byref(P), C.byref(DynLqrTrajectory._lqr_io(cfg, T, dict(ins, **outs))), E, D, S, eff,
              device=planes0.device)
        ctx.save_for_backward(*ins.values(), *outs.values())
        ctx.cfg = cfg
        return outs["states"], outs["rpm"]

    @staticmethod
    def jvp(ctx, *tangents):
        raise ValueError("differentiable_rollout(controller=Tracker): the tracker loop has reverse mode only; forward-mode "
                         "(dual tensor) derivatives are not implemented for it")

    @staticmethod
    def backward(ctx, g_states, g_rpm):
        _no_double_backward()
        saved = ctx.saved_tensors
        ins = dict(zip(LQR_INS, saved[:6]))
        outs = dict(zip(("states", "rpm"), saved[6:]))
        P, E, D, S, eff, tick0, box = ctx.cfg
        T, n = outs["rpm"].shape[0], E * D
        f64 = dict(dtype=torch.float64, device=outs["rpm"].device)
        grads = dict(g_state0=torch.empty((13 * n,), **f64), g_last_rpm=torch.empty((n, 4), **f64), g_phys=torch.empty((n, 16), **f64),
                     g_rpm_nom=torch.zeros_like(ins["rpm_nom"]) if ctx.needs_input_grad[3] else None,
                     g_K=torch.zeros_like(ins["K"]) if ctx.needs_input_grad[4] else None,
                     g_z_nom=torch.zeros_like(ins["z_nom"]) if ctx.needs_input_grad[5] else None)
        ptrs = dict(ins, **outs, **grads, g_states=g_states.to(torch.float64).contiguous(),
                    g_rpm=None if g_rpm is None else g_rpm.to(torch.float64).contiguous(), scratch=torch.empty((S, 13, n), **f64))
        _call("qs_dyn_lqr_traj_vjp", C.byref(P), C.byref(DynLqrTrajectory._lqr_io(ctx.cfg, T, ptrs)), E, D, S, eff, device=outs["rpm"].device)
        g = grads
        return (g["g_state0"], g["g_last_rpm"], g["g_phys"].view(E, D, 16).sum(dim=1), g["g_rpm_nom"], g["g_K"], g["g_z_nom"], None,
                None)


def _tracker_inputs(env, trk, plan, state, last_rpm, phys, num_steps=None, **schedule):
    """The checked arguments of differentiable_rollout(controller=Tracker, plan=): (cfg, T, inputs), inputs = (planes0,
    last_rpm, rows, rpm_nom, K, z_nom) as DynLqrTrajectory takes them."""
    E, D, dev = env._E, env._D, env.device
    given = sorted(k for k, v in schedule.items() if v is not None)
    if given:
        raise ValueError("a Tracker flies its plan: %s do not apply (no waypoints, start, offset, targets, gains, pid_state or "
                         "control_timestep)" % ", ".join(given))
    T = trk.ticks(env, num_steps, last_rpm)
    plan = dict(plan or {})
    bad = set(plan) - set(PLAN_KEYS)
    if bad:
        raise ValueError("unknown plan keys %s (expected some of rpm, K, z)" % sorted(bad))
    shapes = dict(rpm=(trk.T, E, D, 4), K=(trk.T, E, D, 4, trk.nz), z=(trk.T, E, D, trk.nz))
    own = dict(rpm=trk.rpm_nom, K=trk.K, z=trk.z_nom)
    tens = [_tensor(plan[k], "plan[%r]" % k, shapes[k], dev).reshape(own[k].shape) if k in plan else own[k] for k in PLAN_KEYS]
    planes0, last_rpm, rows = _start_state(env, state, last_rpm, phys)
    cfg = (*dyn_cfg(env), trk.tick, trk.box)
    return cfg, T, (planes0, last_rpm, rows, *tens)


def _tracker_loop(env, trk, plan, state, last_rpm, phys, **schedule):
    E, D, dev = env._E, env._D, env.device
    cfg, T, ins = _tracker_inputs(env, trk, plan, state, last_rpm, phys, **schedule)
    with torch.cuda.device(dev):
        states, rpm = DynLqrTrajectory.apply(*ins, cfg, T)
    out = unpack_traj(states, T, E, D)
    out["rpm"] = rpm.reshape(T, E, D, 4)
    return out


def actor64(params, activation, obs, noise=None):
    """The raw action [..., out] of the MlpPolicy actor with float64 `params` = [W1, b1, ..., Wout, bout, log_std] on observation
    rows obs [..., in]: mean + exp(log_std) * noise (noise=None: the mean)."""
    act = torch.tanh if activation == "tanh" else torch.relu
    h = obs
    for k in range(0, len(params) - 3, 2):
        h = act(h @ params[k] + params[k + 1])
    raw = h @ params[-3] + params[-2]
    return raw if noise is None else raw + torch.exp(params[-1]) * noise


def actor64_jvp(params, t_params, activation, obs, noise=None, t_noise=None):
    """The tangent of actor64(params, activation, obs, noise) along t_params (None: zero) and t_noise (None: zero), obs held
    constant: one batched forward-mode pass written out (forward-mode AD cannot nest inside the jvp of an autograd.Function).
    ReLU passes the tangent where the unit is positive, as torch.relu's derivative does."""
    z = lambda t, x: torch.zeros_like(x) if t is None else t
    h, th = obs, None
    for k in range(0, len(params) - 3, 2):
        W, b = params[k], params[k + 1]
        pre = h @ W + b
        tz = h @ z(t_params[k], W) + z(t_params[k + 1], b) + (0.0 if th is None else th @ W)
        h = torch.tanh(pre) if activation == "tanh" else torch.relu(pre)
        th = tz * (1.0 - h * h) if activation == "tanh" else torch.where(h > 0, tz, torch.zeros_like(tz))
    W, b = params[-3], params[-2]
    t_raw = h @ z(t_params[-3], W) + z(t_params[-2], b) + th @ W
    if noise is not None:
        scale = torch.exp(params[-1])
        t_raw = t_raw + scale * (z(t_params[-1], params[-1]) * noise + z(t_noise, noise))
    return t_raw


def _policy_io(cls, cfg, T, theta, ptrs):
    """The QsDynPolicyTrajIO (or QsDynPolicyTrajJvpIO: `cls`) of PolicyTrajectory: the actor's layers from the float64
    parameters theta, the tensors of `ptrs`."""
    activation, B = cfg[2], cfg[3]
    io = _io(cls, T, dict(ptrs, log_std=theta[-1]), act_buffer_size=B, depth=len(theta) // 2 - 1,
             activation=N.MLP_TANH if activation == "tanh" else N.MLP_RELU, in_dim=theta[0].shape[0], out_dim=theta[-3].shape[1])
    for l in range(io.depth + 1):
        io.w[l], io.b[l] = theta[2 * l].data_ptr(), theta[2 * l + 1].data_ptr()
        if l < io.depth:
            io.width[l] = theta[2 * l].shape[1]
    return io


class PolicyTrajectory(torch.autograd.Function):
    """(states [T, 13 N], raw actions [T, N, A], obs [T, E, in]) = the T ticks of qs_dyn_policy_traj from planes0 [13 N] and the
    action buffer abuf [N, B, A], with last_rpm [N, 4], the per-aviary rows [E, 16], noise [T, E, out] (or None) and the actor's
    float64 parameters `theta` ([W1, b1, ..., Wout, bout, log_std]).  backward = qs_dyn_policy_traj_vjp, which carries the
    sequential dependency and returns g_raw, the cotangent of every raw action; the gradients of theta and noise are then one
    batched autograd pass of the actor over the T * E saved observation rows (deterministic, any architecture).  jvp
    (torch.autograd.forward_ad) = one batched forward-mode pass of the actor over the same rows for the tangent that theta and
    the noise add to each raw action (actor64_jvp), then qs_dyn_policy_traj_jvp.  obs is not differentiable.  `cfg` = (QsParams, act_type,
    activation, B, E, D, A, substeps, effects, T).  Double backward and tangents that require grad raise ValueError."""

    @staticmethod
    def _saved(ctx):
        """({state0, last_rpm, phys, action_buffer, noise (or None)}, {states, actions, obs}, theta) of the forward"""
        saved = list(ctx.saved_tensors)
        keys = ["state0", "last_rpm", "phys", "action_buffer"] + (["noise"] if ctx.has_noise else [])
        ins = dict(zip(keys, saved[:len(keys)]))
        ins.setdefault("noise", None)
        outs = dict(zip(("states", "actions", "obs"), saved[len(keys):len(keys) + 3]))
        return ins, outs, saved[len(keys) + 3:]

    @staticmethod
    def forward(ctx, planes0, last_rpm, rows, abuf, noise, cfg, *theta):
        theta = tuple(t.contiguous() for t in theta)
        ins = dict(state0=planes0.contiguous(), last_rpm=last_rpm.contiguous(), phys=rows.contiguous(), action_buffer=abuf.contiguous(),
                   noise=None if noise is None else noise.contiguous())
        P, act_type, activation, B, E, D, A, S, eff, T = cfg
        n = E * D
        f64 = dict(dtype=torch.float64, device=planes0.device)
        outs = dict(states=torch.empty((T, 13 * n), **f64), actions=torch.empty((T, n, A), **f64),
                    obs=torch.empty((T, E, theta[0].shape[0]), **f64))
        io = _policy_io(N.QsDynPolicyTrajIO, cfg, T, theta, dict(ins, **outs))
        _call("qs_dyn_policy_traj", C.byref(P), C.byref(io), act_type, E, D, S, eff, device=planes0.device)
        ctx.save_for_backward(*(x for x in ins.values() if x is not None), *outs.values(), *theta)
        ctx.save_for_forward(*(x for x in ins.values() if x is not None), *outs.values(), *theta)
        ctx.cfg, ctx.has_noise = cfg, noise is not None
        ctx.mark_non_differentiable(outs["obs"])
        return outs["states"], outs["actions"], outs["obs"]

    @staticmethod
    def jvp(ctx, t_planes0, t_last_rpm, t_rows, t_abuf, t_noise, _t_cfg, *t_theta):
        """Forward mode: the tangents (t_states [T, 13 N], t_actions [T, N, A]) along the inputs' tangents; obs has none.  The
        tangent theta and the noise add to raw action k, t_raw_in = J_theta t_theta + exp(log_std) (t_log_std noise + t_noise),
        is one batched forward-mode pass of the actor over the saved observations (actor64_jvp); qs_dyn_policy_traj_jvp carries
        the rest, linearising each tick at the forward's stored states.  A tangent that requires grad raises ValueError."""
        tangents = (t_planes0, t_last_rpm, t_rows, t_abuf, t_noise) + tuple(t_theta)
        if any(t is not None and t.requires_grad for t in tangents):
            raise ValueError("differentiable_rollout: a tangent that requires grad (reverse mode over forward mode) is not supported: "
                             "the JVP kernel has no derivative of its own")
        ins, outs, theta = PolicyTrajectory._saved(ctx)
        cfg = ctx.cfg
        P, act_type, activation, B, E, D, A, S, eff, T = cfg
        n = E * D
        f64 = lambda t: None if t is None else t.to(torch.float64).contiguous()
        t_raw_in = None
        t_eps = f64(t_noise) if ctx.has_noise else None
        if t_eps is not None or any(t is not None for t in t_theta):
            t_raw_in = actor64_jvp(theta, [f64(t) for t in t_theta], activation, outs["obs"], ins["noise"], t_eps).reshape(T, n, A).contiguous()
        t_phys = f64(t_rows)
        if t_phys is not None and t_phys.data_ptr() % 16:          # the kernel reads t_phys rows as 16-byte pairs
            t_phys = t_phys.clone()
        t_states, t_actions = torch.empty_like(outs["states"]), torch.empty_like(outs["actions"])
        ptrs = dict(ins, **outs, t_state0=f64(t_planes0), t_last_rpm=f64(t_last_rpm), t_phys=t_phys, t_action_buffer=f64(t_abuf),
                    t_raw_in=t_raw_in, t_states=t_states, t_actions=t_actions)
        io = _policy_io(N.QsDynPolicyTrajJvpIO, cfg, T, theta, ptrs)
        _call("qs_dyn_policy_traj_jvp", C.byref(P), C.byref(io), act_type, E, D, S, eff, device=t_states.device)
        return t_states, t_actions, None

    @staticmethod
    def backward(ctx, g_states, g_actions, _g_obs):
        _no_double_backward()
        ins, outs, theta = PolicyTrajectory._saved(ctx)
        cfg = ctx.cfg
        P, act_type, activation, B, E, D, A, S, eff, T = cfg
        n = E * D
        f64 = dict(dtype=torch.float64, device=outs["states"].device)
        grads = dict(g_raw=torch.empty((T, n, A), **f64), g_state0=torch.empty((13 * n,), **f64), g_last_rpm=torch.empty((n, 4), **f64),
                     g_phys=torch.empty((n, 16), **f64), g_action_buffer=torch.empty((n, B, A), **f64))
        outs.update(g_states=g_states.to(torch.float64).contiguous(), g_actions=g_actions.to(torch.float64).contiguous(),
                    scratch=torch.empty((S, 13, n), **f64))
        io = _policy_io(N.QsDynPolicyTrajIO, cfg, T, theta, dict(ins, **outs, **grads))
        _call("qs_dyn_policy_traj_vjp", C.byref(P), C.byref(io), act_type, E, D, S, eff, device=outs["states"].device)
        # the parameters' (and the noise's) gradients: raw[k, e] = actor(obs[k, e]) + exp(log_std) noise[k, e] with cotangent g_raw
        g_raw = grads["g_raw"].view(T, E, D * A)
        need = [j for j in range(len(theta)) if ctx.needs_input_grad[6 + j]]
        g_theta, g_noise = [None] * len(theta), None
        want_noise = ctx.has_noise and ctx.needs_input_grad[4]
        if need or want_noise:
            with torch.enable_grad():
                leaves = [t.detach().requires_grad_(j in need) for j, t in enumerate(theta)]
                eps = ins["noise"].detach().requires_grad_(True) if want_noise else ins["noise"]
                raw = actor64(leaves, activation, outs["obs"], eps)
                got = torch.autograd.grad(raw, [leaves[j] for j in need] + ([eps] if want_noise else []), g_raw, allow_unused=True)
            for j, g in zip(need, got):
                g_theta[j] = g
            if want_noise:
                g_noise = got[-1]
        return (grads["g_state0"], grads["g_last_rpm"], grads["g_phys"].view(E, D, 16).sum(dim=1), grads["g_action_buffer"], g_noise, None,
                *g_theta)


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


def _per_drone(x, name, width, E, D, dev, T=None):
    """An input of `width` values per drone as [E * D, width]: from [width] (every drone) or [E, D, width], and where T is given
    from [T, E, D, width] too, as [T, E * D, width].  Anything else raises ValueError naming `name`."""
    if isinstance(x, torch.Tensor) and x.dim() == 1:
        return _tensor(x, name, (width,), dev).expand(E * D, width)
    if T is not None and isinstance(x, torch.Tensor) and x.dim() == 4:
        if x.shape[0] != T:
            raise ValueError("%s has %d ticks but the horizon is T = %d" % (name, x.shape[0], T))
        return _tensor(x, name, (T, E, D, width), dev).reshape(T, E * D, width)
    return _tensor(x, name, (E, D, width), dev).reshape(E * D, width)


def _start_state(env, state, last_rpm, phys):
    """The planes [13 N] of the initial state, last_rpm [N, 4] and the per-aviary rows [E, 16] of differentiable_rollout."""
    from .params import PHYS_KEYS, physical_rows
    E, D, n, dev = env._E, env._D, env._N, env.device
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
    return planes0, last_rpm, rows


MAX_DW_DRONES = 128                  # downwash: whole aviaries per 128-thread CTA


def _check_downwash(env, policy, controller):
    """The refusals of differentiable_rollout(downwash=True)."""
    from .ilqr import Tracker
    if not env._effects & N.EFFECT_DW:
        raise ValueError("differentiable_rollout(downwash=True): the env has no downwash to differentiate (use PYB_DW or "
                         "PYB_GND_DRAG_DW, or leave downwash=False)")
    if env._EXTERNAL_DOWNWASH:
        raise ValueError("differentiable_rollout(downwash=True): the downwash of a formation sharded over devices is not available")
    if env._D > MAX_DW_DRONES:
        raise ValueError("differentiable_rollout(downwash=True): an aviary has at most %d drones, got %d" % (MAX_DW_DRONES, env._D))
    if policy is not None or isinstance(controller, Tracker):
        raise ValueError("differentiable_rollout(downwash=True) takes rpm= or controller=DSLPIDControl: the policy and tracker "
                         "loops have no downwash adjoint")


def _refuse_downwash(env, caller, derivative):
    if env._effects & N.EFFECT_DW or env._EXTERNAL_DOWNWASH:
        raise ValueError("%s does not support downwash: the pairwise term has no %s (use Physics.DYN, PYB, PYB_GND or PYB_DRAG)"
                         % (caller, derivative))


def _rpm_ticks(env, rpm):
    """T of an rpm [T, E, D, 4] float64 tensor on the env's device; anything else raises ValueError."""
    if not isinstance(rpm, torch.Tensor) or rpm.dim() != 4:
        raise ValueError("rpm must be a [T, %d, %d, 4] float64 CUDA tensor" % (env._E, env._D))
    T = rpm.shape[0]
    if T <= 0:
        raise ValueError("rpm must hold at least one tick")
    _tensor(rpm, "rpm", (T, env._E, env._D, 4), env.device)
    return T


def differentiable_rollout(env, rpm=None, controller=None, state=None, last_rpm=None, phys=None, policy=None, params=None, noise=None,
                           action_buffer=None, plan=None, downwash=False, **schedule):
    """BaseAviary.differentiable_rollout (see there)."""
    from .ilqr import Tracker
    if downwash:
        _check_downwash(env, policy, controller)
    else:
        _refuse_downwash(env, "differentiable_rollout()", "adjoint")
    if (rpm is not None) + (controller is not None) + (policy is not None) != 1:
        raise ValueError("differentiable_rollout() takes exactly one of rpm [T, E, D, 4] (open loop), controller= (closed loop) or "
                         "policy= (an MlpPolicy in the loop)")
    if plan is not None and not isinstance(controller, Tracker):
        raise ValueError("plan= is the plan of a tracker loop: it needs controller=ilqr.Tracker(sol), got %s"
                         % ("controller=%s" % type(controller).__name__ if controller is not None else
                            "policy=" if policy is not None else "rpm="))
    if policy is not None:
        given = sorted(k for k, v in schedule.items() if v is not None and k != "num_steps")
        if given:
            raise ValueError("%s apply to a controller rollout only" % ", ".join(given))
        return _policy_loop(env, policy, params, noise, action_buffer, schedule.get("num_steps"), state, last_rpm, phys)
    given = sorted(k for k, v in (("params", params), ("noise", noise), ("action_buffer", action_buffer)) if v is not None)
    if given:
        raise ValueError("%s apply to a policy rollout only" % ", ".join(given))
    if isinstance(controller, Tracker):
        return _tracker_loop(env, controller, plan, state, last_rpm, phys, **schedule)
    if controller is not None:
        return _closed_loop(env, controller, state, last_rpm, phys, **schedule)
    given = sorted(k for k, v in schedule.items() if v is not None)
    if given:
        raise ValueError("%s apply to a controller rollout only" % ", ".join(given))
    E, D, n, dev = env._E, env._D, env._N, env.device
    T = _rpm_ticks(env, rpm)
    planes0, last_rpm, rows = _start_state(env, state, last_rpm, phys)
    with torch.cuda.device(dev):
        states = DynTrajectory.apply(rpm.reshape(T, n, 4).contiguous(), planes0, last_rpm.contiguous(), rows.contiguous(), dyn_cfg(env))
    return unpack_traj(states, T, E, D)


def schedule_targets(waypoints, start, offset, T, E, D, dev):
    """target_pos [T, E * D, 3] of CtrlAviary.rollout's schedule: waypoints[(start[i] + k) % W][i or 0] + offset[i], built from
    gathers, expands and sums so that its backward is deterministic (every gather index is hit once per drone)."""
    n = E * D
    if not isinstance(waypoints, torch.Tensor):
        raise ValueError("waypoints must be a float64 tensor [W, 3] or [W, %d, %d, 3]" % (E, D))
    if waypoints.dim() == 2:
        W = waypoints.shape[0]
        wp = _tensor(waypoints, "waypoints", (W, 3), dev)[:, None, :].expand(W, n, 3)
    else:
        W = waypoints.shape[0] if waypoints.dim() == 4 else 0
        wp = _tensor(waypoints, "waypoints", (W, E, D, 3), dev).reshape(W, n, 3)
    if W == 0:
        raise ValueError("waypoints must hold at least one row")
    if start is None:
        st0 = torch.zeros((n,), dtype=torch.int64, device=dev)
    else:
        st0 = start if isinstance(start, torch.Tensor) else torch.as_tensor(start)
        if st0.dtype.is_floating_point or st0.dtype == torch.bool or st0.numel() not in (1, n):
            raise ValueError("start must be an integer or integers [%d, %d]" % (E, D))
        st0 = st0.to(device=dev, dtype=torch.int64).reshape(-1).expand(n)
    idx = torch.remainder(st0[None, :] + torch.arange(W, device=dev)[:, None], W)           # [W, n]: row of tick k' of drone i
    rot = torch.gather(wp, 0, idx[:, :, None].expand(W, n, 3))                               # [W, n, 3]: tick k' (k' < W)
    tpos = rot[:T] if T <= W else rot.repeat((T + W - 1) // W, 1, 1)[:T]
    if offset is not None:                  # no zero offset when there is none: -0.0 + 0.0 would change the sign of a zero target
        tpos = tpos + _per_drone(offset, "offset", 3, E, D, dev)
    return tpos


def _closed_loop_inputs(env, controller, state, last_rpm, phys, caller, derivative, waypoints=None, start=None, offset=None,
                        target_rpy=None, target_vel=None, target_rpy_rates=None, control_timestep=None, num_steps=None, gains=None,
                        pid_state=None):
    """The checked arguments of a closed-loop call (differentiable_rollout(controller=) or linearise(controller=)): (cfg, T,
    inputs), inputs = (planes0, pid0, target_pos, target_vel, target_rpy, target_rpy_rates, last_rpm, rows, gains) as
    DynCtrlTrajectory takes them.  `caller` / `derivative` name the call and its derivative in the MRAC refusal."""
    from .control.DSLPIDControl import DSLPIDControl
    from .control.MRAC import MRAC
    E, D, n, dev = env._E, env._D, env._N, env.device
    if isinstance(controller, MRAC):
        raise ValueError("%s has no %s of MRAC: pass a DSLPIDControl" % (caller, derivative))
    if not isinstance(controller, DSLPIDControl):
        raise ValueError("controller must be a DSLPIDControl, got %s" % type(controller).__name__)
    if controller.num_drones != n:
        raise ValueError("the controller must be a DSLPIDControl for the env's %d drones (num_drones=%d)" % (n, controller.num_drones))
    if torch.device(controller.device) != dev:
        raise ValueError("the controller's state is on %s, the env's on %s" % (controller.device, dev))
    if waypoints is None:
        raise ValueError("a controller rollout needs waypoints [W, 3] or [W, %d, %d, 3]" % (E, D))
    T = (waypoints.shape[0] if isinstance(waypoints, torch.Tensor) else 0) if num_steps is None else int(num_steps)
    if T <= 0:
        raise ValueError("num_steps must be > 0")
    tpos = schedule_targets(waypoints, start, offset, T, E, D, dev)
    tvel, trpy, trr = (torch.zeros((n, 3), dtype=torch.float64, device=dev) if x is None else _per_drone(x, k, 3, E, D, dev)
                       for x, k in ((target_vel, "target_vel"), (target_rpy, "target_rpy"), (target_rpy_rates, "target_rpy_rates")))
    CP = controller._P
    gains = dict(gains or {})
    bad = set(gains) - set(GAIN_KEYS)
    if bad:
        raise ValueError("unknown gains %s (expected some of %s)" % (sorted(bad), ", ".join(GAIN_KEYS)))
    cols = []
    for k, f in zip(GAIN_KEYS, ("pid_p_for", "pid_i_for", "pid_d_for", "pid_p_tor", "pid_i_tor", "pid_d_tor")):
        if k not in gains:
            cols.append(torch.tensor(list(getattr(CP, f)), dtype=torch.float64, device=dev).expand(E, 3))
        elif isinstance(gains[k], torch.Tensor) and gains[k].dim() == 1:
            cols.append(_tensor(gains[k], "gains[%r]" % k, (3,), dev).expand(E, 3))
        else:
            cols.append(_tensor(gains[k], "gains[%r]" % k, (E, 3), dev))
    table = torch.cat(cols, dim=1)
    pid_state = dict(pid_state or {})
    bad = set(pid_state) - set(PID_KEYS)
    if bad:
        raise ValueError("unknown pid_state keys %s (expected some of %s)" % (sorted(bad), ", ".join(PID_KEYS)))
    pid0 = torch.cat([_tensor(pid_state[k], "pid_state[%r]" % k, (E, D, 3), dev).reshape(n, 3).t() if k in pid_state
                      else controller._state[3 * j:3 * j + 3].detach().clone() for j, k in enumerate(PID_KEYS)])
    planes0, last_rpm, rows = _start_state(env, state, last_rpm, phys)
    dt = float(env.CTRL_TIMESTEP if control_timestep is None else control_timestep)
    cfg = (env._P, CP, dt, E, D, env.PYB_STEPS_PER_CTRL, env._effects)
    return cfg, T, (planes0, pid0, tpos, tvel, trpy, trr, last_rpm, rows, table)


def _closed_loop(env, controller, state, last_rpm, phys, **schedule):
    E, D, dev = env._E, env._D, env.device
    cfg, T, ins = _closed_loop_inputs(env, controller, state, last_rpm, phys, "differentiable_rollout()", "adjoint", **schedule)
    with torch.cuda.device(dev):
        states, rpm = DynCtrlTrajectory.apply(*ins, cfg)
    out = unpack_traj(states, T, E, D)
    out["rpm"] = rpm.reshape(T, E, D, 4)
    return out


def _policy_inputs(env, policy, params, noise, action_buffer, num_steps, state, last_rpm, phys, caller):
    """The checked arguments of a policy-loop call (differentiable_rollout(policy=) or linearise(policy=), named by `caller`):
    (cfg, inputs, theta), inputs = (planes0, last_rpm, rows, action_buffer, noise) as PolicyTrajectory takes them."""
    from .policy import MlpPolicy
    E, D, n, dev = env._E, env._D, env._N, env.device
    if not isinstance(policy, MlpPolicy):
        raise ValueError("policy must be an MlpPolicy, got %s" % type(policy).__name__)
    act_type = env._act_type()
    if act_type not in (N.ACT_RPM, N.ACT_ONE_D_RPM):
        raise ValueError("%s supports ActionType.RPM and ONE_D_RPM: PID, VEL and ONE_D_PID run the embedded "
                         "DSLPID controller inside the policy loop, which has no adjoint yet" % caller)
    A, B, od = env._A, env._B, env._obs_dim
    if B == 0:
        raise ValueError("%s needs an action buffer: ctrl_freq=%d gives ACTION_BUFFER_SIZE = 0" % (caller, env.CTRL_FREQ))
    if policy.in_dim != D * od or policy.out_dim != D * A:
        raise ValueError("policy must map %d inputs to %d outputs, not %d to %d" % (D * od, D * A, policy.in_dim, policy.out_dim))
    if torch.device(policy.device) != dev:
        raise ValueError("the policy's weights are on %s, the env's state on %s" % (policy.device, dev))
    shapes = [tuple(t.shape) for wb in policy.actor for t in wb] + [tuple(policy.log_std.shape)]
    if params is None:
        theta = [t.detach().double() for wb in policy.actor for t in wb] + [policy.log_std.detach().double()]
    else:
        theta = list(params)
        if len(theta) != len(shapes):
            raise ValueError("params must be the %d tensors of policy.parameters64() (weight and bias per actor layer, then log_std), "
                             "got %d" % (len(shapes), len(theta)))
        for j, (t, sh) in enumerate(zip(theta, shapes)):
            _tensor(t, "params[%d]" % j, sh, dev)
    if noise is None:
        if num_steps is None:
            raise ValueError("a policy rollout needs num_steps (or noise [T, %d, %d])" % (E, D * A))
        T = int(num_steps)
    else:
        T = noise.shape[0] if isinstance(noise, torch.Tensor) and noise.dim() == 3 else 0
        if num_steps is not None and int(num_steps) != T:
            raise ValueError("noise must be [num_steps, %d, %d]" % (E, D * A))
        _tensor(noise, "noise", (T, E, D * A), dev)
    if T <= 0:
        raise ValueError("num_steps must be > 0")
    if action_buffer is None:
        action_buffer = env._by_id(env._obs_buf[env._cur][:, 12:]).detach().double().reshape(n, B, A)
    else:
        action_buffer = _tensor(action_buffer, "action_buffer", (E, D, B, A), dev).reshape(n, B, A)
    planes0, last_rpm, rows = _start_state(env, state, last_rpm, phys)
    cfg = (env._P, act_type, policy.activation, B, E, D, A, env.PYB_STEPS_PER_CTRL, env._effects, T)
    return cfg, (planes0, last_rpm, rows, action_buffer, noise), theta


def _policy_out(env, cfg, states, actions, obs):
    """{pos, quat, vel, rpy_rates, actions, obs} of a policy loop as differentiable_rollout(policy=) returns them"""
    E, D = env._E, env._D
    T, A, od = cfg[9], cfg[6], env._obs_dim
    out = unpack_traj(states, T, E, D)
    out["actions"] = actions.reshape(T, E, D, A)
    out["obs"] = obs.reshape(T, E, D, od)
    return out


def _policy_loop(env, policy, params, noise, action_buffer, num_steps, state, last_rpm, phys):
    cfg, ins, theta = _policy_inputs(env, policy, params, noise, action_buffer, num_steps, state, last_rpm, phys,
                                     "differentiable_rollout(policy=)")
    with torch.cuda.device(env.device):
        states, actions, obs = PolicyTrajectory.apply(*ins, cfg, *theta)
    return _policy_out(env, cfg, states, actions, obs)


def tick_jacobians(cfg, rpm, planes0, last_rpm, rows):
    """(states [T, 13 N], jac [T, N, 13, C]) of qs_dyn_traj and qs_dyn_tick_jac from dense rpm [T, N, 4], planes0 [13 N],
    last_rpm [N, 4] and rows [E, 16]; `cfg` = (QsParams, E, D, substeps, effects), C = 17 or 21 with drag (include/quadsim.h)."""
    P, E, D, S, eff = cfg
    states = _dyn_traj(cfg, rpm, planes0, last_rpm, rows)
    jac = torch.empty((rpm.shape[0], E * D, 13, 21 if eff & N.EFFECT_DRAG else 17), dtype=torch.float64, device=rpm.device)
    io = _io(N.QsDynTrajJvpIO, rpm.shape[0], dict(_traj_ptrs(rpm, planes0, last_rpm, rows, states), jac=jac))
    _call("qs_dyn_tick_jac", C.byref(P), C.byref(io), E, D, S, eff, device=rpm.device)
    return states, jac


def ctrl_tick_jacobians(cfg, ins):
    """({states, rpm, pid_states} of qs_dyn_ctrl_traj, jac [T, N, 26, C]) of qs_dyn_ctrl_tick_jac from the dense inputs `ins`
    (CTRL_INS); `cfg` as DynCtrlTrajectory's, C = 25 or 29 with drag (include/quadsim.h)."""
    P, CP, dt, E, D, S, eff = cfg
    outs = _dyn_ctrl_traj(cfg, ins)
    T, dev = ins["target_pos"].shape[0], ins["target_pos"].device
    jac = torch.empty((T, E * D, 26, 29 if eff & N.EFFECT_DRAG else 25), dtype=torch.float64, device=dev)
    io = _io(N.QsDynCtrlTrajJvpIO, T, dict(ins, **outs, jac=jac), control_timestep=dt)
    _call("qs_dyn_ctrl_tick_jac", C.byref(P), C.byref(CP), C.byref(io), E, D, S, eff, device=dev)
    return outs, jac


def _linearise_closed_loop(env, controller, state, last_rpm, phys, **schedule):
    E, D, dev = env._E, env._D, env.device
    with torch.no_grad():
        cfg, T, ins = _closed_loop_inputs(env, controller, state, last_rpm, phys, "linearise()", "tangent", **schedule)
        with torch.cuda.device(dev):
            outs, jac = ctrl_tick_jacobians(cfg, dict(zip(CTRL_INS, (x.detach().contiguous() for x in ins))))
    out = unpack_traj(outs["states"], T, E, D)
    out["rpm"] = outs["rpm"].view(T, E, D, 4)
    out["pid_state"] = outs["pid_states"].transpose(1, 2).reshape(T, E, D, 9)
    nz = 26 if cfg[6] & N.EFFECT_DRAG else 22
    jac = jac.view(T, E, D, 26, jac.shape[-1])
    out["A"], out["B"] = jac[..., :nz, :nz], jac[..., :nz, nz:]
    out["K"], out["K_target"] = jac[..., 22:26, :nz], jac[..., 22:26, nz:]
    return out


def policy_tick_jacobians(cfg, ins, theta):
    """({states, actions, obs} of qs_dyn_policy_traj, jac [T, E, R, R]) of qs_dyn_policy_tick_jac from the dense inputs `ins`
    (planes0, last_rpm, rows, action_buffer, noise) and the float64 parameters theta; `cfg` as PolicyTrajectory's, R = n_z + D A
    (include/quadsim.h)."""
    P, act_type, activation, B, E, D, A, S, eff, T = cfg
    planes0 = ins[0]
    n, dev = E * D, planes0.device
    f64 = dict(dtype=torch.float64, device=dev)
    outs = dict(states=torch.empty((T, 13 * n), **f64), actions=torch.empty((T, n, A), **f64), obs=torch.empty((T, E, theta[0].shape[0]), **f64))
    ptrs = dict(zip(("state0", "last_rpm", "phys", "action_buffer", "noise"), ins), **outs)
    io = _policy_io(N.QsDynPolicyTrajIO, cfg, T, theta, ptrs)
    _call("qs_dyn_policy_traj", C.byref(P), C.byref(io), act_type, E, D, S, eff, device=dev)
    R = D * (16 + B * A + (4 if eff & N.EFFECT_DRAG else 0)) + D * A
    jac = torch.empty((T, E, R, R), **f64)
    io = _policy_io(N.QsDynPolicyTrajJvpIO, cfg, T, theta, dict(ptrs, jac=jac))
    _call("qs_dyn_policy_tick_jac", C.byref(P), C.byref(io), act_type, E, D, S, eff, device=dev)
    return outs, jac


def _linearise_policy(env, policy, params, noise, action_buffer, num_steps, state, last_rpm, phys):
    with torch.no_grad():
        cfg, ins, theta = _policy_inputs(env, policy, params, noise, action_buffer, num_steps, state, last_rpm, phys, "linearise(policy=)")
        dense = lambda x: None if x is None else x.detach().contiguous()
        with torch.cuda.device(env.device):
            outs, jac = policy_tick_jacobians(cfg, [dense(x) for x in ins], [dense(t) for t in theta])
    out = _policy_out(env, cfg, outs["states"], outs["actions"], outs["obs"])
    nz = jac.shape[-1] - env._D * env._A
    out["A"], out["B"], out["K"] = jac[..., :nz, :nz], jac[..., :nz, nz:], jac[..., nz:, :nz]
    return out


def linearise(env, rpm=None, controller=None, state=None, last_rpm=None, phys=None, policy=None, params=None, noise=None,
              action_buffer=None, **schedule):
    """BaseAviary.linearise (see there)."""
    _refuse_downwash(env, "linearise()", "tangent")
    if policy is not None:
        if rpm is not None or controller is not None:
            raise ValueError("linearise() takes exactly one of rpm [T, E, D, 4] (open loop), controller= (closed loop) or policy= (an "
                             "MlpPolicy in the loop)")
        given = sorted(k for k, v in schedule.items() if v is not None and k != "num_steps")
        if given:
            raise ValueError("%s apply to a controller linearisation only" % ", ".join(given))
        return _linearise_policy(env, policy, params, noise, action_buffer, schedule.get("num_steps"), state, last_rpm, phys)
    given = sorted(k for k, v in (("params", params), ("noise", noise), ("action_buffer", action_buffer)) if v is not None)
    if given:
        raise ValueError("%s apply to a policy linearisation only" % ", ".join(given))
    if (rpm is not None) + (controller is not None) != 1:
        raise ValueError("linearise() takes exactly one of rpm [T, E, D, 4] (open loop) or controller= (closed loop)")
    if controller is not None:
        return _linearise_closed_loop(env, controller, state, last_rpm, phys, **schedule)
    given = sorted(k for k, v in schedule.items() if v is not None)
    if given:
        raise ValueError("%s apply to a controller linearisation only" % ", ".join(given))
    E, D, n = env._E, env._D, env._N
    T = _rpm_ticks(env, rpm)
    with torch.no_grad():
        planes0, last_rpm, rows = _start_state(env, state, last_rpm, phys)
        states, jac = tick_jacobians(dyn_cfg(env), *(x.detach().contiguous() for x in (rpm.reshape(T, n, 4), planes0, last_rpm, rows)))
    cols = jac.shape[-1]
    out = unpack_traj(states, T, E, D)
    jac = jac.view(T, E, D, 13, cols)
    out["A"], out["B"] = jac[..., :13], jac[..., 13:17]
    if cols == 21:
        out["B_last"] = jac[..., 17:21]
    return out
