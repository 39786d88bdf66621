"""Batched iLQR of raw-RPM trajectories of Physics.DYN (DESIGN.md 4.5.1): Gauss-Newton DDP for every drone at once, one
independent problem per drone, on the per-tick Jacobians of qs_dyn_tick_jac and the kernels qs_ilqr_backward,
qs_ilqr_line_search and qs_ilqr_commit (include/quadsim.h), or with rpm_bounds their control-limited variants qs_ilqr_box_*.
BaseAviary.ilqr is the public entry point; Problem holds one solve's device buffers and runs its steps, so that each step can
also be called on its own.  Tracker flies a solution's LQR tracker in CtrlAviary.rollout() (qs_ctrl_rollout_lqr).
differentiable_ilqr (BaseAviary.differentiable_ilqr) is the same solve with gradients of the solution: IlqrSolution, whose
backward is one adjoint LQR pass on the device (qs_ilqr_adjoint, qs_ilqr_adjoint_rollout)."""
import contextlib
import ctypes as C

import torch

from . import _native as N
from .diff import (STATE_KEYS, _call, _dyn_traj_vjp, _io, _per_drone, _refuse_downwash, _start_state, _tensor, _traj_ptrs, dyn_cfg,
                   pack_state, unpack_states, unpack_traj)

ALPHAS = tuple(2.0 ** -j for j in range(10))               # the line search's step sizes, largest first
DEFAULT_Q = (1.0,) * 3 + (1.0,) * 4 + (0.1,) * 3 + (0.01,) * 3   # pos, quat, vel, rpy_rates
DEFAULT_R = (1e-2,) * 4                                    # on the command relative to HOVER_RPM
FINAL_SCALE = 100.0                                        # Q_final = FINAL_SCALE * Q by default
HOVER_TARGET = {"quat": (0.0, 0.0, 0.0, 1.0), "vel": (0.0, 0.0, 0.0), "rpy_rates": (0.0, 0.0, 0.0)}
# one aviary's row of the packed weights [E, 30] (QsIlqrIO.weights): [Q | Q_final | R]
W_Q, W_Q_FINAL, W_R = slice(0, 13), slice(13, 26), slice(26, 30)


def pack_traj(pos, quat, vel, w):
    """[T, N, 3], [T, N, 4], [T, N, 3], [T, N, 3] -> [T, 13 N]: pack_state of every tick."""
    T = pos.shape[0]
    return torch.cat([torch.cat([pos, w[..., 0:1]], -1).reshape(T, -1), quat.reshape(T, -1),
                      torch.cat([vel, w[..., 1:2]], -1).reshape(T, -1), w[..., 2]], dim=1)


def _target_ticks(target):
    """The time axes of the [T, E, D, k] entries of `target` (a set)."""
    return {x.shape[0] for x in target.values() if isinstance(x, torch.Tensor) and x.dim() == 4}


def _rpm_box(rpm_bounds, T, E, D, dev, max_rpm=None):
    """rpm_bounds (None, "motor" or a pair (lo, hi) of [4], [E, D, 4] or [T, E, D, 4]) as None or (lo, hi, per_tick, ok): owned
    contiguous lo, hi [N, 4] or, per tick, [T, N, 4], and a 0-dim bool ok (not read here): no NaN, lo <= hi and, with each drone's
    max_rpm [N, 4], 0 <= lo, hi <= max_rpm.  "motor" is the box [0, max_rpm], or None (the env's clip only) without max_rpm."""
    if rpm_bounds is None or (isinstance(rpm_bounds, str) and rpm_bounds == "motor" and max_rpm is None):
        return None
    if isinstance(rpm_bounds, str) and rpm_bounds == "motor":
        return torch.zeros_like(max_rpm), max_rpm.clone(), False, torch.ones((), dtype=torch.bool, device=dev)
    if not isinstance(rpm_bounds, (tuple, list)) or len(rpm_bounds) != 2:
        raise ValueError("rpm_bounds must be None, 'motor' or a pair (lo, hi) of float64 CUDA tensors in raw RPM")
    lo = _per_drone(rpm_bounds[0], "rpm_bounds[0] (lo)", 4, E, D, dev, T)
    hi = _per_drone(rpm_bounds[1], "rpm_bounds[1] (hi)", 4, E, D, dev, T)
    per_tick = lo.dim() == 3 or hi.dim() == 3
    if per_tick:
        lo, hi = lo.expand(T, E * D, 4), hi.expand(T, E * D, 4)
    lo, hi = lo.detach().clone(memory_format=torch.contiguous_format), hi.detach().clone(memory_format=torch.contiguous_format)
    ok = ~(torch.isnan(lo).any() | torch.isnan(hi).any()) & (lo <= hi).all()
    if max_rpm is not None:
        ok = ok & (lo >= 0).all() & (hi <= max_rpm).all()
    return lo, hi, per_tick, ok


def _clampd(v, lo, hi):
    """qs::clampd elementwise: v < lo ? lo : (v > hi ? hi : v)"""
    return torch.where(v < lo, lo, torch.where(v > hi, hi, v))


def _weight(x, name, default, E, dev):
    """A weight vector as [E, width]: from [width] or [E, width]; None -> `default`."""
    width = len(default)
    if x is None:
        return torch.tensor(default, dtype=torch.float64, device=dev).expand(E, width)
    if isinstance(x, torch.Tensor) and x.dim() == 1:
        return _tensor(x, name, (width,), dev).expand(E, width)
    return _tensor(x, name, (E, width), dev)


def check_iters(iters):
    """A planner's iteration count (ilqr(), differentiable_ilqr(), mppi()): an integer >= 0, else ValueError."""
    if isinstance(iters, bool) or not isinstance(iters, int) or iters < 0:
        raise ValueError("iters must be an integer >= 0, got %r" % (iters,))


def horizon(env, target, num_steps, rpm, what):
    """T of a planner's call (ilqr(), mppi()) from num_steps, the target's time axis and rpm, every one that is given agreeing,
    after checking the target's keys; anything else raises ValueError naming `what`."""
    E, D = env._E, env._D
    if not isinstance(target, dict) or "pos" not in target:
        raise ValueError("target must be a dict with 'pos' ([3], [%d, %d, 3] or [T, %d, %d, 3]) and optionally quat, vel and "
                         "rpy_rates" % (E, D, E, D))
    bad = set(target) - {k for k, _ in STATE_KEYS}
    if bad:
        raise ValueError("unknown target keys %s (expected pos, quat, vel, rpy_rates)" % sorted(bad))
    given = {}
    if num_steps is not None:
        given["num_steps"] = {int(num_steps)}
    if _target_ticks(target):
        given["target"] = _target_ticks(target)
    if rpm is not None:
        if not isinstance(rpm, torch.Tensor) or rpm.dim() != 4:
            raise ValueError("rpm must be a [T, %d, %d, 4] float64 CUDA tensor" % (E, D))
        given["rpm"] = {rpm.shape[0]}
    if not given:
        raise ValueError("%s needs the horizon: num_steps, a target with a time axis [T, %d, %d, k] or rpm [T, %d, %d, 4]"
                         % (what, E, D, E, D))
    ticks = set().union(*given.values())
    if len(ticks) != 1:
        raise ValueError("%s: the horizons of %s disagree (%s)" % (what, ", ".join(sorted(given)), sorted(ticks)))
    T = ticks.pop()
    if T <= 0:
        raise ValueError("%s: the horizon T must be > 0, got %d" % (what, T))
    return T


def pack_inputs(env, target, T, rpm, Q, R, Q_final, rpm_ref, state, last_rpm, phys, rpm_bounds, what, checks=(), graph=False):
    """The packed inputs of a planner's problem over T ticks (arguments as BaseAviary.ilqr), as a dict: targets [T, 13 N],
    weights [E, 30], rpm_ref [N, 4], the guess rpm [T, N, 4] (owned, projected into the box), box None or (lo, hi, per_tick),
    planes0 [13 N], last_rpm [N, 4], rows [E, 16] and graph (with `graph`: the recorded (targets, weights, rpm_ref, planes0,
    last_rpm, rows), else None).  The values of the weights, of the bounds and of every (ok, message) of `checks` (0-dim bool
    tensors) are read in one synchronisation; the first that fails raises ValueError."""
    E, D, n, dev = env._E, env._D, env._N, env.device
    out = {}
    with contextlib.nullcontext() if graph else torch.no_grad():
        planes0, last_rpm, rows = _start_state(env, state, last_rpm, phys)
        parts = [_per_drone(target[k], "target[%r]" % k, w, E, D, dev, T) if k in target
                 else _per_drone(torch.tensor(HOVER_TARGET[k], dtype=torch.float64, device=dev), k, w, E, D, dev)
                 for k, w in STATE_KEYS]
        parts = [x if x.dim() == 3 else x.expand(T, n, x.shape[-1]) for x in parts]
        targets = pack_traj(*parts)
        out["targets"] = targets.detach().contiguous()
        q = _weight(Q, "Q", DEFAULT_Q, E, dev)
        qf = FINAL_SCALE * q if Q_final is None else _weight(Q_final, "Q_final", DEFAULT_Q, E, dev)
        r = _weight(R, "R", DEFAULT_R, E, dev)
        weights = torch.cat([q, qf, r], dim=1)                 # W_Q, W_Q_FINAL, W_R
        out["weights"] = weights.detach().contiguous()
        oks = [(torch.isfinite(out["weights"]).all() & (out["weights"] >= 0).all() & (r > 0).all(),
                "%s: Q and Q_final must be finite and >= 0, R finite and > 0" % what)]
        max_rpm = rows[:, 13].reshape(E, 1, 1).expand(E, D, 4).reshape(n, 4)
        box = _rpm_box(rpm_bounds, T, E, D, dev, max_rpm)
        if box is not None:
            oks.append((box[3], "%s: rpm_bounds must not be NaN and must satisfy 0 <= lo <= hi <= MAX_RPM of each drone's row" % what))
        oks += list(checks)
        # the one synchronisation of a solve: the weights', the bounds' and the checks' values
        vals = [bool(oks[0][0].item())] if len(oks) == 1 else torch.stack([ok for ok, _ in oks]).tolist()
        for v, (_, msg) in zip(vals, oks):
            if not v:
                raise ValueError(msg)
        out["box"] = None if box is None else box[:3]                # "motor": MAX_RPM is a constant
        hover = rows[:, 12].reshape(E, 1, 1).expand(E, D, 4)
        ref = hover.reshape(n, 4) if rpm_ref is None else _per_drone(rpm_ref, "rpm_ref", 4, E, D, dev)
        out["rpm_ref"] = ref.detach().contiguous()
        if rpm is None:
            rpm = hover.reshape(1, n, 4).expand(T, n, 4)
        else:
            rpm = _tensor(rpm, "rpm", (T, E, D, 4), dev).reshape(T, n, 4)
        out["rpm"] = rpm.detach().clone().contiguous()
        if out["box"] is not None:                           # the guess projected into the box
            lo, hi, per_tick = out["box"]
            torch.minimum(torch.maximum(out["rpm"], lo), hi, out=out["rpm"])
    out["planes0"], out["last_rpm"], out["rows"] = planes0, last_rpm, rows
    out["graph"] = (targets, weights, ref, planes0, last_rpm, rows) if graph else None
    return out


class Problem:
    """The device buffers of one batched iLQR solve and its steps.  Arguments as BaseAviary.ilqr; `alphas` are the line
    search's step sizes (1 to 16).  `feedback = False` runs the line search and the commit with K = 0 (an open-loop line
    search along k).  With `rpm_bounds` every step runs the control-limited kernels qs_ilqr_box_*, the guess is projected into
    the box before the first nominal, and `active` holds the held rotors of the last backward pass.  With `graph` the inputs
    are packed with autograd recording (the solve's buffers stay detached) and `graph` holds the recorded packed (targets, weights,
    rpm_ref, planes0, last_rpm, rows): the inputs of IlqrSolution."""

    def __init__(self, env, target, num_steps=None, rpm=None, Q=None, R=None, Q_final=None, rpm_ref=None, state=None, last_rpm=None,
                 phys=None, alphas=ALPHAS, rpm_bounds=None, graph=False):
        _refuse_downwash(env, "ilqr()", "Jacobian")
        E, D, n, dev = env._E, env._D, env._N, env.device
        T = horizon(env, target, num_steps, rpm, "ilqr()")
        alphas = tuple(float(a) for a in alphas)
        if not 1 <= len(alphas) <= 16:
            raise ValueError("alphas must hold 1 to 16 step sizes")
        pk = pack_inputs(env, target, T, rpm, Q, R, Q_final, rpm_ref, state, last_rpm, phys, rpm_bounds, "ilqr()", graph=graph)
        self.targets, self.weights, self.rpm_ref, self.rpm, self.box = pk["targets"], pk["weights"], pk["rpm_ref"], pk["rpm"], pk["box"]
        planes0, last_rpm, rows = pk["planes0"], pk["last_rpm"], pk["rows"]
        self.env_shape = (E, D)
        self.graph = pk["graph"]
        self.planes0, self.last_rpm, self.rows = planes0.detach().contiguous(), last_rpm.detach().contiguous(), rows.detach().contiguous()
        self.cfg = dyn_cfg(env)
        self.T, self.n, self.dev = T, n, dev
        self.nz = 17 if env._effects & N.EFFECT_DRAG else 13
        f64 = dict(dtype=torch.float64, device=dev)
        self.alphas = torch.tensor(alphas, **f64)
        self.states = torch.empty((T, 13 * n), **f64)
        self.jac = torch.empty((T, n, 13, 21 if self.nz == 17 else 17), **f64)
        self.K = torch.zeros((T, n, 4, self.nz), **f64)
        self.k = torch.zeros((T, n, 4), **f64)
        self.dV = torch.zeros((n, 2), **f64)
        self.J = torch.empty((len(alphas), n), **f64)
        self.mu = torch.zeros((n,), **f64)
        self.status = torch.zeros((n,), dtype=torch.int32, device=dev)
        self.converged = torch.zeros((n,), dtype=torch.uint8, device=dev)
        self.active = None if self.box is None else torch.zeros((T, n, 4), dtype=torch.int8, device=dev)
        self.feedback = True

    def _ilqr(self, name, alpha=None, **ptrs):
        P, E, D, S, eff = self.cfg
        alpha = self.alphas if alpha is None else alpha
        base = dict(jac=self.jac, state0=self.planes0, last_rpm=self.last_rpm, phys=self.rows, targets=self.targets, weights=self.weights,
                    rpm_ref=self.rpm_ref, alpha=alpha, states=self.states, rpm=self.rpm, mu=self.mu,
                    K=self.K if self.feedback or name == "qs_ilqr_backward" else None, k=self.k, dV=self.dV, J=self.J, status=self.status,
                    converged=self.converged)
        base.update(ptrs)
        io = _io(N.QsIlqrIO, self.T, base, n_alpha=alpha.numel())
        if self.box is not None:
            lo, hi, per_tick = self.box
            io = N.QsIlqrBoxIO(base=io, rpm_lo=lo.data_ptr(), rpm_hi=hi.data_ptr(), per_tick=int(per_tick),
                               active=None if self.active is None else self.active.data_ptr())
            name = name.replace("qs_ilqr_", "qs_ilqr_box_")
        _call(name, C.byref(P), C.byref(io), E, D, S, eff, device=self.dev)

    def nominal(self):
        """states = qs_dyn_traj(rpm)"""
        P, E, D, S, eff = self.cfg
        io = _io(N.QsDynTrajIO, self.T, _traj_ptrs(self.rpm, self.planes0, self.last_rpm, self.rows, self.states))
        _call("qs_dyn_traj", C.byref(P), C.byref(io), E, D, S, eff, device=self.dev)

    def jacobians(self):
        """jac = qs_dyn_tick_jac at the nominal (states, rpm)"""
        P, E, D, S, eff = self.cfg
        io = _io(N.QsDynTrajJvpIO, self.T, dict(_traj_ptrs(self.rpm, self.planes0, self.last_rpm, self.rows, self.states), jac=self.jac))
        _call("qs_dyn_tick_jac", C.byref(P), C.byref(io), E, D, S, eff, device=self.dev)

    def backward(self):
        """K, k, dV, status and mu of qs_ilqr_backward at jac"""
        self._ilqr("qs_ilqr_backward")

    def line_search(self, alpha=None, out=None):
        """J(alpha) [n_alpha, N] of qs_ilqr_line_search (alpha: a float64 tensor, default the Problem's step sizes)"""
        self._ilqr("qs_ilqr_line_search", alpha=alpha, J=self.J if out is None else out)
        return self.J if out is None else out

    def cost(self, out):
        """out [N] = J of the nominal: the line search at alpha = 0 without gains, the nominal's own rollout"""
        self._ilqr("qs_ilqr_line_search", alpha=torch.zeros((1,), dtype=torch.float64, device=self.dev), J=out, K=None, k=None,
                   status=None, converged=None)

    def commit(self, cost_in, cost_out):
        """qs_ilqr_commit from the line search's J: the nominal's cost cost_in [N], the new one into cost_out [N]"""
        self._ilqr("qs_ilqr_commit", cost_in=cost_in, cost_out=cost_out)

    def result(self, cost):
        E, D = self.env_shape
        T = self.T
        out = unpack_traj(self.states, T, E, D)
        out["rpm"] = self.rpm.view(T, E, D, 4)
        out["K"] = self.K.view(T, E, D, 4, self.nz)
        out["z"] = self.loop_states().view(T, E, D, self.nz)
        out["k"] = self.k.view(T, E, D, 4)
        out["cost"] = cost.view(cost.shape[0], E, D)
        out["mu"] = self.mu.view(E, D)
        out["converged"] = self.converged.view(E, D).bool()
        if self.active is not None:
            out["active"] = self.active.view(T, E, D, 4)
        return out


    def loop_states(self):
        """z_nom [T, N, n_z]: the state before each tick in drone_vec's order (px py pz qx qy qz qw vx vy vz wx wy wz), tick 0 the
        start, and with drag the clipped RPMs of the tick before (last_rpm at tick 0): what the rollouts difference against"""
        T, n = self.T, self.n
        x = unpack_states(torch.cat([self.planes0.view(1, -1), self.states[:-1]]), n)
        z = [x[k] for k, _ in STATE_KEYS]
        if self.nz == 17:
            E, D = self.env_shape
            mr = self.rows[:, 13].reshape(E, 1, 1).expand(E, D, 4).reshape(1, n, 4)
            z.append(torch.cat([self.last_rpm.view(1, n, 4), _clampd(self.rpm[:-1], torch.zeros_like(mr), mr)]))
        return torch.cat(z, dim=-1)


def solve(p, iters):
    """Runs `iters` iterations of Problem p and returns BaseAviary.ilqr's result.  Before the loop the nominal is qs_dyn_traj(rpm)
    and its cost row 0; each iteration is the line search and the commit along the gains of the last backward pass, then the
    Jacobians and the backward pass at the new nominal, so the returned K and k are always those of the returned trajectory.
    Nothing is read back to the host."""
    with torch.no_grad(), torch.cuda.device(p.dev):
        cost = torch.empty((iters + 1, p.n), dtype=torch.float64, device=p.dev)
        p.nominal()
        p.cost(cost[0])
        p.jacobians()
        p.backward()
        for it in range(iters):
            p.line_search()
            p.commit(cost[it], cost[it + 1])
            p.jacobians()
            p.backward()
    return p.result(cost)


def ilqr(env, target, num_steps=None, rpm=None, Q=None, R=None, Q_final=None, rpm_ref=None, iters=20, state=None, last_rpm=None, phys=None,
         rpm_bounds=None):
    """BaseAviary.ilqr (see there)."""
    check_iters(iters)
    p = Problem(env, target, num_steps=num_steps, rpm=rpm, Q=Q, R=R, Q_final=Q_final, rpm_ref=rpm_ref, state=state, last_rpm=last_rpm,
                phys=phys, rpm_bounds=rpm_bounds)
    return solve(p, iters)


def adjoint(p, g_states, g_rpm):
    """The adjoint LQR of Problem p's solution (DESIGN.md 4.5.1 "Gradients of the solution") for the cotangents g_states
    [T, 13 N] and g_rpm [T, N, 4] (either None: zeros): qs_dyn_tick_jac at (p.rpm, p.states) into a buffer freed on return, then
    qs_ilqr_adjoint and qs_ilqr_adjoint_rollout, with p.active as the held set when p has bounds.  Returns (w [T, N, 4],
    dx [T, 13 N], K [T, N, 4, n_z], k [T, N, 4], status [N] int32); w and dx are NaN on drones with status 1."""
    P, E, D, S, eff = p.cfg
    T, n, dev = p.T, p.n, p.dev
    f64 = dict(dtype=torch.float64, device=dev)
    with torch.no_grad(), torch.cuda.device(dev):
        p.jac = torch.empty((T, n, 13, 21 if p.nz == 17 else 17), **f64)
        try:
            p.jacobians()
            out = dict(K=torch.empty((T, n, 4, p.nz), **f64), k=torch.empty((T, n, 4), **f64),
                       status=torch.empty((n,), dtype=torch.int32, device=dev), w=torch.empty((T, n, 4), **f64),
                       dx=torch.empty((T, 13 * n), **f64))
            g_states = torch.zeros((T, 13 * n), **f64) if g_states is None else g_states.to(torch.float64).contiguous()
            g_rpm = None if g_rpm is None else g_rpm.to(torch.float64).reshape(T, n, 4).contiguous()
            io = _io(N.QsIlqrAdjointIO, T, dict(jac=p.jac, rpm=p.rpm, phys=p.rows, weights=p.weights, active=p.active,
                                                g_states=g_states, g_rpm=g_rpm, **out))
            for name in ("qs_ilqr_adjoint", "qs_ilqr_adjoint_rollout"):
                _call(name, C.byref(P), C.byref(io), E, D, S, eff, device=dev)
        finally:
            p.jac = None
    return out["w"], out["dx"], out["K"], out["k"], out["status"]


def state_weights(weights, E, D, T):
    """W [T, 13 N] in the planes layout of the states: each aviary's Q for ticks < T - 1 and Q_final for the last, from the
    packed weights [E, 30]."""
    n = E * D
    planes = lambda q: pack_state(q[:, 0:3], q[:, 3:7], q[:, 7:10], q[:, 10:13])
    q = weights[:, W_Q].repeat_interleave(D, dim=0)
    qf = weights[:, W_Q_FINAL].repeat_interleave(D, dim=0)
    return torch.cat([planes(q).reshape(1, 13 * n).expand(T - 1, 13 * n), planes(qf).reshape(1, 13 * n)])


def _refuse_forward_ad(xs):
    from torch.autograd import forward_ad
    if any(x is not None and forward_ad.unpack_dual(x).tangent is not None for x in xs):
        raise ValueError("differentiable_ilqr() is reverse mode only: forward-mode AD (dual tensors) is not supported")


class IlqrSolution(torch.autograd.Function):
    """(states [T, 13 N], rpm [T, N, 4]) of solve(p, iters) as a function of the packed inputs of Problem p built with
    graph=True: targets [T, 13 N], weights [E, 30], rpm_ref [N, 4], planes0 [13 N], last_rpm [N, 4] and rows [E, 16] (p's own
    detached buffers are what the kernels read).  `out` receives the whole result of solve().  The forward frees p's Jacobian
    buffer; the backward recomputes it once at the solution (adjoint()), so nothing of size T N 13 C is held in between.

    Backward, with w and dx the adjoint LQR's solution for the cotangents: the cost-side inputs (targets, weights, rpm_ref, the
    rows through HOVER_RPM) get the gradient of the surrogate
        s = -sum_k [W_k (X*_k - r_k) . dx_k + Rt (U*_k - u_ref) . w_k]
    (X*, U*, dx and w constant) by torch autograd, and the dynamics-side inputs (planes0, last_rpm, rows) qs_dyn_traj_vjp at the
    solution with the cotangent g_X - W dx.  Double backward and forward-mode AD raise ValueError."""

    @staticmethod
    def forward(ctx, targets, weights, rpm_ref, planes0, last_rpm, rows, p, iters, out):
        out.update(solve(p, iters))
        states, rpm = p.states, p.rpm
        # the outputs live on ctx through save_for_backward only: p keeps no reference to them (no cycle through the graph)
        p.states = p.rpm = p.jac = None
        ctx.save_for_backward(states, rpm)
        ctx.p = p
        return states, rpm

    @staticmethod
    def jvp(ctx, *tangents):
        raise ValueError("differentiable_ilqr() is reverse mode only: forward-mode AD (dual tensors) is not supported")

    @staticmethod
    def backward(ctx, g_states, g_rpm):
        if torch.is_grad_enabled():
            raise ValueError("differentiable_ilqr(): double backward (create_graph=True) is not supported: the adjoint LQR has no "
                             "derivative of its own")
        p = ctx.p
        states, rpm = ctx.saved_tensors
        E, D = p.env_shape
        T, n = p.T, p.n
        p.states, p.rpm = states, rpm
        try:
            w, dx, _, _, _ = adjoint(p, g_states, g_rpm)
        finally:
            p.states = p.rpm = None
        need = ctx.needs_input_grad
        W = state_weights(p.weights, E, D, T)
        grads = [None] * 6
        # cost side: the surrogate s(theta), by autograd over detached leaves
        cost_ins = [j for j in (0, 1, 2, 5) if need[j]]
        if cost_ins:
            tg, wt, ref, rows = (x.detach().requires_grad_(j in cost_ins)
                                 for j, x in ((0, p.targets), (1, p.weights), (2, p.rpm_ref), (5, p.rows)))
            with torch.enable_grad():
                Rt = (wt[:, W_R] / (rows[:, 12:13] * rows[:, 12:13])).repeat_interleave(D, dim=0)
                s = -((state_weights(wt, E, D, T) * (states - tg) * dx).sum() + (Rt * (rpm - ref) * w).sum())
                got = torch.autograd.grad(s, [x for j, x in zip((0, 1, 2, 5), (tg, wt, ref, rows)) if j in cost_ins])
            for j, g in zip(cost_ins, got):
                grads[j] = g
        # dynamics side: one VJP with the direct cotangent g_X and the Gauss-Newton implicit term -W dx
        if need[3] or need[4] or need[5]:
            cot = -(W * dx) if g_states is None else g_states - W * dx
            _, g0, glast, grows = _dyn_traj_vjp(p.cfg, rpm, p.planes0, p.last_rpm, p.rows, states, cot)
            grads[3], grads[4] = g0, glast
            grads[5] = grows if grads[5] is None else grads[5] + grows
        return (*grads, None, None, None)


def differentiable_ilqr(env, target, num_steps=None, rpm=None, Q=None, R=None, Q_final=None, rpm_ref=None, iters=20, state=None,
                        last_rpm=None, phys=None, rpm_bounds=None):
    """BaseAviary.differentiable_ilqr (see there)."""
    _refuse_downwash(env, "differentiable_ilqr()", "Jacobian")
    check_iters(iters)
    if isinstance(rpm_bounds, (tuple, list)) and any(isinstance(b, torch.Tensor) and b.requires_grad for b in rpm_bounds):
        raise ValueError("differentiable_ilqr(): rpm_bounds are constants: a bound tensor must not require grad (detach it)")
    p = Problem(env, target, num_steps=num_steps, rpm=rpm, Q=Q, R=R, Q_final=Q_final, rpm_ref=rpm_ref, state=state, last_rpm=last_rpm,
                phys=phys, rpm_bounds=rpm_bounds, graph=True)
    _refuse_forward_ad(p.graph)
    out = {}
    states, rpm_out = IlqrSolution.apply(*p.graph, p, iters, out)
    E, D = p.env_shape
    sol = unpack_traj(states, p.T, E, D)
    sol["rpm"] = rpm_out.view(p.T, E, D, 4)
    for k in ("K", "z", "k", "cost", "mu", "converged", "active"):
        if k in out:
            sol[k] = out[k]
    return sol


class Tracker:
    """The time-varying LQR tracker of an ilqr() solution, flown by CtrlAviary.rollout(controller=Tracker(sol)) in one launch
    (qs_ctrl_rollout_lqr, DESIGN.md 4.1e).  Plan tick p of drone i applies
        u = rpm[p] + K[p] (z - z[p]),   then clamp(u, lo[p], hi[p]) with rpm_bounds,   then the env's clip to [0, MAX_RPM]
    where z is the drone's state before the tick in drone_vec's order, with n_z = 17 followed by the RPMs the env applied at the tick
    before (its last_clipped_action), and z[p], rpm[p], K[p] are sol's.  From the solve's own start, on the plant it planned on,
    every tick reproduces sol's trajectory bit for bit (z - z[p] = 0).  The plant may differ from the plan: any Physics mode
    (downwash up to 128 drones per aviary) and any set_physical_params table; the tracker runs the plan's n_z whatever the
    plant's effects.  The result of ilqr() does not record the control rate: flying a plan at a rate other than the env's
    CTRL_FREQ it was solved at is the caller's error and is not detected.

    sol: the result of BaseAviary.ilqr (its rpm, K and z; float64 CUDA tensors of one device).  The plan is copied once (ilqr's
    layout is the kernel's), so later changes to sol do not reach the tracker.  rpm_bounds: None (default) or "motor" (the env's own
    clip only), or the pair (lo, hi) the plan was solved with, each [4], [E, D, 4] or [T, E, D, 4] float64 on sol's device
    (NaN or lo > hi raise ValueError).

    tick: the plan tick of the next rollout's first tick, 0 at construction.  Each rollout of R ticks advances it by R, so calls
    of R and T - R ticks fly the plan as one call of T ticks, bit for bit; the caller may set it.

    sol's K is the gain of the solve's last backward pass at each drone's final regularisation: K = -(Quu + mu diag(Quu))^-1 Qux,
    about 1 / (1 + mu) of the unregularised gain.  A drone whose last steps were rejected ends with a large mu (1e3 to 1e5 is
    common after 30 iterations) and its tracker barely acts.  To fly with the unregularised gains at the returned trajectory,
    solve through Problem and recompute them at mu = 0 (Quu is positive definite for R > 0):
        p = Problem(env, target, ...); sol = solve(p, iters); p.mu.zero_(); p.backward(); sol = p.result(sol["cost"])

    Gains are not screened on the device (that would synchronise every call).  For a drone whose last backward pass failed
    (an exhausted restart ladder, e.g. mu = +inf), K at tick t holds the gains of the last attempt that factorised tick t: the
    pass runs from tick T - 1 down and every attempt, the failing ones included, writes the ticks above the one where its
    factorisation failed, at its own (largest) mu.  A tick that no attempt of any pass reached holds 0 (sol's K starts at zero);
    with mu = +inf no attempt factorises any tick, so K is what earlier passes left.  The tracker applies those gains as they
    are.  A non-finite gain gives a NaN command, which the clip does not
    remove: that drone's state becomes NaN, the others are unaffected."""

    def __init__(self, sol, rpm_bounds=None):
        if not isinstance(sol, dict) or not all(isinstance(sol.get(k), torch.Tensor) for k in ("rpm", "K", "z")):
            raise ValueError("Tracker(sol): sol must be the result of ilqr(), with tensors rpm, K and z")
        rpm, K, z = sol["rpm"], sol["K"], sol["z"]
        if rpm.dim() != 4 or rpm.shape[-1] != 4 or rpm.shape[0] <= 0 or not rpm.is_cuda:
            raise ValueError("Tracker(sol): sol['rpm'] must be a [T, E, D, 4] float64 CUDA tensor")
        T, E, D = rpm.shape[:3]
        dev = rpm.device
        nz = K.shape[-1] if K.dim() == 5 else -1
        if nz not in (13, 17):
            raise ValueError("Tracker(sol): sol['K'] must be [%d, %d, %d, 4, n_z] with n_z 13 or 17" % (T, E, D))
        _tensor(rpm, "sol['rpm']", (T, E, D, 4), dev)
        _tensor(K, "sol['K']", (T, E, D, 4, nz), dev)
        _tensor(z, "sol['z']", (T, E, D, nz), dev)
        n = E * D
        with torch.no_grad():
            # owned, C-contiguous copies whatever sol's strides (clone alone keeps a permuted tensor's strides)
            dense = dict(memory_format=torch.contiguous_format)
            self.K = K.detach().reshape(T, n, 4, nz).clone(**dense)                     # [T][N][4][n_z]
            self.z_nom = z.detach().reshape(T, n, nz).clone(**dense)                    # [T][N][n_z]
            self.rpm_nom = rpm.detach().reshape(T, n, 4).clone(**dense)                 # [T][N][4]: one 32-byte load per drone
            box = _rpm_box(rpm_bounds, T, E, D, dev)                                  # owned, 32-byte aligned
            if box is not None and not bool(box[3].item()):
                raise ValueError("Tracker: rpm_bounds must not be NaN and must satisfy lo <= hi")
            self.box = None if box is None else box[:3]
        self.T, self.env_shape, self.nz, self.device = T, (E, D), nz, dev
        self.tick = 0

    def _io(self, tick):
        """The QsLqrRolloutIO of a launch from plan tick `tick`"""
        lo, hi, per_tick = self.box if self.box is not None else (None, None, False)
        return N.QsLqrRolloutIO(K=self.K.data_ptr(), z_nom=self.z_nom.data_ptr(), rpm_nom=self.rpm_nom.data_ptr(),
                                lo=None if lo is None else lo.data_ptr(), hi=None if hi is None else hi.data_ptr(),
                                per_tick=int(per_tick), n_z=self.nz, T_plan=self.T, tick0=tick)

    def ticks(self, env, num_steps=None, last_rpm=None):
        """The ticks of a rollout of `env` from plan tick self.tick (num_steps, or the rest of the plan), after checking this plan
        against env; `last_rpm` (differentiable_rollout()'s) stands in for env's last_clipped_action for an n_z = 17 plan."""
        E, D = env._E, env._D
        if self.env_shape != (E, D):
            raise ValueError("the Tracker's plan is for %d x %d drones, the env has %d x %d" % (*self.env_shape, E, D))
        if self.device != env.device:
            raise ValueError("the Tracker's plan is on %s, the env's state on %s" % (self.device, env.device))
        if isinstance(self.tick, bool) or not isinstance(self.tick, int) or self.tick < 0:
            raise ValueError("Tracker.tick must be an integer >= 0, got %r" % (self.tick,))
        T = self.T - self.tick if num_steps is None else int(num_steps)
        if num_steps is not None and T <= 0:
            raise ValueError("num_steps must be > 0")
        if T <= 0 or self.tick + T > self.T:
            raise ValueError("the Tracker's plan has %d ticks: ticks [%d, %d) do not fit" % (self.T, self.tick, self.tick + T))
        if env._order is not None:
            raise ValueError("a Tracker indexes drones by id: not available on a formation reordered by reorder_by_morton()")
        if self.nz == 17 and last_rpm is None and not env._track_last_action:
            raise ValueError("an n_z = 17 plan (solved with drag) needs the RPMs applied before tick 0: the env's last_clipped_action, "
                             "which this env does not keep (differentiable_rollout() also takes last_rpm=)")
        return T
