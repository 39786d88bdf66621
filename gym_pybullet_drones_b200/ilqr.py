"""Batched iLQR of raw-RPM trajectories of Physics.DYN (DESIGN.md 4.5.1): Gauss-Newton DDP for every drone at once, one
independent problem per drone, on the per-tick Jacobians of qs_dyn_tick_jac and the kernels qs_ilqr_backward,
qs_ilqr_line_search and qs_ilqr_commit (include/quadsim.h), or with rpm_bounds their control-limited variants qs_ilqr_box_*.
BaseAviary.ilqr is the public entry point; Problem holds one solve's device buffers and runs its steps, so that each step can
also be called on its own.  Tracker flies a solution's LQR tracker in CtrlAviary.rollout() (qs_ctrl_rollout_lqr)."""
import ctypes as C

import torch

from . import _native as N
from .diff import STATE_KEYS, _call, _io, _refuse_downwash, _start_state, _tensor, _traj_ptrs, unpack_states

ALPHAS = tuple(2.0 ** -j for j in range(10))               # the line search's step sizes, largest first
DEFAULT_Q = (1.0,) * 3 + (1.0,) * 4 + (0.1,) * 3 + (0.01,) * 3   # pos, quat, vel, rpy_rates
DEFAULT_R = (1e-2,) * 4                                    # on the command relative to HOVER_RPM
FINAL_SCALE = 100.0                                        # Q_final = FINAL_SCALE * Q by default
HOVER_TARGET = {"quat": (0.0, 0.0, 0.0, 1.0), "vel": (0.0, 0.0, 0.0), "rpy_rates": (0.0, 0.0, 0.0)}


def pack_traj(pos, quat, vel, w):
    """[T, N, 3], [T, N, 4], [T, N, 3], [T, N, 3] -> [T, 13 N]: pack_state of every tick."""
    T = pos.shape[0]
    return torch.cat([torch.cat([pos, w[..., 0:1]], -1).reshape(T, -1), quat.reshape(T, -1),
                      torch.cat([vel, w[..., 1:2]], -1).reshape(T, -1), w[..., 2]], dim=1)


def _target_ticks(target):
    """The time axes of the [T, E, D, k] entries of `target` (a set)."""
    return {x.shape[0] for x in target.values() if isinstance(x, torch.Tensor) and x.dim() == 4}


def _target_part(x, name, width, T, E, D, dev):
    """target[name] as [T, E * D, width]: from [width], [E, D, width] or [T, E, D, width]."""
    if not isinstance(x, torch.Tensor):
        raise ValueError("%s must be a float64 tensor [%d], [%d, %d, %d] or [%d, %d, %d, %d]" % (name, width, E, D, width, T, E, D, width))
    if x.dim() == 1:
        return _tensor(x, name, (width,), dev).expand(T, E * D, width)
    if x.dim() == 3:
        return _tensor(x, name, (E, D, width), dev).reshape(1, E * D, width).expand(T, E * D, width)
    return _tensor(x, name, (T, E, D, width), dev).reshape(T, E * D, width)


def _bound(x, name, T, E, D, dev):
    """One side of rpm_bounds as ([E * D, 4] or [T, E * D, 4], has a time axis): from [4], [E, D, 4] or [T, E, D, 4]."""
    if not isinstance(x, torch.Tensor) or x.dim() not in (1, 3, 4):
        raise ValueError("%s must be a float64 CUDA tensor [4], [%d, %d, 4] or [%d, %d, %d, 4]" % (name, E, D, T, E, D))
    if x.dim() == 1:
        return _tensor(x, name, (4,), dev).expand(E * D, 4), False
    if x.dim() == 3:
        return _tensor(x, name, (E, D, 4), dev).reshape(E * D, 4), False
    if x.shape[0] != T:
        raise ValueError("ilqr(): %s has %d ticks but the horizon is T = %d" % (name, x.shape[0], T))
    return _tensor(x, name, (T, E, D, 4), dev).reshape(T, E * D, 4), True


def _rpm_box(rpm_bounds, rows, T, E, D, dev):
    """rpm_bounds as (lo, hi, per_tick, ok): lo and hi [N, 4] (per_tick False) or [T, N, 4] (True), contiguous, and ok a 0-dim
    bool tensor (not read here) that is true when no bound is NaN, lo <= hi and 0 <= lo, hi <= MAX_RPM of each drone's row."""
    n = E * D
    max_rpm = rows[:, 13].reshape(E, 1, 1).expand(E, D, 4).reshape(n, 4)
    if isinstance(rpm_bounds, str) and rpm_bounds == "motor":
        lo = torch.zeros((n, 4), dtype=torch.float64, device=dev)
        return lo, max_rpm.contiguous(), False, torch.ones((), dtype=torch.bool, device=dev)
    if not isinstance(rpm_bounds, (tuple, list)) or len(rpm_bounds) != 2:
        raise ValueError("rpm_bounds must be None, 'motor' or a pair (lo, hi) of float64 CUDA tensors in raw RPM")
    lo, lo_t = _bound(rpm_bounds[0], "rpm_bounds[0] (lo)", T, E, D, dev)
    hi, hi_t = _bound(rpm_bounds[1], "rpm_bounds[1] (hi)", T, E, D, dev)
    per_tick = lo_t or hi_t
    if per_tick:
        lo, hi = lo.expand(T, n, 4), hi.expand(T, n, 4)
    lo, hi = lo.detach().contiguous(), hi.detach().contiguous()
    ok = ~(torch.isnan(lo).any() | torch.isnan(hi).any()) & (lo <= hi).all() & (lo >= 0).all() & (hi <= max_rpm).all()
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


class Problem:
    """The device buffers of one batched iLQR solve and its steps.  Arguments as BaseAviary.ilqr; `alphas` are the line
    search's step sizes (1 to 16).  `feedback = False` runs the line search and the commit with K = 0 (an open-loop line
    search along k).  With `rpm_bounds` every step runs the control-limited kernels qs_ilqr_box_*, the guess is projected into
    the box before the first nominal, and `active` holds the held rotors of the last backward pass."""

    def __init__(self, env, target, num_steps=None, rpm=None, Q=None, R=None, Q_final=None, rpm_ref=None, state=None, last_rpm=None,
                 phys=None, alphas=ALPHAS, rpm_bounds=None):
        _refuse_downwash(env, "ilqr()", "Jacobian")
        E, D, n, dev = env._E, env._D, env._N, env.device
        if not isinstance(target, dict) or "pos" not in target:
            raise ValueError("target must be a dict with 'pos' ([3], [%d, %d, 3] or [T, %d, %d, 3]) and optionally quat, vel and "
                             "rpy_rates" % (E, D, E, D))
        bad = set(target) - {k for k, _ in STATE_KEYS}
        if bad:
            raise ValueError("unknown target keys %s (expected pos, quat, vel, rpy_rates)" % sorted(bad))
        # T from num_steps, the target's time axis and rpm: every one that is given must agree
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
            raise ValueError("ilqr() needs the horizon: num_steps, a target with a time axis [T, %d, %d, k] or rpm [T, %d, %d, 4]"
                             % (E, D, E, D))
        ticks = set().union(*given.values())
        if len(ticks) != 1:
            raise ValueError("ilqr(): the horizons of %s disagree (%s)" % (", ".join(sorted(given)), sorted(ticks)))
        T = ticks.pop()
        if T <= 0:
            raise ValueError("ilqr(): the horizon T must be > 0, got %d" % T)
        alphas = tuple(float(a) for a in alphas)
        if not 1 <= len(alphas) <= 16:
            raise ValueError("alphas must hold 1 to 16 step sizes")
        with torch.no_grad():
            planes0, last_rpm, rows = _start_state(env, state, last_rpm, phys)
            parts = [_target_part(target[k], "target[%r]" % k, w, T, E, D, dev) if k in target
                     else _target_part(torch.tensor(HOVER_TARGET[k], dtype=torch.float64, device=dev), k, w, T, E, D, dev)
                     for k, w in STATE_KEYS]
            self.targets = pack_traj(*parts).contiguous()
            q = _weight(Q, "Q", DEFAULT_Q, E, dev)
            qf = FINAL_SCALE * q if Q_final is None else _weight(Q_final, "Q_final", DEFAULT_Q, E, dev)
            r = _weight(R, "R", DEFAULT_R, E, dev)
            self.weights = torch.cat([q, qf, r], dim=1).contiguous()
            w_ok = torch.isfinite(self.weights).all() & (self.weights >= 0).all() & (r > 0).all()
            if rpm_bounds is None:
                # the one synchronisation of a solve: the weights' values
                if not bool(w_ok.item()):
                    raise ValueError("ilqr(): Q and Q_final must be finite and >= 0, R finite and > 0")
                self.box = None
            else:
                lo, hi, per_tick, b_ok = _rpm_box(rpm_bounds, rows, T, E, D, dev)
                # the one synchronisation of a solve: the weights' and the bounds' values
                w_ok, b_ok = torch.stack([w_ok, b_ok]).tolist()
                if not w_ok:
                    raise ValueError("ilqr(): Q and Q_final must be finite and >= 0, R finite and > 0")
                if not b_ok:
                    raise ValueError("ilqr(): rpm_bounds must not be NaN and must satisfy 0 <= lo <= hi <= MAX_RPM of each "
                                     "drone's row")
                self.box = (lo, hi, per_tick)
            hover = rows[:, 12].reshape(E, 1, 1).expand(E, D, 4)
            if rpm_ref is None:
                ref = hover.reshape(n, 4)
            elif isinstance(rpm_ref, torch.Tensor) and rpm_ref.dim() == 1:
                ref = _tensor(rpm_ref, "rpm_ref", (4,), dev).expand(n, 4)
            else:
                ref = _tensor(rpm_ref, "rpm_ref", (E, D, 4), dev).reshape(n, 4)
            self.rpm_ref = ref.detach().contiguous()
            if rpm is None:
                rpm = hover.reshape(1, n, 4).expand(T, n, 4)
            else:
                rpm = _tensor(rpm, "rpm", (T, E, D, 4), dev).reshape(T, n, 4)
            self.rpm = rpm.detach().clone().contiguous()
            if self.box is not None:                             # the guess projected into the box
                lo, hi, per_tick = self.box
                torch.minimum(torch.maximum(self.rpm, lo), hi, out=self.rpm)
        self.env_shape = (E, D)
        self.planes0, self.last_rpm, self.rows = planes0.contiguous(), last_rpm.detach().contiguous(), rows.contiguous()
        self.cfg = (env._P, E, D, env.PYB_STEPS_PER_CTRL, env._effects)
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
        T, n = self.T, self.n
        out = {k: v.reshape(T, E, D, v.shape[-1]) for k, v in unpack_states(self.states, n).items()}
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
    if isinstance(iters, bool) or not isinstance(iters, int) or iters < 0:
        raise ValueError("iters must be an integer >= 0, got %r" % (iters,))
    p = Problem(env, target, num_steps=num_steps, rpm=rpm, Q=Q, R=R, Q_final=Q_final, rpm_ref=rpm_ref, state=state, last_rpm=last_rpm,
                phys=phys, rpm_bounds=rpm_bounds)
    return solve(p, iters)


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
            self.box = None
            if not (rpm_bounds is None or (isinstance(rpm_bounds, str) and rpm_bounds == "motor")):
                if not isinstance(rpm_bounds, (tuple, list)) or len(rpm_bounds) != 2:
                    raise ValueError("rpm_bounds must be None, 'motor' or a pair (lo, hi) of float64 CUDA tensors in raw RPM")
                lo, lo_t = _bound(rpm_bounds[0], "rpm_bounds[0] (lo)", T, E, D, dev)
                hi, hi_t = _bound(rpm_bounds[1], "rpm_bounds[1] (hi)", T, E, D, dev)
                per_tick = lo_t or hi_t
                if per_tick:
                    lo, hi = lo.expand(T, n, 4), hi.expand(T, n, 4)
                lo, hi = lo.detach().clone().contiguous(), hi.detach().clone().contiguous()      # owned, 32-byte aligned
                if not bool((~(torch.isnan(lo).any() | torch.isnan(hi).any()) & (lo <= hi).all()).item()):
                    raise ValueError("Tracker: rpm_bounds must not be NaN and must satisfy lo <= hi")
                self.box = (lo, hi, per_tick)
        self.T, self.env_shape, self.nz, self.device = T, (E, D), nz, dev
        self.tick = 0

    def _io(self, tick):
        """The QsLqrRolloutIO of a launch from plan tick `tick`"""
        lo, hi, per_tick = self.box if self.box is not None else (None, None, False)
        return N.QsLqrRolloutIO(K=self.K.data_ptr(), z_nom=self.z_nom.data_ptr(), rpm_nom=self.rpm_nom.data_ptr(),
                                lo=None if lo is None else lo.data_ptr(), hi=None if hi is None else hi.data_ptr(),
                                per_tick=int(per_tick), n_z=self.nz, T_plan=self.T, tick0=tick)
