"""Sampling-based trajectory optimisation (MPPI, model predictive path integral) of raw-RPM trajectories for every Physics mode of
the DYN family, downwash included (DESIGN.md 4.5.2), on the kernels qs_mppi_sample, qs_mppi_update and qs_mppi_commit
(include/quadsim.h).  The problem, its cost J and its checks are ilqr()'s (ilqr.horizon, ilqr.pack_inputs).  BaseAviary.mppi
is the public entry point."""
import ctypes as C
import math
import numbers

import torch

from . import _native as N
from .diff import MAX_DW_DRONES, _call, _io, dyn_cfg, unpack_traj
from .ilqr import check_iters, horizon, pack_inputs

MAX_SAMPLES = 1024


def _sigma(sigma, E, dev):
    """sigma as an owned [E] float64 tensor and its check (None for a Python number, checked here; else a 0-dim bool tensor)."""
    if isinstance(sigma, numbers.Real) and not isinstance(sigma, bool):
        if not (math.isfinite(sigma) and sigma > 0):
            raise ValueError("mppi(): sigma must be finite and > 0, got %r" % (sigma,))
        return torch.full((E,), float(sigma), dtype=torch.float64, device=dev), None
    if not isinstance(sigma, torch.Tensor) or sigma.dtype != torch.float64 or sigma.device != dev or \
            tuple(sigma.shape) not in ((), (E,)):
        raise ValueError("mppi(): sigma must be a number or a float64 tensor of shape () or [%d] on %s" % (E, dev))
    s = sigma.detach().expand(E).clone()
    return s, torch.isfinite(s).all() & (s > 0).all()


def _check_scalars(env, samples, temperature, seed):
    if isinstance(samples, bool) or not isinstance(samples, int) or not 2 <= samples <= MAX_SAMPLES:
        raise ValueError("mppi(): samples must be an integer in [2, %d], got %r" % (MAX_SAMPLES, samples))
    if isinstance(temperature, bool) or not isinstance(temperature, numbers.Real) or not (math.isfinite(temperature) and temperature > 0):
        raise ValueError("mppi(): temperature must be finite and > 0, got %r" % (temperature,))
    if isinstance(seed, bool) or not isinstance(seed, int) or not 0 <= seed < 2 ** 64:
        raise ValueError("mppi(): seed must be an integer in [0, 2^64), got %r" % (seed,))
    if env._EXTERNAL_DOWNWASH:
        raise ValueError("mppi(): the downwash of a formation sharded over devices is not available (plan one device's aviaries)")
    if env._effects & N.EFFECT_DW:
        if env._order is not None:
            raise ValueError("mppi(): with downwash the pair sum runs in storage order: not available on a formation reordered by "
                             "reorder_by_morton()")
        if env._D > MAX_DW_DRONES:
            raise ValueError("mppi(): with downwash an aviary has at most %d drones, got %d" % (MAX_DW_DRONES, env._D))


class Mppi:
    """The device buffers of one mppi() call and its launches (each can also be called on its own): sample(it), update(it),
    commit(it, cost_out) and nominal(cost_out).  Arguments as BaseAviary.mppi."""

    def __init__(self, env, target, num_steps=None, rpm=None, Q=None, R=None, Q_final=None, rpm_ref=None, samples=64, sigma=0.02,
                 temperature=0.1, seed=0, state=None, last_rpm=None, phys=None, rpm_bounds=None):
        _check_scalars(env, samples, temperature, seed)
        E, D, n, dev = env._E, env._D, env._N, env.device
        T = horizon(env, target, num_steps, rpm, "mppi()")
        self.sigma, s_ok = _sigma(sigma, E, dev)
        checks = [] if s_ok is None else [(s_ok, "mppi(): sigma must be finite and > 0")]
        pk = pack_inputs(env, target, T, rpm, Q, R, Q_final, rpm_ref, state, last_rpm, phys, rpm_bounds, "mppi()", checks=checks)
        self.targets, self.weights, self.rpm_ref, self.rpm, self.box = pk["targets"], pk["weights"], pk["rpm_ref"], pk["rpm"], pk["box"]
        self.planes0, self.last_rpm = pk["planes0"].contiguous(), pk["last_rpm"].contiguous()
        self.rows = pk["rows"].contiguous()
        self.cfg = dyn_cfg(env)
        self.T, self.n, self.dev, self.env_shape = T, n, dev, (E, D)
        self.K, self.seed, self.temperature = samples, seed, float(temperature)
        f64 = dict(dtype=torch.float64, device=dev)
        self.states = torch.empty((T, 13 * n), **f64)
        self.J = torch.empty((samples, n), **f64)
        self.cand = torch.empty((T, n, 4), **f64)
        self.pick = torch.empty((E if env._effects & N.EFFECT_DW else n,), dtype=torch.int32, device=dev)

    def io(self, iteration, **ptrs):
        lo, hi, per_tick = self.box if self.box is not None else (None, None, False)
        base = dict(state0=self.planes0, last_rpm=self.last_rpm, phys=self.rows, targets=self.targets, weights=self.weights,
                    rpm_ref=self.rpm_ref, sigma=self.sigma, rpm_lo=lo, rpm_hi=hi, rpm=self.rpm, states=self.states, J=self.J,
                    cand=self.cand, pick=self.pick)
        base.update(ptrs)
        return _io(N.QsMppiIO, self.T, base, K=self.K, iteration=iteration, per_tick=int(per_tick), seed=self.seed,
                   temperature=self.temperature)

    def _launch(self, name, io):
        P, E, D, S, eff = self.cfg
        _call(name, C.byref(P), C.byref(io), E, D, S, eff, device=self.dev)

    def nominal(self, cost_out):
        """states and cost_out [N] of the nominal's own rollout"""
        self._launch("qs_mppi_commit", self.io(0, cand=None, cost_out=cost_out, pick=None))

    def sample(self, it):
        """J [K, N] of every sample of iteration `it`"""
        self._launch("qs_mppi_sample", self.io(it))

    def update(self, it):
        """cand [T, N, 4] from J"""
        self._launch("qs_mppi_update", self.io(it))

    def commit(self, it, cost_out):
        """the new nominal (rpm, states), its cost_out [N] and pick"""
        self._launch("qs_mppi_commit", self.io(it, cost_out=cost_out))

    def noise(self, it):
        """eps [K, T, N, 4] of iteration `it`"""
        out = torch.empty((self.K, self.T, self.n, 4), dtype=torch.float64, device=self.dev)
        E, D = self.env_shape
        _call("qs_mppi_noise", C.byref(self.io(it, noise=out)), E, D, device=self.dev)
        return out

    def result(self, cost):
        E, D = self.env_shape
        out = unpack_traj(self.states, self.T, E, D)
        out["rpm"] = self.rpm.view(self.T, E, D, 4)
        out["cost"] = cost.view(cost.shape[0], E, D)
        return out


def solve(m, iters):
    """`iters` iterations of Mppi m: the nominal's trajectory and cost row 0 once, then per iteration sample, update and
    commit.  Nothing is read back to the host."""
    with torch.no_grad(), torch.cuda.device(m.dev):
        cost = torch.empty((iters + 1, m.n), dtype=torch.float64, device=m.dev)
        m.nominal(cost[0])
        for it in range(iters):
            m.sample(it)
            m.update(it)
            m.commit(it, cost[it + 1])
    return m.result(cost)


def mppi(env, target, num_steps=None, rpm=None, Q=None, R=None, Q_final=None, rpm_ref=None, iters=30, samples=64, sigma=0.02,
         temperature=0.1, seed=0, state=None, last_rpm=None, phys=None, rpm_bounds=None):
    """BaseAviary.mppi (see there)."""
    check_iters(iters)
    m = Mppi(env, target, num_steps=num_steps, rpm=rpm, Q=Q, R=R, Q_final=Q_final, rpm_ref=rpm_ref, samples=samples, sigma=sigma,
             temperature=temperature, seed=seed, state=state, last_rpm=last_rpm, phys=phys, rpm_bounds=rpm_bounds)
    return solve(m, iters)
