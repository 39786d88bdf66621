"""Shared helpers for the parity tests (test infrastructure)."""
import ctypes as C
import os
import re
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ("pos", "quat", "rpy", "vel", "ang_v", "rpy_rates")

# north-star tolerance: |a-b| <= 1e-5 * max(|b|, 1) element-wise on the kinematic state
RTOL = 1e-5
# what the float64 state planes actually deliver on non-chaotic trajectories (the kernels differ from the float64
# reference only in operation order, series vs libm in _integrateQ, and 1/|q| renormalisation): used where the
# observation's float32 cast is not in the way
TIGHT = 1e-9


def relerr(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1.0))) if a.size else 0.0


def quat_err(a, b):
    """sign-insensitive quaternion comparison (q and -q are the same rotation)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    s = np.sign(np.sum(a * b, axis=-1, keepdims=True))
    s[s == 0] = 1
    return relerr(a * s, b)


def pack_planes(pos, quat, vel, w):
    """float64 [n,3],[n,4],[n,3],[n,3] -> float64 planes [13 n] in the layout of include/quadsim.h."""
    n = pos.shape[0]
    pl = np.zeros((13 * n,), np.float64)
    p = pl[:12 * n].reshape(3, n, 4)
    p[0, :, 0:3], p[0, :, 3] = pos, w[:, 0]
    p[1] = quat
    p[2, :, 0:3], p[2, :, 3] = vel, w[:, 1]
    pl[12 * n:] = w[:, 2]
    return pl


def unpack_planes(pl):
    pl = np.asarray(pl, np.float64).reshape(-1)
    n = pl.size // 13
    p = pl[:12 * n].reshape(3, n, 4)
    w = np.stack([p[0, :, 3], p[2, :, 3], pl[12 * n:]], axis=1)
    return p[0, :, 0:3], p[1], p[2, :, 0:3], w


_INCLUDE = re.compile(r'^\s*#\s*include\s*"([^"]+)"', re.M)
_HARNESSES = {}


def _sources(path, seen=None):
    """path and every file it reaches through #include "..." lines (resolved against the including file's directory)."""
    seen = set() if seen is None else seen
    path = os.path.normpath(path)
    if path not in seen:
        seen.add(path)
        with open(path) as f:
            for inc in _INCLUDE.findall(f.read()):
                _sources(os.path.join(os.path.dirname(path), inc), seen)
    return seen


def harness(name):
    """Builds (g++, when the library is older than tests/host_harness/<name>.cpp or any file it includes) and loads
    tests/host_harness/lib<name>.so: kernel code compiled for the host."""
    if name not in _HARNESSES:
        src = os.path.join(ROOT, "tests", "host_harness", name + ".cpp")
        out = os.path.join(ROOT, "tests", "host_harness", "lib%s.so" % name)
        if not os.path.isfile(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in _sources(src)):
            subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", "-o", out, src], check=True)
        _HARNESSES[name] = C.CDLL(out)
    return _HARNESSES[name]


def drone_model(name):
    from gym_pybullet_drones_b200.utils.enums import DroneModel
    return {"cf2x": DroneModel.CF2X, "cf2p": DroneModel.CF2P, "race": DroneModel.RACE}[name]


def host_harness():
    """tests/host_harness/core_host.cpp: the CUDA kernels' per-drone core compiled for the host."""
    L = harness("core_host")
    L.hh_downwash_pair.restype = C.c_double
    L.hh_downwash_pair.argtypes = [C.c_void_p, C.c_double, C.c_double]
    L.hh_downwash_acts.argtypes = [C.c_double, C.c_double]
    L.hh_downwash_fz.restype = C.c_double
    L.hh_downwash_fz.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double]
    L.hh_half_angle.argtypes = [C.c_double, C.c_double, C.POINTER(C.c_double), C.POINTER(C.c_double)]
    L.hh_tick.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p]
    L.hh_pid.argtypes = [C.c_void_p] + [C.c_void_p, C.c_double] + [C.c_void_p] * 4 + [C.c_double] + [C.c_void_p] * 5
    L.hh_quat_to_euler.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    L.hh_upright.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.hh_hover_terms.argtypes = [C.c_void_p] * 4 + [C.c_int, C.c_int, C.c_void_p]
    return L


def ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class PolicyRef:
    """Float64 NumPy restatement of the on-device policy (`MlpPolicy` evaluated by rollout_kernel<.,.,kNetClassic>): actor mean,
    sampled action, log-probability and critic value from the fp32 weights the policy holds, plus the accuracy criterion the
    kernel is held to.

    Criterion, per output element (actor mean or critic value) of a batch of observations:
        |kernel - float64| <= FP32_MULTIPLE * e32[j] + floor[j]
    * e32[j] = max over the batch of |fp32 - float64| for output j, where fp32 is the same network evaluated in NumPy float32
      (BLAS sgemm, libm tanhf).  That is the error of a plain fp32 evaluation at these inputs: it grows with |x| and with K
      the way the kernel's does.  The kernel's products carry ~2^-21 relative error (the two-term split drops x_lo' w_lo' and
      rounds each lo' part to 11 bits) against fp32's 2^-24 rounding of each product and partial sum; the accumulators are fp32
      in both.  FP32_MULTIPLE = 16 allows for that 8x and a factor 2 for the two accumulator sets the kernel adds at the end.
    * floor[j] covers tanh_fast's absolute error e = TANH_FAST_ABS_ERR (1 - 2 / (exp(2x) + 1) with __expf and __fdividef),
      which the fp32 yardstick does not have.  The errors of different hidden units are uncorrelated (each depends on the low
      bits of its own argument), so they add through the following layers as a root sum of squares: an error of size e in
      every unit of layer 1 gives layer 2's pre-activation k a standard deviation of at most e sqrt(sum_i W2[i,k]^2), tanh' <= 1
      passes it on, layer 2's own tanh adds e, and layer 3 weights both by W3[k,j]:
          floor[j] = TANH_SIGMAS * e * sqrt(sum_k W3[k,j]^2 (1 + sum_i W2[i,k]^2)).
      TANH_SIGMAS = 6 standard deviations, with e the worst-case error standing in for the RMS one.  The worst-case sum
      e sum_k |W3[k,j]| (1 + sum_i |W2[i,k]|) is 5x larger for these 64-unit layers; the kernel stays below 0.15 of it at every
      shape tested, and a kernel that dropped w_lo' would miss it by only ~3x.
    * The sampled action r = fmaf(expf(log_std), eps, mean) adds expf's 2 ulp on std * eps and one rounding of r:
      2^-22 (|mean| + |std eps|) on top of the mean's bound.  The log-probability is a float32 sum of n = D*A terms
      -0.5 eps^2 - log_std - log(2 pi)/2 of three roundings each: (n + 3) 2^-24 sum_j (0.5 eps_j^2 + |log_std_j| + log(2 pi)/2).
    Removing the fp16 low part of either operand costs up to 2^-11 relative per product; the negative controls in
    test_gpu_policy.py check that the criterion misses such a kernel by a factor of more than 10."""
    TANH_FAST_ABS_ERR = 2e-7
    TANH_SIGMAS = 6.0
    FP32_MULTIPLE = 16.0
    HALF_LOG_2PI = 0.91893853320467274
    # rollout.cu splits an observation x into fp16 parts with saturating conversions: x_hi = 65504 and x_lo' = 65504 for every
    # x >= 65504 + 65504 / 2048, so the network sees x_hi + x_lo' / 2048 = 65535.984375 (and symmetrically below zero)
    OBS_SATURATION = 65504.0 + 65504.0 / 2048.0

    def __init__(self, pol):
        f64 = lambda net: None if net is None else [(w.detach().cpu().double().numpy(), b.detach().cpu().double().numpy()) for w, b in net]   # noqa: E731
        self.actor, self.critic = f64(pol.actor), f64(pol.critic)
        self.log_std = pol.log_std.detach().cpu().double().numpy()
        self.in_dim, self.out_dim = pol.in_dim, pol.out_dim
        self.floor_actor = self._floor(self.actor)
        self.floor_critic = None if self.critic is None else self._floor(self.critic)

    @classmethod
    def _floor(cls, net):
        w2, w3 = net[1][0] ** 2, net[2][0] ** 2
        return cls.TANH_SIGMAS * cls.TANH_FAST_ABS_ERR * np.sqrt((w3 * (1.0 + w2.sum(axis=0))[:, None]).sum(axis=0))

    @staticmethod
    def mlp(net, x, dtype=np.float64):
        h = np.asarray(x).astype(dtype)
        for k, (w, b) in enumerate(net):
            h = h @ w.astype(dtype) + b.astype(dtype)
            if k < 2:
                h = np.tanh(h)
        return h

    def flat(self, obs):
        x = np.asarray(obs.detach().cpu().numpy() if hasattr(obs, "detach") else obs, np.float32)
        return x.reshape(-1, self.in_dim)

    def forward(self, obs, noise=None):
        """obs [E, D, obs_dim] or [E, in_dim] (float32) -> float64 (mean, raw action, log-prob, value or None)."""
        x = self.flat(obs).astype(np.float64)
        mean = self.mlp(self.actor, x)
        eps = np.zeros_like(mean) if noise is None else self._eps(noise, mean.shape)
        raw = mean + np.exp(self.log_std) * eps
        logp = (-0.5 * eps * eps - self.log_std - self.HALF_LOG_2PI).sum(axis=1)
        val = None if self.critic is None else self.mlp(self.critic, x)[:, 0]
        return mean, raw, logp, val

    @staticmethod
    def _eps(noise, shape):
        e = noise.detach().cpu().numpy() if hasattr(noise, "detach") else np.asarray(noise)
        return e.astype(np.float32).astype(np.float64).reshape(shape)

    def tolerance(self, net, floor, x):
        """(float64 output [B, out], tolerance [B, out]) of one network on the float32 rows x [B, in_dim]."""
        y64 = self.mlp(net, x.astype(np.float64))
        y32 = self.mlp(net, x.astype(np.float32), np.float32).astype(np.float64)
        e32 = np.abs(y32 - y64).max(axis=0)
        return y64, np.broadcast_to(self.FP32_MULTIPLE * e32 + floor, y64.shape)

    def check(self, obs, noise, actions, log_probs, values=None, ref_obs=None):
        """Worst |kernel - float64| / tolerance of one tick: dict(actions=..., log_probs=..., values=...).  `ref_obs` (default
        obs) is what the reference evaluates, e.g. the observation as the kernel's saturating conversion sees it."""
        x = self.flat(obs)
        xr = x if ref_obs is None else self.flat(ref_obs)
        mean, tol_m = self.tolerance(self.actor, self.floor_actor, xr)
        eps = np.zeros_like(mean) if noise is None else self._eps(noise, mean.shape)
        se = np.exp(self.log_std) * eps
        raw = mean + se
        tol_a = tol_m + 2.0 ** -22 * (np.abs(mean) + np.abs(se))
        got_a = np.asarray(actions.detach().cpu().numpy() if hasattr(actions, "detach") else actions, np.float64).reshape(raw.shape)
        out = dict(actions=float((np.abs(got_a - raw) / tol_a).max()))
        terms = -0.5 * eps * eps - self.log_std - self.HALF_LOG_2PI
        tol_lp = (terms.shape[1] + 3) * 2.0 ** -24 * (0.5 * eps * eps + np.abs(self.log_std) + self.HALF_LOG_2PI).sum(axis=1)
        got_lp = np.asarray(log_probs.detach().cpu().numpy() if hasattr(log_probs, "detach") else log_probs, np.float64).reshape(-1)
        out["log_probs"] = float((np.abs(got_lp - terms.sum(axis=1)) / tol_lp).max())
        if self.critic is not None and values is not None:
            v, tol_v = self.tolerance(self.critic, self.floor_critic, xr)
            got_v = np.asarray(values.detach().cpu().numpy() if hasattr(values, "detach") else values, np.float64).reshape(-1)
            out["values"] = float((np.abs(got_v - v[:, 0]) / tol_v[:, 0]).max())
        return out

    @classmethod
    def saturate(cls, x):
        """An observation as the kernel's fp16 split sees it (see OBS_SATURATION)."""
        return np.clip(np.asarray(x, np.float64), -cls.OBS_SATURATION, cls.OBS_SATURATION)


class HostSim:
    """n independent drones stepped by the host build of the kernel core (float64 planes like the CUDA kernels)."""

    def __init__(self, params, n, act_type, A, substeps, effects=0, pid=False):
        self.L = host_harness()
        self.P, self.n, self.act_type, self.A, self.S, self.effects = params, n, act_type, A, substeps, effects
        self.planes = np.zeros((13 * n,), np.float64)
        self.last_rpm = np.zeros((n, 4), np.float64)
        self.pid = np.zeros((9, n), np.float64) if pid else None
        self.rec = np.zeros((n, 23), np.float64)

    def set_state(self, pos, quat, vel, w):
        self.planes[...] = pack_planes(np.asarray(pos, np.float64).reshape(self.n, 3), np.asarray(quat, np.float64).reshape(self.n, 4),
                                       np.asarray(vel, np.float64).reshape(self.n, 3), np.asarray(w, np.float64).reshape(self.n, 3))

    def tick(self, action):
        a = np.ascontiguousarray(np.asarray(action, np.float32).reshape(self.n, self.A))
        self.L.hh_tick(C.addressof(self.P), ptr(self.planes), self.n, ptr(a), self.A, self.act_type, self.S, self.effects,
                       ptr(self.last_rpm), ptr(self.pid), ptr(self.rec))
        r = self.rec
        return dict(pos=r[:, 0:3], quat=r[:, 3:7], rpy=r[:, 7:10], vel=r[:, 10:13], ang_v=r[:, 13:16], rpy_rates=r[:, 16:19], rpm=r[:, 19:23])
