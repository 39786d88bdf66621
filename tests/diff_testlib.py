"""Shared helpers of the differentiable-trajectory tests (test infrastructure): the g++ build of dyn_adjoint.cuh (the adjoint core
of the dyn_traj kernels) and the drone batches the tests differentiate at."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = ("cf2x", "cf2p", "race")

_HH = None


def diff_harness():
    """Builds (g++) and loads tests/host_harness/diff_host.cpp: the kernels' tick adjoint compiled for the host."""
    global _HH
    if _HH is not None:
        return _HH
    src = os.path.join(ROOT, "tests", "host_harness", "diff_host.cpp")
    out = os.path.join(ROOT, "tests", "host_harness", "libdiff_host.so")
    csrc = os.path.join(ROOT, "gym_pybullet_drones_b200", "csrc")
    deps = [src, os.path.join(csrc, "dyn_adjoint.cuh"), os.path.join(csrc, "quad_core.cuh"), os.path.join(ROOT, "include", "quadsim.h")]
    if not os.path.isfile(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", "-o", out, src], check=True)
    L = C.CDLL(out)
    L.dh_tick_vjp.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_int, C.c_int] + [C.c_void_p] * 9
    L.dh_half_angle_grad.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_void_p]
    _HH = L
    return L


def drone_model(name):
    from gym_pybullet_drones_b200.utils.enums import DroneModel
    return {"cf2x": DroneModel.CF2X, "cf2p": DroneModel.CF2P, "race": DroneModel.RACE}[name]


def params_of(model, pyb_freq=240, ctrl_freq=240):
    """(QsParams, AviaryConstants) of a drone model."""
    from gym_pybullet_drones_b200.params import AviaryConstants, fill_params
    c = AviaryConstants(drone_model(model), pyb_freq, ctrl_freq)
    return fill_params(c), c


def quat_from_rpy(rpy):
    from gym_pybullet_drones_b200.params import quaternion_from_euler
    return quaternion_from_euler(np.asarray(rpy, dtype=np.float64))


def scenarios(c, rng, n=4):
    """{name: (state [n, 13], raw rpm [n, 4], previous clipped rpm [n, 4])} at the decision points of DESIGN.md 4.5.  c: the
    model's AviaryConstants."""
    hover, mx = float(c.HOVER_RPM), float(c.MAX_RPM)
    clip = float(c.GND_EFF_H_CLIP)

    def state(pos, rpy, vel, w):
        q = quat_from_rpy(rpy)
        return np.concatenate([pos, q, vel, w], axis=1)

    def rnd(lo, hi, shape):
        return rng.uniform(lo, hi, shape)

    z3 = np.zeros((n, 3))
    out = {}
    # exact hover: level, at rest, equal RPMs -- w = 0 in every substep (the isclose branch of the forward)
    out["hover"] = (state(np.tile([0.0, 0.0, 1.0], (n, 1)), z3, z3, z3), np.full((n, 4), hover), np.full((n, 4), hover))
    # generic flight
    out["flight"] = (state(rnd(-1, 1, (n, 3)) + [0, 0, 1.5], rnd(-0.4, 0.4, (n, 3)), rnd(-1, 1, (n, 3)), rnd(-3, 3, (n, 3))),
                     hover * rnd(0.8, 1.2, (n, 4)), hover * rnd(0.8, 1.2, (n, 4)))
    # tumbling: |w| dt / 2 beyond 1/2 (the sqrt / sincos range of half_angle_terms) at 240 Hz, mostly about the body z axis (about
    # a transverse axis the explicit Euler step of w x Jw amplifies the rates by ~1.7 per substep at these speeds)
    w = np.concatenate([rnd(-5, 5, (n, 2)), rnd(250, 300, (n, 1)) * np.sign(rnd(-1, 1, (n, 1)))], 1)
    out["tumbling"] = (state(rnd(-1, 1, (n, 3)) + [0, 0, 2], rnd(-3, 3, (n, 3)), rnd(-2, 2, (n, 3)), w),
                       hover * rnd(0.5, 1.5, (n, 4)), hover * rnd(0.5, 1.5, (n, 4)))
    # propellers below the ground-effect height clip (and some above it)
    out["ground"] = (state(np.concatenate([rnd(-1, 1, (n, 2)), rnd(0.1 * clip, 1.5 * clip, (n, 1))], 1), rnd(-0.2, 0.2, (n, 3)),
                           rnd(-0.5, 0.5, (n, 3)), rnd(-2, 2, (n, 3))), hover * rnd(0.8, 1.2, (n, 4)), hover * rnd(0.8, 1.2, (n, 4)))
    # RPM commands beyond the clip on both sides
    raw = hover * rnd(0.8, 1.2, (n, 4))
    raw[:, 0] = mx * rnd(1.01, 1.5, n)
    raw[:, 2] = -hover * rnd(0.01, 0.5, n)
    out["clipped"] = (state(rnd(-1, 1, (n, 3)) + [0, 0, 0.05], rnd(-0.3, 0.3, (n, 3)), rnd(-1, 1, (n, 3)), rnd(-3, 3, (n, 3))),
                      raw, np.clip(hover * rnd(0.8, 1.2, (n, 4)), 0, mx))
    # tilted past the upright switch (|roll| > pi/2), near the ground
    rpy = np.concatenate([rnd(1.7, 2.8, (n, 1)) * np.sign(rnd(-1, 1, (n, 1))), rnd(-0.3, 0.3, (n, 2))], 1)
    out["tilted"] = (state(np.concatenate([rnd(-1, 1, (n, 2)), rnd(0.02, 0.2, (n, 1))], 1), rpy, rnd(-1, 1, (n, 3)), rnd(-3, 3, (n, 3))),
                     hover * rnd(0.8, 1.2, (n, 4)), hover * rnd(0.8, 1.2, (n, 4)))
    return out


def host_tick_vjp(P, effects, S, state, raw, up, g_out, rows=None):
    """The host-built kernel core: one tick and its VJP.  Returns (out, g_state, g_raw, g_up, g_row)."""
    L = diff_harness()
    n = state.shape[0]
    a = lambda x: np.ascontiguousarray(x, dtype=np.float64)
    state, raw, up, g_out = a(state), a(raw), a(up), a(g_out)
    rows = None if rows is None else a(rows)
    outs = [np.zeros((n, 13)), np.zeros((n, 13)), np.zeros((n, 4)), np.zeros((n, 4)), np.zeros((n, 16))]
    p = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)
    L.dh_tick_vjp(C.addressof(P), p(rows), effects, S, n, p(state), p(raw), p(up), p(g_out), *[p(o) for o in outs])
    return outs

