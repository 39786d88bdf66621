"""Times the backward of differentiable_ilqr() (ilqr.IlqrSolution, DESIGN.md 4.5.1 "Gradients of the solution") on one GPU
against one iLQR iteration in the same call, and prints one JSON line per (physics, bounds) with the card name and power limit.
CtrlAviary, 65 536 drones (E = 16 384 aviaries of D = 4), T = 48 ticks at 240 / 48 Hz, targets within 0.5 m, --iters
iterations of the forward.  CUDA events around each launch, [min, median, max] ms over --reps after --warmup:
  * iteration: one iLQR iteration (line search, commit, Jacobians, backward pass) of the same problem;
  * the backward's parts: jac (qs_dyn_tick_jac at the solution), adjoint (qs_ilqr_adjoint), rollout
    (qs_ilqr_adjoint_rollout), vjp (qs_dyn_traj_vjp with g_X - W dx), torch (the surrogate's autograd and the elementwise
    terms);
  * backward: the whole autograd backward of l = <g_X, states> + <g_U, rpm> w.r.t. every packed input."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from jvp_bench import card  # noqa: E402


def stats(ts):
    ts = sorted(ts)
    return [round(ts[0], 3), round(ts[len(ts) // 2], 3), round(ts[-1], 3)]


def timed(fns, reps, warmup):
    """{name: [min, median, max] ms} of each fn, launched in order per rep"""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(fns) + 1)]
    times = {k: [] for k, _ in fns}
    for it in range(warmup + reps):
        ev[0].record()
        for j, (_, fn) in enumerate(fns):
            fn()
            ev[j + 1].record()
        torch.cuda.synchronize()
        if it >= warmup:
            for j, (k, _) in enumerate(fns):
                times[k].append(ev[j].elapsed_time(ev[j + 1]))
    return {k: stats(v) for k, v in times.items()}


def run(physics, E, D, T, iters, reps, warmup, rpm_bounds):
    from gym_pybullet_drones_b200 import _native as N
    from gym_pybullet_drones_b200.diff import _call, _dyn_traj_vjp, _io
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.ilqr import IlqrSolution, Problem, state_weights
    from gym_pybullet_drones_b200.utils.enums import Physics
    rng = np.random.default_rng(0)
    xyz = np.stack([rng.uniform(-1, 1, D), rng.uniform(-1, 1, D), rng.uniform(0.5, 1.5, D)], 1)
    env = CtrlAviary(num_drones=D, physics=getattr(Physics, physics), pyb_freq=240, ctrl_freq=48, initial_xyzs=xyz, num_envs=E)
    env.reset()
    dev = env.device
    target = {"pos": torch.tensor(rng.uniform(-0.5, 0.5, (E, D, 3)) + np.array([0.0, 0.0, 1.0]), device=dev)}
    # the whole backward through autograd
    p = Problem(env, target, num_steps=T, rpm_bounds=rpm_bounds, graph=True)
    leaves = [x.detach().clone().requires_grad_() for x in p.graph]
    states, rpm = IlqrSolution.apply(*leaves, p, iters, {})
    gX, gU = torch.randn_like(states), 1e-4 * torch.randn_like(rpm)
    loss = (states * gX).sum() + (rpm * gU).sum()
    out = timed([("backward", lambda: torch.autograd.grad(loss, leaves, retain_graph=True))], reps, warmup)
    # its parts, on the solved problem
    P, _, _, S, eff = p.cfg
    n = p.n
    p.states, p.rpm = states.detach(), rpm.detach()
    f64 = dict(dtype=torch.float64, device=dev)
    p.jac = torch.empty((T, n, 13, 21 if p.nz == 17 else 17), **f64)
    bufs = dict(K=torch.empty((T, n, 4, p.nz), **f64), k=torch.empty((T, n, 4), **f64), status=torch.empty((n,), dtype=torch.int32, device=dev),
                w=torch.empty((T, n, 4), **f64), dx=torch.empty((T, 13 * n), **f64))
    io = _io(N.QsIlqrAdjointIO, T, dict(jac=p.jac, rpm=p.rpm, phys=p.rows, weights=p.weights, active=p.active, g_states=gX, g_rpm=gU, **bufs))
    W = state_weights(p.weights, E, D, T)

    def surrogate():
        tg, wt, ref, rows = (x.detach().requires_grad_() for x in (p.targets, p.weights, p.rpm_ref, p.rows))
        Rt = (wt[:, 26:30] / (rows[:, 12:13] * rows[:, 12:13])).repeat_interleave(D, dim=0)
        s = -((state_weights(wt, E, D, T) * (p.states - tg) * bufs["dx"]).sum() + (Rt * (p.rpm - ref) * bufs["w"]).sum())
        torch.autograd.grad(s, [tg, wt, ref, rows])
        return gX - W * bufs["dx"]

    parts = [("jac", p.jacobians),
             ("adjoint", lambda: _call("qs_ilqr_adjoint", C.byref(P), C.byref(io), E, D, S, eff, device=dev)),
             ("rollout", lambda: _call("qs_ilqr_adjoint_rollout", C.byref(P), C.byref(io), E, D, S, eff, device=dev)),
             ("vjp", lambda: _dyn_traj_vjp(p.cfg, p.rpm, p.planes0, p.last_rpm, p.rows, p.states, gX - W * bufs["dx"])),
             ("torch", surrogate)]
    out.update(timed(parts, reps, warmup))
    # one iLQR iteration of the same problem (line search, commit, Jacobians, backward pass)
    cost = torch.empty((2, n), **f64)
    p.cost(cost[0])
    p.converged.zero_()
    it = [("line", p.line_search), ("commit", lambda: p.commit(cost[0], cost[1])), ("it_jac", p.jacobians), ("it_backward", p.backward)]
    t_it = timed(it, reps, warmup)
    out["iteration"] = [round(sum(v[j] for v in t_it.values()), 3) for j in range(3)]
    out["iteration_backward_pass"] = t_it["it_backward"]
    med = {k: out[k][1] for k in ("jac", "adjoint", "rollout", "vjp", "torch")}
    held = None if p.active is None else round(float((p.active != 0).float().mean()), 4)
    return {"physics": physics, "rpm_bounds": rpm_bounds, "held_share": held, "drones": n, "T": T, "nz": p.nz, "ms": out,
            "parts_sum_ms": round(sum(med.values()), 3), "backward_over_iteration": round(out["backward"][1] / out["iteration"][1], 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=16384)
    ap.add_argument("--drones", type=int, default=4)
    ap.add_argument("--T", type=int, default=48)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--physics", default="DYN,PYB_DRAG")
    ap.add_argument("--rpm-bounds", default="none,motor")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ilqr_grad_bench: no CUDA device")
    name = card()
    for physics in a.physics.split(","):
        for b in a.rpm_bounds.split(","):
            r = run(physics, a.envs, a.drones, a.T, a.iters, a.reps, a.warmup, None if b == "none" else b)
            r["card"] = name
            print(json.dumps(r), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
