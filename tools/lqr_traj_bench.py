"""differentiable_rollout(controller=ilqr.Tracker, plan=) (qs_dyn_lqr_traj / qs_dyn_lqr_traj_vjp) against the rollouts beside it.

  fwd          the tracker loop's forward, plan rpm and K requiring grad (what a training step runs)
  fwd_bwd      the forward and the backward of a scalar loss over every output
  rollout      CtrlAviary.rollout(controller=Tracker), record=False (the production tracker; it refuses GND|DRAG)
  open_fwd     the open loop, differentiable_rollout(rpm) with rpm requiring grad
  open_fwd_bwd its forward and backward

65 536 drones as aviaries of D = 4, T = 48, Physics.DYN (a plan of n_z = 13) and GND|DRAG (n_z = 17).  The plan is synthetic
(hover RPMs plus noise, small random gains, z the start state): its values do not change what the kernels read.  Times are CUDA
events in milliseconds per call, the best of --runs runs of --reps calls each after a warm-up, the variants alternating.  Prints
the card and its power limit, one line per case, then one JSON line.

    python tools/lqr_traj_bench.py [--runs 3] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

KEYS = ("pos", "quat", "vel", "rpy_rates")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip().splitlines()[0]
        return [c.strip() for c in out.split(",")]
    except Exception:
        return [torch.cuda.get_device_name(), "unknown", "unknown"]


def timed(fn, reps):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ev0.record()
    for _ in range(reps):
        fn()
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / reps


def case(physics, n, T, runs, reps):
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.ilqr import Tracker
    from gym_pybullet_drones_b200.utils.enums import Physics
    D = 4
    E = n // D
    env = CtrlAviary(num_drones=D, physics=Physics.PYB_GND_DRAG_DW if physics == "GND|DRAG" else Physics.DYN, num_envs=E)
    env.reset()
    if physics == "GND|DRAG":
        env._effects = 3                          # ground effect and drag without downwash, as ilqr plans
    nz = 17 if physics == "GND|DRAG" else 13
    dev = env.device
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.cat([getattr(env, k) for k in KEYS], dim=-1)
    if nz == 17:
        x = torch.cat([x, env._last_rpm.view(E, D, 4)], dim=-1)
    h = float(env.HOVER_RPM)
    sol = {"rpm": h * (1 + 0.01 * torch.randn((T, E, D, 4), generator=g, dtype=torch.float64, device=dev)),
           "K": 1e-3 * torch.randn((T, E, D, 4, nz), generator=g, dtype=torch.float64, device=dev),
           "z": x[None].expand(T, E, D, nz).contiguous()}
    trk = Tracker(sol)
    plan = {k: sol[k].clone().requires_grad_() for k in ("rpm", "K")}
    rpm = sol["rpm"].clone().requires_grad_()

    def loss(out):
        return sum(out[k].sum() for k in out)

    def fwd():
        env.differentiable_rollout(controller=trk, plan=plan)

    def fwd_bwd():
        loss(env.differentiable_rollout(controller=trk, plan=plan)).backward()

    def open_fwd():
        env.differentiable_rollout(rpm)

    def open_fwd_bwd():
        loss(env.differentiable_rollout(rpm)).backward()

    def rollout():
        env.rollout(controller=trk, record=False)
        trk.tick = 0

    fns = dict(fwd=fwd, fwd_bwd=fwd_bwd, open_fwd=open_fwd, open_fwd_bwd=open_fwd_bwd)
    if physics != "GND|DRAG":
        fns["rollout"] = rollout
    snap = {k: getattr(env, k).clone() for k in KEYS}
    for f in fns.values():
        f()
    best = {k: float("inf") for k in fns}
    for _ in range(runs):
        for k, f in fns.items():
            best[k] = min(best[k], timed(f, reps))
    env.set_state(**snap)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--drones", type=int, default=65536)
    ap.add_argument("--ticks", type=int, default=48)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lqr_traj_bench.py needs a CUDA device")
    name, plim, clk = card()
    print("card: %s, power limit %s, max SM clock %s" % (name, plim, clk))
    res = {}
    for physics in ("DYN", "GND|DRAG"):
        r = case(physics, a.drones, a.ticks, a.runs, a.reps)
        res[physics] = r
        print("%-8s %d drones T=%d: %s" % (physics, a.drones, a.ticks, "  ".join("%s %.3f ms" % kv for kv in r.items())))
    print(json.dumps(dict(card=name, power_limit=plim, drones=a.drones, T=a.ticks, ms=res)))


if __name__ == "__main__":
    main()
