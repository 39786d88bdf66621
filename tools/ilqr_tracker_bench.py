"""CtrlAviary.rollout(controller=ilqr.Tracker(plan)) (qs_ctrl_rollout_lqr) against the rollouts and the loop it sits beside.

  lqr          the tracker rollout, record=False, n_z 13 and 17 (a plan of drones with drag carries the previous RPMs)
  raw          CtrlAviary.rollout(actions) with float64 RPMs, record=False: the open-loop plan
  track        CtrlAviary.rollout(controller=DSLPIDControl, waypoints), record=False
  loop         (65 536 drones only) per tick: the tracker's law in torch on the env's planes, then rollout(actions=u, 1 tick)

The plan is synthetic (hover RPMs, gains of 1e-6, z_nom the start state): its values do not change what the kernel reads, and
ilqr()'s Jacobians would not fit in memory at 1 048 576 drones.  Sizes: 65 536 and 1 048 576 drones as aviaries of D = 4;
T = 48 at 65 536 and T = 16 at 1 048 576 (the plan and its kernel-layout copy take 2 x 8.7 GB there with n_z = 17).  Physics.DYN
and PYB_GND_DRAG_DW.  `plan_GBs` is the plan's bytes per tick, 8 (4 n_z + n_z + 4) per drone, over the lqr time and `of_peak`
its share of the data sheet's 3.35 TB/s.  The variants alternate, --runs runs each, the best is kept; times are CUDA events in
microseconds per tick.  Prints the card and its power limit, one line per case, then one JSON line.

    python tools/ilqr_tracker_bench.py [--runs 3] [--reps 4]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_BPS = 3.35e12
SIZES = ((65536, 48), (1 << 20, 16))
PHYSICS = ("DYN", "PYB_GND_DRAG_DW")
D = 4


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip().splitlines()[0]
        return [c.strip() for c in out.split(",")]
    except Exception:
        return [torch.cuda.get_device_name(), "unknown", "unknown"]


def timed(fn, reps, T):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ev0.record()
    for _ in range(reps):
        fn()
    ev1.record()
    torch.cuda.synchronize()
    return 1e3 * ev0.elapsed_time(ev1) / (reps * T)


def synthetic_plan(env, T, nz):
    """an ilqr()-shaped result: hover RPMs, gains of 1e-6, z_nom the env's state (and its last RPMs)"""
    E, n, dev = env._E, env._N, env.device
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.cat([getattr(env, k) for k in ("pos", "quat", "vel", "rpy_rates")], dim=-1)
    if nz == 17:
        x = torch.cat([x, env._last_rpm.view(E, D, 4)], dim=-1)
    return {"rpm": torch.full((T, E, D, 4), float(env.HOVER_RPM), dtype=torch.float64, device=dev),
            "K": 1e-6 * torch.randn((T, E, D, 4, nz), dtype=torch.float64, device=dev, generator=g),
            "z": x.unsqueeze(0).expand(T, E, D, nz).contiguous()}


def plan_bytes(n, nz):
    return 8 * n * (4 * nz + nz + 4)


def bench(n, T, physics, runs, reps, variants=("lqr13", "lqr17", "raw", "track", "loop")):
    from gym_pybullet_drones_b200.control import DSLPIDControl
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.ilqr import Tracker
    from gym_pybullet_drones_b200.utils.enums import DroneModel, Physics
    E = n // D
    env = CtrlAviary(num_drones=D, physics=Physics[physics], pyb_freq=240, ctrl_freq=48, num_envs=E)
    env.reset()
    fns = {}
    for nz in (13, 17):
        if "lqr%d" % nz in variants:
            trk = Tracker(synthetic_plan(env, T, nz))
            torch.cuda.empty_cache()

            def f(trk=trk):
                trk.tick = 0
                env.rollout(controller=trk, record=False)
            fns["lqr%d" % nz] = f
    if "raw" in variants:
        raw = torch.full((T, E, D, 4), float(env.HOVER_RPM), dtype=torch.float64, device=env.device)
        fns["raw"] = lambda: env.rollout(actions=raw, record=False)
    if "track" in variants:
        ctrl = DSLPIDControl(DroneModel.CF2X, num_drones=n)
        wp = env.pos.unsqueeze(0).expand(T, E, D, 3).contiguous()          # hold position: per-drone device waypoints
        fns["track"] = lambda: env.rollout(controller=ctrl, waypoints=wp, num_steps=T, record=False)
    if "loop" in variants and n <= 65536:
        from gym_pybullet_drones_b200.diff import unpack_states
        plan = synthetic_plan(env, T, 13)
        K, z, rpm = plan["K"].reshape(T, n, 4, 13), plan["z"].reshape(T, n, 13), plan["rpm"].reshape(T, n, 4)

        def loop():
            for k in range(T):
                s = unpack_states(env._planes, n)
                x = torch.cat([s[q] for q in ("pos", "quat", "vel", "rpy_rates")], dim=-1)
                u = rpm[k] + torch.einsum("njq,nq->nj", K[k], x - z[k])
                env.rollout(actions=u.view(1, E, D, 4), record=False)
        fns["loop"] = loop
    best = {k: float("inf") for k in fns}
    for k, f in fns.items():                                              # warm-up
        f()
    for _ in range(runs):
        for k, f in fns.items():
            best[k] = min(best[k], timed(f, reps if k != "loop" else 1, T))
    res = {k: round(v, 2) for k, v in best.items()}
    for nz in (13, 17):
        if "lqr%d" % nz in res:
            t = res["lqr%d" % nz] * 1e-6
            res["plan_GBs_%d" % nz] = round(plan_bytes(n, nz) / t / 1e9, 1)
            res["of_peak_%d" % nz] = round(plan_bytes(n, nz) / t / PEAK_BPS, 3)
    del fns, env
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=4)
    args = ap.parse_args()
    name, power, sm = card()
    print("card: %s, power limit %s, max SM clock %s" % (name, power, sm))
    out = {"card": name, "power_limit": power, "lib": os.environ.get("QS_LIBQUADSIM", "default")}
    for n, T in SIZES:
        for physics in PHYSICS:
            r = bench(n, T, physics, args.runs, args.reps)
            print("%8d drones  T=%2d  %-16s %s" % (n, T, physics, "  ".join("%s %s" % kv for kv in r.items())), flush=True)
            out["%d_%s" % (n, physics)] = r
    print(json.dumps(out))


if __name__ == "__main__":
    main()
