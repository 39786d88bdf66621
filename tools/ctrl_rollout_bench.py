"""rollout() of the control envs (qs_ctrl_rollout) against the per-tick loops it replaces.

  track_roll   CtrlAviary.rollout(controller=DSLPIDControl, waypoints=pid.py's circle, per-drone phase, z offset), record=False
  track_rows   the same with record=True (the [T, E, D, 20] state vectors written every tick)
  track_loop   T x (computeControlFromEnv(env, targets[k], target_rpy) + step(rpm)): the pid.py loop, targets precomputed on the device
  vel_roll     VelocityAviary.rollout(actions), record=False       vel_steps   T x step(actions[k])
  raw_roll     CtrlAviary.rollout(actions), record=False           raw_steps   T x step(actions[k])

The inputs keep the drones flying (the circle, zero velocity commands, hover RPMs), so the cost does not drift with the state.
Sizes: E = 4 096 x D = 1, the pid.py shape E = 32 768 x D = 3, and E = 1 048 576 x D = 1; T = 48; Physics.DYN and
PYB_GND_DRAG_DW (all three effects).  The variants alternate, --runs runs each; times are CUDA events on the stream in
microseconds per tick.  Prints the card, its power limit and SM clock limit, one line per size, then one JSON line.

    python tools/ctrl_rollout_bench.py [--runs 3] [--reps 4]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

T = 48
SIZES = ((4096, 1), (32768, 3), (1 << 20, 1))
PHYSICS = ("DYN", "PYB_GND_DRAG_DW")
VARIANTS = ("track_roll", "track_rows", "track_loop", "vel_roll", "vel_steps", "raw_roll", "raw_steps")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip().splitlines()[0]
        return [c.strip() for c in out.split(",")]
    except Exception:
        return [torch.cuda.get_device_name(), "unknown", "unknown", "unknown"]


def timed(fn, reps):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ev0.record()
    for _ in range(reps):
        fn()
    ev1.record()
    torch.cuda.synchronize()
    return 1e3 * ev0.elapsed_time(ev1) / (reps * T)


def bench(E, D, physics, runs, reps):
    from gym_pybullet_drones_b200.control import DSLPIDControl
    from gym_pybullet_drones_b200.envs import CtrlAviary, VelocityAviary
    from gym_pybullet_drones_b200.utils.enums import DroneModel, Physics
    n, dev = E * D, torch.device("cuda")
    kw = dict(num_drones=D, physics=Physics[physics], pyb_freq=240, ctrl_freq=48, num_envs=E)
    ctrl_env, vel_env = CtrlAviary(**kw), VelocityAviary(**kw)
    ctrl_env.reset(); vel_env.reset()
    ctrl = DSLPIDControl(DroneModel.CF2X, num_drones=n)
    W = 48 * 10                                                           # pid.py: NUM_WP = ctrl_freq * 10
    i = np.arange(W)
    wp = np.stack([0.3 * np.cos(2 * np.pi * i / W + np.pi / 2), 0.3 * np.sin(2 * np.pi * i / W + np.pi / 2) - 0.3, np.zeros(W)], axis=1)
    start = (np.arange(n) * W // 6 % W).astype(np.int32)
    offset = np.zeros((n, 3))
    offset[:, 2] = ctrl_env.pos.reshape(n, 3)[:, 2].cpu().numpy()
    trpy = torch.zeros((n, 3), dtype=torch.float64, device=dev)
    tk = dict(waypoints=wp, start=start, offset=offset, target_rpy=trpy, num_steps=T)
    tp_dev = torch.from_numpy(CtrlAviary.schedule_targets(wp, start, offset, T)).to(dev)        # [T, n, 3]: every call flies the same T ticks
    vel_act = torch.zeros((T, E, D, 4), device=dev)
    raw_act = torch.full((T, E, D, 4), float(ctrl_env.HOVER_RPM), dtype=torch.float32, device=dev)
    outs = {}

    def track(record):
        def f():
            key = "rows" if record else "roll"
            outs[key] = ctrl_env.rollout(controller=ctrl, record=record, out=outs.get(key), **tk)
        return f

    def track_loop():
        for k in range(T):
            rpm = ctrl.computeControlFromEnv(ctrl_env, tp_dev[k], target_rpy=trpy)
            ctrl_env.step(rpm)

    def vel_roll():
        outs["vel"] = vel_env.rollout(vel_act, record=False, out=outs.get("vel"))

    def vel_steps():
        for k in range(T):
            vel_env.step(vel_act[k])

    def raw_roll():
        outs["raw"] = ctrl_env.rollout(raw_act, record=False, out=outs.get("raw"))

    def raw_steps():
        for k in range(T):
            ctrl_env.step(raw_act[k])

    fns = dict(track_roll=track(False), track_rows=track(True), track_loop=track_loop, vel_roll=vel_roll, vel_steps=vel_steps,
               raw_roll=raw_roll, raw_steps=raw_steps)
    for v in VARIANTS:                                   # warm-up: allocations, first launches
        fns[v]()
    res = {v: [] for v in VARIANTS}
    for _ in range(runs):
        for v in VARIANTS:
            res[v].append(round(timed(fns[v], reps), 2))
    del ctrl_env, vel_env, ctrl, outs, tp_dev
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=4, help="calls of T = 48 ticks per timed run")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ctrl_rollout_bench.py needs a CUDA device")
    name, pl, smax, scur = card()
    print("card: %s, power limit %s, max SM clock %s, SM clock at start %s" % (name, pl, smax, scur), flush=True)
    out = {"card": name, "power_limit": pl, "max_sm_clock": smax, "ticks_per_call": T, "runs": a.runs, "unit": "us per tick",
           "results": {}}
    for E, D in SIZES:
        for physics in PHYSICS:
            key = "E%d_D%d_%s" % (E, D, physics)
            out["results"][key] = bench(E, D, physics, a.runs, a.reps)
            print(key, json.dumps(out["results"][key]), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
