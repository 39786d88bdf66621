"""CtrlAviary.rollout(controller=MRAC(...)) (qs_ctrl_rollout_mrac) against the per-tick loop it replaces and the DSLPID rollout.

  mrac_roll    CtrlAviary.rollout(controller=MRAC, waypoints=one hover point per drone), record=False
  mrac_loop    T x (computeControlFromEnv(env, target) + step(rpm)): the mrac.py loop
  pid_roll     CtrlAviary.rollout(controller=DSLPIDControl, same schedule), record=False

CF2X, Physics.DYN, 240/120 Hz, T = 120, E = 65 536 and 1 048 576 aviaries of one drone; every drone starts at rest at its
target's height minus 0.1 m, so the controllers work and stay away from saturation.  The variants alternate, --runs runs each;
times are CUDA events on the stream in microseconds per tick.  Prints the card and its power limit, one line per size, then one
JSON line.

    python tools/mrac_rollout_bench.py [--runs 3] [--reps 2]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

T = 120
SIZES = (65536, 1 << 20)
VARIANTS = ("mrac_roll", "mrac_loop", "pid_roll")


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
    return 1e3 * ev0.elapsed_time(ev1) / (reps * T)


def bench(E, runs, reps):
    from gym_pybullet_drones_b200.control import MRAC, DSLPIDControl
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils.enums import DroneModel, Physics
    dev = torch.device("cuda")
    rng = np.random.default_rng(0)
    init = np.concatenate([rng.uniform(-1, 1, (E, 2)), rng.uniform(0.5, 1.0, (E, 1))], axis=1)
    envs = {}
    for v in VARIANTS:
        envs[v] = CtrlAviary(num_drones=1, physics=Physics.DYN, pyb_freq=240, ctrl_freq=120, num_envs=E)
        envs[v].reset()
        envs[v].set_state(pos=init.reshape(E, 1, 3))
    mrac_r, mrac_l = MRAC(DroneModel.CF2X, num_drones=E), MRAC(DroneModel.CF2X, num_drones=E)
    pid = DSLPIDControl(DroneModel.CF2X, num_drones=E)
    wp = np.zeros((1, 3))
    offset = init + [0, 0, 0.1]
    tk = dict(waypoints=wp, offset=offset, num_steps=T, record=False)
    tgt = torch.from_numpy(offset).to(dev)
    outs = {}

    def mrac_roll():
        outs["m"] = envs["mrac_roll"].rollout(controller=mrac_r, out=outs.get("m"), **tk)

    def mrac_loop():
        env = envs["mrac_loop"]
        for _ in range(T):
            env.step(mrac_l.computeControlFromEnv(env, tgt))

    def pid_roll():
        outs["p"] = envs["pid_roll"].rollout(controller=pid, out=outs.get("p"), **tk)

    fns = dict(mrac_roll=mrac_roll, mrac_loop=mrac_loop, pid_roll=pid_roll)
    for v in VARIANTS:                                   # warm-up: allocations, first launches
        fns[v]()
    res = {v: [] for v in VARIANTS}
    for _ in range(runs):
        for v in VARIANTS:
            res[v].append(round(timed(fns[v], reps), 2))
    z = envs["mrac_roll"].pos[:, 0, 2].cpu().numpy()
    res["mrac_z_error_after_warmup_and_runs"] = float(np.max(np.abs(z - offset[:, 2])))
    del envs, mrac_r, mrac_l, pid, outs
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=2, help="calls of T = 120 ticks per timed run")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("mrac_rollout_bench.py needs a CUDA device")
    name, pl, smax = card()
    print("card: %s, power limit %s, max SM clock %s" % (name, pl, smax), flush=True)
    out = {"card": name, "power_limit": pl, "max_sm_clock": smax, "ticks_per_call": T, "runs": a.runs, "unit": "us per tick",
           "results": {}}
    for E in SIZES:
        key = "E%d_D1_DYN" % E
        out["results"][key] = bench(E, a.runs, a.reps)
        print(key, json.dumps(out["results"][key]), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
