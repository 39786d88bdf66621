"""Times BaseAviary.differentiable_rollout on one GPU: the forward (qs_dyn_traj) and forward + backward (qs_dyn_traj_vjp), next
to CtrlAviary.rollout(actions=float64, record=False) of the same ticks, at E = 32 768 aviaries of D = 2 drones, T = 64 ticks of
S = 8 substeps (240 / 30 Hz), for Physics.DYN and GND|DRAG (the latter through the C ABI's effects; no Physics member has both).
Prints one JSON line with the card name and power limit read in the same call.  CUDA events, median of --reps."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def timed(fn, reps):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=32768)
    ap.add_argument("--drones", type=int, default=2)
    ap.add_argument("--ticks", type=int, default=64)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    from gym_pybullet_drones_b200 import _native as N
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils.enums import Physics
    E, D, T = args.envs, args.drones, args.ticks
    res = {"card": card(), "E": E, "D": D, "T": T, "S": 8}
    for name, physics, eff in (("dyn", Physics.DYN, 0), ("gnd_drag", Physics.PYB_DRAG, N.EFFECT_GND | N.EFFECT_DRAG)):
        env = CtrlAviary(num_drones=D, physics=physics, pyb_freq=240, ctrl_freq=30, num_envs=E)
        env.reset()
        env._effects = eff                       # GND|DRAG is reachable through the C ABI only
        g = torch.Generator(device=env.device).manual_seed(0)
        rpm = env.HOVER_RPM * (1 + 0.05 * (2 * torch.rand((T, E, D, 4), generator=g, device=env.device, dtype=torch.float64) - 1))
        r = rpm.clone().requires_grad_(True)
        fwd = timed(lambda: env.differentiable_rollout(rpm), args.reps)

        def fb():
            out = env.differentiable_rollout(r)
            torch.autograd.grad(out["pos"].sum(), r)
        both = timed(fb, args.reps)
        res[name] = {"forward_ms": fwd, "forward_backward_ms": both}
        if eff in (0, N.EFFECT_DRAG):
            env._effects = 0 if eff == 0 else N.EFFECT_DRAG
            state = env._planes.clone()
            res[name]["ctrl_rollout_f64_ms"] = timed(lambda: (env._planes.copy_(state), env.rollout(actions=rpm, record=False)), args.reps)
        n = E * D
        # forward: rpm 32 B and the state 104 B per drone-tick written (+ state0 once); backward: rpm (tick and previous) 64 B,
        # the start state and the cotangent 208 B, g_rpm 32 B, the substep records 2 x 104 B x (S - 1) per drone-tick
        res[name]["bytes_per_drone_tick"] = {"forward": 32 + 104, "backward": 64 + 208 + 32 + 2 * 104 * 7}
        res[name]["drone_ticks_per_s_forward"] = n * T / (fwd * 1e-3)
        del env
    print(json.dumps(res))


if __name__ == "__main__":
    main()
