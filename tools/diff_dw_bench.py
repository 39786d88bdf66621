"""Times BaseAviary.differentiable_rollout(downwash=True) on one GPU: the forward (qs_dyn_traj_dw) and forward + backward
(qs_dyn_traj_dw_vjp) at N = 65 536 drones, T = 48 ticks of S = 5 substeps (240 / 48 Hz), on Physics.PYB_DW with D = 2, 8, 32
and 128 drones per aviary, next to the per-drone kernels (qs_dyn_traj, qs_dyn_traj_vjp) on Physics.PYB_DRAG at the same N.
The configurations are timed in rounds, each round one repeat of every configuration in turn, so that drift on a shared card
spreads over all of them; the median over rounds is reported.  Prints one JSON line with the card name and power limit read in
the same call.  CUDA events around each call (the host waits for the device before the end event is read)."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from diff_bench import card                                  # noqa: E402


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--drones", type=int, default=65536)
    ap.add_argument("--ticks", type=int, default=48)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--sizes", default="2,8,32,128")
    args = ap.parse_args()
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils.enums import Physics
    n, T = args.drones, args.ticks
    configs = [("drag_per_drone", Physics.PYB_DRAG, 2, False)] + [("dw_D%d" % D, Physics.PYB_DW, D, True)
                                                                   for D in (int(s) for s in args.sizes.split(","))]
    runs = {}
    for name, physics, D, dw in configs:
        E = n // D
        k = torch.arange(D, dtype=torch.float64)
        xyz = torch.stack([0.3 * ((k // 4) % 6), 0.3 * (k // 24), 0.5 + 0.9 * (k % 4)], 1).numpy()    # columns of 4, 0.9 m apart
        env = CtrlAviary(num_drones=D, physics=physics, pyb_freq=240, ctrl_freq=48, num_envs=E, initial_xyzs=xyz)
        env.reset()
        g = torch.Generator(device=env.device).manual_seed(0)
        rpm = env.HOVER_RPM * (1 + 0.05 * (2 * torch.rand((T, E, D, 4), generator=g, device=env.device, dtype=torch.float64) - 1))
        r = rpm.clone().requires_grad_(True)

        def fwd(env=env, rpm=rpm, dw=dw):
            env.differentiable_rollout(rpm, downwash=dw)

        def both(env=env, r=r, dw=dw):
            out = env.differentiable_rollout(r, downwash=dw)
            torch.autograd.grad(out["pos"].sum(), r)

        for _ in range(2):                                   # warm-up: module load, allocator
            fwd()
            both()
        runs[name] = (fwd, both, {"E": E, "D": D})
    times = {name: {"forward_ms": [], "forward_backward_ms": []} for name in runs}
    for _ in range(args.rounds):
        for name, (fwd, both, _) in runs.items():
            times[name]["forward_ms"].append(event_ms(fwd))
            times[name]["forward_backward_ms"].append(event_ms(both))
    res = {"card": card(), "N": n, "T": T, "S": 5, "rounds": args.rounds}
    for name, (_, _, shape) in runs.items():
        med = {k: sorted(v)[len(v) // 2] for k, v in times[name].items()}
        spread = {k.replace("_ms", "_spread_ms"): max(v) - min(v) for k, v in times[name].items()}
        res[name] = dict(shape, **med, **spread, backward_ms=med["forward_backward_ms"] - med["forward_ms"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
