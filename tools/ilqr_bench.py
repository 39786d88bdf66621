"""Times one iLQR iteration of BaseAviary.ilqr on one GPU (DESIGN.md 4.5.1) and prints one JSON line per physics with the card
name and power limit read in the same call.  CtrlAviary, 65 536 drones (E = 16 384 aviaries of D = 4), T = 48 ticks at 240 / 48 Hz
(S = 5 substeps), Physics.DYN and PYB_DRAG, hover guess, targets within 0.5 m.  Each step of an iteration is timed with CUDA
events around its launch, [min, median, max] ms over --reps iterations after --warmup:
  * jac:      qs_dyn_tick_jac at the nominal;
  * backward: qs_ilqr_backward, with the bytes it must move computed from the shapes (the Jacobian read, K and k written, the
              states, targets and rpm read once) over its time, and that rate as a share of the H100 SXM data sheet's 3.35 TB/s;
  * line:     qs_ilqr_line_search over the 10 step sizes;
  * commit:   qs_ilqr_commit.
--rpm-bounds motor times the control-limited kernels (qs_ilqr_box_*) with the box (0, MAX_RPM), and reports the share of
rotor-ticks the last backward pass held.  --task picks the targets: spread (within 0.5 m of (0, 0, 1), the default), hover
(within 2 mm of each drone's start: no bound binds, the backward takes the fast path at every tick) or climb (1 m straight up:
rotors saturate)."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from jvp_bench import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def stats(ts):
    ts = sorted(ts)
    return [round(ts[0], 3), round(ts[len(ts) // 2], 3), round(ts[-1], 3)]


def run(physics, E, D, T, reps, warmup, task="spread", rpm_bounds=None):
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.ilqr import Problem
    from gym_pybullet_drones_b200.utils.enums import Physics
    rng = np.random.default_rng(0)
    xyz = np.stack([rng.uniform(-1, 1, D), rng.uniform(-1, 1, D), rng.uniform(0.5, 1.5, D)], 1)
    env = CtrlAviary(num_drones=D, physics=getattr(Physics, physics), pyb_freq=240, ctrl_freq=48, initial_xyzs=xyz, num_envs=E)
    env.reset()
    if task == "spread":
        target = {"pos": torch.tensor(rng.uniform(-0.5, 0.5, (E, D, 3)) + np.array([0.0, 0.0, 1.0]), device=env.device)}
    else:
        pos = env.pos.to(torch.float64).clone()
        if task == "climb":
            pos[..., 2] += 1.0
        else:
            pos += torch.as_tensor(rng.uniform(-2e-3, 2e-3, tuple(pos.shape)), dtype=torch.float64, device=env.device)
        target = {"pos": pos}
    p = Problem(env, target, num_steps=T, rpm_bounds=rpm_bounds)
    n = p.n
    cost = torch.empty((2, n), dtype=torch.float64, device=env.device)
    p.nominal()
    p.cost(cost[0])
    steps = (("jac", p.jacobians), ("backward", p.backward), ("line", p.line_search), ("commit", lambda: p.commit(cost[0], cost[1])))
    times = {k: [] for k, _ in steps}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(steps) + 1)]
    for it in range(warmup + reps):
        ev[0].record()
        for j, (_, fn) in enumerate(steps):
            fn()
            ev[j + 1].record()
        torch.cuda.synchronize()
        accepted = int((cost[1] < cost[0]).sum().item())
        cost[0].copy_(cost[1])
        if it >= warmup:
            for j, (k, _) in enumerate(steps):
                times[k].append(ev[j].elapsed_time(ev[j + 1]))
    C = p.jac.shape[-1]
    nz = p.nz
    # the backward's compulsory traffic: the Jacobian, the nominal states, targets and rpm read, K and k written
    bwd_bytes = 8 * T * n * (13 * C + 13 + 13 + 4 + 4 * nz + 4)
    med = {k: stats(v)[1] for k, v in times.items()}
    held = None if p.active is None else round(float((p.active != 0).float().mean()), 4)
    return {"physics": physics, "task": task, "rpm_bounds": rpm_bounds, "held_share": held, "drones": n, "T": T, "nz": nz,
            "ms": {k: stats(v) for k, v in times.items()},
            "iteration_ms": round(sum(med.values()), 3), "backward_GB": round(bwd_bytes / 1e9, 3),
            "backward_TB_per_s": round(bwd_bytes / (med["backward"] * 1e-3) / 1e12, 3),
            "backward_share_of_3.35TB_per_s": round(bwd_bytes / (med["backward"] * 1e-3) / HBM_BYTES_PER_S, 3),
            "accepted_in_last_iteration": accepted}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=16384)
    ap.add_argument("--drones", type=int, default=4)
    ap.add_argument("--T", type=int, default=48)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--physics", default="DYN,PYB_DRAG")
    ap.add_argument("--task", default="spread", choices=["spread", "hover", "climb"])
    ap.add_argument("--rpm-bounds", default=None, choices=["motor"])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ilqr_bench: no CUDA device")
    name = card()
    for physics in a.physics.split(","):
        r = run(physics, a.envs, a.drones, a.T, a.reps, a.warmup, a.task, a.rpm_bounds)
        r["card"] = name
        print(json.dumps(r))
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
