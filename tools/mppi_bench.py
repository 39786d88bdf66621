"""Times one mppi() iteration (DESIGN.md 4.5.2) per kernel on one GPU next to one ilqr() iteration of the same problem, and prints
one JSON line per physics with the card name and power limit.  CtrlAviary, 65 536 drones (E = 16 384 aviaries of D = 4; with
downwash 4-drone stacks), T = 48 ticks at 240 / 48 Hz, K = --samples.  CUDA events around each launch, [min, median, max] ms over
--reps after --warmup:
  * sample / update / commit: qs_mppi_sample, qs_mppi_update, qs_mppi_commit, and mppi_iter their sum;
  * ilqr_iter: one iLQR iteration (line search, commit, Jacobians, backward pass), without downwash only;
  * sample_substeps_per_s: drone-substeps per second of the sample kernel (N K T substeps per tick / its median)."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from ilqr_grad_bench import timed  # noqa: E402
from jvp_bench import card  # noqa: E402


def run(physics, E, D, T, K, reps, warmup):
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.ilqr import Problem
    from gym_pybullet_drones_b200.mppi import Mppi
    from gym_pybullet_drones_b200.utils.enums import Physics
    rng = np.random.default_rng(0)
    if physics == "PYB_DW":
        xyz = np.array([[0.0, 0.0, 0.5], [0.03, 0.0, 2.0], [0.0, 0.03, 3.5], [0.03, 0.03, 5.0]])
    else:
        xyz = np.stack([rng.uniform(-1, 1, D), rng.uniform(-1, 1, D), rng.uniform(0.5, 1.5, D)], 1)
    env = CtrlAviary(num_drones=D, physics=getattr(Physics, physics), pyb_freq=240, ctrl_freq=48, initial_xyzs=xyz, num_envs=E)
    env.reset()
    dev = env.device
    target = {"pos": env.pos.clone() + torch.tensor(rng.uniform(-0.5, 0.5, (E, D, 3)), device=dev)}
    m = Mppi(env, target, num_steps=T, samples=K)
    cost = torch.empty((2, m.n), dtype=torch.float64, device=dev)
    m.nominal(cost[0])
    out = timed([("sample", lambda: m.sample(0)), ("update", lambda: m.update(0)), ("commit", lambda: m.commit(0, cost[1]))], reps, warmup)
    it = timed([("mppi_iter", lambda: (m.sample(0), m.update(0), m.commit(0, cost[1])))], reps, warmup)
    out.update(it)
    if physics != "PYB_DW":
        p = Problem(env, target, num_steps=T)
        c = torch.empty((2, p.n), dtype=torch.float64, device=dev)
        p.nominal()
        p.cost(c[0])
        p.jacobians()
        p.backward()
        out.update(timed([("ilqr_iter", lambda: (p.line_search(), p.commit(c[0], c[1]), p.jacobians(), p.backward()))], reps, warmup))
    S = env.PYB_STEPS_PER_CTRL
    out["sample_substeps_per_s"] = float("%.4g" % (m.n * K * T * S / (out["sample"][1] * 1e-3)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--E", type=int, default=16384)
    ap.add_argument("--D", type=int, default=4)
    ap.add_argument("--T", type=int, default=48)
    ap.add_argument("--samples", type=int, default=64)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--physics", default="DYN,PYB_DRAG,PYB_DW")
    a = ap.parse_args()
    gpu = card()
    for physics in a.physics.split(","):
        res = run(physics, a.E, a.D, a.T, a.samples, a.reps, a.warmup)
        print(json.dumps(dict(physics=physics, gpu=gpu, drones=a.E * a.D, T=a.T, K=a.samples, **res)))


if __name__ == "__main__":
    main()
