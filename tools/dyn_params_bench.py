"""Cost of the per-aviary physical-constants table (QsState.phys, env.set_physical_params) on the device-resident step and
rollout: three variants timed in alternation, three runs each, in one process.

  none    : no table (the kernels of ABI 3, constants in QsParams)
  nominal : set_physical_params() -- every row holds the constructor's model
  random  : m, J x U[0.7, 1.3], kf, km x U[0.8, 1.2], arm, thrust2weight x U[0.9, 1.1] per aviary

Workloads: the headline one of bench.py (MultiHoverAviary 32 768 x 2, RPM, 240/30, same-step autoreset, R rotating batches,
fresh uniform actions, CUDA events around K steps), the same with ONE_D_RPM (A = 1), and rollout() of 32 ticks with device
actions and with an on-device policy (random weights).  Prints the card and its power limit, then one JSON line.

    python tools/dyn_params_bench.py [--steps 400] [--batches 8] [--runs 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

D, E = 2, 32768
VARIANTS = ("none", "nominal", "random")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=20).stdout.strip().splitlines()[0]
        name, pl = [c.strip() for c in out.split(",")]
        return name, pl
    except Exception:
        return torch.cuda.get_device_name(), "unknown"


def randomise(env, gen):
    def u(lo, hi):
        return lo + (hi - lo) * torch.rand((env.num_envs,), device=env.device, dtype=torch.float64, generator=gen)
    nom = env.physical_params()
    env.set_physical_params(m=nom["m"] * u(0.7, 1.3), ixx=nom["ixx"] * u(0.7, 1.3), iyy=nom["iyy"] * u(0.7, 1.3),
                            izz=nom["izz"] * u(0.7, 1.3), kf=nom["kf"] * u(0.8, 1.2), km=nom["km"] * u(0.8, 1.2),
                            arm=nom["arm"] * u(0.9, 1.1), thrust2weight=nom["thrust2weight"] * u(0.9, 1.1))


def make(variant, act, R, gen):
    from gym_pybullet_drones_b200.envs import MultiHoverAviary
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    envs = [MultiHoverAviary(num_drones=D, physics=Physics.DYN, act=act, num_envs=E, autoreset="same_step") for _ in range(R)]
    for e in envs:
        if variant == "nominal":
            e.set_physical_params()
        elif variant == "random":
            randomise(e, gen)
        e.reset()
    return envs


def time_steps(envs, acts, steps):
    R = len(envs)
    for k in range(20):
        envs[k % R].step(acts[k % R][0])
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ev0.record()
    for k in range(steps):
        envs[k % R].step(acts[k % R][(k // R) % len(acts[0])])
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / steps


def time_rollout(envs, T, reps, policy=None, noise=None):
    outs = [None] * len(envs)
    for i, e in enumerate(envs):
        outs[i] = e.rollout(num_steps=T, seed=i, policy=policy, noise=noise)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ev0.record()
    for k in range(reps):
        i = k % len(envs)
        outs[i] = envs[i].rollout(num_steps=T, seed=k, out=outs[i], policy=policy, noise=noise)
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / (reps * T)


def random_policy(in_dim, out_dim, gen):
    from gym_pybullet_drones_b200.policy import MlpPolicy
    dev = torch.device("cuda")

    def lin(i, o):
        return ((torch.randn((i, o), device=dev, generator=gen) / i ** 0.5).float(), (0.01 * torch.randn((o,), device=dev, generator=gen)).float())
    actor = [lin(in_dim, 64), lin(64, 64), lin(64, out_dim)]
    critic = [lin(in_dim, 64), lin(64, 64), lin(64, 1)]
    return MlpPolicy(actor, torch.full((out_dim,), -0.5, device=dev), critic)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--rollout-reps", type=int, default=8)
    a = ap.parse_args()
    from gym_pybullet_drones_b200.utils.enums import ActionType
    name, pl = card()
    print("card: %s, power limit %s" % (name, pl), flush=True)
    gen = torch.Generator(device="cuda").manual_seed(7)
    res = {"card": name, "power_limit": pl, "drones": E * D, "steps": a.steps, "batches": a.batches}
    for label, act, width in (("step_rpm", ActionType.RPM, 4), ("step_one_d_rpm", ActionType.ONE_D_RPM, 1)):
        sets = {v: make(v, act, a.batches, gen) for v in VARIANTS}
        acts = [[torch.rand((E, D, width), device="cuda", generator=gen) * 2 - 1 for _ in range(8)] for _ in range(a.batches)]
        ms = {v: [] for v in VARIANTS}
        for r in range(a.runs):
            for v in VARIANTS:
                ms[v].append(time_steps(sets[v], acts, a.steps))
        res[label] = {v: {"us_per_step": [round(1e3 * x, 2) for x in ms[v]]} for v in VARIANTS}
        print(label, json.dumps(res[label]), flush=True)
        del sets, acts
        torch.cuda.empty_cache()
    for label, pol in (("rollout32_actions", False), ("rollout32_policy", True)):
        sets = {v: make(v, ActionType.RPM, 2, gen) for v in VARIANTS}
        policy = noise = None
        if pol:
            e0 = sets["none"][0]
            policy = random_policy(D * e0._obs_dim, D * 4, gen)
            noise = torch.randn((32, E, D * 4), device="cuda", generator=gen)
        ms = {v: [] for v in VARIANTS}
        for r in range(a.runs):
            for v in VARIANTS:
                ms[v].append(time_rollout(sets[v], 32, a.rollout_reps, policy, noise))
        res[label] = {v: {"us_per_tick": [round(1e3 * x, 2) for x in ms[v]]} for v in VARIANTS}
        print(label, json.dumps(res[label]), flush=True)
        del sets
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
