"""Cost of the on-device policy rollout with the embedded controller (PID, VEL, ONE_D_PID) and with the DYN+ effects, against
the physics alone and against the per-tick path a user has without it.

Bench size: MultiHoverAviary, 32 768 aviaries x 2 drones, 240/30 Hz, same-step autoreset, T = 16 ticks per rollout() call, R
envs rotating (every launch finds its state in HBM, as tools/policy_quick.py does).  Per workload (action type, physics):

  actor         rollout(policy=actor only, noise)
  actor_critic  rollout(policy=actor + critic, noise)
  actions       rollout() with device-generated actions: the physics alone
  torch_step    forward_torch (actor + critic) on the current observation + step() of the clipped actions, per tick, on CUDA
                tensors (what collect_rollouts does without the fused rollout)

Control in the same process: the RPM / DYN policy rollout (DESIGN.md 6: 43.3 us actor, 63.2 us with the critic on a 400 W card).
The variants of a workload alternate, --runs runs each; times are CUDA events in microseconds per tick of 65 536 drones.
Prints the card and its power limit, one line per workload, then one JSON line.

    python tools/policy_actions_bench.py [--runs 3] [--reps 12] [--envs 4]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

D, E, T = 2, 32768, 16
WORKLOADS = (("RPM", "DYN"), ("PID", "DYN"), ("VEL", "DYN"), ("ONE_D_PID", "DYN"), ("RPM", "PYB_GND_DRAG_DW"), ("PID", "PYB_GND_DRAG_DW"))
VARIANTS = ("actor", "actor_critic", "actions", "torch_step")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=20).stdout.strip().splitlines()[0]
        name, pl = [c.strip() for c in out.split(",")]
        return name, pl
    except Exception:
        return torch.cuda.get_device_name(), "unknown"


def policies(in_dim, out_dim, gen):
    """(actor only, actor + critic) with random weights: the cost does not depend on the values."""
    from gym_pybullet_drones_b200.policy import MlpPolicy
    dev = torch.device("cuda")

    def lin(i, o):
        return ((torch.randn((i, o), device=dev, generator=gen) / i ** 0.5).float(), (0.01 * torch.randn((o,), device=dev, generator=gen)).float())
    actor = [lin(in_dim, 64), lin(64, 64), lin(64, out_dim)]
    critic = [lin(in_dim, 64), lin(64, 64), lin(64, 1)]
    log_std = torch.full((out_dim,), -0.5, device=dev)
    return MlpPolicy(actor, log_std), MlpPolicy(actor, log_std, critic)


def timed(fn, reps, ticks_per_rep):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ev0.record()
    for k in range(reps):
        fn(k)
    ev1.record()
    torch.cuda.synchronize()
    return 1e3 * ev0.elapsed_time(ev1) / (reps * ticks_per_rep)


def bench_workload(act, physics, runs, reps, R, gen):
    from gym_pybullet_drones_b200.envs import MultiHoverAviary
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    envs = [MultiHoverAviary(num_drones=D, physics=Physics[physics], act=ActionType[act], num_envs=E, autoreset="same_step")
            for _ in range(R)]
    for e in envs:
        e.reset()
    A, od = envs[0]._A, envs[0]._obs_dim
    actor, actor_critic = policies(D * od, D * A, gen)
    noise = torch.randn((T, E, D * A), device="cuda", generator=gen)
    outs = {v: [None] * R for v in VARIANTS}

    def roll(v, pol):
        def f(k):
            i = k % R
            outs[v][i] = envs[i].rollout(num_steps=T, seed=k, out=outs[v][i], policy=pol, noise=None if pol is None else noise)
        return f

    def torch_step(k):
        i = k % R
        env = envs[i]
        for t in range(T):
            raw, _, _ = actor_critic.forward_torch(env._obs_buf[env._cur].view(E, D, od), noise[t])
            env.step(raw.clamp(-1, 1).view(E, D, A))

    fns = {"actor": roll("actor", actor), "actor_critic": roll("actor_critic", actor_critic), "actions": roll("actions", None),
           "torch_step": torch_step}
    for v in VARIANTS:                                       # warm-up: allocations, carve-out, first launches
        for k in range(R):
            fns[v](k)
    res = {v: [] for v in VARIANTS}
    for _ in range(runs):
        for v in VARIANTS:
            res[v].append(round(timed(fns[v], reps if v != "torch_step" else max(2, reps // 4), T), 2))
    del envs, outs
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=12, help="rollout() calls of T = 16 ticks per timed run")
    ap.add_argument("--envs", type=int, default=4, help="envs rotating through the timed loop")
    a = ap.parse_args()
    name, pl = card()
    print("card: %s, power limit %s" % (name, pl), flush=True)
    gen = torch.Generator(device="cuda").manual_seed(7)
    out = {"card": name, "power_limit": pl, "drones": E * D, "ticks_per_rollout": T, "runs": a.runs, "envs": a.envs,
           "unit": "us per tick", "workloads": {}}
    for act, physics in WORKLOADS:
        key = "%s/%s" % (act, physics)
        out["workloads"][key] = bench_workload(act, physics, a.runs, a.reps, a.envs, gen)
        print(key, json.dumps(out["workloads"][key]), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
