"""Cost of the on-device policy rollout per network shape (SB3 net_arch and activation), against the per-tick path a user has
without it, at the bench shape.

Bench size: MultiHoverAviary, 32 768 aviaries x 2 drones, 240/30 Hz, same-step autoreset, T = 16 ticks per rollout() call, R envs
rotating (every launch finds its state in HBM, as tools/policy_actions_bench.py does).  Per workload (action type, architecture):

  actor         rollout(policy=actor only, noise)
  actor_critic  rollout(policy=actor + critic, noise)
  torch_step    forward_torch (actor + critic) on the current observation + step() of the clipped actions, per tick, on CUDA
                tensors (what collect_rollouts does without the fused rollout)

Architectures: [64, 64] Tanh (the control: qs_rollout's register-resident evaluator, DESIGN.md 6: ~43 / ~63 us on a 400 W card),
the same network forced through qs_rollout_mlp ("general"), [64, 64] ReLU, [128, 128], [256, 256] and [256, 128, 64, 32] Tanh.
The width cap of qs_rollout_mlp is the widest width whose actor_critic is not slower than torch_step here.
The variants of a workload alternate, --runs runs each; times are CUDA events in microseconds per tick of 65 536 drones.
Prints the card and its power limit, one line per workload, then one JSON line.

    python tools/policy_arch_bench.py [--runs 3] [--reps 12] [--envs 4]
"""
import argparse
import copy
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from policy_actions_bench import card, timed  # noqa: E402

D, E, T = 2, 32768, 16
# (name, action type, net_arch, activation, force the general path)
WORKLOADS = (("tanh64x2", "RPM", [64, 64], "tanh", False), ("tanh64x2-general", "RPM", [64, 64], "tanh", True),
             ("relu64x2", "RPM", [64, 64], "relu", False), ("tanh128x2", "RPM", [128, 128], "tanh", False),
             ("tanh256x2", "RPM", [256, 256], "tanh", False), ("tanh256-128-64-32", "RPM", [256, 128, 64, 32], "tanh", False),
             ("pid-tanh64x2", "PID", [64, 64], "tanh", False), ("pid-tanh256x2", "PID", [256, 256], "tanh", False))
VARIANTS = ("actor", "actor_critic", "torch_step")


def policies(in_dim, out_dim, arch, activation, general, seed):
    """(actor only, actor + critic) with random weights: the cost does not depend on the values."""
    from gym_pybullet_drones_b200.policy import MlpPolicy
    ac = MlpPolicy.random(in_dim, out_dim, seed=seed, critic=True, log_std=-0.5, net_arch=arch, activation=activation)
    a = MlpPolicy(ac.actor, ac.log_std, None, activation=activation)
    if general:
        a, ac = copy.copy(a), copy.copy(ac)
        a.classic = ac.classic = False
    return a, ac


def bench_workload(act, arch, activation, general, runs, reps, R, gen):
    from gym_pybullet_drones_b200.envs import MultiHoverAviary
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    envs = [MultiHoverAviary(num_drones=D, physics=Physics.DYN, act=ActionType[act], num_envs=E, autoreset="same_step") for _ in range(R)]
    for e in envs:
        e.reset()
    A, od = envs[0]._A, envs[0]._obs_dim
    actor, actor_critic = policies(D * od, D * A, arch, activation, general, seed=7)
    noise = torch.randn((T, E, D * A), device="cuda", generator=gen)
    outs = {v: [None] * R for v in VARIANTS}

    def roll(v, pol):
        def f(k):
            i = k % R
            outs[v][i] = envs[i].rollout(num_steps=T, out=outs[v][i], policy=pol, noise=noise)
        return f

    def torch_step(k):
        env = envs[k % R]
        for t in range(T):
            raw, _, _ = actor_critic.forward_torch(env._obs_buf[env._cur].view(E, D, od), noise[t])
            env.step(raw.clamp(-1, 1).view(E, D, A))

    fns = {"actor": roll("actor", actor), "actor_critic": roll("actor_critic", actor_critic), "torch_step": torch_step}
    for v in VARIANTS:                                       # warm-up: allocations, carve-out, first launches, cuBLAS
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
    for key, act, arch, activation, general in WORKLOADS:
        out["workloads"][key] = bench_workload(act, arch, activation, general, a.runs, a.reps, a.envs, gen)
        print(key, json.dumps(out["workloads"][key]), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
