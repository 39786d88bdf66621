"""Cost of the terminal observations and their critic values in rollout() (final_obs / final_values, same-step autoreset).

Bench size: MultiHoverAviary, 32 768 aviaries x 2 drones, 240/30 Hz, same-step autoreset, T = 16 ticks per rollout() call, R envs
rotating (every launch finds its state in HBM).  The step counters start spread over the 8 s episode (242 ticks), so about 1/242
of the aviaries finish per tick, as in steady state, as long as the drones stay inside the bounds.  Two action sources:

  hover   every action is 0 (action rollouts: a zero action tensor; policy rollouts: an actor whose output layer is zero and no
          noise), so the drones hover and only the time-out ends an episode: about 1/242 of the aviaries finish per tick
  random  uniform device-generated actions / a random actor with Gaussian noise, as bench.py: the drones leave the bounds within
          a few ticks, about 10 % of the aviaries finish per tick and nearly every CTA runs the critic pass (the worst case)

Per action type (RPM, PID) and source:

  actions            rollout() with the actions
  actions_final_obs  the same with final_obs=True
  critic             rollout(policy=actor + critic, noise)
  critic_final_vals  the same with final_values=True
  critic_final_both  the same with final_obs=True and final_values=True

The variants alternate, --runs runs each; times are CUDA events in microseconds per tick of 65 536 drones.  Also printed: the
share of aviaries that finished per tick and the share of policy CTA-ticks (32 aviaries per CTA) that held a finished aviary,
i.e. ran the critic pass.  Prints the card and its power limit, one line per workload, then one JSON line.

    python tools/rollout_final_bench.py [--runs 3] [--reps 12] [--envs 4]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

D, E, T = 2, 32768, 16
EPISODE_TICKS = 242                       # ticks until the 8 s time-out at 240/30 Hz (the first with sc / 240 > 8)
WORKLOADS = (("RPM", "hover"), ("PID", "hover"), ("RPM", "random"), ("PID", "random"))
VARIANTS = ("actions", "actions_final_obs", "critic", "critic_final_vals", "critic_final_both")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=20).stdout.strip().splitlines()[0]
        name, pl = [c.strip() for c in out.split(",")]
        return name, pl
    except Exception:
        return torch.cuda.get_device_name(), "unknown"


def actor_critic(in_dim, out_dim, gen, zero_actions):
    """Random weights (the cost does not depend on the values); zero_actions: the actor's output layer is zero."""
    from gym_pybullet_drones_b200.policy import MlpPolicy
    dev = torch.device("cuda")

    def lin(i, o):
        return ((torch.randn((i, o), device=dev, generator=gen) / i ** 0.5).float(), (0.01 * torch.randn((o,), device=dev, generator=gen)).float())
    out = lin(64, out_dim)
    if zero_actions:
        out = (torch.zeros_like(out[0]), torch.zeros_like(out[1]))
    return MlpPolicy([lin(in_dim, 64), lin(64, 64), out], torch.full((out_dim,), -0.5, device=dev),
                     [lin(in_dim, 64), lin(64, 64), lin(64, 1)])


def timed(fn, reps):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ev0.record()
    for k in range(reps):
        fn(k)
    ev1.record()
    torch.cuda.synchronize()
    return 1e3 * ev0.elapsed_time(ev1) / (reps * T)


def bench_workload(act, source, runs, reps, R, gen):
    from gym_pybullet_drones_b200.envs import MultiHoverAviary
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    rng = np.random.default_rng(0)
    envs = [MultiHoverAviary(num_drones=D, physics=Physics.DYN, act=ActionType[act], num_envs=E, autoreset="same_step")
            for _ in range(R)]
    for env in envs:
        env.reset()
        env.set_state(step_counter=rng.integers(0, EPISODE_TICKS, E) * env.PYB_STEPS_PER_CTRL)
    A, od = envs[0]._A, envs[0]._obs_dim
    hover = source == "hover"
    pol = actor_critic(D * od, D * A, gen, hover)
    noise = None if hover else torch.randn((T, E, D * A), device="cuda", generator=gen)
    zeros = torch.zeros((T, E, D, A), device="cuda")
    outs = {v: [None] * R for v in VARIANTS}
    act_opts = dict(actions=zeros) if hover else dict(num_steps=T)
    opts = {"actions": act_opts, "actions_final_obs": dict(final_obs=True, **act_opts), "critic": dict(policy=pol, noise=noise),
            "critic_final_vals": dict(policy=pol, noise=noise, final_values=True),
            "critic_final_both": dict(policy=pol, noise=noise, final_obs=True, final_values=True)}

    def roll(v):
        def f(k):
            i = k % R
            o = dict(opts[v])
            if "policy" in o:
                o["num_steps"] = T
            outs[v][i] = envs[i].rollout(seed=k, out=outs[v][i], **o)
        return f

    fns = {v: roll(v) for v in VARIANTS}
    for v in VARIANTS:                                       # warm-up: allocations, carve-out, first launches
        for k in range(R):
            fns[v](k)
    res = {v: [] for v in VARIANTS}
    for _ in range(runs):
        for v in VARIANTS:
            res[v].append(round(timed(fns[v], reps), 2))
    # how often aviaries finished, and how often a policy CTA (64 // D aviaries) held one, over the last critic_final_vals outputs
    done = torch.stack([o["terminated"] | o["truncated"] for o in outs["critic_final_vals"]])      # [R, T, E]
    res["finished_per_tick"] = round(float(done.float().mean()), 5)
    res["cta_ticks_with_critic_pass"] = round(float(done.view(R, T, E // (64 // D), 64 // D).any(-1).float().mean()), 4)
    del envs, outs
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=12, help="rollout() calls of T = 16 ticks per timed run")
    ap.add_argument("--envs", type=int, default=4, help="envs rotating through the timed loop")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("rollout_final_bench.py needs a CUDA device")
    name, pl = card()
    print("card: %s, power limit %s" % (name, pl), flush=True)
    gen = torch.Generator(device="cuda").manual_seed(7)
    out = {"card": name, "power_limit": pl, "drones": E * D, "ticks_per_rollout": T, "runs": a.runs, "envs": a.envs,
           "unit": "us per tick", "workloads": {}}
    for act, source in WORKLOADS:
        key = "%s/%s" % (act, source)
        out["workloads"][key] = bench_workload(act, source, a.runs, a.reps, a.envs, gen)
        print(key, json.dumps(out["workloads"][key]), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
