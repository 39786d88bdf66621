"""Cost of next-step autoreset in rollout(), against same-step rollouts and against T x step().

Bench size: MultiHoverAviary, 32 768 aviaries x 2 drones, 240/30 Hz, T = 16 ticks per rollout() call, R envs per autoreset mode
rotating (every launch finds its state in HBM).  The step counters start spread over the 8 s episode (242 ticks), so about 1/242
of the aviaries finish per tick, as in steady state, as long as the drones stay inside the bounds.  Two action sources, as
tools/rollout_final_bench.py:

  hover   every action is 0 (action rollouts: a zero action tensor; policy rollouts: an actor whose output layer is zero and no
          noise): only the time-out ends an episode
  random  uniform device-generated actions / a random actor with Gaussian noise, as bench.py: most aviaries leave the bounds
          within a few ticks

Per action type (RPM, PID) and source:

  same_actions        same-step env, rollout() with the actions
  next_actions        next-step env, rollout() with the actions
  same_critic         same-step env, rollout(policy=actor + critic, noise)
  same_critic_final   the same with final_values=True (the time-out bootstrap values of same-step autoreset)
  next_critic         next-step env, rollout(policy=actor + critic, noise): the bootstrap values are values[k+1]
  next_steps          next-step env, T calls of step() (the actions from a tensor: zeros, or uniform for random)

The variants alternate, --runs runs each; times are CUDA events in microseconds per tick of 65 536 drones.  Also printed: the
share of aviaries reset per tick under next-step autoreset.  Prints the card and its power limit, one line per workload, then one
JSON line.

    python tools/rollout_next_bench.py [--runs 3] [--reps 12] [--envs 4]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.rollout_final_bench import EPISODE_TICKS, actor_critic, card  # noqa: E402

D, E, T = 2, 32768, 16
WORKLOADS = (("RPM", "hover"), ("PID", "hover"), ("RPM", "random"), ("PID", "random"))
VARIANTS = ("same_actions", "next_actions", "same_critic", "same_critic_final", "next_critic", "next_steps")


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
    envs = {}
    for mode in ("same_step", "next_step"):
        envs[mode] = [MultiHoverAviary(num_drones=D, physics=Physics.DYN, act=ActionType[act], num_envs=E, autoreset=mode)
                      for _ in range(R)]
        for env in envs[mode]:
            env.reset()
            env.set_state(step_counter=rng.integers(0, EPISODE_TICKS, E) * env.PYB_STEPS_PER_CTRL)
    A, od = envs["same_step"][0]._A, envs["same_step"][0]._obs_dim
    hover = source == "hover"
    pol = actor_critic(D * od, D * A, gen, hover)
    noise = None if hover else torch.randn((T, E, D * A), device="cuda", generator=gen)
    zeros = torch.zeros((T, E, D, A), device="cuda")
    step_actions = zeros if hover else (torch.rand((T, E, D, A), device="cuda", generator=gen) * 2 - 1)
    act_opts = dict(actions=zeros) if hover else dict(num_steps=T)
    critic = dict(policy=pol, noise=noise, num_steps=T)
    plan = {"same_actions": ("same_step", act_opts), "next_actions": ("next_step", act_opts),
            "same_critic": ("same_step", critic), "same_critic_final": ("same_step", dict(critic, final_values=True)),
            "next_critic": ("next_step", critic)}
    outs = {v: [None] * R for v in VARIANTS}

    def roll(v):
        mode, o = plan[v]

        def f(k):
            i = k % R
            outs[v][i] = envs[mode][i].rollout(seed=k, out=outs[v][i], **o)
        return f

    def steps(k):
        env = envs["next_step"][k % R]
        for j in range(T):
            env.step(step_actions[j])

    fns = {v: roll(v) for v in plan}
    fns["next_steps"] = steps
    for v in VARIANTS:                                       # warm-up: allocations, carve-out, first launches
        for k in range(R):
            fns[v](k)
    res = {v: [] for v in VARIANTS}
    for _ in range(runs):
        for v in VARIANTS:
            res[v].append(round(timed(fns[v], reps), 2))
    reset = torch.stack([o["autoreset"] for o in outs["next_critic"]])         # [R, T, E]
    res["reset_per_tick"] = round(float(reset.float().mean()), 5)
    del envs, outs
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=12, help="rollout() calls of T = 16 ticks per timed run")
    ap.add_argument("--envs", type=int, default=4, help="envs per autoreset mode rotating through the timed loop")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("rollout_next_bench.py needs a CUDA device")
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
