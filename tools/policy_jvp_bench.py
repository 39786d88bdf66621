"""Times the forward mode of the policy loop on one GPU (DESIGN.md 4.5) and prints one JSON line with the card name and power
limit read in the same call.  MultiHoverAviary, ActionType.RPM at 30 Hz control (B = 15 buffered actions, S = 8 substeps of
240 Hz), E = 256 and 4 096 aviaries of D = 1 and 2 drones, T = 32 ticks, [64, 64] Tanh and [256, 256] ReLU actors, Physics.DYN and
PYB_DRAG:
  * linearise: BaseAviary.linearise(policy=) (qs_dyn_policy_traj + qs_dyn_policy_tick_jac), all of A, B, K for the T ticks;
  * jvp: one forward-AD pass of differentiable_rollout(policy=) along a direction of the initial state, the noise and every
    parameter of the actor, forward included;
  * jacfwd_tick: the baseline, the same Jacobian of ONE tick from torch.func.jacfwd of the float64 reference tick
    (tests/policy_jvp_testlib.ref_tick: the state, ang_v, history, drag's rpm and delta columns), vmapped over the aviaries,
    at the tick's inputs; multiply by T for a trajectory (every tick costs the same).
linearise and jacfwd_tick are timed in alternating windows.  CUDA events around each call (each ends in the device's work for that
call), [min, median, max] ms over --reps after warm-up."""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.autograd.forward_ad as fwAD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from jvp_bench import card  # noqa: E402

KEYS = ("pos", "quat", "vel", "rpy_rates")


def stats(ts):
    ts = sorted(ts)
    return [round(ts[0], 3), round(ts[len(ts) // 2], 3), round(ts[-1], 3)]


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def baseline(env, pol, theta, lin):
    """fn() -> the tick-0 Jacobians of every aviary from vmap(jacfwd(reference tick))"""
    from policy_jvp_testlib import ref_tick
    E, D, A, B, dev = env._E, env._D, env._A, env._B, env.device
    tick = ref_tick(env._P, env._effects, env.PYB_STEPS_PER_CTRL, pol.activation, [t.detach() for t in theta], None, device=dev)
    x = torch.cat([lin[k][0] for k in KEYS], dim=-1)                                  # [E, D, 13]
    obs = lin["obs"][0]                                                                # [E, D, od]
    ang, hist = obs[..., 9:12], obs[..., 12:].reshape(E, D, B, A)
    up = torch.full((E, D, 4), float(env.HOVER_RPM), dtype=torch.float64, device=dev)
    from gym_pybullet_drones_b200.params import physical_rows
    with torch.cuda.device(dev):
        rows = physical_rows(env.DRONE_MODEL, env.physical_params(), env.G)
    raw_in = torch.zeros((E, D * A), dtype=torch.float64, device=dev)
    J = torch.func.vmap(torch.func.jacfwd(tick, argnums=(0, 1, 2, 3, 5)))
    return lambda: J(x, ang, hist, up, rows, raw_in)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[256, 4096])
    ap.add_argument("--drones", type=int, nargs="+", default=[1, 2])
    ap.add_argument("--ticks", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-baseline", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("policy_jvp_bench.py measures on a GPU: none found")
    from gym_pybullet_drones_b200.envs import MultiHoverAviary
    from gym_pybullet_drones_b200.policy import MlpPolicy
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    T = args.ticks
    res = {"card": card(), "ctrl_hz": 30, "S": 8, "T": T, "runs": []}
    for E in args.envs:
        for D in args.drones:
            for physics in ("DYN", "PYB_DRAG"):
                xyz = np.stack([0.5 * np.arange(D), np.zeros(D), np.full(D, 1.0)], 1)
                env = MultiHoverAviary(num_drones=D, initial_xyzs=xyz, act=ActionType.RPM, physics=Physics[physics], pyb_freq=240,
                                       ctrl_freq=30, num_envs=E)
                env.reset()
                for arch, act in (([64, 64], "tanh"), ([256, 256], "relu")):
                    pol = MlpPolicy.random(D * env._obs_dim, D * env._A, seed=1, critic=False, log_std=-1.0, net_arch=arch,
                                           activation=act)
                    theta = [t.detach() for t in pol.parameters64()]
                    noise = torch.randn((T, E, D * env._A), dtype=torch.float64, device=env.device)
                    row = {"E": E, "D": D, "physics": physics, "actor": "%s %s" % (arch, act)}
                    lin_fn = lambda: env.linearise(policy=pol, params=theta, noise=noise, num_steps=T)
                    lin = lin_fn()
                    row["jac_doubles"] = int(lin["A"].shape[-1] + lin["B"].shape[-1]) ** 2 * T * E
                    base = None
                    if not args.no_baseline:
                        try:
                            base = baseline(env, pol, theta, lin)
                            base()
                        except (RuntimeError, torch.cuda.OutOfMemoryError) as err:
                            row["jacfwd_tick_error"] = str(err).splitlines()[0][:200]
                            base = None
                    for _ in range(2):
                        lin_fn()
                    torch.cuda.synchronize()
                    t_lin, t_base = [], []
                    for _ in range(args.reps):
                        t_lin.append(event_ms(lin_fn))
                        if base is not None:
                            t_base.append(event_ms(base))
                    row["linearise_ms"] = stats(t_lin)
                    if t_base:
                        row["jacfwd_tick_ms"] = stats(t_base)
                        row["jacfwd_T_ticks_ms_est"] = round(stats(t_base)[1] * T, 3)
                    V = {"state": {k: torch.randn_like(getattr(env, k)) for k in KEYS}, "noise": torch.randn_like(noise),
                         "params": [torch.randn_like(t) for t in theta]}

                    def jvp():
                        with fwAD.dual_level():
                            st = {k: fwAD.make_dual(getattr(env, k).clone(), V["state"][k]) for k in KEYS}
                            out = env.differentiable_rollout(policy=pol, params=[fwAD.make_dual(t, v) for t, v in zip(theta, V["params"])],
                                                             noise=fwAD.make_dual(noise, V["noise"]), num_steps=T, state=st)
                            return fwAD.unpack_dual(out["pos"]).tangent
                    for _ in range(2):
                        jvp()
                    torch.cuda.synchronize()
                    row["jvp_ms"] = stats([event_ms(jvp) for _ in range(args.reps)])
                    res["runs"].append(row)
                    print(json.dumps(row), file=sys.stderr, flush=True)
                    del lin, base
                    torch.cuda.empty_cache()
                del env
    print(json.dumps(res))


if __name__ == "__main__":
    main()
