"""Times the forward mode of the differentiable trajectories on one GPU (DESIGN.md 4.5) and prints one JSON line with the card name
and power limit read in the same call.  At E = 4 096 and 65 536 aviaries of one drone, T = 1 and 32 ticks of S = 8 substeps
(240 / 30 Hz), Physics.DYN and GND|DRAG (the latter through the C ABI's effects; no Physics member has both):
  * linearise: BaseAviary.linearise (qs_dyn_traj + qs_dyn_tick_jac), all of A, B (and B_last);
  * per_tick_vjp: the same Jacobians from the existing VJP, per tick a T = 1 differentiable_rollout from the stored state and
    13 torch.autograd.grad calls with unit cotangents (rows of A, B, B_last for every drone at once) -- at T = 32 the 32 ticks;
  * jvp / vjp: one forward-mode product (torch.autograd.forward_ad through differentiable_rollout) against one reverse-mode
    product (torch.autograd.grad) of the same T-tick trajectory, forward included in both.
CUDA events around each call (each ends in the device's work for that call), [min, median, max] ms over --reps after warm-up."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.autograd.forward_ad as fwAD

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

KEYS = ("pos", "quat", "vel", "rpy_rates")


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
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return [round(ts[0], 3), round(ts[len(ts) // 2], 3), round(ts[-1], 3)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[4096, 65536])
    ap.add_argument("--ticks", type=int, nargs="+", default=[1, 32])
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("jvp_bench.py measures on a GPU: none found")
    from gym_pybullet_drones_b200 import _native as N
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils.enums import Physics
    res = {"card": card(), "D": 1, "S": 8, "runs": []}
    for E in args.envs:
        for name, physics, eff in (("dyn", Physics.DYN, 0), ("gnd_drag", Physics.PYB_DRAG, N.EFFECT_GND | N.EFFECT_DRAG)):
            env = CtrlAviary(num_drones=1, physics=physics, pyb_freq=240, ctrl_freq=30, num_envs=E)
            env.reset()
            env._effects = eff                       # GND|DRAG is reachable through the C ABI only
            for T in args.ticks:
                g = torch.Generator(device=env.device).manual_seed(T)
                rpm = env.HOVER_RPM * (1 + 0.05 * (2 * torch.rand((T, E, 1, 4), generator=g, device=env.device, dtype=torch.float64) - 1))
                row = {"E": E, "T": T, "effects": name}
                row["linearise_ms"] = timed(lambda: env.linearise(rpm), args.reps)
                lin = env.linearise(rpm)
                start = {k: torch.cat([getattr(env, k)[None], lin[k][:-1]]) for k in KEYS}
                drag = eff & N.EFFECT_DRAG

                def per_tick():
                    last = env._last_rpm.clone().reshape(E, 1, 4)
                    for k in range(T):
                        r = rpm[k:k + 1].clone().requires_grad_(True)
                        st = {key: v[k].clone().requires_grad_(True) for key, v in start.items()}
                        lr = last.clone().requires_grad_(bool(drag))
                        out = env.differentiable_rollout(r, state=st, last_rpm=lr)
                        flat = torch.cat([out[key] for key in KEYS], dim=-1)
                        leaves = [st[key] for key in KEYS] + [r] + ([lr] if drag else [])
                        for j in range(13):
                            cot = torch.zeros_like(flat)
                            cot[..., j] = 1.0
                            torch.autograd.grad(flat, leaves, cot, retain_graph=j < 12)
                        last = rpm[k].clamp(0.0, env.MAX_RPM)
                row["per_tick_vjp_ms"] = timed(per_tick, max(2, args.reps // 2))
                v = torch.randn(rpm.shape, generator=g, device=env.device, dtype=torch.float64)

                def jvp():
                    with fwAD.dual_level():
                        out = env.differentiable_rollout(fwAD.make_dual(rpm, v))
                        return fwAD.unpack_dual(out["pos"]).tangent

                r = rpm.clone().requires_grad_(True)
                row["jvp_ms"] = timed(jvp, args.reps)
                row["vjp_ms"] = timed(lambda: torch.autograd.grad(env.differentiable_rollout(r)["pos"].sum(), r), args.reps)
                res["runs"].append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
                del lin, start
            del env
            torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
