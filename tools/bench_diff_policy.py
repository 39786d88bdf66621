"""Times BaseAviary.differentiable_rollout(policy=) forward + backward (two kernel launches and one batched actor pass) against
the per-tick composition a user could write without it: differentiable_rollout(rpm[k:k+1]) + the observation and the actor in
torch, T times (the composition has no access to R_last, so it feeds the body rates as ang_v, and it leaves last_rpm out: the
same launches and shapes, not the same numbers).  HoverAviary with RPM actions, D = 1, T = 32 ticks at 240 / 30 Hz, E = 4 096 and 32 768 aviaries, a
[64, 64] Tanh actor and a [256, 256] one.  CUDA events around windows of about 0.4 s of whole forward + backward calls, the two sides alternating, after a
warm-up of every shape; QS_LIBQUADSIM selects the library (an A/B build of the kernels);
the card's name and power limit are read in the same run.  Prints one JSON line.

    python tools/bench_diff_policy.py [--windows 5] [--envs 4096 32768]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

T = 32


def fused(env, pol, theta, target):
    out = env.differentiable_rollout(policy=pol, params=theta, num_steps=T)
    (((out["pos"] - target) ** 2).sum() + 1e-3 * (out["actions"] ** 2).sum()).backward()


def per_tick(env, pol, theta, target):
    from gym_pybullet_drones_b200.diff import actor64
    E = env._E
    st = {k: getattr(env, k).clone() for k in ("pos", "quat", "vel", "rpy_rates")}
    hist = env._obs_buf[env._cur][:, 12:].double().reshape(E, 1, env._B, env._A)
    loss = 0.0
    for _ in range(T):
        q = st["quat"]
        x, y, z, w = q.unbind(-1)
        rpy = torch.stack([torch.atan2(2 * (y * z + w * x), w * w - x * x - y * y + z * z), torch.asin(-2 * (x * z - w * y)),
                           torch.atan2(2 * (x * y + w * z), w * w + x * x - y * y - z * z)], dim=-1)
        obs = torch.cat([st["pos"], rpy, st["vel"], st["rpy_rates"], hist.reshape(E, 1, -1)], dim=-1)   # ang_v ~ body rates
        raw = actor64(theta, pol.activation, obs.reshape(E, -1)).reshape(E, 1, env._A)
        a = raw.clamp(-1, 1)
        hist = torch.cat([hist[:, :, 1:], a[:, :, None, :]], dim=2)
        st = {k: v[0] for k, v in env.differentiable_rollout((env.HOVER_RPM * (1 + 0.05 * a))[None], state=st).items()}
        loss = loss + ((st["pos"] - target) ** 2).sum() + 1e-3 * (raw ** 2).sum()
    loss.backward()


def window_ms(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def alternate(f, c, windows, target_ms=400.0):
    """Per-call times [min, median, max] over `windows` timed windows of each side, the two sides alternating; a window holds
    enough calls for about target_ms of device time."""
    f(); c()
    torch.cuda.synchronize()
    rf, rc = (max(1, int(target_ms / window_ms(g, 1))) for g in (f, c))
    tf, tc = [], []
    for _ in range(windows):
        tf.append(window_ms(f, rf))
        tc.append(window_ms(c, rc))
    stat = lambda t: [round(x, 3) for x in (min(t), sorted(t)[len(t) // 2], max(t))]
    return stat(tf), stat(tc), rf, rc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--envs", type=int, nargs="+", default=[4096, 32768])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_diff_policy.py measures on a CUDA device; none is available")
    from gym_pybullet_drones_b200.envs import HoverAviary
    from gym_pybullet_drones_b200.policy import MlpPolicy
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    card = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    from gym_pybullet_drones_b200 import _native
    res = {"card": card, "library": os.path.basename(_native.LIB_PATH), "T": T, "windows": args.windows, "ms": "[min, median, max] per call", "cases": []}
    for E in args.envs:
        env = HoverAviary(act=ActionType.RPM, physics=Physics.DYN, pyb_freq=240, ctrl_freq=30, num_envs=E)
        env.reset()
        target = torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64, device=env.device)
        for arch in ([64, 64], [256, 256]):
            pol = MlpPolicy.random(env._obs_dim, env._A, seed=0, critic=False, net_arch=arch)
            theta = pol.parameters64()
            f, c, rf, rc = alternate(lambda: fused(env, pol, theta, target), lambda: per_tick(env, pol, theta, target), args.windows)
            res["cases"].append({"E": E, "arch": arch, "fused_fwd_bwd_ms": f, "per_tick_fwd_bwd_ms": c, "calls_per_window": [rf, rc],
                                 "speedup_of_medians": round(c[1] / f[1], 2)})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
