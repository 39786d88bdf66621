"""Times BaseAviary.differentiable_rollout(controller=DSLPIDControl) on one GPU: the forward (qs_dyn_ctrl_traj) and forward +
backward (qs_dyn_ctrl_traj_vjp, gradients to the gains, the waypoints and the initial state), next to
CtrlAviary.rollout(controller=..., record=False) of the same ticks, at E = 32 768 aviaries of D = 2 drones, T = 64 ticks of S = 8
substeps (240 / 30 Hz), for Physics.DYN and GND|DRAG (the latter through the C ABI's effects; no Physics member has both).
Prints one JSON line with the card name and power limit read in the same call.  CUDA events, median of --reps."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.diff_bench import card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=32768)
    ap.add_argument("--drones", type=int, default=2)
    ap.add_argument("--ticks", type=int, default=64)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    from gym_pybullet_drones_b200 import _native as N
    from gym_pybullet_drones_b200.control import DSLPIDControl
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils.enums import DroneModel, Physics
    E, D, T = args.envs, args.drones, args.ticks
    res = {"card": card(), "E": E, "D": D, "T": T, "S": 8}
    for name, physics, eff in (("dyn", Physics.DYN, 0), ("gnd_drag", Physics.PYB_DRAG, N.EFFECT_GND | N.EFFECT_DRAG)):
        env = CtrlAviary(num_drones=D, physics=physics, pyb_freq=240, ctrl_freq=30, num_envs=E)
        env.reset()
        env._effects = eff                       # GND|DRAG is reachable through the C ABI only
        ctl = DSLPIDControl(DroneModel.CF2X, num_drones=E * D, device=env.device)
        i = np.arange(T)
        wp = torch.tensor(np.stack([0.3 * np.cos(2 * np.pi * i / T), 0.3 * np.sin(2 * np.pi * i / T), np.zeros(T)], 1), device=env.device)
        offset = env.pos.clone()
        fwd = timed(lambda: env.differentiable_rollout(controller=ctl, waypoints=wp, offset=offset), args.reps)
        kp = torch.tensor(list(ctl._P.pid_p_for), dtype=torch.float64, device=env.device).expand(E, 3).clone().requires_grad_(True)
        w = wp.clone().requires_grad_(True)

        def fb():
            out = env.differentiable_rollout(controller=ctl, waypoints=w, offset=offset, gains={"P_COEFF_FOR": kp})
            torch.autograd.grad(out["pos"].sum(), (kp, w))
        both = timed(fb, args.reps)
        res[name] = {"forward_ms": fwd, "forward_backward_ms": both}
        if eff in (0, N.EFFECT_DRAG):
            env._effects = 0 if eff == 0 else N.EFFECT_DRAG
            state, pid = env._planes.clone(), ctl._state.clone()
            res[name]["ctrl_rollout_ms"] = timed(lambda: (env._planes.copy_(state), ctl._state.copy_(pid),
                                                          env.rollout(controller=ctl, waypoints=wp, offset=offset, record=False)), args.reps)
        res[name]["drone_ticks_per_s_forward"] = E * D * T / (fwd * 1e-3)
        del env, ctl
    print(json.dumps(res))


if __name__ == "__main__":
    main()
