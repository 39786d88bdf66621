"""Times the forward mode of the closed-loop (DSLPIDControl) trajectories on one GPU (DESIGN.md 4.5) and prints one JSON line with
the card name and power limit read in the same call.  At E = 4 096 and 32 768 aviaries of D = 1 and 2 drones, T = 1 and 32 ticks
of S = 1 substep (240 / 240 Hz), Physics.DYN and GND|DRAG (the latter through the C ABI's effects; no Physics member has both):
  * linearise: BaseAviary.linearise(controller=) (qs_dyn_ctrl_traj + qs_dyn_ctrl_tick_jac), all of A, B, K, K_target;
  * per_tick_vjp: the same Jacobians from the existing VJP, per tick a T = 1 differentiable_rollout(controller=) from the stored
    state, controller state and (drag) RPMs, and one torch.autograd.grad call per output row of x_{k+1} and u_k (17) with unit
    cotangents -- the controller-state rows are not outputs of differentiable_rollout, so this does less than linearise;
  * jvp / vjp: one forward-mode product (torch.autograd.forward_ad on the waypoints) against one reverse-mode product
    (torch.autograd.grad) of the same T-tick closed loop, forward included in both.
With --circle it prints instead the spectral radius of the product of the closed-loop A's over one period of a circle flown at
48 Hz and at 240 Hz control (the claim of DESIGN.md 4.5, "Horizon and control rate"), without the two integral_rpy_e states
that the default gains never read (each adds an eigenvalue of exactly 1).
CUDA events around each call (each ends in the device's work for that call), [min, median, max] ms over --reps after warm-up."""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.autograd.forward_ad as fwAD

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from jvp_bench import card, timed  # noqa: E402

KEYS = ("pos", "quat", "vel", "rpy_rates")
PID_KEYS = ("integral_pos_e", "last_rpy", "integral_rpy_e")


def circle(W, dev):
    i = np.arange(W)
    c = np.stack([0.3 * np.cos(2 * np.pi * i / W), 0.3 * np.sin(2 * np.pi * i / W), 1.0 + 0.2 * np.sin(4 * np.pi * i / W)], 1)
    return torch.tensor(c, device=dev)


def spectral_radii():
    """rho(A_{P-1} ... A_0) over one period of the circle after one settling period, per control rate, for 16 aviaries"""
    from gym_pybullet_drones_b200.control import DSLPIDControl
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils.enums import DroneModel, Physics
    out = {}
    for ctrl in (48, 240):
        E, W = 16, 2 * ctrl                                   # a 2 s circle, as DESIGN.md 4.5's gradient comparison flies it
        env = CtrlAviary(drone_model=DroneModel.CF2X, num_drones=1, physics=Physics.DYN, pyb_freq=240, ctrl_freq=ctrl, num_envs=E,
                         initial_xyzs=np.array([[0.3, 0.0, 1.0]]))
        env.reset()
        ctl = DSLPIDControl(DroneModel.CF2X, num_drones=E, device=env.device)
        wp = circle(W, env.device)
        env.rollout(controller=ctl, waypoints=wp, num_steps=W, record=False)
        lin = env.linearise(controller=ctl, waypoints=wp, num_steps=W)
        rho = []
        for e in range(E):
            M = torch.eye(lin["A"].shape[-1], dtype=torch.float64)
            for k in range(W):
                M = lin["A"][k, e, 0].cpu() @ M
            live = [j for j in range(M.shape[0]) if j not in (19, 20)]   # integral_rpy_e x, y: I_COEFF_TOR = 0, nothing reads them
            rho.append(float(torch.linalg.eigvals(M[live][:, live]).abs().max()))
        out["%d_hz" % ctrl] = {"period_ticks": W, "rho_min": min(rho), "rho_median": float(np.median(rho)), "rho_max": max(rho)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[4096, 32768])
    ap.add_argument("--drones", type=int, nargs="+", default=[1, 2])
    ap.add_argument("--ticks", type=int, nargs="+", default=[1, 32])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--circle", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ctrl_jvp_bench.py measures on a GPU: none found")
    if args.circle:
        print(json.dumps({"card": card(), "circle": spectral_radii()}))
        return
    from gym_pybullet_drones_b200 import _native as N
    from gym_pybullet_drones_b200.control import DSLPIDControl
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils.enums import DroneModel, Physics
    res = {"card": card(), "S": 1, "runs": []}
    for E in args.envs:
        for D in args.drones:
            for name, physics, eff in (("dyn", Physics.DYN, 0), ("gnd_drag", Physics.PYB_DRAG, N.EFFECT_GND | N.EFFECT_DRAG)):
                xyz = np.stack([0.5 * np.arange(D), np.zeros(D), np.full(D, 1.0)], 1)
                env = CtrlAviary(num_drones=D, physics=physics, pyb_freq=240, ctrl_freq=240, num_envs=E, initial_xyzs=xyz)
                env.reset()
                env._effects = eff                   # GND|DRAG is reachable through the C ABI only
                ctl = DSLPIDControl(DroneModel.CF2X, num_drones=E * D, device=env.device)
                drag = bool(eff & N.EFFECT_DRAG)
                for T in args.ticks:
                    wp = circle(max(T, 2), env.device)
                    row = {"E": E, "D": D, "T": T, "effects": name}
                    row["linearise_ms"] = timed(lambda: env.linearise(controller=ctl, waypoints=wp, num_steps=T), args.reps)
                    lin = env.linearise(controller=ctl, waypoints=wp, num_steps=T)
                    start = {k: torch.cat([getattr(env, k)[None], lin[k][:-1]]) for k in KEYS}

                    def per_tick():
                        last = env._last_rpm.clone().reshape(E, D, 4)
                        for k in range(T):
                            st = {key: v[k].clone().requires_grad_(True) for key, v in start.items()}
                            ps = {key: lin["pid_state"][k][..., 3 * j:3 * j + 3].clone().requires_grad_(True) for j, key in enumerate(PID_KEYS)}
                            lr = last.clone().requires_grad_(drag)
                            off = torch.zeros((E, D, 3), dtype=torch.float64, device=env.device, requires_grad=True)
                            out = env.differentiable_rollout(controller=ctl, waypoints=wp, start=k, num_steps=1, offset=off, state=st,
                                                             pid_state=ps, last_rpm=lr)
                            flat = torch.cat([out[key] for key in KEYS] + [out["rpm"]], dim=-1)
                            leaves = list(st.values()) + list(ps.values()) + [off] + ([lr] if drag else [])
                            for j in range(17):
                                cot = torch.zeros_like(flat)
                                cot[..., j] = 1.0
                                torch.autograd.grad(flat, leaves, cot, retain_graph=j < 16)
                            last = lin["rpm"][k]
                    row["per_tick_vjp_ms"] = timed(per_tick, max(2, args.reps // 2))
                    v = torch.randn(wp.shape, device=env.device, dtype=torch.float64)

                    def jvp():
                        with fwAD.dual_level():
                            out = env.differentiable_rollout(controller=ctl, waypoints=fwAD.make_dual(wp, v), num_steps=T)
                            return fwAD.unpack_dual(out["pos"]).tangent

                    w = wp.clone().requires_grad_(True)
                    row["jvp_ms"] = timed(jvp, args.reps)
                    row["vjp_ms"] = timed(lambda: torch.autograd.grad(
                        env.differentiable_rollout(controller=ctl, waypoints=w, num_steps=T)["pos"].sum(), w), args.reps)
                    res["runs"].append(row)
                    print(json.dumps(row), file=sys.stderr, flush=True)
                    del lin, start
                del env
                torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
