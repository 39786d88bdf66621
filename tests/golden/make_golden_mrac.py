"""Regenerates tests/golden/mrac.npz from the UNMODIFIED reference MRAC (control/MRAC.py) under the test stand-ins
(oracle/standins: pybullet, and python-control's `place` as scipy's YT pole placement -- parity unpinned at that boundary).

    python tests/golden/make_golden_mrac.py            (needs a reference checkout, QS_REFERENCE_ROOT)

Inputs are rounded to float32 values before the reference sees them (stored as float32, exact in float64), and each controller's
calls are chained, so the state between calls needs no storage.  Contents, for model in cf2x / cf2p / race:
  {model}_K, _Am, _P, _Kr_ref_gain, _Kx0, _Kr0          the synthesised gains (MRAC._compute_K)
  {model}_kat_in     float32 [3, 256, 13]    256 controllers, 3 consecutive computeControl calls each (call 0 sets Xm):
                                             pos, quat, vel, ang_vel of each call
  {model}_kat_tgt    float32 [256, 12]       target_pos, target_rpy, target_vel, target_rpy_rates of each controller
  {model}_kat_rpm, _kat_rpy_e  [3, 256, .]   the outputs of each call (pos_e is target_pos - cur_pos, exact)
  {model}_kat_Kx, _Kr, _Xm     [64, .]       the controller state after the third call of controllers STATE_KEPT (32 near
                                             their target, 32 anywhere)
  loop_*   examples/mrac.py's loop (CtrlAviary, DYN, 240/120 Hz, one CF2X from (0,0,0) to (0,0,1)): after one step(zeros),
           600 x (computeControlFromState on the state vector, step(rpm)).  loop_state [600, 13] is what each call received
           (pos, quat, vel, ang_v of the state vector), loop_rpm [600, 4] its output, loop_Kx / _Kr / _Xm [6, .] the controller
           state after calls 99, 199, ..., 599
  p_*      the same loop for one CF2P from (0.3, -0.2, 0.5) to (-0.5, 0.4, 1.2), 1800 ticks, kept at every 10th call
           (p_state [180, 13], p_rpm [180, 4]: calls 0, 10, ...), and the controller state after calls 99, 199, ... (p_Kx [18, .])
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle.ref_loader import load_reference, quiet  # noqa: E402

DT = 1.0 / 120
N_KAT, CALLS = 256, 3
STATE_KEPT = np.r_[0:32, 128:160]


def random_quat(rng, n, spread):
    q = np.concatenate([rng.normal(0, spread, (n, 3)), np.ones((n, 1))], axis=1)
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def f32(x):
    return np.asarray(x, dtype=np.float32).astype(np.float64)


def kat(MRAC, model, rng):
    with quiet():
        c = MRAC(model)
    Kx0, Kr0 = c.Kx.copy(), c.Kr.copy()
    n = N_KAT
    tgt = f32(np.concatenate([rng.uniform(-1, 1, (n, 2)), rng.uniform(0.2, 1.5, (n, 1)), rng.uniform(-0.3, 0.3, (n, 3)),
                              rng.uniform(-0.5, 0.5, (n, 3)), rng.uniform(-0.5, 0.5, (n, 3))], axis=1))
    # half of the controllers near their target (unsaturated PWM), half anywhere
    near = np.arange(n) < n // 2
    pos = np.where(near[None, :, None], tgt[None, :, 0:3] + rng.normal(0, 0.02, (CALLS, n, 3)), rng.uniform(-2, 2, (CALLS, n, 3)))
    quat = np.stack([np.where(near[:, None], random_quat(rng, n, 0.02), random_quat(rng, n, 0.5)) for _ in range(CALLS)])
    vel = np.where(near[None, :, None], rng.normal(0, 0.05, (CALLS, n, 3)), rng.uniform(-1, 1, (CALLS, n, 3)))
    angv = np.where(near[None, :, None], rng.normal(0, 0.1, (CALLS, n, 3)), rng.uniform(-3, 3, (CALLS, n, 3)))
    inp = f32(np.concatenate([pos, quat, vel, angv], axis=2))
    rpm, rpy_e = np.zeros((CALLS, n, 4)), np.zeros((CALLS, n, 3))
    Kx, Kr, Xm = np.zeros((n, 12, 4)), np.zeros((n, 4, 4)), np.zeros((n, 12))
    for j in range(n):
        c.Kx, c.Kr, c.Xm = Kx0.copy(), Kr0.copy(), np.zeros(12)
        c.reset()
        for k in range(CALLS):
            x = inp[k, j]
            rpm[k, j], _, rpy_e[k, j] = c.computeControl(DT, x[0:3], x[3:7], x[7:10], x[10:13], tgt[j, 0:3], tgt[j, 3:6], tgt[j, 6:9],
                                                         tgt[j, 9:12])
        Kx[j], Kr[j], Xm[j] = c.Kx, c.Kr, np.asarray(c.Xm).reshape(12)
    return dict(K=-Kx0.T, Am=c.Am, P=c.P, Kr_ref_gain=c.Kr_ref_gain, Kx0=Kx0, Kr0=Kr0, kat_in=inp.astype(np.float32),
                kat_tgt=tgt.astype(np.float32), kat_rpm=rpm, kat_rpy_e=rpy_e, kat_Kx=Kx[STATE_KEPT], kat_Kr=Kr[STATE_KEPT], kat_Xm=Xm[STATE_KEPT])


def loop(R, MRAC, model, init, target, T):
    with quiet():
        env = R.CtrlAviary(drone_model=model, num_drones=1, initial_xyzs=np.array([init], dtype=float), initial_rpys=np.zeros((1, 3)),
                           physics=R.Physics.DYN, neighbourhood_radius=10, pyb_freq=240, ctrl_freq=120)
        c = MRAC(model)
    a = np.zeros((1, 4))
    rec = {k: [] for k in ("state", "rpm", "Kx", "Kr", "Xm")}
    for _ in range(T):
        obs, *_ = env.step(a)
        rpm, _, _ = c.computeControlFromState(control_timestep=env.CTRL_TIMESTEP, state=obs[0], target_pos=np.array(target),
                                                target_rpy=np.array([0, 0, 0]))
        a[0] = rpm
        st = np.concatenate([obs[0][0:7], obs[0][10:16]])                       # pos, quat, vel, ang_v
        for k, v in (("state", st), ("rpm", rpm), ("Kx", c.Kx), ("Kr", c.Kr), ("Xm", np.asarray(c.Xm).reshape(12))):
            rec[k].append(np.array(v, dtype=np.float64))
    return {k: np.array(v) for k, v in rec.items()}


def main():
    R = load_reference()
    with quiet():
        from gym_pybullet_drones.control.MRAC import MRAC
    rng = np.random.default_rng(20261016)
    out = {}
    for name, m in (("cf2x", R.DroneModel.CF2X), ("cf2p", R.DroneModel.CF2P), ("race", R.DroneModel.RACE)):
        out.update({name + "_" + k: v for k, v in kat(MRAC, m, rng).items()})
    lx = loop(R, MRAC, R.DroneModel.CF2X, [0, 0, 0], [0, 0, 1], 600)
    out.update({"loop_state": lx["state"], "loop_rpm": lx["rpm"]})
    out.update({"loop_" + k: lx[k][99::100] for k in ("Kx", "Kr", "Xm")})
    lp = loop(R, MRAC, R.DroneModel.CF2P, [0.3, -0.2, 0.5], [-0.5, 0.4, 1.2], 1800)
    out.update({"p_state": lp["state"][::10], "p_rpm": lp["rpm"][::10]})
    out.update({"p_" + k: lp[k][99::100] for k in ("Kx", "Kr", "Xm")})
    path = os.path.join(ROOT, "tests", "golden", "mrac.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "%.0f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
