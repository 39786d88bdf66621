"""Shared helpers of the MRAC tests (test infrastructure): the g++ build of mrac_core.cuh, the golden fixture's inputs and the
comparisons against it, and the free-running horizon derived from the tier-2 oracle."""
import ctypes as C

import numpy as np

from qs_testlib import drone_model, harness  # noqa: F401  (drone_model: re-exported for the MRAC tests)

MODELS = ("cf2x", "cf2p", "race")
DT = 1.0 / 120
# agreement with the reference's float64 MRAC, |a - b| <= tol * max(|b|, 1) on rpm, Kx, Kr, Xm, pos_e, rpy_e and the state:
# TOL for free-running loops (within the horizon of free_running_horizon), TF_TOL for the controller fed the reference's states
# (the KAT, the calls of a loop).  The controller alone does not amplify rounding, so the chained calls stay within TF_TOL.
TOL = 1e-9
TF_TOL = 1e-12

def mrac_harness():
    """tests/host_harness/mrac_host.cpp: the kernels' MRAC core compiled for the host."""
    L = harness("mrac_host")
    L.hh_mrac.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double] + [C.c_void_p] * 8
    L.hh_mrac_ang_v.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    L.hh_sizeof_mrac_params.restype = C.c_int
    return L


def gains_of(g, model):
    """The golden's gains of `model` as the dict of oracle.mrac_oracle.gains (Bm, which is exact, from the oracle)."""
    from oracle.mrac_oracle import gains
    G = gains(model)
    G.update(K=g[model + "_K"], Am=g[model + "_Am"], P=g[model + "_P"], Kr_ref_gain=g[model + "_Kr_ref_gain"], Kx=g[model + "_Kx0"],
             Kr=g[model + "_Kr0"])
    return G


def pack_state(Kx, Kr, Xm):
    """[n, 12, 4], [n, 4, 4], [n, 12] -> the [76][n] planes."""
    n = Kx.shape[0]
    return np.ascontiguousarray(np.concatenate([Kx.reshape(n, 48), Kr.reshape(n, 16), Xm.reshape(n, 12)], axis=1).T)


def unpack_state(s):
    n = s.shape[1]
    return s[0:48].T.reshape(n, 12, 4), s[48:64].T.reshape(n, 4, 4), s[64:76].T.reshape(n, 12)


def err(a, b):
    """max |a - b| / max(|b|, 1)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1.0))) if a.size else 0.0


def loop_inputs(state):
    """The computeControlFromState arguments stored in the fixture's [T, 13] rows: pos, quat, vel, ang_v."""
    return state[:, 0:3], state[:, 3:7], state[:, 7:10], state[:, 10:13]


def kat_inputs(g, m):
    """The KAT of model m as float64: (pos, quat, vel, ang_vel) [3, 256, .] and the targets [256, 12]."""
    x = g[m + "_kat_in"].astype(np.float64)
    return (x[..., 0:3], x[..., 3:7], x[..., 7:10], x[..., 10:13]), g[m + "_kat_tgt"].astype(np.float64)


# the KAT controllers whose final state the fixture keeps (make_golden_mrac.STATE_KEPT)
STATE_KEPT = np.r_[0:32, 128:160]


def _worse(worst, **kv):
    for k, v in kv.items():
        worst[k] = max(worst.get(k, 0.0), v)


def kat_worst(ctrl, g, m):
    """Worst error per output of the KAT of model m: the three calls of every controller chained on `ctrl` (a fresh controller for
    256 drones: ctrl.call(pos, quat, vel, ang_vel, targets [n, 12]) -> rpm, pos_e, rpy_e; ctrl.state() -> Kx, Kr, Xm).  pos_e is
    held to target_pos - cur_pos, which is exact."""
    (pos, quat, vel, angv), tgt = kat_inputs(g, m)
    worst = {}
    for k in range(pos.shape[0]):
        rpm, pe, re = ctrl.call(pos[k], quat[k], vel[k], angv[k], tgt)
        _worse(worst, rpm=err(rpm, g[m + "_kat_rpm"][k]), rpy_e=err(re, g[m + "_kat_rpy_e"][k]), pos_e=err(pe, tgt[:, 0:3] - pos[k]))
    Kx, Kr, Xm = ctrl.state()
    _worse(worst, Kx=err(Kx[STATE_KEPT], g[m + "_kat_Kx"]), Kr=err(Kr[STATE_KEPT], g[m + "_kat_Kr"]), Xm=err(Xm[STATE_KEPT], g[m + "_kat_Xm"]))
    return worst


def loop_worst(ctrl, g):
    """Worst error of every call of mrac.py's CF2X loop fed the reference's states, chained on `ctrl` (one drone, as kat_worst):
    the RPMs of all 600 calls and the controller state after calls 99, 199, ..., 599."""
    pos, quat, vel, angv = loop_inputs(g["loop_state"])
    tgt = np.zeros((1, 12))
    tgt[0, 2] = 1.0
    worst = {}
    for k in range(pos.shape[0]):
        rpm, _, _ = ctrl.call(pos[k][None], quat[k][None], vel[k][None], angv[k][None], tgt)
        _worse(worst, rpm=err(rpm, g["loop_rpm"][k][None]))
        if k % 100 == 99:
            Kx, Kr, Xm = ctrl.state()
            j = k // 100
            _worse(worst, Kx=err(Kx[0], g["loop_Kx"][j]), Kr=err(Kr[0], g["loop_Kr"][j]), Xm=err(Xm[0], g["loop_Xm"][j]))
    return worst


# the fixture's closed loops (make_golden_mrac.py): model, initial position, target, ticks
LOOPS = {"cf2x": ("cf2x", (0.0, 0.0, 0.0), (0.0, 0.0, 1.0), 600), "cf2p": ("cf2p", (0.3, -0.2, 0.5), (-0.5, 0.4, 1.2), 1800)}


def free_running_horizon(case="cf2x"):
    """A closed loop of the fixture (mrac.py's CF2X loop, or the CF2P offset case; DYN, 240/120 Hz) run twice by the tier-2
    oracle, the twin with the controller's z input moved by one ulp at every tick.  Returns (first tick at which the twins'
    states or RPMs differ by more than TOL, or the loop's length; the horizon = half of it, or the whole loop if the twins never
    part): rounding differences of one ulp per tick grow past TOL after the first value whatever the implementation, so a
    free-running comparison with the reference is meaningful only below it."""
    from oracle.dyn_oracle import OracleAviary
    from oracle.mrac_oracle import OracleMRAC, ang_v_from_state
    model, init, target, ticks = LOOPS[case]

    def run(eps):
        env = OracleAviary("ctrl", 1, 1, model, 240, 120, initial_xyzs=np.array([init]))
        c = OracleMRAC(1, model)
        a = np.zeros((1, 1, 4))
        out = []
        for _ in range(ticks):
            env.step(a)
            pos = env.pos[0].copy()
            if eps:
                pos[:, 2] = np.nextafter(pos[:, 2], np.inf)
            av = ang_v_from_state(env.quat[0], env.rpy_rates[0])
            rpm, _, _ = c.compute(env.P.CTRL_TIMESTEP, pos, env.quat[0], env.vel[0], av, np.array([target]))
            a = rpm.reshape(1, 1, 4)
            out.append(np.concatenate([env.pos[0, 0], env.quat[0, 0], env.vel[0, 0], rpm[0]]))
        return np.array(out)
    x, y = run(False), run(True)
    d = np.max(np.abs(x - y) / np.maximum(np.abs(x), 1.0), axis=1)
    over = np.nonzero(d > TOL)[0]
    if not over.size:
        return ticks, ticks
    return int(over[0]), int(over[0]) // 2
