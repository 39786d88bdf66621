"""Regenerates tests/golden/dyn_params.npz: the UNMODIFIED reference flying drones whose physical constants were changed after
construction, the way a reference user randomises the dynamics between episodes.

Needs a checkout of the reference (oracle/ref_loader.py, QS_REFERENCE_ROOT):
    python tests/golden/make_golden_dyn_params.py
The other fixtures stay as they are (tests/golden/make_golden.py writes those; its recording helpers are reused here).

Each case constructs a reference env, then overwrites M, L, J, J_INV, KF, KM, GRAVITY, HOVER_RPM and MAX_RPM (and
THRUST2WEIGHT_RATIO) before reset(), with values derived by the reference's own formulas (BaseAviary.py:117-119, J_INV =
np.linalg.inv(J) as in _parseURDFParameters).  The reference reads them from the env at call time: _dynamics
(BaseAviary.py:838-858), _preprocessAction (BaseRLAviary.py:192,225), CtrlAviary's clip (CtrlAviary.py:140).  Its embedded
DSLPIDControl keeps the constants of its own URDF (BaseControl.py:35-40).  `<key>_props` holds the eight properties in
gym_pybullet_drones_b200.params.PHYS_KEYS order: m, ixx, iyy, izz, kf, km, arm, thrust2weight.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import R, flat, quiet, run_env, save  # noqa: E402  (loads the reference)

PHYS_KEYS = ("m", "ixx", "iyy", "izz", "kf", "km", "arm", "thrust2weight")

# key, env kind, drone count, model, pyb, ctrl, action, ticks, factors on the nominal properties, action seed
DYN_PARAMS_CASES = [
    dict(key="cf2x_heavy_rpm", kind="hover", nd=1, model="cf2x", pyb=240, ctrl=30, act="rpm", T=120, seed=201,
         scale=dict(m=1.25, ixx=1.15, iyy=1.2, izz=1.1, kf=1.05, km=0.95)),
    dict(key="cf2p_light_one_d_rpm", kind="hover", nd=1, model="cf2p", pyb=240, ctrl=30, act="one_d_rpm", T=120, seed=202,
         scale=dict(m=0.8, ixx=0.85, iyy=0.9, izz=0.8, kf=0.9, km=1.1, thrust2weight=1.05)),
    dict(key="race_long_arm_rpm", kind="hover", nd=1, model="racer", pyb=240, ctrl=30, act="rpm", T=120, seed=203,
         scale=dict(arm=1.1, m=1.05, kf=0.95)),
    dict(key="multi3_rpm", kind="multihover", nd=3, model="cf2x", pyb=240, ctrl=30, act="rpm", T=150, seed=204,
         scale=dict(m=1.1, ixx=0.9, iyy=1.1, izz=1.05, kf=1.1, km=1.2, arm=0.95)),
    # thrust-to-weight 1.6 instead of 2.25: MAX_RPM = 1.26 HOVER_RPM, below most of the commanded RPMs
    dict(key="ctrl_low_t2w_clip", kind="ctrl", nd=2, model="cf2x", pyb=240, ctrl=240, act="raw", T=120, seed=205,
         scale=dict(m=1.1, kf=0.95, thrust2weight=1.6 / 2.25)),
    dict(key="pid_48", kind="hover", nd=1, model="cf2x", pyb=240, ctrl=48, act="pid", T=96, seed=206,
         scale=dict(m=1.15, ixx=1.1, iyy=0.9, izz=1.2, kf=0.9, km=1.1)),
]


def properties(env, scale):
    """The env's nominal properties times `scale` (PHYS_KEYS order)."""
    nom = dict(m=env.M, ixx=env.J[0, 0], iyy=env.J[1, 1], izz=env.J[2, 2], kf=env.KF, km=env.KM, arm=env.L,
               thrust2weight=env.THRUST2WEIGHT_RATIO)
    return np.array([float(nom[k]) * scale.get(k, 1.0) for k in PHYS_KEYS])


def overwrite(env, p):
    """The constants a reference user changes, derived as BaseAviary.__init__ derives them."""
    m, ixx, iyy, izz, kf, km, arm, t2w = (float(x) for x in p)
    env.M, env.L, env.KF, env.KM, env.THRUST2WEIGHT_RATIO = m, arm, kf, km, t2w
    env.J = np.diag([ixx, iyy, izz])
    env.J_INV = np.linalg.inv(env.J)
    env.GRAVITY = env.G * env.M                                                     # BaseAviary.py:117
    env.HOVER_RPM = np.sqrt(env.GRAVITY / (4 * env.KF))                             # :118
    env.MAX_RPM = np.sqrt((env.THRUST2WEIGHT_RATIO * env.GRAVITY) / (4 * env.KF))   # :119


def case_actions(c, env):
    rng = np.random.default_rng(c["seed"])
    nd = c["nd"]
    if c["act"] == "raw":            # float64 RPMs from 0.9 to 1.5 x the new HOVER_RPM: the clip at 1.26 x binds often
        return env.HOVER_RPM * rng.uniform(0.9, 1.5, (c["T"], nd, 4))
    if c["act"] == "pid":            # piecewise-constant set-points inside the truncation box
        seg = (np.array([0, 0, 1.0], np.float32) + 0.5 * rng.uniform(-1, 1, (4, nd, 3)).astype(np.float32)).astype(np.float32)
        return np.repeat(seg, c["T"] // 4, axis=0)
    aw = 1 if c["act"] == "one_d_rpm" else 4
    return rng.uniform(-1, 1, (c["T"], nd, aw)).astype(np.float32)


def dyn_params_fixture():
    A = R.ActionType
    acts_enum = {"rpm": A.RPM, "one_d_rpm": A.ONE_D_RPM, "pid": A.PID}
    models = {"cf2x": R.DroneModel.CF2X, "cf2p": R.DroneModel.CF2P, "racer": R.DroneModel.RACE}
    out = {"cases": np.array(json.dumps(DYN_PARAMS_CASES))}
    for c in DYN_PARAMS_CASES:
        kw = dict(drone_model=models[c["model"]], physics=R.Physics.DYN, pyb_freq=c["pyb"], ctrl_freq=c["ctrl"])
        with quiet():
            if c["kind"] == "ctrl":
                env = R.CtrlAviary(num_drones=c["nd"], **kw)
            elif c["kind"] == "hover":
                env = R.HoverAviary(act=acts_enum[c["act"]], **kw)
            else:
                env = R.MultiHoverAviary(num_drones=c["nd"], act=acts_enum[c["act"]], **kw)
        p = properties(env, c["scale"])
        overwrite(env, p)
        acts = case_actions(c, env)
        with quiet():
            rec = run_env(env, acts, record_obs_every=1)
        rec["props"] = p
        rec["HOVER_RPM"], rec["MAX_RPM"] = np.float64(env.HOVER_RPM), np.float64(env.MAX_RPM)
        if c["kind"] == "multihover":
            rec["TARGET_POS"] = np.asarray(env.TARGET_POS)
        if c["kind"] == "ctrl":
            rec["clipped_fraction"] = np.float64(np.mean(acts > env.MAX_RPM))
        out.update(flat(c["key"], rec))
    save("dyn_params", **out)


if __name__ == "__main__":
    dyn_params_fixture()
