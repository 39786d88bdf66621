"""The per-aviary oracle (tests/dyn_params_lib.py) and the row builder against the UNMODIFIED reference flying drones whose
constants were overwritten after construction (tests/golden/dyn_params.npz, make_golden_dyn_params.py).  CPU only.

What this pins: the reference reads M, L, J, J_INV, KF, KM, GRAVITY, HOVER_RPM and MAX_RPM at call time and keeps no other
derived copy that the step uses (else the overwritten reference would leave the oracle); the oracle's per-aviary constants
follow the reference's paths for the arm (L/sqrt(2) in the CF2X / RACE torques, L in CF2P's), HOVER_RPM (RPM and ONE_D_RPM
decode), MAX_RPM (CtrlAviary clip) and the embedded controller (nominal CF2X, not the overwritten constants)."""
import json

import numpy as np
import pytest
import torch

from dyn_params_lib import PerAviaryOracle
from gym_pybullet_drones_b200.params import PHYS_KEYS, physical_rows
from gym_pybullet_drones_b200.utils.enums import DroneModel
from oracle import dyn_oracle as O
from test_oracle_golden import FIELDS, force_state, relerr, replay

MODELS = {"cf2x": DroneModel.CF2X, "cf2p": DroneModel.CF2P, "racer": DroneModel.RACE}


def cases(g):
    return {c["key"]: c for c in json.loads(str(g["cases"]))}


def oracle_for(g, c):
    kind = {"hover": "hover", "multihover": "multihover", "ctrl": "ctrl"}[c["kind"]]
    act = "rpm" if c["act"] == "raw" else c["act"]
    p = g[c["key"] + "_props"]
    return PerAviaryOracle(kind, 1, c["nd"], drone_model=c["model"], pyb_freq=c["pyb"], ctrl_freq=c["ctrl"], act=act,
                           props={k: p[j:j + 1] for j, k in enumerate(PHYS_KEYS)})


FREE = ["cf2x_heavy_rpm", "cf2p_light_one_d_rpm", "race_long_arm_rpm", "multi3_rpm", "ctrl_low_t2w_clip"]


@pytest.mark.parametrize("key", FREE)
def test_oracle_replays_the_overwritten_reference(golden, key):
    """Whole trajectories at 1e-10: state, reward, flags, observations."""
    g = golden("dyn_params")
    c = cases(g)[key]
    env = oracle_for(g, c)
    assert float(env.P.HOVER_RPM.ravel()[0]) == float(g[key + "_HOVER_RPM"])
    assert float(env.P.MAX_RPM.ravel()[0]) == float(g[key + "_MAX_RPM"])
    if c["kind"] == "multihover":
        assert relerr(env.TARGET_POS[0], g[key + "_TARGET_POS"]) == 0
    if c["kind"] == "ctrl":
        assert float(g[key + "_clipped_fraction"]) > 0.2                      # the MAX_RPM clip binds
    replay(env, g, key, 1)


def test_oracle_replays_the_overwritten_reference_pid_teacher_forced(golden):
    """PID at 48 Hz: the drone's constants are overwritten, the embedded controller keeps its URDF's; each tick from the
    reference's previous state and controller integrals, at 1e-11."""
    key = "pid_48"
    g = golden("dyn_params")
    env = oracle_for(g, cases(g)[key])
    acts = g[key + "_actions"]
    env.reset()
    for t in range(acts.shape[0]):
        force_state(env, g, key, t - 1)
        obs, r, te, tr = env.step(acts[t][None])
        for f in FIELDS:
            assert relerr(getattr(env, f)[0], g[key + "_" + f][t]) < 1e-11, (key, f, t)
        assert relerr(env.ctrl.integral_rpy_e, g[key + "_pid_integral_rpy_e"][t]) < 1e-11
        assert relerr(env.ctrl.integral_pos_e, g[key + "_pid_integral_pos_e"][t]) < 1e-11
        assert abs(r[0] - g[key + "_reward"][t]) < 1e-10
        assert bool(tr[0]) == bool(g[key + "_truncated"][t])


def test_nominal_constants_do_not_reproduce_the_fixture(golden):
    """Negative control: the oracle with the model's nominal constants leaves the overwritten reference within a few ticks."""
    g = golden("dyn_params")
    c = cases(g)["cf2x_heavy_rpm"]
    env = O.OracleAviary("hover", 1, 1, drone_model="cf2x", act="rpm")
    env.reset()
    for t in range(10):
        env.step(g["cf2x_heavy_rpm_actions"][t][None])
    assert relerr(env.pos[0], g["cf2x_heavy_rpm_pos"][9]) > 1e-4
    assert c["scale"]["m"] != 1.0


@pytest.mark.parametrize("key", FREE + ["pid_48"])
def test_rows_carry_the_reference_hover_and_max_rpm(golden, key):
    """physical_rows of the fixture's properties gives the reference's HOVER_RPM and MAX_RPM bit for bit."""
    g = golden("dyn_params")
    c = cases(g)[key]
    p = g[key + "_props"]
    row = physical_rows(MODELS[c["model"]], {k: torch.tensor([float(p[j])], dtype=torch.float64) for j, k in enumerate(PHYS_KEYS)})[0]
    assert float(row[12]) == float(g[key + "_HOVER_RPM"]) and float(row[13]) == float(g[key + "_MAX_RPM"])
