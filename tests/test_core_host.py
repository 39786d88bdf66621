"""The CUDA kernels' per-drone core (csrc/quad_core.cuh) compiled for the host and checked against the golden
vectors of the unmodified reference -- same source as the GPU build, same float32-storage/float64-register
split, no GPU needed.  The GPU suite (-m gpu) repeats these through the C ABI."""
import ctypes as C

import numpy as np
import pytest

from gym_pybullet_drones_b200 import _native as N
from gym_pybullet_drones_b200.params import AviaryConstants, fill_params, quaternion_from_euler
from gym_pybullet_drones_b200.utils.enums import DroneModel
from qs_testlib import FIELDS, HostSim, RTOL, host_harness, ptr, quat_err, relerr


def check_fields(out, g, key, t, tol=RTOL, idx=slice(None)):
    for f in FIELDS:
        ref = g[key + "_" + f][t][idx]
        e = quat_err(out[f], ref) if f == "quat" else relerr(out[f], ref)
        assert e <= tol, (key, f, t, e)


@pytest.mark.parametrize("cf,steps", [(240, 1000), (30, 125)])
@pytest.mark.parametrize("stream", ["zeros", "rand", "sine", "const"])
def test_hover_rpm_1000_physics_steps(golden, cf, steps, stream):
    """BASELINE config 1: HoverAviary, 1 drone, DYN, 240 Hz, 1000 physics steps, <= 1e-5 rel on every state element."""
    g = golden("hover_rpm_1000")
    key = "cf%d_%s" % (cf, stream)
    c = AviaryConstants(DroneModel.CF2X, 240, cf)
    sim = HostSim(fill_params(c), 1, N.ACT_RPM, 4, c.PYB_STEPS_PER_CTRL)
    sim.set_state(c.default_init_xyzs(1), quaternion_from_euler(np.zeros((1, 3))), np.zeros((1, 3)), np.zeros((1, 3)))
    acts = g[key + "_actions"]
    tol = RTOL if stream != "const" else 1e-4      # constant torque: |w| reaches 40 rad/s, divergent trajectory
    for t in range(min(steps, acts.shape[0])):
        out = sim.tick(acts[t])
        check_fields(out, g, key, t, tol)


def test_hover_rpm_long_horizon_report(golden):
    """Informational bound for 1000 control ticks at 30 Hz (8000 physics steps, 33 s of open-loop tumbling)."""
    g = golden("hover_rpm_1000")
    c = AviaryConstants(DroneModel.CF2X, 240, 30)
    worst = 0.0
    for stream in ("rand", "sine"):
        key = "cf30_" + stream
        sim = HostSim(fill_params(c), 1, N.ACT_RPM, 4, 8)
        sim.set_state(c.default_init_xyzs(1), quaternion_from_euler(np.zeros((1, 3))), np.zeros((1, 3)), np.zeros((1, 3)))
        acts = g[key + "_actions"]
        for t in range(acts.shape[0]):
            out = sim.tick(acts[t])
            for f in FIELDS:
                ref = g[key + "_" + f][t]
                worst = max(worst, quat_err(out[f], ref) if f == "quat" else relerr(out[f], ref))
    assert worst < 2e-4, worst


@pytest.mark.parametrize("model", [DroneModel.CF2P, DroneModel.RACE])
def test_other_models_raw_rpm(golden, model):
    g = golden("ctrl_models_300")
    key = model.value
    c = AviaryConstants(model, 240, 120)
    sim = HostSim(fill_params(c), 2, N.ACT_RAW_RPM, 4, 2)
    sim.set_state(c.default_init_xyzs(2), quaternion_from_euler(np.zeros((2, 3))), np.zeros((2, 3)), np.zeros((2, 3)))
    acts = g[key + "_actions"]
    for t in range(acts.shape[0]):
        # raw RPM enters the ABI as float32: give both sides the same float32-representable sequence? The
        # golden used float64 rpm, so allow the 6e-8 input rounding on top of the state tolerance.
        out = sim.tick(acts[t])
        obs = g[key + "_obs"][t]
        assert relerr(out["pos"], obs[:, 0:3]) < 3e-5 and quat_err(out["quat"], obs[:, 3:7]) < 3e-5, t
        assert relerr(out["vel"], obs[:, 10:13]) < 3e-5 and relerr(out["ang_v"], obs[:, 13:16]) < 1e-4, t
        assert relerr(out["rpm"], obs[:, 16:20]) < 1e-7


@pytest.mark.parametrize("model", [DroneModel.CF2X, DroneModel.CF2P])
def test_pid_known_answers(golden, model):
    g = golden("pid_kat")
    k = model.value + "_"
    L = host_harness()
    P = fill_params(AviaryConstants(model), pid_model=model)
    n = g[k + "pos"].shape[0]
    st = np.zeros((n, 9))
    for call in range(3):
        for i in range(n):
            rpm, pe, ye = np.zeros(4), np.zeros(3), C.c_double()
            pos = g[k + "pos"][i] + 0.01 * call
            L.hh_pid(C.addressof(P), ptr(st[i]), 1 / 48, ptr(pos), ptr(g[k + "quat"][i].copy()), ptr(g[k + "vel"][i].copy()),
                     ptr(g[k + "target_pos"][i].copy()), float(g[k + "target_rpy"][i, 2]), ptr(g[k + "target_vel"][i].copy()),
                     ptr(g[k + "target_rpy_rates"][i].copy()), ptr(rpm), ptr(pe), C.addressof(ye))
            assert relerr(rpm, g[k + "rpm"][call][i]) < 1e-9, (call, i)
            assert relerr(pe, g[k + "pos_e"][call][i]) < 1e-12 and abs(ye.value - g[k + "yaw_e"][call][i]) < 1e-10
        assert relerr(st[:, 0:3], g[k + "integral_pos_e"][call]) < 1e-12
        assert relerr(st[:, 3:6], g[k + "last_rpy"][call]) < 1e-12
        assert relerr(st[:, 6:9], g[k + "integral_rpy_e"][call]) < 1e-10


ACTS = {"pid": (N.ACT_PID, 3), "vel": (N.ACT_VEL, 4), "one_d_pid": (N.ACT_ONE_D_PID, 1)}


@pytest.mark.parametrize("key,nd,act", [("hover_d1_pid", 1, "pid"), ("hover_d1_vel", 1, "vel"), ("hover_d1_one_d_pid", 1, "one_d_pid"), ("multi_d2_pid", 2, "pid")])
def test_rl_pid_actions_teacher_forced(golden, key, nd, act):
    """240/30 Hz RL envs with the embedded PID: each tick starts from the reference's previous state (the free-running
    30 Hz loop is chaotic in the reference itself, see tests/test_oracle_golden.py)."""
    g = golden("rl_pid_cf30")
    c = AviaryConstants(DroneModel.CF2X, 240, 30)
    at, A = ACTS[act]
    sim = HostSim(fill_params(c), nd, at, A, 8, pid=True)
    acts = g[key + "_actions"]
    for t in range(acts.shape[0]):
        if t == 0:
            sim.set_state(c.default_init_xyzs(nd), quaternion_from_euler(np.zeros((nd, 3))), np.zeros((nd, 3)), np.zeros((nd, 3)))
        else:
            sim.set_state(g[key + "_pos"][t - 1], g[key + "_quat"][t - 1], g[key + "_vel"][t - 1], g[key + "_rpy_rates"][t - 1])
            sim.pid[0:3] = g[key + "_pid_integral_pos_e"][t - 1].T
            sim.pid[3:6] = g[key + "_pid_last_rpy"][t - 1].T
            sim.pid[6:9] = g[key + "_pid_integral_rpy_e"][t - 1].T
        out = sim.tick(acts[t])
        check_fields(out, g, key, t, 2e-5)


@pytest.mark.parametrize("key,nd,act", [("hover_d1_pid", 1, "pid"), ("hover_d1_vel", 1, "vel"), ("hover_d1_one_d_pid", 1, "one_d_pid"), ("multi_d2_pid", 2, "pid")])
def test_rl_pid_actions_trajectory_120hz(golden, key, nd, act):
    """240/120 Hz: contractive closed loop, whole 480-tick trajectories compared."""
    g = golden("rl_pid_cf120")
    c = AviaryConstants(DroneModel.CF2X, 240, 120)
    at, A = ACTS[act]
    sim = HostSim(fill_params(c), nd, at, A, 2, pid=True)
    sim.set_state(c.default_init_xyzs(nd), quaternion_from_euler(np.zeros((nd, 3))), np.zeros((nd, 3)), np.zeros((nd, 3)))
    acts = g[key + "_actions"]
    for t in range(acts.shape[0]):
        out = sim.tick(acts[t])
        check_fields(out, g, key, t, 5e-5)


def test_half_angle_series_matches_libm():
    L = host_harness()
    rng = np.random.default_rng(0)
    for n in np.concatenate([rng.uniform(0, 500, 200), [1e-7, 1e-3, 239.9, 240.1, 1e4]]):
        c, s = C.c_double(), C.c_double()
        L.hh_half_angle(float(n * n), 1 / 240, C.byref(c), C.byref(s))
        th = n / 480
        assert abs(c.value - np.cos(th)) < 3e-16 and abs(s.value - np.sin(th) / n) < 3e-19 + 1e-15 * abs(np.sin(th) / n)


def test_downwash_predicate_is_the_references_sqrt():
    """qs::downwash_acts is BaseAviary._downwash's `dz > 0 and norm(dxy) < 10` as the oracle states it, sqrt(dx*dx + dy*dy) < 10
    (oracle/dyn_oracle.py, downwash_body_z), at the boundary and on random pairs within a few ulps of 10 m apart"""
    L = host_harness()
    # the least double whose correctly rounded sqrt is 10: the kernels' constant, 100 - 2^-46 (dxy2 < 100 differs right there)
    limit = next(x for x in (100.0 - k * 2.0 ** -46 for k in range(8)) if np.sqrt(np.nextafter(x, 0.0)) < 10.0)
    assert limit == 99.99999999999999 and np.sqrt(limit) == 10.0
    for dxy2 in (np.nextafter(limit, 0.0), limit, 100.0, np.nextafter(100.0, 200.0), 0.0, 25.0):
        want = bool(np.sqrt(dxy2) < 10.0)
        assert L.hh_downwash_acts(1.0, dxy2) == want, dxy2
        assert L.hh_downwash_acts(0.0, dxy2) == 0 and L.hh_downwash_acts(-1.0, dxy2) == 0
    assert L.hh_downwash_acts(1.0, limit) == 0 and limit < 100.0              # the pair `dxy2 < 100` would keep
    rng = np.random.default_rng(0)
    xy0 = rng.uniform(-5, 5, (20000, 2))
    th = rng.uniform(0, 2 * np.pi, 20000)
    xy1 = xy0 + (10.0 + rng.uniform(-4e-15, 4e-15, 20000))[:, None] * np.stack([np.cos(th), np.sin(th)], 1)
    d = xy1 - xy0
    dxy2 = d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]
    want = np.sqrt(dxy2) < 10.0
    got = np.array([L.hh_downwash_acts(1.0, float(x)) for x in dxy2], dtype=bool)
    assert np.array_equal(got, want)
    assert (want != (dxy2 < 100.0)).sum() > 100                               # the old compare disagrees on many of these


@pytest.mark.parametrize("D", [1, 3, 5, 32])
def test_downwash_fz_is_the_pair_sum_in_drone_order(D):
    """qs::downwash_fz, the in-CTA pair sum of every downwash kernel, against mppi_ref.dw_fz on random aviaries of D drones,
    with drone 1 of aviary 0 above drone 0 at dx*dx + dy*dy = 100 - 2^-46: that pair does not act, and the reference that
    tests dxy2 < 100 (a negative control) counts it"""
    import torch
    import mppi_ref as MR
    L = host_harness()
    P = fill_params(AviaryConstants(DroneModel.CF2X))
    rng = np.random.default_rng(D)
    G = 8
    # drones within 0.3 m in xy, where the pair terms are large, and about half of them 12 m away in x, where pairs do not act
    pos = np.concatenate([rng.uniform(-0.3, 0.3, (G, D, 2)), rng.uniform(0.1, 3, (G, D, 1))], axis=2)
    pos[:, :, 0] += 12.0 * rng.integers(0, 2, (G, D))
    if D > 1:
        # above every other drone, so that only drone 1 could act on drone 0; 60 m apart in z, where a pair 10 m apart in xy
        # has a term of -1.2e-5
        x, y = 1.0402010050251256, 9.945751950915763
        assert x * x + y * y == 99.99999999999999
        pos[0, 0], pos[0, 1] = (0.0, 0.0, 100.0), (x, y, 160.0)
    flat = np.ascontiguousarray(pos.reshape(-1))
    got = np.array([[L.hh_downwash_fz(C.addressof(P), ptr(flat), g * D, D, *pos[g, j]) for j in range(D)] for g in range(G)])
    want = MR.dw_fz(P, torch.from_numpy(pos)).numpy()
    assert np.all(np.abs(got - want) <= 1e-14 * np.abs(want)), np.max(np.abs(got - want))
    if D > 1:
        assert (want < -1e-3).sum() >= want.size // 8                         # large sums, not only underflowed terms
        lt100 = MR.dw_fz(P, torch.from_numpy(pos), lt100=True).numpy()
        assert got[0, 0] == 0.0 and lt100[0, 0] < -1e-5
