"""Every threshold decision of csrc/quad_core.cuh at its boundary, on the CPU build of the same source (tests/host_harness).
The host libm is the reference's libm, so every float64 decision must equal the reference's predicate -- evaluated with the
Bullet stand-in, drone by drone -- exactly, with no band.  The GPU suite repeats these sweeps through the kernels
(test_gpu_thresholds.py), where CUDA's 2-ulp atan2/asin need a band of a few ulps."""
import ctypes as C
import math

import numpy as np
import torch

import threshold_sweeps as S
from gym_pybullet_drones_b200.params import AviaryConstants, euler_from_quaternion, fill_params
from gym_pybullet_drones_b200.utils.enums import DroneModel
from qs_testlib import host_harness, ptr


def _hover_terms(pos, q, tgt, f32, **bounds):
    L = host_harness()
    P = fill_params(AviaryConstants(DroneModel.CF2X, 240, 30), **bounds)
    n = q.shape[0]
    out = np.zeros((n, 5))
    L.hh_hover_terms(C.addressof(P), ptr(np.ascontiguousarray(pos, np.float64)), ptr(np.ascontiguousarray(q, np.float64)),
                     ptr(np.ascontiguousarray(tgt, np.float64)), n, int(f32), ptr(out))
    return out


def _k2e(q, f32):
    out = np.zeros((q.shape[0], 3))
    host_harness().hh_quat_to_euler(ptr(np.ascontiguousarray(q, np.float64)), q.shape[0], int(f32), ptr(out))
    return out


def test_s1_tilt_truncation_is_decided_on_float64_angles():
    """HoverAviary.py:110-111 on the reference's float64 rpy.  With RPY_F32 the reported angles are float32 (atan2f/asinf), yet
    the decision must still be the float64 one: the sweep holds angles that round to 0.4f from below, where a float32 decision
    reads 0.40000000596 > 0.4 and truncates although the reference does not."""
    q = S.quat(S.tilt_poses())
    n = q.shape[0]
    pos, tgt = np.tile([0.0, 0.0, 1.0], (n, 1)), np.tile([0.0, 0.0, 5.0], (n, 1))
    want = S.tilted(q)
    assert 0 < want.sum() < n
    f32_wrong = 0
    for f32 in (False, True):
        out = _hover_terms(pos, q, tgt, f32)
        got = out[:, 2] != 0
        bad = np.nonzero(got != want)[0]
        assert bad.size == 0, ("rpy_f32=%s" % f32, len(bad), S.euler(q[bad[:4]]))
        if f32:
            f32_wrong = int(((np.abs(out[:, 3]) > S.TILT) | (np.abs(out[:, 4]) > S.TILT) != want).sum())
    # the sweep reaches the float32 window: a decision on the reported float32 angles would have been wrong there
    assert f32_wrong > 100, f32_wrong
    print("S1 host: %d poses, %d truncated, %d where the float32 angles decide wrongly" % (n, want.sum(), f32_wrong))


def test_s1_negative_control_one_ulp_of_tilt_bound():
    """The sweep resolves single ulps: moving tilt_bound by one ulp changes decisions."""
    q = S.quat(S.tilt_poses())
    n = q.shape[0]
    pos, tgt = np.tile([0.0, 0.0, 1.0], (n, 1)), np.tile([0.0, 0.0, 5.0], (n, 1))
    base = _hover_terms(pos, q, tgt, False)[:, 2]
    for k in (1, -1):
        moved = _hover_terms(pos, q, tgt, False, tilt_bound=S.ulps(S.TILT, k))[:, 2]
        assert (moved != base).sum() > 0
        assert np.array_equal(moved != 0, S.tilted(q, S.ulps(S.TILT, k)))


def test_s2_position_bounds_exact():
    ident = np.tile([0.0, 0.0, 0.0, 1.0], (1, 1))
    for task in ("hover", "multihover"):
        pos = S.bound_positions(task)
        n = pos.shape[0]
        q = np.repeat(ident, n, axis=0)
        out = _hover_terms(pos, q, np.zeros((n, 3)), True, xy_bound=S.XY_BOUND[task])
        assert np.array_equal(out[:, 2] != 0, S.out_of_bounds(pos, task)), task


def test_s3_distance_is_the_reference_norm():
    """The per-drone distance hover_terms feeds to `dist < 1e-4` (HoverAviary.py:91): np.linalg.norm of the reference, to the ulp."""
    rng = np.random.default_rng(1)
    ks = np.arange(-32, 33)
    d = S.TERM_DIST * (1 + ks * 2.0 ** -40)
    u = rng.normal(size=(ks.size, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    tgt = np.tile([0.1, -0.2, 1.0], (ks.size, 1))
    pos = tgt - u * d[:, None]
    q = np.tile([0.0, 0.0, 0.0, 1.0], (ks.size, 1))
    out = _hover_terms(pos, q, tgt, True)
    ref = np.array([np.linalg.norm(tgt[i] - pos[i]) for i in range(ks.size)])
    assert np.max(np.abs(out[:, 1] - ref) / np.spacing(ref)) <= 1.0
    near = np.abs(ref - S.TERM_DIST) <= 4 * np.spacing(S.TERM_DIST)
    assert np.array_equal((out[:, 1] < S.TERM_DIST)[~near], (ref < S.TERM_DIST)[~near])
    assert 0 < (ref < S.TERM_DIST).sum() < ks.size


def test_s4_gimbal_guard_float64_euler_is_bullets():
    """quat_to_euler<false> is Bullet's getEulerFromQuaternion bit for bit, on both sides of the +-0.99999 guard."""
    q = S.guard_quats()
    sa = S.sarg(q)
    near = np.abs(np.abs(sa) - S.GUARD) <= 8 * np.spacing(S.GUARD)
    inside = np.abs(sa) >= S.GUARD
    assert near.sum() >= 8 and (near & inside).sum() >= 2 and (near & ~inside).sum() >= 2, (near.sum(), (near & inside).sum())
    assert np.array_equal(_k2e(q, False), S.euler(q))


def test_s4_gimbal_guard_float32_euler():
    """RPY_F32: in the guard branch roll == 0 and pitch == +-pi/2 exactly (float32(pitch) is float32(pi/2)); yaw = 2 atan2f of
    the float32-rounded x, y: within 2 (2^-24 + 2 ulp(float32)) rad of the float64 yaw.  Off the guard every angle is within the
    bound the tilt decision's band is derived from (quad_core.cuh, qs::tilted): 2^-24 for rounding the arguments of atan2f, times
    tan|pitch| for asinf's, plus 3 ulp(float32)."""
    q = S.guard_quats()
    ref, got = S.euler(q), _k2e(q, True)
    g = np.abs(S.sarg(q)) >= S.GUARD
    assert g.sum() > 0 and (~g).sum() > 0
    assert np.all(got[g, 0] == 0.0) and np.array_equal(got[g, 1], ref[g, 1])
    assert np.array_equal(np.float32(got[g, 1]), np.float32(np.sign(ref[g, 1]) * np.float32(math.pi / 2)))
    dy = np.abs(np.angle(np.exp(1j * (got[g, 2] - ref[g, 2]))))
    assert np.all(dy <= 2 * (2.0 ** -24 + 2 * np.spacing(np.float32(np.pi)))), dy.max()
    off = np.abs(got[~g] - ref[~g])
    off = np.minimum(off, 2 * np.pi - off)
    arg = np.ones_like(off) * 2.0 ** -24
    arg[:, 1] *= np.tan(np.abs(ref[~g, 1]))
    bound = arg + 3 * np.spacing(np.abs(ref[~g]).astype(np.float32)).astype(np.float64)
    assert np.all(off <= bound), np.max(off / bound)


def test_s4_state_vector_euler_has_the_guard():
    """`_getDroneStateVectors()` (and render(), and user _computeTruncated hooks) take rpy from params.euler_from_quaternion:
    roll == 0 and pitch == +-pi/2 exactly in the guard branch, yaw Bullet's 2 atan2(-+x, +-y); elsewhere within a few ulps of
    Bullet (torch's CPU atan2/asin are not glibc's)."""
    q = S.guard_quats()
    ref = S.euler(q)
    got = euler_from_quaternion(torch.from_numpy(q)).numpy()
    g = np.abs(S.sarg(q)) >= S.GUARD
    assert np.all(got[g, 0] == 0.0) and np.array_equal(got[g, 1], ref[g, 1])
    d = np.abs(got - ref)
    d = np.minimum(d, 2 * np.pi - d)
    assert np.all(d <= 8 * np.spacing(np.pi)), d.max()
    # and shape handling of the [E, D, 4] tensors the env passes
    assert euler_from_quaternion(torch.from_numpy(q[:6]).view(2, 3, 4)).shape == (2, 3, 3)


def test_s5_ground_effect_switch_is_the_references():
    """qs::upright equals |RN(atan2(ra, rb))| < fl(pi/2) and |pitch| < fl(pi/2) of the stand-in exactly, at roll = +-pi/2 with
    rb tiny positive, zero and negative, and at the gimbal guard."""
    q = np.concatenate([S.upright_quats(), S.guard_quats()])
    got = np.zeros(q.shape[0], np.uint8)
    host_harness().hh_upright(ptr(np.ascontiguousarray(q)), q.shape[0], ptr(got))
    want = S.upright(q)
    assert np.array_equal(got != 0, want), int(((got != 0) != want).sum())
    # negative control: the plain `rb > 0` rule disagrees on this sweep (it reaches the rounding window of atan2)
    x, y, z, w = q.T
    rb = w * w - x * x - y * y + z * z
    naive = (np.abs(S.sarg(q)) < S.GUARD) & ((rb > 0) | ((rb == 0) & (2 * (y * z + w * x) == 0)))
    assert (naive != want).sum() > 50, int((naive != want).sum())
    print("S5 host: %d quaternions, %d upright, the rb > 0 rule differs on %d" % (q.shape[0], want.sum(), (naive != want).sum()))


def test_s6_pid_at_the_guard_and_the_yaw_wrap():
    """DSLPIDControl.computeControl (qc pid_control) with pitch at the gimbal guard and yaw at +-pi with last_rpy across the
    wrap, teacher-forced against the oracle's controller, at the 1e-7 of the other PID tests.  A wrong guard branch moves the
    D term by ~(pi/2)/dt * kd, far outside it."""
    L = host_harness()
    st = S.pid_states()
    dt = 1 / 48
    P = fill_params(AviaryConstants(DroneModel.CF2X), pid_model=DroneModel.CF2X)
    want_rpm, want_last = S.oracle_pid(st, dt)
    n = st["pos"].shape[0]
    for i in range(n):
        s9 = np.zeros(9)
        s9[3:6] = st["last_rpy"][i]
        rpm, pe, ye = np.zeros(4), np.zeros(3), C.c_double()
        c = lambda k: np.ascontiguousarray(st[k][i])      # noqa: E731
        L.hh_pid(C.addressof(P), ptr(s9), dt, ptr(c("pos")), ptr(c("quat")), ptr(c("vel")), ptr(c("target_pos")),
                 float(st["target_rpy"][i, 2]), ptr(np.zeros(3)), ptr(np.zeros(3)), ptr(rpm), ptr(pe), C.addressof(ye))
        assert np.max(np.abs(rpm - want_rpm[i]) / np.abs(want_rpm[i])) < 1e-7, (i, rpm, want_rpm[i])
        assert np.max(np.abs(s9[3:6] - want_last[i])) < 1e-7, i


def test_s5_ground_effect_tick_uses_the_switch():
    """One PYB_GND tick of dyn_tick_k (240/240 Hz: one substep) from S5 states, below, near and above GND_EFF_H_CLIP, against
    the float64 oracle's substep with the stand-in's upright decision, at TIGHT: this pins how dyn_tick_k wires qs::upright
    (which quaternion, the arguments, the per-propeller force).  Negative control: the oracle with the other decision misses
    by far more than TIGHT."""
    from gym_pybullet_drones_b200 import _native as N
    from qs_testlib import TIGHT, HostSim, relerr
    pos, q = S.ground_effect_states()
    n = q.shape[0]
    sim = HostSim(fill_params(AviaryConstants(DroneModel.CF2X, 240, 240)), n, N.ACT_RPM, 4, 1, effects=N.EFFECT_GND)
    sim.set_state(pos, q, np.zeros((n, 3)), np.zeros((n, 3)))
    out = sim.tick(np.full((n, 4), 0.3, np.float32))
    p1, _, v1, w1 = S.oracle_ground_effect_tick(pos, q, 0.3)
    assert relerr(out["pos"], p1) < TIGHT and relerr(out["vel"], v1) < TIGHT and relerr(out["rpy_rates"], w1) < TIGHT
    _, _, v2, w2 = S.oracle_ground_effect_tick(pos, q, 0.3, flip=True)
    assert relerr(out["vel"], v2) > 1e5 * TIGHT and relerr(out["rpy_rates"], w2) > 1e5 * TIGHT
    up = S.upright(q)
    assert 0 < up.sum() < n
