"""Every threshold decision of the step and rollout kernels at its boundary (-m gpu): tilt and position truncation, termination,
the gimbal guard of the reported angles (KIN rows, [N][20] state rows, the Logger ring, _getDroneStateVectors), the
ground-effect switch inside the tick, the PID controller at the guard and at the yaw wrap, and the observation a reset writes.

Each check compares a decision with the reference's predicate evaluated on the kernel's OWN post-tick float64 state
(env._plane, autoreset off), drone by drone with the Bullet stand-in and the host libm (tests/threshold_sweeps.py).  That
separates the decision from the dynamics, which other tests pin, so no window of 1e-4 is needed: positions allow no band at all,
angles and the distance a band of BAND_ULPS ulps of 0.4 and of 1e-4.  The band covers CUDA's 2-ulp float64 atan2/asin against
glibc's, and the renormalisation of the stored quaternion after the kernel has decided (one rounding per component moves an
angle by up to ~4 ulps of 0.4).  Every run reports how many samples fell inside the band.

States: all four rotor speeds equal and the body rate zero keep the attitude exactly through a tick (the torque sums cancel, and
_integrateQ is skipped); ONE_D_RPM gives equal rotor speeds for any action, RPM for four equal components.  So every tick of a
rollout decides on the attitude of the final planes."""
import contextlib
import math
import os

import numpy as np
import pytest
import torch

import threshold_sweeps as S

pytestmark = pytest.mark.gpu

BAND_ULPS = 16
MODES = {"pipe4": {"QS_FAST_PIPE": "4"}, "pipe2": {"QS_FAST_PIPE": "2"}, "classic": {"QS_FAST_PIPE": "0"}, "general": {"QS_FAST": "0"}}


@contextlib.contextmanager
def _env_vars(values):
    keys = ("QS_FAST", "QS_FAST_PIPE")
    old = {k: os.environ.get(k) for k in keys}
    try:
        for k in keys:
            os.environ.pop(k, None)
        os.environ.update(values)
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _make(kind, E, act="RPM", rpy_f32=True, autoreset=None, physics="DYN", D=2, **kw):
    from gym_pybullet_drones_b200.envs import HoverAviary, MultiHoverAviary
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    args = dict(physics=Physics[physics], act=ActionType[act], num_envs=E, rpy_f32=rpy_f32, autoreset=autoreset, **kw)
    env = HoverAviary(**args) if kind == "hover" else MultiHoverAviary(num_drones=D, **args)
    env.reset()
    return env


def _place(env, pos, quat):
    n = env._N
    env.set_state(pos=pos, quat=quat, vel=np.zeros((n, 3)), rpy_rates=np.zeros((n, 3)))


def _zero(env, T=None):
    shape = (env._E, env._D, env._A) if T is None else (T, env._E, env._D, env._A)
    return torch.zeros(shape, device="cuda")


def _planes(env):
    return env._plane[0, :, 0:3].cpu().numpy().copy(), env._plane[1].cpu().numpy().copy()


def _truncation_predicate(env, kind):
    """[E] the reference's truncation on the planes, and [E] whether an angle sits within the band of the bound."""
    pos, q = _planes(env)
    drone = S.out_of_bounds(pos, kind) | S.tilted(q)
    near = S.tilt_margin(q) <= BAND_ULPS
    D = env._D
    return drone.reshape(-1, D).any(axis=1), near.reshape(-1, D).any(axis=1)


def _check_flags(name, got, want, near, counts):
    """Outside the band the flags equal the predicate; counts[name] = (samples in the band, of which the kernel and the
    predicate disagree)."""
    got = np.asarray(got, bool)
    bad = np.nonzero((got != want) & ~near)[0]
    assert bad.size == 0, (name, bad.size, bad[:8])
    counts[name] = (int(near.sum()), int(((got != want) & near).sum()))


def _tilt_state(kind, E):
    """S1 poses, cycled over E aviaries (both drones of a MultiHover aviary get the same pose, 1 m apart in x)."""
    q = S.quat(S.tilt_poses())
    idx = np.arange(E) % q.shape[0]
    D = 1 if kind == "hover" else 2
    qq = np.repeat(q[idx], D, axis=0)
    pos = np.tile([0.0, 0.0, 0.5], (E * D, 1))                     # off the target: nothing terminates
    if D == 2:
        pos[1::2, 0] = 1.0
    return pos, qq


# ---------------------------------------------------------------------------------------------------------------
# S1 tilt and S2 position bounds: truncated / done of every step kernel
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rpy_f32", [True, False])
@pytest.mark.parametrize("kind", ["hover", "multihover"])
def test_s1_s2_step_truncation_every_kernel(kind, rpy_f32):
    counts = {}
    E = 3040
    pos_t, q_t = _tilt_state(kind, E)
    D = 1 if kind == "hover" else 2
    pos_b = S.bound_positions(kind)
    nb = pos_b.shape[0]
    pos_b_full = np.repeat(pos_b, D, axis=0)
    if D == 2:
        pos_b_full[1::2] = [0.0, 0.0, 1.0]                       # the aviary's other drone well inside
    # S2 rows replace the first nb aviaries, at the identity attitude (x and y are kept bit for bit by the tick)
    pos_t[:nb * D], q_t[:nb * D] = pos_b_full, np.tile([0.0, 0.0, 0.0, 1.0], (nb * D, 1))
    for mode, values in MODES.items():
        for act in (("RPM", "ONE_D_RPM") if mode == "classic" else ("RPM",)):
            with _env_vars(values):
                env = _make(kind, E, act=act, rpy_f32=rpy_f32)
                _place(env, pos_t, q_t)
                env.step(_zero(env))
                torch.cuda.synchronize()
            want, near = _truncation_predicate(env, kind)
            tr, dn = env._truncated.cpu().numpy(), env._done.cpu().numpy()
            _check_flags("%s/%s truncated" % (mode, act), tr, want, near, counts)
            _check_flags("%s/%s done" % (mode, act), dn, want | env._terminated.cpu().numpy(), near, counts)
            pos, _ = _planes(env)
            assert np.array_equal(pos[:nb * D, 0:2], pos_b_full[:, 0:2])      # x, y of the S2 rows untouched
            assert (mode == "general") != bool(env._warp_ticket.any()), mode
    assert min(c[0] for c in counts.values()) > 0, counts
    print("S1/S2 %s rpy_f32=%s: (in band, of which disagreeing) per run %s" % (kind, rpy_f32, counts))


def test_s1_general_kernel_pid_actions():
    """The general kernel with the embedded PID (PID, VEL, ONE_D_PID): the attitude moves during the tick, but the flags must
    still equal the predicate on the planes the tick leaves."""
    counts = {}
    E = 3040
    pos, q = _tilt_state("hover", E)
    for act in ("PID", "VEL", "ONE_D_PID"):
        with _env_vars(MODES["general"]):
            env = _make("hover", E, act=act)
            _place(env, pos, q)
            a = _zero(env)
            if act == "PID":
                a[..., 2] = 1.0
            env.step(a)
            torch.cuda.synchronize()
        want, near = _truncation_predicate(env, "hover")
        _check_flags(act, env._truncated.cpu().numpy(), want, near, counts)
    print("S1 PID actions: in band %s" % counts)


def test_s1_per_aviary_constants_row():
    """A per-aviary constants table (set_physical_params) does not change the decision."""
    counts = {}
    E = 3040
    pos, q = _tilt_state("hover", E)
    for mode in ("pipe4", "general"):
        with _env_vars(MODES[mode]):
            env = _make("hover", E)
            m = torch.full((E,), 0.027, dtype=torch.float64, device="cuda")
            m[::3] = 0.03
            env.set_physical_params(m=m)
            _place(env, pos, q)
            env.step(_zero(env))
            torch.cuda.synchronize()
        assert env._st.phys                                              # the PHYS instantiations ran
        assert (mode == "general") != bool(env._warp_ticket.any()), mode
        want, near = _truncation_predicate(env, "hover")
        _check_flags(mode, env._truncated.cpu().numpy(), want, near, counts)
        assert want[~near].sum() > 0 and (~want[~near]).sum() > 0 and near.sum() > 0
    print("S1 per-aviary table: (in band, of which disagreeing) %s" % counts)


def test_s1_negative_control_one_ulp():
    """Moving tilt_bound by one ulp changes at least one S1 decision: the sweep resolves single ulps."""
    E = 3040
    pos, q = _tilt_state("hover", E)
    res = []
    for bound in (S.TILT, S.ulps(S.TILT, 1)):
        env = _make("hover", E)
        env._P.tilt_bound = bound
        _place(env, pos, q)
        env.step(_zero(env))
        res.append(env._truncated.cpu().numpy().copy())
    assert (res[0] != res[1]).sum() > 0


# ---------------------------------------------------------------------------------------------------------------
# S1 through rollout(): actions, the default policy, a non-default net_arch, next-step and same-step autoreset
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rpy_f32", [True, False])
def test_s1_rollout_truncation(rpy_f32):
    from gym_pybullet_drones_b200.policy import MlpPolicy
    counts, T, E = {}, 3, 3040
    pos, q = _tilt_state("hover", E)
    runs = {}
    for name, act, autoreset, pol in (("actions", "RPM", None, None), ("policy", "ONE_D_RPM", None, "default"),
                                      ("mlp", "ONE_D_RPM", None, [32]), ("next_step", "ONE_D_RPM", "next_step", "default"),
                                      ("same_step", "RPM", "same_step", None), ("same_step_twin", "RPM", None, None)):
        env = _make("hover", E, act=act, rpy_f32=rpy_f32, autoreset=autoreset)
        _place(env, pos, q)
        if pol is None:
            out = env.rollout(_zero(env, T))
        else:
            kw = {} if pol == "default" else dict(net_arch=pol)
            policy = MlpPolicy.random(env._obs_dim, env._A, seed=5, **kw)
            out = env.rollout(policy=policy, num_steps=T if autoreset != "next_step" else 1)
        torch.cuda.synchronize()
        tr = out["truncated"].cpu().numpy()
        runs[name] = tr
        if autoreset is None:
            want, near = _truncation_predicate(env, "hover")
            for k in range(T if pol is None or autoreset is None else 1):
                _check_flags("%s tick %d" % (name, k), tr[k], want, near, counts)
        elif autoreset == "next_step":
            want, near = _truncation_predicate(env, "hover")      # tick 0 of a next-step rollout leaves the terminal state
            _check_flags(name, tr[0], want, near, counts)
    # same-step autoreset gives the flag bits of its autoreset-off twin at the first tick
    assert np.array_equal(runs["same_step"][0], runs["same_step_twin"][0])
    print("S1 rollout rpy_f32=%s: in band %s" % (rpy_f32, counts))


# ---------------------------------------------------------------------------------------------------------------
# S3 termination: the summed distance at 1e-4 (1 +- k 2^-40)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,D", [("hover", 1), ("multihover", 2), ("multihover", 4)])
def test_s3_termination(kind, D):
    ks = np.arange(-64, 65)
    E = ks.size
    counts = {}
    for mode in ("pipe4", "classic", "general"):
        with _env_vars(MODES[mode]):
            env = _make(kind, E, D=D)
            tgt = env._target[:, 0:3].cpu().numpy()          # [D, 3]
            rng = np.random.default_rng(7)
            u = rng.normal(size=(E, D, 3))
            u /= np.linalg.norm(u, axis=2, keepdims=True)
            d = S.TERM_DIST * (1 + ks * 2.0 ** -40) / D
            pos = tgt[None] - u * d[:, None, None]
            _place(env, pos.reshape(-1, 3), np.tile([0.0, 0.0, 0.0, 1.0], (E * D, 1)))
            env.step(_zero(env))
            torch.cuda.synchronize()
        p, _ = _planes(env)
        dist = np.array([sum(np.linalg.norm(tgt[j] - p[e * D + j]) for j in range(D)) for e in range(E)])
        want = dist < S.TERM_DIST
        near = np.abs(dist - S.TERM_DIST) <= BAND_ULPS * np.spacing(S.TERM_DIST)
        assert 0 < want.sum() < E
        _check_flags(mode, env._terminated.cpu().numpy(), want, near, counts)
    print("S3 %s D=%d: (in band, of which disagreeing) %s" % (kind, D, counts))


# ---------------------------------------------------------------------------------------------------------------
# S4 the gimbal guard in the reported angles
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rpy_f32", [True, False])
def test_s4_reported_angles_at_the_guard(rpy_f32):
    """KIN rows and _getDroneStateVectors(): in the guard branch roll == 0 and pitch == float32(+-pi/2) exactly; yaw within
    2 (2^-24 + 2 ulp) of the stand-in's (rpy_f32) or a float32 ulp (float64 angles)."""
    q = S.guard_quats()
    E = q.shape[0]
    env = _make("hover", E, rpy_f32=rpy_f32)
    _place(env, np.tile([0.0, 0.0, 1.0], (E, 1)), q)
    obs, *_ = env.step(_zero(env))
    torch.cuda.synchronize()
    _, qp = _planes(env)
    ref = S.euler(qp)
    sa = np.abs(S.sarg(qp))
    # the kernel takes the branch on the quaternion before the store renormalises it: a sample within a few ulps of the guard
    # may sit on the other side in the planes (the state-vector rows below come from the planes themselves: no band there)
    near = np.abs(sa - S.GUARD) <= BAND_ULPS * np.spacing(S.GUARD)
    g = (sa >= S.GUARD) & ~near
    assert g.sum() > 10 and (sa < S.GUARD).sum() > 10
    print("S4 rpy_f32=%s: %d in the guard branch, %d within %d ulps of it" % (rpy_f32, g.sum(), near.sum(), BAND_ULPS))
    head = obs.cpu().numpy().reshape(E, -1)[:, 3:6]
    assert np.all(head[g, 0] == 0.0)
    assert np.array_equal(head[g, 1], np.float32(ref[g, 1]))
    dy = np.abs(np.angle(np.exp(1j * (head[g, 2].astype(np.float64) - ref[g, 2]))))
    assert np.all(dy <= 2 * (2.0 ** -24 + 2 * np.spacing(np.float32(np.pi))) + np.spacing(np.float32(np.pi))), dy.max()
    sv = env._getDroneStateVectors().reshape(E, 20)
    gp = sa >= S.GUARD
    assert np.all(sv[gp, 7] == 0.0) and np.array_equal(sv[gp, 8], ref[gp, 1])
    d = np.abs(sv[:, 7:10] - ref)
    d = np.minimum(d, 2 * np.pi - d)
    assert np.all(d <= 8 * np.spacing(np.pi)), d.max()


# ---------------------------------------------------------------------------------------------------------------
# S7 the observation a reset writes
# ---------------------------------------------------------------------------------------------------------------
def _reset_rpys(E):
    rng = np.random.default_rng(3)
    base = np.concatenate([S.euler(S.guard_quats()), S.tilt_poses()[::7], rng.uniform(-3, 3, (64, 3)) * [0.5, 0.5, 1.0]])
    return base[np.arange(E) % base.shape[0]].reshape(E, 1, 3)


@pytest.mark.parametrize("rpy_f32", [True, False])
def test_s7_reset_observation_every_path(rpy_f32):
    """reset(), same-step autoreset (pipelined, classic, general step, rollout) and next-step autoreset (general step, rollout)
    write the same head bits: float32 of the stand-in's float64 angles of the initial quaternion."""
    E = 640
    rpys = _reset_rpys(E)
    far = np.tile([10.0, 0.0, 1.0], (E, 1))                          # out of bounds: every aviary truncates at once
    heads = {}
    env = _make("hover", E, rpy_f32=rpy_f32, initial_rpys=rpys)
    obs, _ = env.reset()
    heads["reset"] = obs.cpu().numpy().reshape(E, -1)[:, 0:12]
    init_q = env._init_quat.cpu().numpy().reshape(-1, 4)[:, 0:4]
    ref = np.float32(S.euler(init_q))
    for mode in ("pipe4", "classic", "general"):
        with _env_vars(MODES[mode]):
            env = _make("hover", E, rpy_f32=rpy_f32, autoreset="same_step", initial_rpys=rpys)
            _place(env, far, env._init_quat.cpu().numpy()[:, 0:4])
            obs, _, _, tr, _ = env.step(_zero(env))
            assert bool(tr.all())
            heads["same_step " + mode] = obs.cpu().numpy().reshape(E, -1)[:, 0:12]
    env = _make("hover", E, rpy_f32=rpy_f32, autoreset="same_step", initial_rpys=rpys)
    _place(env, far, env._init_quat.cpu().numpy()[:, 0:4])
    out = env.rollout(_zero(env, 1))
    heads["same_step rollout"] = out["obs"][0].cpu().numpy().reshape(E, -1)[:, 0:12]
    with _env_vars(MODES["general"]):
        env = _make("hover", E, rpy_f32=rpy_f32, autoreset="next_step", initial_rpys=rpys)
        _place(env, far, env._init_quat.cpu().numpy()[:, 0:4])
        env.step(_zero(env))
        obs, *_ = env.step(_zero(env))
        heads["next_step general"] = obs.cpu().numpy().reshape(E, -1)[:, 0:12]
    env = _make("hover", E, rpy_f32=rpy_f32, autoreset="next_step", initial_rpys=rpys)
    _place(env, far, env._init_quat.cpu().numpy()[:, 0:4])
    out = env.rollout(_zero(env, 2))
    heads["next_step rollout"] = out["obs"][1].cpu().numpy().reshape(E, -1)[:, 0:12]
    for k, h in heads.items():
        assert np.array_equal(h[:, 3:6], ref), (k, int((h[:, 3:6] != ref).any(axis=1).sum()))
        assert np.array_equal(h, heads["reset"]), k
    assert math.isfinite(float(ref.sum()))


# ---------------------------------------------------------------------------------------------------------------
# S5 the ground-effect switch inside the device tick
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("physics", ["PYB_GND", "PYB_GND_DRAG_DW"])
def test_s5_ground_effect_tick(physics):
    """One PYB_GND tick (240/240 Hz: one substep; from rest, so drag and the single drone's downwash add nothing) from S5 states
    against the float64 oracle's substep with the stand-in's upright decision, at TIGHT.  The states have |q|^2 == 1 exactly in
    the kernels' arithmetic, so the renormalisation on entry leaves the bits the switch sees untouched.  Negative control: the
    oracle with the other decision misses by far more than TIGHT."""
    from qs_testlib import TIGHT, relerr
    pos, q = S.ground_effect_states()
    E = q.shape[0]
    env = _make("hover", E, physics=physics, pyb_freq=240, ctrl_freq=240)
    assert env.PYB_STEPS_PER_CTRL == 1
    _place(env, pos, q)
    env.step(torch.full((E, 1, 4), 0.3, device="cuda"))
    torch.cuda.synchronize()
    p, _ = _planes(env)
    v = env._plane[2, :, 0:3].cpu().numpy()
    w = np.stack([env._plane[0, :, 3].cpu().numpy(), env._plane[2, :, 3].cpu().numpy(), env._wz.cpu().numpy()], axis=1)
    p1, _, v1, w1 = S.oracle_ground_effect_tick(pos, q, 0.3)
    assert relerr(p, p1) < TIGHT and relerr(v, v1) < TIGHT and relerr(w, w1) < TIGHT, (relerr(v, v1), relerr(w, w1))
    _, _, v2, w2 = S.oracle_ground_effect_tick(pos, q, 0.3, flip=True)
    assert relerr(v, v2) > 1e5 * TIGHT and relerr(w, w2) > 1e5 * TIGHT
    up = S.upright(q)
    assert 0 < up.sum() < E
    print("S5 %s: %d states, %d upright" % (physics, E, up.sum()))


# ---------------------------------------------------------------------------------------------------------------
# S6 the PID controller at the gimbal guard and at the yaw wrap
# ---------------------------------------------------------------------------------------------------------------
def test_s6_pid_at_the_guard_and_the_yaw_wrap():
    """DSLPIDControl.computeControl on the device (pid_kernel) with pitch at the guard and yaw at +-pi with last_rpy across the
    wrap, one call teacher-forced against the oracle's controller at 1e-7 (the bound of the other device PID tests): a wrong
    guard branch moves the D term by ~(pi/2)/dt * kd."""
    from gym_pybullet_drones_b200.control import DSLPIDControl
    from gym_pybullet_drones_b200.utils.enums import DroneModel
    st = S.pid_states()
    n, dt = st["pos"].shape[0], 1 / 48
    ctl = DSLPIDControl(DroneModel.CF2X, num_drones=n)
    ctl.set_state(last_rpy=st["last_rpy"])
    rpm, _, _ = ctl.computeControl(dt, st["pos"], st["quat"], st["vel"], None, st["target_pos"], target_rpy=st["target_rpy"])
    want_rpm, want_last = S.oracle_pid(st, dt)
    assert np.max(np.abs(rpm - want_rpm) / np.abs(want_rpm)) < 1e-7
    assert np.max(np.abs(ctl.last_rpy.reshape(n, 3) - want_last)) < 1e-7
    g = np.abs(S.sarg(st["quat"])) >= S.GUARD
    assert g.sum() > 10


# ---------------------------------------------------------------------------------------------------------------
# S4 the guard in the [N][20] state rows (CtrlAviary.step, qs_ctrl_rollout) and in the Logger ring (float64)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rpy_f32", [True, False])
def test_s4_guard_in_state_rows_and_logger(rpy_f32, tmp_path):
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils import Logger
    from gym_pybullet_drones_b200.utils.enums import Physics
    q = S.guard_quats()[:128]                                                # one aviary of at most one CTA
    D = q.shape[0]
    rows = {}
    env = CtrlAviary(num_drones=D, physics=Physics.DYN, num_envs=1, rpy_f32=rpy_f32)
    lg = Logger(logging_freq_hz=240, output_folder=str(tmp_path), num_drones=D).attach(env, capacity=4)
    env.reset()
    _place(env, np.tile([0.0, 0.0, 1.0], (D, 1)), q)
    rpm = np.full((1, D, 4), 14000.0, np.float32)                            # equal rotor speeds: the attitude is kept
    obs, *_ = env.step(torch.from_numpy(rpm).cuda())
    torch.cuda.synchronize()
    rows["step"] = obs.cpu().numpy().reshape(D, 20)
    _, qp = _planes(env)
    assert lg.flush() == 1
    logged = lg.states[:, 6:9, 0]                                            # Logger.py order: pos3 vel3 rpy3 (float64)
    env2 = CtrlAviary(num_drones=D, physics=Physics.DYN, num_envs=1, rpy_f32=rpy_f32)
    env2.reset()
    _place(env2, np.tile([0.0, 0.0, 1.0], (D, 1)), q)
    out = env2.rollout(actions=torch.from_numpy(rpm[None]).cuda())
    rows["ctrl_rollout"] = out["obs"][0].cpu().numpy().reshape(D, 20)
    assert np.array_equal(_planes(env2)[1], qp)
    sa = np.abs(S.sarg(qp))
    ref = S.euler(qp)
    near = np.abs(sa - S.GUARD) <= BAND_ULPS * np.spacing(S.GUARD)
    g = (sa >= S.GUARD) & ~near
    assert g.sum() > 10
    for k, r in rows.items():
        assert np.all(r[g, 7] == 0.0) and np.array_equal(r[g, 8], np.float32(ref[g, 1])), k
    # the Logger ring carries float64 angles from the planes: Bullet's branch exactly, by the planes' own sarg
    gp = sa >= S.GUARD
    assert np.all(logged[gp, 0] == 0.0) and np.array_equal(logged[gp, 1], ref[gp, 1])
    d = np.abs(logged - ref)
    assert np.all(np.minimum(d, 2 * np.pi - d) <= 8 * np.spacing(np.pi)), d.max()
