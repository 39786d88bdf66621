"""-m gpu: a formation re-binned by reorder_by_morton() keeps the caller's drone ids through every drone-indexed API.

reorder_by_morton() permutes the STORAGE order of a large downwash formation.  Env A is stored scrambled and reordered before
its first tick (twice in a row) and then every 3 ticks; twin B has the same arguments and is never reordered.  Everything is
compared in drone-id order: A against B up to the float32 summation order of the downwash pair term (1e-6 on positions, 1e-5
on float32 observation fields), and B (so A) against the float64 tier-2 oracle at RTOL.  Negative control in every test: the
permutation is far from the identity, and the same comparison made on A's storage order misses its bound by at least 10^3
(any two drones of the formation are >= 1.5 m apart), so a surface that forgets to map ids fails loudly."""
import functools

import numpy as np
import pytest
import torch

from mrac_testlib import TF_TOL, err, gains_of
from qs_testlib import RTOL, quat_err, relerr
from test_gpu_formation import stacks

pytestmark = pytest.mark.gpu

SIZES = [1024, 333]              # 32 full chunks, and a ragged last chunk (the first 333 drones of stacks(10, 9))
POS_TOL, OBS_TOL = 1e-6, 1e-5
MRAC_TOL = 1e-4                  # Kx / Kr / Xm after 12 free-running ticks (measured 1.5e-5 between A and B at 1 024 drones)
T = 12                           # free-running ticks at 240 / 240 Hz


def _imports():
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils.enums import Physics
    from oracle import dyn_oracle as O
    return CtrlAviary, Physics, O


def _formation(D):
    """stacks() scrambled by a fixed permutation (the storage order the caller hands over)."""
    xyz = stacks(16, 16) if D == 1024 else stacks(10, 9)[:D]
    perm = np.random.default_rng(5).permutation(D)
    assert np.count_nonzero(perm == np.arange(D)) < D // 10
    return xyz[perm]


def _twins(cls, xyz, **kw):
    _, Physics, _ = _imports()
    kw = dict(dict(physics=Physics.PYB_GND_DRAG_DW, pyb_freq=240, ctrl_freq=240, num_envs=1), **kw)
    envs = [cls(num_drones=len(xyz), initial_xyzs=xyz, **kw) for _ in range(2)]
    for e in envs:
        e.reset()
    return envs


def _reorder(env, t):
    """A's schedule: two reorders in a row before the first tick, then one every 3 ticks."""
    if t == 0:
        env.reorder_by_morton()
    elif t % 3:
        return
    o = env.reorder_by_morton().cpu().numpy()
    assert np.array_equal(np.sort(o), np.arange(len(o)))
    assert np.count_nonzero(o == np.arange(len(o))) < len(o) // 10          # far from the identity


def _hover_actions(rng, D):
    _, _, O = _imports()
    return (O.OracleParams().HOVER_RPM * (1 + 0.05 * rng.uniform(-1, 1, (1, D, 4)))).astype(np.float32)


def _np(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _agree(got, want, tol, storage, what):
    """A's rows (drone ids) within `tol` of B's; A's storage-order rows miss by >= 10^3 x tol (negative control)."""
    assert relerr(got, want) < tol, (what, relerr(got, want))
    assert relerr(storage, want) > 1e3 * tol, (what, "negative control", relerr(storage, want))


def _same_obs(a, oa, ob):
    """[D, k] observations of A and B: positions at POS_TOL, the other float32 fields at OBS_TOL."""
    storage = _np(a._obs_buf[a._cur])
    _agree(oa[:, 0:3], ob[:, 0:3], POS_TOL, storage[:, 0:3], "obs pos")
    assert relerr(oa[:, 3:], ob[:, 3:]) < OBS_TOL


def _state20_vs_oracle(o, ref):
    """[D, 20] state rows against the oracle's state vectors."""
    assert relerr(o[:, 0:3], ref[:, 0:3]) < RTOL and quat_err(o[:, 3:7], ref[:, 3:7]) < RTOL
    assert relerr(o[:, 7:16], ref[:, 7:16]) < RTOL and relerr(o[:, 16:20], ref[:, 16:20]) < RTOL


def _same_state(a, b):
    """State views and state vectors of A (drone ids) against B's."""
    _agree(_np(a.pos[0]), _np(b.pos[0]), POS_TOL, _np(a._plane[0, :, 0:3]), "pos")
    for name in ("quat", "vel", "rpy_rates"):
        assert relerr(_np(getattr(a, name)), _np(getattr(b, name))) < OBS_TOL, name
    assert torch.equal(a.last_clipped_action, b.last_clipped_action)           # the same clipped actions, bit for bit
    sa, sb = a._getDroneStateVectors()[0], b._getDroneStateVectors()[0]
    _agree(sa[:, 0:3], sb[:, 0:3], POS_TOL, _np(a._plane[0, :, 0:3]), "state vector pos")
    assert relerr(sa[:, 3:16], sb[:, 3:16]) < OBS_TOL and np.array_equal(sa[:, 16:20], sb[:, 16:20])
    for j in (0, 1, len(sa) // 2, len(sa) - 1):
        assert np.array_equal(a._getDroneStateVector(j), sa[j]), j
    return sb


def _set_oracle_state(ora, O, pos, quat, vel, w):
    ora.pos, ora.quat, ora.vel, ora.rpy_rates = (np.array(x, dtype=np.float64)[None] for x in (pos, quat, vel, w))
    ora.rpy = O.quat_to_euler(ora.quat)


# ---------------------------------------------------------------------------------------------------------------------
# 1. state views and set_state

@pytest.mark.parametrize("D", SIZES)
def test_state_views_and_set_state(D):
    CtrlAviary, _, O = _imports()
    xyz = _formation(D)
    a, b = _twins(CtrlAviary, xyz, track_last_action=True)
    ora = O.OracleAviary("ctrl", 1, D, ctrl_freq=240, initial_xyzs=xyz, effects=7)
    rng = np.random.default_rng(1)
    for t in range(T):
        _reorder(a, t)
        act = _hover_actions(rng, D)
        a.step(torch.from_numpy(act).cuda()); b.step(torch.from_numpy(act).cuda()); ora.step(act)
        sb = _same_state(a, b)
        _state20_vs_oracle(sb, ora.state_vector()[0])
    # set_state with drone-id arrays: drone `hi` is put 0.4 m above drone `lo`, into its downwash
    pos, quat, vel, w = (_np(getattr(b, k)[0]).copy() for k in ("pos", "quat", "vel", "rpy_rates"))
    lo, hi = int(np.argmin(pos[:, 2] + 1e-3 * pos[:, 0])), int(np.argmax(pos[:, 2] + 1e-3 * pos[:, 0]))
    fz_before = O.downwash_body_z(ora.P, pos[None])[0]
    pos[hi] = pos[lo] + [0.02, -0.01, 0.4]
    for env in (a, b):
        env.set_state(pos=pos[None], quat=quat[None], vel=vel[None], rpy_rates=w[None])
    _set_oracle_state(ora, O, pos, quat, vel, w)
    for name in ("pos", "quat", "vel", "rpy_rates"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name
    # the float32 mirror the downwash kernels read was written in storage order
    assert torch.equal(a._pos_f32[a._inv, 0:3], a.pos[0].float())
    assert relerr(_np(a._pos_f32[:, 0:3]), pos) > 1e3 * POS_TOL
    ref_fz = O.downwash_body_z(ora.P, ora.pos)[0]
    assert abs(ref_fz[lo]) > 2 * abs(fz_before[lo])
    act = _hover_actions(rng, D)
    a.step(torch.from_numpy(act).cuda()); b.step(torch.from_numpy(act).cuda()); ora.step(act)
    scale = np.max(np.abs(ref_fz))
    fa, fb, fs = _np(a._dw_fz[a._inv]), _np(b._dw_fz), _np(a._dw_fz)
    assert np.max(np.abs(fa - ref_fz)) < 1e-5 * scale and np.max(np.abs(fb - ref_fz)) < 1e-5 * scale
    assert np.max(np.abs(fs - ref_fz)) > 1e-2 * scale                                      # negative control
    sb = _same_state(a, b)
    _state20_vs_oracle(sb, ora.state_vector()[0])


# ---------------------------------------------------------------------------------------------------------------------
# 2. every step path

PATHS = ["torch_f32", "numpy_f32", "numpy_f64", "torch_f64", "single_env", "formation_shard"]


@functools.lru_cache(maxsize=None)
def _oracle_run(D):
    _, _, O = _imports()
    ora = O.OracleAviary("ctrl", 1, D, ctrl_freq=240, initial_xyzs=_formation(D), effects=7)
    rng = np.random.default_rng(2)
    acts, obs = [], []
    for _ in range(T):
        act = _hover_actions(rng, D)
        acts.append(act)
        obs.append(ora.step(act)[0][0])
    return acts, obs


def _path_twins(path, xyz):
    CtrlAviary, Physics, _ = _imports()
    if path == "formation_shard":
        from gym_pybullet_drones_b200.formation import FormationShard
        envs = [FormationShard(xyz, physics=Physics.PYB_GND_DRAG_DW, exchange="local", rank=0, world=1, pyb_freq=240, ctrl_freq=240)
                for _ in range(2)]
        for e in envs:
            e.reset()
        return envs
    return _twins(CtrlAviary, xyz, num_envs=None) if path == "single_env" else _twins(CtrlAviary, xyz)


def _step_path(env, path, act):
    """One tick through `path`; -> the [D, 20] observation as the path returns it (NumPy or tensor)."""
    D = act.shape[1]
    if path in ("torch_f32", "formation_shard"):
        o = env.step(torch.from_numpy(act).cuda())[0]
        assert isinstance(o, torch.Tensor)
    elif path == "numpy_f32":
        o = env.step(act)[0]
        assert isinstance(o, np.ndarray)
    elif path == "numpy_f64":
        o = env.step(act.astype(np.float64))[0]
    elif path == "torch_f64":
        o = env.step(torch.from_numpy(act.astype(np.float64)).cuda())[0]
    else:
        o = env.step(act[0])[0]
        assert isinstance(o, np.ndarray) and o.shape == (D, 20)
    return _np(o).reshape(D, 20)


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("D", SIZES)
def test_step_paths(D, path):
    xyz = _formation(D)
    a, b = _path_twins(path, xyz)
    acts, ref = _oracle_run(D)
    for t in range(T):
        _reorder(a, t)
        oa, ob = _step_path(a, path, acts[t]), _step_path(b, path, acts[t])
        _same_obs(a, oa, ob)
        _state20_vs_oracle(ob, ref[t])
        _state20_vs_oracle(oa, ref[t])


# ---------------------------------------------------------------------------------------------------------------------
# 3. / 4. the controller loops (DSLPIDControl, MRAC) with a different target per drone

def _targets(xyz, seed):
    rng = np.random.default_rng(seed)
    D = len(xyz)
    tgt = xyz + rng.uniform(-0.3, 0.3, (D, 3))
    trpy = np.concatenate([np.zeros((D, 2)), rng.uniform(-0.5, 0.5, (D, 1))], axis=1)      # saturates the yaw torque
    return tgt, trpy


@pytest.mark.parametrize("D", SIZES)
def test_dslpid_loop(D):
    CtrlAviary, _, O = _imports()
    from gym_pybullet_drones_b200.control import DSLPIDControl
    from gym_pybullet_drones_b200.utils.enums import DroneModel
    xyz = _formation(D)
    a, b = _twins(CtrlAviary, xyz)
    ca, cb = (DSLPIDControl(DroneModel.CF2X, num_drones=D) for _ in range(2))
    opid = O.OraclePID(D)
    tgt, trpy = _targets(xyz, 3)
    for t in range(T):
        _reorder(a, t)
        pos, quat, vel = (_np(getattr(b, k)[0]) for k in ("pos", "quat", "vel"))
        rpm_o, _, _ = opid.compute(b.CTRL_TIMESTEP, pos, quat, vel, tgt, target_rpy=trpy)        # teacher-forced on B's state
        rpm_a, rpm_b = ca.computeControlFromEnv(a, tgt, target_rpy=trpy), cb.computeControlFromEnv(b, tgt, target_rpy=trpy)
        ra, rb = _np(rpm_a).reshape(D, 4), _np(rpm_b).reshape(D, 4)
        _agree(ra, rb, OBS_TOL, ra[_np(a._order)], "rpm")
        assert relerr(rb, rpm_o) < RTOL
        sa, sb = _np(ca._state), _np(cb._state)                               # integral_pos_e, last_rpy, integral_rpy_e
        assert relerr(sa, sb) < OBS_TOL
        assert relerr(sb, np.concatenate([opid.integral_pos_e.T, opid.last_rpy.T, opid.integral_rpy_e.T])) < RTOL
        oa, ob = a.step(rpm_a)[0], b.step(rpm_b)[0]
        _same_obs(a, _np(oa)[0], _np(ob)[0])


@pytest.mark.parametrize("D", SIZES)
def test_mrac_loop(D, golden):
    CtrlAviary, _, O = _imports()
    from gym_pybullet_drones_b200.control import MRAC
    from gym_pybullet_drones_b200.utils.enums import DroneModel
    from oracle.mrac_oracle import OracleMRAC, ang_v_from_state
    xyz = _formation(D)
    a, b = _twins(CtrlAviary, xyz)
    ca, cb = (MRAC(DroneModel.CF2X, num_drones=D) for _ in range(2))
    G = gains_of(golden("mrac"), "cf2x")
    tgt, trpy = _targets(xyz, 4)

    def oracle_from(c, env):
        o = OracleMRAC(D, "cf2x", gains_=G)
        o.Kx, o.Kr, o.Xm, o.control_counter = c.Kx.copy(), c.Kr.copy(), c.Xm.copy(), c.control_counter
        pos, quat, vel, w = (_np(getattr(env, k)[0]) for k in ("pos", "quat", "vel", "rpy_rates"))
        rpm, _, _ = o.compute(env.CTRL_TIMESTEP, pos, quat, vel, ang_v_from_state(quat, w), tgt, trpy)
        return o, np.clip(rpm, 0, env.MAX_RPM)

    for t in range(T):
        _reorder(a, t)
        tf = t == T // 2
        if tf:
            (oa_, rpm_oa), (ob_, rpm_ob) = oracle_from(ca, a), oracle_from(cb, b)
        rpm_a, rpm_b = ca.computeControlFromEnv(a, tgt, target_rpy=trpy), cb.computeControlFromEnv(b, tgt, target_rpy=trpy)
        ra, rb = _np(rpm_a).reshape(D, 4), _np(rpm_b).reshape(D, 4)
        _agree(ra, rb, OBS_TOL, ra[_np(a._order)], "rpm")
        # the adaptation law amplifies the last-bit differences of the states (P = 600 I scale); Kx and Kr start equal for
        # every drone (no adaptation while Xm = X), so the negative control is Xm's (it holds the positions)
        for k in ("Kx", "Kr"):
            assert relerr(getattr(ca, k), getattr(cb, k)) < MRAC_TOL, k
        _agree(ca.Xm, cb.Xm, MRAC_TOL, ca.Xm[_np(a._order)], "Xm")
        assert relerr(_np(ca.last_pos_e), _np(cb.last_pos_e)) < OBS_TOL
        if tf:                                                          # one tick teacher-forced, A and B each on its own state
            for c, o, r, ro in ((ca, oa_, ra, rpm_oa), (cb, ob_, rb, rpm_ob)):
                assert err(r, ro) <= TF_TOL and err(c.Kx, o.Kx) <= TF_TOL and err(c.Kr, o.Kr) <= TF_TOL and err(c.Xm, o.Xm) <= TF_TOL
        oa, ob = a.step(rpm_a)[0], b.step(rpm_b)[0]
        _same_obs(a, _np(oa)[0], _np(ob)[0])


# ---------------------------------------------------------------------------------------------------------------------
# 5. the embedded PID of VelocityAviary, and the terminal / reset observations of same-step autoreset

@pytest.mark.parametrize("D", SIZES)
def test_velocity_aviary_pid_state(D):
    _, _, O = _imports()
    from gym_pybullet_drones_b200.envs import VelocityAviary
    xyz = _formation(D)
    a, b = _twins(VelocityAviary, xyz)
    ora = O.OracleAviary("velocity", 1, D, ctrl_freq=240, initial_xyzs=xyz, effects=7)
    rng = np.random.default_rng(7)
    for t in range(T):
        _reorder(a, t)
        act = np.concatenate([rng.uniform(-1, 1, (1, D, 3)), rng.uniform(0, 1, (1, D, 1))], axis=-1).astype(np.float32)
        oa, ob = _np(a.step(torch.from_numpy(act).cuda())[0])[0], _np(b.step(torch.from_numpy(act).cuda())[0])[0]
        ora.step(act)
        _same_obs(a, oa, ob)
        _state20_vs_oracle(ob, ora.state_vector()[0])
        pa, pb = _np(a.pid_state), _np(b.pid_state)                            # integral_pos_e, last_rpy, integral_rpy_e
        assert relerr(pa, pb) < OBS_TOL
        assert relerr(pb, np.concatenate([ora.ctrl.integral_pos_e.T, ora.ctrl.last_rpy.T, ora.ctrl.integral_rpy_e.T])) < RTOL


def test_rl_envs_refuse_large_downwash_aviaries():
    """The RL tasks reduce over one aviary inside a CTA: MultiHoverAviary with downwash takes at most 128 drones per aviary, so
    a reorderable hover formation does not exist; the refusal is a clear ValueError."""
    _, Physics, _ = _imports()
    from gym_pybullet_drones_b200.envs import MultiHoverAviary
    env = MultiHoverAviary(num_drones=333, initial_xyzs=_formation(333), physics=Physics.PYB_DW, num_envs=1, autoreset="same_step")
    env.reset()
    with pytest.raises(ValueError, match="128"):
        env.step(torch.zeros((1, 333, 4), device="cuda"))


@pytest.mark.parametrize("D", SIZES)
def test_same_step_autoreset_final_and_reset_obs(D):
    """Same-step autoreset of a formation with a task hook: set_state pushes one named drone out of bounds; info["final_obs"]
    and the reset observation are in drone-id order, the reset rows exactly the initial poses."""
    CtrlAviary, _, O = _imports()

    class Fenced(CtrlAviary):
        def _computeTruncated(self):                # the formation spans 25 m in x
            return (self.pos[..., 0].abs() > 30).any(dim=1)

    xyz = _formation(D)
    a, b = _twins(Fenced, xyz, autoreset="same_step")
    ora = O.OracleAviary("ctrl", 1, D, ctrl_freq=240, initial_xyzs=xyz, effects=7)
    rng = np.random.default_rng(8)
    _reorder(a, 0)
    act = _hover_actions(rng, D)
    ra, rb = a.step(torch.from_numpy(act).cuda()), b.step(torch.from_numpy(act).cuda())
    o_obs = ora.step(act)[0][0]
    assert not bool(ra[3][0]) and not bool(rb[3][0])
    oa, ob = _np(ra[0])[0], _np(rb[0])[0]
    _same_obs(a, oa, ob)
    _state20_vs_oracle(ob, o_obs)
    # drone j leaves the fence: the aviary truncates and resets in the same step
    j = D // 3
    pos = _np(b.pos[0]).copy()
    pos[j, 0] = 40.0
    for env in (a, b):
        env.set_state(pos=pos[None])
    ora.pos = pos[None].copy()
    act = _hover_actions(rng, D)
    ra, rb = a.step(torch.from_numpy(act).cuda()), b.step(torch.from_numpy(act).cuda())
    o_obs = ora.step(act)[0][0]
    assert bool(ra[3][0]) and bool(rb[3][0])
    fa, fb = _np(ra[4]["final_obs"])[0], _np(rb[4]["final_obs"])[0]
    _agree(fa[:, 0:3], fb[:, 0:3], POS_TOL, fa[_np(a._order), 0:3], "final_obs pos")
    assert relerr(fa[:, 3:], fb[:, 3:]) < OBS_TOL and fa[j, 0] > 39.0
    _state20_vs_oracle(fb, o_obs)
    _state20_vs_oracle(fa, o_obs)
    # the reset observation: the initial pose of every drone, by drone id, exactly
    oa, ob = _np(ra[0])[0], _np(rb[0])[0]
    init = ora.reset()[0].astype(np.float32)
    assert np.array_equal(oa, init) and np.array_equal(ob, init)
    assert relerr(_np(a._obs_buf[a._cur])[:, 0:3], xyz) > 1e3 * POS_TOL


# ---------------------------------------------------------------------------------------------------------------------
# 6. adjacency, judged on A's own float64 positions

def _check_adjacency(a, radius):
    _, _, O = _imports()
    pos = _np(a._plane[0, :, 0:3][a._inv])[None]           # the kernel's own float64 positions, gathered into drone ids
    ref = O.adjacency_matrix(pos, radius)[0]
    adj = _np(a.adjacency())[0]
    assert np.array_equal(adj, ref.astype(np.uint8))
    assert np.array_equal(a._getAdjacencyMatrix(), ref)
    o = _np(a._order)
    assert np.count_nonzero(adj[o][:, o] != adj) > len(o)                     # the storage-slot matrix is another one


@pytest.mark.parametrize("D", SIZES)
def test_adjacency_formation(D):
    CtrlAviary, _, _ = _imports()
    a, _ = _twins(CtrlAviary, _formation(D), neighbourhood_radius=2.0)
    rng = np.random.default_rng(9)
    for t in range(4):
        _reorder(a, t)
        a.step(torch.from_numpy(_hover_actions(rng, D)).cuda())
        _check_adjacency(a, 2.0)


def test_adjacency_threshold_lattice():
    """The 0.25 m lattice of test_adjacency_pairs_on_the_threshold (thousands of pairs on or within float32 ulps of the 1.0 m
    threshold), stored scrambled and reordered: bit-exact by drone id."""
    CtrlAviary, Physics, _ = _imports()
    D = 864
    k = np.arange(D)
    pos = np.stack([0.25 * (k % 12), 0.25 * ((k // 12) % 12), 0.25 * (k // 144)], axis=1).astype(np.float64)
    rng = np.random.default_rng(11)
    pos = pos + rng.choice([0.0, 1e-9, -1e-9, 3e-8, -3e-8, 1e-6, -1e-6], size=pos.shape, p=[0.4, 0.1, 0.1, 0.1, 0.1, 0.1, 0.1])
    pos = pos[rng.permutation(D)]
    a = CtrlAviary(num_drones=D, neighbourhood_radius=1.0, initial_xyzs=pos, physics=Physics.PYB_DW, num_envs=1)
    a.reset()
    _reorder(a, 0)
    assert np.array_equal(_np(a._plane[0, :, 0:3][a._inv]), pos)
    d = np.sqrt(np.sum((pos[:, None, :] - pos[None, :, :]) ** 2, axis=-1))
    assert np.count_nonzero(np.abs(d - 1.0) < 1e-5) > 2000
    _check_adjacency(a, 1.0)


# ---------------------------------------------------------------------------------------------------------------------
# 7. Logger: the device ring records storage slots, so the combination is refused

def test_logger_refuses_a_reordered_env(tmp_path):
    CtrlAviary, _, _ = _imports()
    from gym_pybullet_drones_b200.utils.Logger import Logger
    D = 333
    xyz = _formation(D)
    a, _ = _twins(CtrlAviary, xyz)
    log = Logger(logging_freq_hz=240, output_folder=str(tmp_path), num_drones=D).attach(a)
    with pytest.raises(ValueError, match="Logger"):
        a.reorder_by_morton()
    assert a._order is None                                                    # refused before anything moved
    obs = _np(a.step(torch.from_numpy(_hover_actions(np.random.default_rng(10), D)).cuda())[0])[0]
    log.detach()
    assert relerr(log.states[:, 0:3, 0], obs[:, 0:3]) < POS_TOL                 # attached before any reorder: drone ids
    _reorder(a, 0)
    with pytest.raises(ValueError, match="reorder_by_morton"):
        Logger(logging_freq_hz=240, output_folder=str(tmp_path), num_drones=D).attach(a)


# ---------------------------------------------------------------------------------------------------------------------
# 8. masked and full reset()

@pytest.mark.parametrize("D", SIZES)
def test_reset_full_and_masked(D):
    CtrlAviary, _, _ = _imports()
    xyz = _formation(D)
    a, b = _twins(CtrlAviary, xyz)
    rng = np.random.default_rng(12)
    for opts in (None, {"reset_mask": np.array([True])}):
        for t in range(5):
            _reorder(a, t)
            act = torch.from_numpy(_hover_actions(rng, D)).cuda()
            a.step(act); b.step(act)
        oa, ob = _np(a.reset(options=opts)[0])[0], _np(b.reset(options=opts)[0])[0]
        assert np.array_equal(oa[:, 0:3], xyz.astype(np.float32)) and np.array_equal(oa, ob)
        assert np.array_equal(_np(a.pos)[0], xyz) and torch.equal(a.quat, b.quat)
        assert relerr(_np(a._obs_buf[a._cur])[:, 0:3], xyz) > 1e3 * POS_TOL
        for _ in range(3):
            act = torch.from_numpy(_hover_actions(rng, D)).cuda()
            oa, ob = _np(a.step(act)[0])[0], _np(b.step(act)[0])[0]
            _same_obs(a, oa, ob)
