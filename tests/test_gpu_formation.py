"""-m gpu: neighbourhood query, culled downwash and the sharded-formation exchange (SURVEY.md 8f rank 3)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from qs_testlib import relerr

pytestmark = pytest.mark.gpu


def _imports():
    from gym_pybullet_drones_b200 import _native as N
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.formation import FormationShard, morton_order
    from gym_pybullet_drones_b200.utils.enums import Physics
    from oracle import dyn_oracle as O
    return N, CtrlAviary, FormationShard, morton_order, Physics, O


def config4_grid(nx, ny, pitch=0.15):
    """BASELINE config 4 geometry (SURVEY.md 8d): grid in xy with 0.15 m pitch, z = 0.1 + 0.05 (i mod 16).  Used for
    STATIC force evaluations only (nearly equal heights make the dynamics ill-conditioned, see stacks())."""
    k = np.arange(nx * ny)
    j, i = np.divmod(k, nx)
    return np.stack([pitch * i, pitch * j, 0.1 + 0.05 * (k % 16)], axis=1).astype(np.float32).astype(np.float64)


def stacks(nx, ny, pitch=1.6):
    """nx x ny stacks of 4 drones 1.5 m apart with small lateral offsets (well-conditioned dynamics: the model's
    1/dz^2 term is singular for nearly equal heights, so drones of one layer never get within the Gaussian's reach)."""
    k = np.arange(nx * ny * 4)
    st, ly = k // 4, k % 4
    return np.stack([pitch * (st % nx) + 0.04 * ly, pitch * (st // nx) - 0.03 * ly, 0.5 + 1.5 * ly], axis=1).astype(np.float32).astype(np.float64)


def _fz(N, env, cull=True, boxed=False):
    D = env._D
    fz = torch.zeros(env._E * D, device="cuda")
    old = os.environ.get("QS_DW_CULL")
    os.environ["QS_DW_CULL"] = "1" if cull else "0"
    sp = torch.cuda.current_stream().cuda_stream
    try:
        if boxed:
            ws = torch.zeros((env._E, (D + 31) // 32, 8), device="cuda")
            N.check(N.lib().qs_downwash_boxed(C.byref(env._P), C.byref(env._st), env._E, D, ws.data_ptr(), fz.data_ptr(), sp), "qs_downwash_boxed")
        else:
            N.check(N.lib().qs_downwash(C.byref(env._P), C.byref(env._st), env._E, D, fz.data_ptr(), sp), "qs_downwash")
    finally:
        if old is None:
            del os.environ["QS_DW_CULL"]
        else:
            os.environ["QS_DW_CULL"] = old
    return fz.cpu().numpy()


def test_adjacency_golden(golden):
    """BaseAviary._getAdjacencyMatrix of the unmodified reference on three random swarms: bit-exact."""
    N, CtrlAviary, _, _, Physics, _ = _imports()
    g = golden("adjacency")
    for k in range(3):
        pos, radius = g["case%d_pos" % k], float(g["case%d_radius" % k])
        env = CtrlAviary(num_drones=pos.shape[0], neighbourhood_radius=radius, initial_xyzs=pos, physics=Physics.DYN)
        adj = env._getAdjacencyMatrix()
        assert adj.dtype == np.float64 and np.array_equal(adj, g["case%d_adjacency" % k])


@pytest.mark.parametrize("E,D,radius", [(3, 1000, 0.7), (1, 4096, 1.1), (5, 37, np.inf), (2, 512, 0.0), (2, 48, -1.0)])
def test_adjacency_vs_oracle(E, D, radius):
    """Vector query [E, D, D] against the NumPy restatement: ragged D (scalar stores), D % 16 == 0 (16-byte stores),
    several column tiles, radius 0 and negative (identity) and inf (all ones)."""
    N, CtrlAviary, _, _, Physics, O = _imports()
    rng = np.random.default_rng(3)
    pos = rng.uniform(-2, 2, (E, D, 3)).astype(np.float32).astype(np.float64)
    env = CtrlAviary(num_drones=D, neighbourhood_radius=radius, initial_xyzs=pos, physics=Physics.DYN, num_envs=E)
    env.reset()
    adj = env.adjacency().cpu().numpy()
    ref = O.adjacency_matrix(pos, radius)
    assert adj.dtype == np.uint8 and np.array_equal(adj, ref.astype(np.uint8))
    assert np.array_equal(adj, adj.transpose(0, 2, 1))


@pytest.mark.parametrize("D", [864, 1000])
def test_adjacency_pairs_on_the_threshold(D):
    """A lattice with 0.25 m pitch and radius 1.0: thousands of pairs sit EXACTLY on the threshold (4 steps along an axis,
    3-4-5 triangles ... -- the reference's `<` says no) and, after perturbing random coordinates by 1e-9 ... 1e-6, within a
    few float32 ulps of it on either side.  The float32 fast decision must hand every such pair to the float64 arithmetic of
    the reference (the kernel's band logic): bit-exact against the float64 restatement."""
    N, CtrlAviary, _, _, Physics, O = _imports()
    k = np.arange(D)
    pos = np.stack([0.25 * (k % 12), 0.25 * ((k // 12) % 12), 0.25 * (k // 144)], axis=1).astype(np.float64)
    rng = np.random.default_rng(11)
    eps = rng.choice([0.0, 1e-9, -1e-9, 3e-8, -3e-8, 1e-6, -1e-6], size=pos.shape, p=[0.4, 0.1, 0.1, 0.1, 0.1, 0.1, 0.1])
    pos = pos + eps
    env = CtrlAviary(num_drones=D, neighbourhood_radius=1.0, initial_xyzs=pos, physics=Physics.DYN, num_envs=1)
    env.reset()
    adj = env.adjacency().cpu().numpy()
    ref = O.adjacency_matrix(pos[None], 1.0).astype(np.uint8)
    d = np.sqrt(np.sum((pos[:, None, :] - pos[None, :, :]) ** 2, axis=-1))
    assert np.count_nonzero(np.abs(d - 1.0) < 1e-5) > 2000              # the case really is full of threshold pairs
    assert np.array_equal(adj, ref)


@pytest.mark.parametrize("order", ["rows", "morton", "shuffled"])
def test_downwash_culling_is_exact(order):
    """Chunk culling only skips pairs that fail the reference's predicate or whose Gaussian is exactly 0.0f: the culled
    kernel is BIT-identical to the all-pairs evaluation, whatever the index order, and both match the oracle."""
    N, CtrlAviary, _, morton_order, Physics, O = _imports()
    xyz = config4_grid(64, 64)
    if order == "morton":
        xyz = xyz[morton_order(xyz[:, :2])]
    elif order == "shuffled":
        xyz = xyz[np.random.default_rng(1).permutation(len(xyz))]
    env = CtrlAviary(num_drones=len(xyz), initial_xyzs=xyz, physics=Physics.PYB_DW, num_envs=1)
    env.reset()
    ref = O.downwash_body_z(O.OracleParams(), xyz[None])[0]
    assert np.count_nonzero(ref) > 0.7 * len(xyz)
    for boxed in (False, True):                      # tiled kernel (qs_downwash) and box-table kernel (qs_downwash_boxed)
        a, b = _fz(N, env, cull=True, boxed=boxed), _fz(N, env, cull=False, boxed=boxed)
        assert np.array_equal(a, b), boxed
        assert relerr(a, ref) < 1e-5, boxed


def test_downwash_cutoff_10m_and_ragged_tiles():
    """Sources beyond the 10 m xy cut-off (BaseAviary.py:800) and a drone count that is no multiple of the tile sizes."""
    N, CtrlAviary, _, _, Physics, O = _imports()
    rng = np.random.default_rng(8)
    D = 777
    xyz = np.stack([rng.uniform(-9, 9, D), rng.uniform(-9, 9, D), 0.5 + 4.0 * rng.integers(0, 6, D) + rng.uniform(0, 0.3, D)], axis=1)
    xyz = xyz.astype(np.float32).astype(np.float64)
    env = CtrlAviary(num_drones=D, initial_xyzs=xyz, physics=Physics.PYB_DW, num_envs=1)
    env.reset()
    ref = O.downwash_body_z(O.OracleParams(), xyz[None])[0]
    for boxed in (False, True):
        a, b = _fz(N, env, cull=True, boxed=boxed), _fz(N, env, cull=False, boxed=boxed)
        assert np.array_equal(a, b), boxed
        assert relerr(a, ref) < 1e-5, boxed


def _run_local(FormationShard, Physics, xyz, acts, **kw):
    env = FormationShard(xyz, physics=Physics.PYB_GND_DRAG_DW, exchange="local", rank=0, world=1, pyb_freq=240, ctrl_freq=48, **kw)
    env.reset()
    for a in acts:
        obs, _, _, _, _ = env.step(torch.from_numpy(a).cuda())
    torch.cuda.synchronize()
    return obs.clone(), (env.pos.clone(), env.quat.clone(), env.vel.clone(), env.rpy_rates.clone())


@pytest.mark.parametrize("world,fused", [(1, True), (2, True), (3, True), (2, False)])
def test_formation_shards_p2p_protocol_one_gpu(world, fused):
    """The push + flag exchange with `world` in-process shards on ONE device, each on its own stream: the states after
    6 ticks x 5 substeps are bit-identical to the unsharded formation (chunks and row groups are 32 consecutive drones of
    the GLOBAL index, so the summation order does not depend on the partition), no wait timed out.  fused: the positions are
    pushed by the dynamics kernel's epilogue (qs_dyn_substeps_pub; one explicit qs_dw_publish after the reset only), else by a
    qs_dw_publish launch per substep."""
    N, _, FormationShard, _, Physics, O = _imports()
    xyz = stacks(16, 12)                                  # 768 drones: 768 / 384 / 256 per rank, all multiples of 32
    n, T = len(xyz), 6
    rng = np.random.default_rng(11)
    hover = O.OracleParams().HOVER_RPM
    acts = [(hover * (1 + 0.05 * rng.uniform(-1, 1, (1, n, 4)))).astype(np.float32) for _ in range(T)]
    obs_ref, planes_ref = _run_local(FormationShard, Physics, xyz, acts)
    shards = [FormationShard(xyz, physics=Physics.PYB_GND_DRAG_DW, exchange="p2p", rank=r, world=world,
                             pyb_freq=240, ctrl_freq=48) for r in range(world)]
    if world > 1:
        for s in shards:
            s.connect(shards)
    for s in shards:
        assert s._fuse_publish
        s._fuse_publish = fused
    streams = [torch.cuda.Stream() for _ in shards]
    torch.cuda.synchronize()
    for s in shards:
        s.reset()
    torch.cuda.synchronize()
    outs = [None] * world
    for a in acts:
        a_dev = torch.from_numpy(a).cuda()
        torch.cuda.synchronize()
        for r, s in enumerate(shards):
            with torch.cuda.stream(streams[r]):
                outs[r] = s.step(a_dev[:, s.shard.start:s.shard.stop].contiguous())[0]
    torch.cuda.synchronize()
    assert not any(s.exchange_timed_out() for s in shards)
    obs = torch.cat(outs, dim=1)
    assert torch.equal(obs, obs_ref)
    for k, name in enumerate(("pos", "quat", "vel", "rpy_rates")):
        assert torch.equal(torch.cat([getattr(s, name) for s in shards], dim=1), planes_ref[k]), name


def test_formation_local_vs_oracle():
    """FormationShard(exchange='local') = CtrlAviary with the external downwash stage, against the O(N^2) oracle."""
    N, _, FormationShard, _, Physics, O = _imports()
    xyz = stacks(16, 8)
    n, T = len(xyz), 8
    env = FormationShard(xyz, physics=Physics.PYB_GND_DRAG_DW, exchange="local", rank=0, world=1, pyb_freq=240, ctrl_freq=48)
    ora = O.OracleAviary("ctrl", 1, n, ctrl_freq=48, initial_xyzs=xyz, effects=7)
    env.reset(); ora.reset()
    rng = np.random.default_rng(2)
    for t in range(T):
        a = (ora.P.HOVER_RPM * (1 + 0.05 * rng.uniform(-1, 1, (1, n, 4)))).astype(np.float32)
        obs, _, _, _, _ = env.step(torch.from_numpy(a).cuda())
        o_obs, _, _, _ = ora.step(a)
        o = obs.cpu().numpy()
        assert relerr(o[..., 0:3], o_obs[..., 0:3]) < 1e-5, t
        assert relerr(o[..., 7:16], o_obs[..., 7:16]) < 1e-5, t


def test_multi_aviary_boxed_downwash_and_ragged_sizes():
    """qs_downwash_boxed over several aviaries with a drone count that is no multiple of 32 (partial last chunk and row
    group), against the oracle and bit-identical to its all-chunks evaluation."""
    N, CtrlAviary, _, _, Physics, O = _imports()
    rng = np.random.default_rng(4)
    E, D = 3, 333
    xyz = np.stack([rng.uniform(-6, 6, (E, D)), rng.uniform(-6, 6, (E, D)), 0.5 + 3.0 * rng.integers(0, 5, (E, D)) + rng.uniform(0, 0.2, (E, D))], axis=2)
    xyz = xyz.astype(np.float32).astype(np.float64)
    env = CtrlAviary(num_drones=D, initial_xyzs=xyz, physics=Physics.PYB_DW, num_envs=E)
    env.reset()
    a, b = _fz(N, env, cull=True, boxed=True), _fz(N, env, cull=False, boxed=True)
    assert np.array_equal(a, b)
    ref = O.downwash_body_z(O.OracleParams(), xyz).reshape(-1)
    assert np.count_nonzero(ref) > 0.5 * E * D and relerr(a, ref) < 1e-5


def test_p2p_needs_chunk_aligned_shards():
    _, _, FormationShard, _, Physics, _ = _imports()
    with pytest.raises(ValueError):
        FormationShard(stacks(5, 5), physics=Physics.PYB_DW, exchange="p2p", rank=0, world=2)


def test_device_morton_resort_keeps_drone_ids_and_trajectories():
    """reorder_by_morton(): a formation stored in a spatially incoherent order is re-binned on the device every few ticks;
    actions and observations keep the caller's drone ids, the trajectories equal those of the untouched env up to the
    float32 summation order of the pair term, and the culled downwash kernel gets cheaper."""
    N, CtrlAviary, _, morton_order, Physics, O = _imports()
    xyz = stacks(16, 16)                                                    # 1024 drones
    rng = np.random.default_rng(3)
    xyz = xyz[rng.permutation(len(xyz))]                                    # scrambled storage order
    n, T = len(xyz), 12
    kw = dict(num_drones=n, initial_xyzs=xyz, physics=Physics.PYB_GND_DRAG_DW, pyb_freq=240, ctrl_freq=48, num_envs=1)
    a, b = CtrlAviary(**kw), CtrlAviary(**kw)
    a.reset(); b.reset()
    hover = O.OracleParams().HOVER_RPM
    for t in range(T):
        if t % 3 == 0:
            order = b.reorder_by_morton()
            assert sorted(order.cpu().tolist()) == list(range(n))
        act = torch.from_numpy((hover * (1 + 0.05 * rng.uniform(-1, 1, (1, n, 4)))).astype(np.float32)).cuda()
        oa, *_ = a.step(act)
        ob, *_ = b.step(act)
        assert relerr(ob[..., 0:3].cpu().numpy(), oa[..., 0:3].cpu().numpy()) < 1e-6 and relerr(ob[..., 10:13].cpu().numpy(), oa[..., 10:13].cpu().numpy()) < 1e-5, t
    # storage order of b is now spatially coherent: its chunk boxes are small
    def box_volume(env):
        p = env._pos_f32[:, 0:3].view(-1, 32, 3)
        return float(((p.max(dim=1).values - p.min(dim=1).values).clamp_min(1e-3)).prod(dim=1).mean())
    assert box_volume(b) < 0.2 * box_volume(a)
