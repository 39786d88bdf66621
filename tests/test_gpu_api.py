"""API conformance on the GPU: the surface examples/learn.py, pid.py and SB3 touch (SURVEY.md 8b)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_sb3_vecenv_protocol_episode_stats():
    """SB3 VecEnv protocol (what make_vec_env + Monitor give learn.py): zero action -> every episode is the reference's
    KAT episode: 242 steps, return 333.8626, time-limit truncation, terminal observation = last obs of the episode."""
    from gym_pybullet_drones_b200.envs import HoverAviary
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    from gym_pybullet_drones_b200.vec import SB3VecAviary
    E = 16
    venv = SB3VecAviary(HoverAviary, E, physics=Physics.DYN, act=ActionType.ONE_D_RPM)
    assert venv.num_envs == E and venv.observation_space.shape == (1, 27) and venv.action_space.shape == (1, 1)
    obs = venv.reset()
    assert obs.shape == (E, 1, 27) and obs.dtype == np.float32
    act = np.zeros((E, 1, 1), np.float32)
    last = None
    for t in range(242):
        last = obs
        venv.step_async(act)
        obs, rews, dones, infos = venv.step_wait()
        assert obs.shape == (E, 1, 27) and rews.shape == (E,) and dones.shape == (E,) and len(infos) == E
        if t < 241:
            assert not dones.any() and infos[0] == {}
    assert dones.all()
    for i in range(E):
        ep = infos[i]["episode"]
        assert ep["l"] == 242 and abs(ep["r"] - 333.862626904298) < 1e-2
        assert infos[i]["TimeLimit.truncated"] is True
        term_obs = infos[i]["terminal_observation"]
        assert term_obs.shape == (1, 27) and abs(term_obs[0, 2] - 0.1125) < 1e-6
    # after the auto-reset the returned obs is the reset observation and the counters restarted
    assert np.allclose(obs[:, 0, :3], [0, 0, 0.1125]) and int(venv.env.step_counter.max()) == 0
    assert venv.env_is_wrapped(type("Monitor", (), {})) == [True] * E
    assert venv.get_attr("CTRL_FREQ") == [30] * E
    venv.close()


def test_reference_attribute_surface():
    """Attributes and methods learn.py / pid.py read (learn.py:143,157,168,189; pid.py:116,132,142)."""
    from gym_pybullet_drones_b200.envs import CtrlAviary, HoverAviary, MultiHoverAviary
    from gym_pybullet_drones_b200.utils.enums import ActionType, DroneModel, ObservationType, Physics
    env = MultiHoverAviary(num_drones=2, obs=ObservationType.KIN, act=ActionType.ONE_D_RPM)      # learn.py's call
    assert env.NUM_DRONES == 2 and env.CTRL_FREQ == 30 and env.PYB_FREQ == 240 and env.EPISODE_LEN_SEC == 8
    assert abs(env.CTRL_TIMESTEP - 1 / 30) < 1e-15 and env.PYB_STEPS_PER_CTRL == 8 and env.ACTION_BUFFER_SIZE == 15
    assert env.action_space.shape == (2, 1) and env.observation_space.shape == (2, 27)
    assert env.action_space.dtype == np.float32 and env.observation_space.dtype == np.float32
    assert np.allclose(env.INIT_XYZS, [[0, 0, 0.1125], [0.1588, 0.1588, 0.1125]])
    assert np.allclose(env.TARGET_POS, [[0, 0, 1.1125], [0.1588, 0.1588, 0.6125]])
    assert abs(env.HOVER_RPM - 14468.429183500699) < 1e-9 and abs(env.MAX_RPM - 21702.64377525105) < 1e-9
    obs, info = env.reset(seed=42, options={})
    assert obs.shape == (2, 27) and info == {"answer": 42}
    obs, r, te, tr, info = env.step(env.action_space.sample())
    assert obs.shape == (2, 27) and isinstance(r, float) and isinstance(te, bool) and isinstance(tr, bool)
    env.render()
    env.close()
    assert env.getPyBulletClient() == -1 and list(env.getDroneIds()) == [0, 1]
    c = CtrlAviary(drone_model=DroneModel.CF2X, num_drones=3, physics=Physics.PYB, neighbourhood_radius=10, pyb_freq=240, ctrl_freq=48)
    assert c.action_space.shape == (3, 4) and c.observation_space.shape == (3, 20) and abs(c.action_space.high[0, 0] - c.MAX_RPM) < 1e-2
    obs, _ = c.reset()
    assert obs.shape == (3, 20) and c._getAdjacencyMatrix().shape == (3, 3)
    assert c._getDroneStateVector(1).shape == (20,)
    with pytest.raises(ValueError):
        HoverAviary(pyb_freq=240, ctrl_freq=7)                       # BaseAviary.py:79-80
    with pytest.raises(NotImplementedError):
        HoverAviary(obs=ObservationType.RGB)
    with pytest.raises(ValueError):
        CtrlAviary(num_drones=2, initial_xyzs=np.zeros((3, 3)))


def test_policy_rollout_on_device_config3_shape():
    """Config 3 shape at test size: an SB3-MlpPolicy-shaped torch network drives the vectorised env entirely on the
    device (no host copies), SAME_STEP autoreset, under a CUDA graph."""
    from gym_pybullet_drones_b200.envs import MultiHoverAviary
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    E, D = 4096, 2
    env = MultiHoverAviary(num_drones=D, physics=Physics.DYN, act=ActionType.RPM, num_envs=E, autoreset="same_step")
    torch.manual_seed(0)
    pi = torch.nn.Sequential(torch.nn.Linear(D * 72, 64), torch.nn.Tanh(), torch.nn.Linear(64, 64), torch.nn.Tanh(),
                             torch.nn.Linear(64, D * 4)).cuda()
    obs, _ = env.reset()
    act = torch.zeros((E, D, 4), device="cuda")
    ret = torch.zeros(E, device="cuda")
    n_done = torch.zeros((), device="cuda")

    def one_step(o):
        with torch.no_grad():
            mean = pi(o.reshape(E, -1))
            act.copy_((mean + 0.3 * torch.randn_like(mean)).clamp(-1, 1).view(E, D, 4))
        o2, rew, term, trunc, info = env.step(act)
        ret.add_(rew)
        n_done.add_(info["_final_obs"].sum())
        return o2
    for _ in range(4):
        obs = one_step(obs)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    static_obs = [env._obs_view[0], env._obs_view[1]]
    with torch.cuda.graph(g):
        one_step(static_obs[env._cur])
        one_step(static_obs[env._cur])
    for _ in range(60):
        g.replay()
    torch.cuda.synchronize()
    assert torch.isfinite(ret).all() and float(ret.mean()) > 0 and float(n_done) > 0
    assert int(env.step_counter.max()) <= 8 * 124


@pytest.mark.parametrize("cls,act,D,phys,T", [("MultiHoverAviary", "RPM", 2, "DYN", 300), ("HoverAviary", "ONE_D_RPM", 1, "DYN", 40),
                                              ("HoverAviary", "PID", 1, "DYN", 40), ("MultiHoverAviary", "RPM", 4, "PYB_GND_DRAG_DW", 24),
                                              ("MultiHoverAviary", "VEL", 3, "PYB_DRAG", 24), ("HoverAviary", "PID+clear", 1, "DYN", 60)])
def test_rollout_is_bit_identical_to_steps(cls, act, D, phys, T):
    """qs_rollout(T) == T x qs_step: observations, rewards, flags, final state planes, PID state and counters, bit for bit
    (state in registers / history in a sliding shared-memory window vs HBM round trips).  T=300 also crosses the
    shared-memory window limit, so the Python side splits the rollout into two launches."""
    import gym_pybullet_drones_b200.envs as envs
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    E = 300
    clear = act.endswith("+clear")
    act = act.split("+")[0]
    kw = dict(physics=Physics[phys], act=ActionType[act], num_envs=E, autoreset="same_step")
    if clear:
        kw.update(autoreset_clears_action_buffer=True, autoreset_clears_controllers=True)
    if cls == "MultiHoverAviary":
        kw["num_drones"] = D
        if phys != "DYN":
            kw["initial_xyzs"] = np.array([[0.05 * k, -0.03 * k, 0.3 + 1.5 * k] for k in range(D)])
    e1, e2 = getattr(envs, cls)(**kw), getattr(envs, cls)(**kw)
    A = e1._A
    g = torch.Generator(device="cuda").manual_seed(11)
    acts = torch.rand((T, E, D, A), device="cuda", generator=g) * 2 - 1
    if act == "PID":
        acts = acts * (torch.tensor([2.5, 2.5, 0.5], device="cuda") if clear else 0.3) + torch.tensor([0.0, 0.0, 0.8], device="cuda")
    e1.reset(); e2.reset()
    obs_l, rew_l, te_l, tr_l = [], [], [], []
    for t in range(T):
        o, r, te, tr, _ = e1.step(acts[t])
        obs_l.append(o.clone()); rew_l.append(r.clone()); te_l.append(te.clone()); tr_l.append(tr.clone())
    out = e2.rollout(acts)
    assert torch.equal(out["obs"], torch.stack(obs_l)) and torch.equal(out["rewards"], torch.stack(rew_l))
    assert torch.equal(out["terminated"], torch.stack(te_l)) and torch.equal(out["truncated"], torch.stack(tr_l))
    assert torch.equal(e1._planes, e2._planes) and torch.equal(e1._step_counter, e2._step_counter)
    assert torch.equal(e1._last_rpm, e2._last_rpm)
    if e1._pid is not None:
        assert torch.equal(e1._pid, e2._pid)
    assert torch.equal(e1._obs_buf[e1._cur], e2._obs_buf[e2._cur])
    if act == "RPM" and phys == "DYN":
        assert bool((torch.stack(te_l) | torch.stack(tr_l)).any())      # autoreset exercised inside the rollout
    # the envs stay interchangeable afterwards
    o1, *_ = e1.step(acts[0]); o2, *_ = e2.step(acts[0])
    assert torch.equal(o1, o2)


def test_rollout_device_action_generator():
    """actions=None: uniform[-1,1) actions from the counter-based device generator == its NumPy restatement, and the
    rollout equals stepping with those actions; consecutive rollouts continue the stream."""
    from gym_pybullet_drones_b200.envs import MultiHoverAviary
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    E, D, T = 256, 2, 20
    kw = dict(num_drones=D, physics=Physics.DYN, act=ActionType.RPM, num_envs=E, autoreset="same_step")
    e1, e2 = MultiHoverAviary(**kw), MultiHoverAviary(**kw)
    e1.reset(); e2.reset()
    outa = e2.rollout(num_steps=T, seed=1234)
    a_ref = MultiHoverAviary.rollout_actions_reference(1234, 0, T, E * D, 4).reshape(T, E, D, 4)
    assert np.array_equal(outa["actions"].cpu().numpy(), a_ref)
    assert float(outa["actions"].min()) >= -1 and float(outa["actions"].max()) < 1 and abs(float(outa["actions"].mean())) < 0.01
    for t in range(T):
        o, *_ = e1.step(outa["actions"][t])
        assert torch.equal(o, outa["obs"][t]), t
    outb = e2.rollout(num_steps=5, seed=1234)
    b_ref = MultiHoverAviary.rollout_actions_reference(1234, T, 5, E * D, 4).reshape(5, E, D, 4)
    assert np.array_equal(outb["actions"].cpu().numpy(), b_ref)


@pytest.mark.parametrize("cls,act,D,E,mode,rpy_f32", [
    ("MultiHoverAviary", "RPM", 2, 1024, "same_step", True), ("MultiHoverAviary", "ONE_D_RPM", 2, 1024, "same_step", True),
    ("HoverAviary", "RPM", 1, 333, "same_step", True), ("HoverAviary", "ONE_D_RPM", 1, 1000, None, False),
    ("MultiHoverAviary", "RPM", 4, 77, "same_step", False), ("MultiHoverAviary", "RPM", 32, 5, None, True),
    ("MultiHoverAviary", "ONE_D_RPM", 8, 300, "same_step", True)])
def test_fast_step_kernels_are_bit_identical_to_the_general_kernel(cls, act, D, E, mode, rpy_f32, monkeypatch):
    """step_fast.cu (warp-per-span kernels, templated on A / task / autoreset / rpy precision) against step_general.cu
    (QS_FAST=0) on the same inputs: observations, rewards, flags, terminal observations, state planes and counters are equal
    bit for bit, ragged last warps and 32-drone aviaries included."""
    import gym_pybullet_drones_b200.envs as envs
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    kw = dict(physics=Physics.DYN, act=ActionType[act], num_envs=E, autoreset=mode, rpy_f32=rpy_f32)
    if cls == "MultiHoverAviary":
        kw["num_drones"] = D
    e1, e2 = getattr(envs, cls)(**kw), getattr(envs, cls)(**kw)
    A = e1._A
    g = torch.Generator(device="cuda").manual_seed(3)
    e1.reset(); e2.reset()
    n_done = 0
    for t in range(150):
        a = torch.rand((E, D, A), device="cuda", generator=g) * 2 - 1
        monkeypatch.setenv("QS_FAST", "1")
        o1, r1, te1, tr1, i1 = e1.step(a)
        monkeypatch.setenv("QS_FAST", "0")
        o2, r2, te2, tr2, i2 = e2.step(a)
        for name, x, y in (("obs", o1, o2), ("reward", r1, r2), ("terminated", te1, te2), ("truncated", tr1, tr2), ("planes", e1._planes, e2._planes),
                           ("step_counter", e1._step_counter, e2._step_counter), ("last_rpm", e1._last_rpm, e2._last_rpm)):
            assert torch.equal(x, y), (name, t, float((x.double() - y.double()).abs().max()))
        if mode == "same_step":
            done = i1["_final_obs"]
            assert torch.equal(done, i2["_final_obs"]) and torch.equal(i1["final_obs"][done], i2["final_obs"][done]), t
            n_done += int(done.sum())
    if mode == "same_step":
        assert n_done > 0


def test_user_subclass_hooks_are_honoured():
    """The reference's template-method seam (BaseAviary.py:1021-1104): a user subclass overriding _computeReward /
    _computeTruncated (single-env and vector API) and _preprocessAction (CtrlAviary) is called after every tick; the
    kernel then only advances the physics.  Checked against the same quantities computed from the built-in env."""
    from gym_pybullet_drones_b200.envs import CtrlAviary, HoverAviary
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics

    class MyHover(HoverAviary):            # reference-style hooks (HoverAviary.py:68-117 rewritten by a user)
        def _computeReward(self):
            state = self._getDroneStateVector(0)
            return -float(np.linalg.norm(self.TARGET_POS - state[0:3]))

        def _computeTruncated(self):
            return bool(self._getDroneStateVector(0)[2] > 0.2)

    env, ref = MyHover(physics=Physics.DYN, act=ActionType.RPM), HoverAviary(physics=Physics.DYN, act=ActionType.RPM)
    assert env._py_hooks and not ref._py_hooks
    env.reset(); ref.reset()
    saw_trunc = False
    for t in range(40):
        a = np.full((1, 4), 0.5, np.float32)
        o, r, te, tr, info = env.step(a)
        o2, r2, te2, tr2, _ = ref.step(a)
        assert np.array_equal(o, o2) and info == {"answer": 42}
        z = ref._getDroneStateVector(0)[2]
        assert abs(r + np.linalg.norm(np.array([0, 0, 1.0]) - ref._getDroneStateVector(0)[0:3])) < 1e-12 and tr == bool(z > 0.2) and te == te2
        saw_trunc |= tr
    assert saw_trunc

    class MyVecHover(HoverAviary):         # vector API: hooks return [E] tensors
        def _computeReward(self):
            return -(self.pos[:, 0, 2] - 1.0).abs().float()

        def _computeTerminated(self):
            return self.pos[:, 0, 2] > 0.15

    E = 64
    venv = MyVecHover(physics=Physics.DYN, act=ActionType.RPM, num_envs=E, autoreset="same_step")
    obs, _ = venv.reset()
    g = torch.Generator(device="cuda").manual_seed(0)
    n_done = 0
    for t in range(60):
        a = torch.rand((E, 1, 4), device="cuda", generator=g)
        obs, r, te, tr, info = venv.step(a)
        z_after = info["final_obs"][:, 0, 2]
        assert r.shape == (E,) and te.dtype == torch.bool and torch.equal(te, z_after > 0.15)
        done = info["_final_obs"]                 # _computeTruncated is not overridden: the kernel's Hover truncation still applies
        assert torch.equal(done, te | tr)
        # finished aviaries were reset by the host side: back at the initial height, terminal observation kept
        assert torch.all(venv.pos[done][:, 0, 2] == venv.INIT_XYZS[0, 2])
        assert torch.all(venv.step_counter[done] == 0)
        n_done += int(done.sum())
    assert n_done > 0

    class MyCtrl(CtrlAviary):              # CtrlAviary._preprocessAction (CtrlAviary.py:121-140) replaced: action = thrust fraction
        def _preprocessAction(self, action):
            return np.repeat(np.asarray(action, np.float64) * self.MAX_RPM, 4, axis=-1)

    c, cref = MyCtrl(num_drones=2, physics=Physics.DYN), CtrlAviary(num_drones=2, physics=Physics.DYN)
    c.reset(); cref.reset()
    for t in range(20):
        frac = np.array([[0.6], [0.7]])
        o, *_ = c.step(frac)
        o2, *_ = cref.step(np.repeat(frac * cref.MAX_RPM, 4, axis=-1))
        assert np.array_equal(o, o2)


def test_device_logger_ring_matches_reference_logger_layout(golden, tmp_path):
    """SURVEY 8f rank 4: a utils.Logger attached to a CtrlAviary logs every tick on the device (qs_log_append); after the
    pid.py circle (teacher-forced from the golden states, like test_pid_circle_workload) its .npy equals what the
    reference's Logger.log(drone, t, state, control) produces when fed the golden state vectors (Logger.py:83-127)."""
    from gym_pybullet_drones_b200.control import DSLPIDControl
    from gym_pybullet_drones_b200.envs import CtrlAviary
    from gym_pybullet_drones_b200.utils import Logger
    from gym_pybullet_drones_b200.utils.enums import DroneModel, Physics
    g = golden("pid_circle_cf2x")
    T = 60
    env = CtrlAviary(num_drones=3, initial_xyzs=g["INIT_XYZS"], initial_rpys=g["INIT_RPYS"], physics=Physics.DYN, pyb_freq=240, ctrl_freq=48)
    lg = Logger(logging_freq_hz=48, output_folder=str(tmp_path), num_drones=3).attach(env, capacity=40)
    host = Logger(logging_freq_hz=48, output_folder=str(tmp_path / "h"), num_drones=3)        # host-side log() of the GOLDEN states
    env.reset()
    for t in range(T):
        if t > 0:
            st = g["obs"][t - 1]
            env.set_state(pos=st[:, 0:3], quat=st[:, 3:7], vel=st[:, 10:13], rpy_rates=g["rpy_rates"][t - 1])
        ctrl = np.hstack([g["target"][t], g["INIT_RPYS"], np.zeros((3, 6))])
        lg.set_controls(ctrl)
        env.step(g["action"][t - 1] if t > 0 else np.zeros((3, 4)))
        for j in range(3):
            host.log(drone=j, timestamp=(t + 1) * 5 / 240, state=g["obs"][t][j], control=ctrl[j])
        if t == 25:
            assert lg.flush() == 26                      # ring of 40 entries: flushed before it wraps (the next 34 wrap around)
    d = np.load(lg.save())
    ts, st, ct = host._trimmed()
    assert d["timestamps"].shape == (3, T) and d["states"].shape == (3, 16, T) and d["controls"].shape == (3, 12, T)
    assert np.allclose(d["timestamps"], ts, atol=1e-12) and np.array_equal(d["controls"], ct.astype(np.float32).astype(np.float64))
    err = np.abs(d["states"] - st) / np.maximum(np.abs(st), 1.0)
    # the RPMs enter CtrlAviary as float32 (6e-8): 2.5e-8 m/s on the velocity of one tick; ang_v is read from the float32 observation
    assert err[:, 0:9].max() < 1e-6 and err[:, 9:12].max() < 2e-6 and err[:, 12:16].max() < 1e-7, err.max(axis=(0, 2))


@pytest.mark.parametrize("act,world", [("RPM", 3), ("ONE_D_RPM", 2)])
def test_fused_observation_gather_in_process(act, world):
    """sharding.ObsGather: every shard's step kernel writes its finished rows, rewards and flags straight into the learner's
    [E_total, D, obs_dim] tensor and raises its flag; after wait() the learner's tensors equal what ONE env over all aviaries
    returns, bit for bit (shards on one device here, each on its own stream; tools/gather_multi_gpu.py runs it across GPUs)."""
    from gym_pybullet_drones_b200.envs import MultiHoverAviary
    from gym_pybullet_drones_b200.sharding import ObsGather, shard_envs
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    E, D, T = 96 * world + 32, 2, 30
    A = 4 if act == "RPM" else 1
    kw = dict(num_drones=D, physics=Physics.DYN, act=ActionType[act], autoreset="same_step")
    ref = MultiHoverAviary(num_envs=E, **kw)
    shards = [shard_envs(E, r, world) for r in range(world)]
    envs = [MultiHoverAviary(num_envs=s.count, **kw) for s in shards]
    gathers = [ObsGather(e, s, learner=0, local=True) for e, s in zip(envs, shards)]
    ObsGather.connect_local(gathers)
    streams = [torch.cuda.Stream() for _ in envs]
    ref.reset()
    for e in envs:
        e.reset()
    g = torch.Generator(device="cuda").manual_seed(1)
    for t in range(T):
        a = torch.rand((E, D, A), device="cuda", generator=g) * 2 - 1
        o, r, te, tr, _ = ref.step(a)
        torch.cuda.synchronize()
        for e, s, st in zip(envs, shards, streams):
            with torch.cuda.stream(st):
                e.step(a[s.start:s.stop].contiguous())
        go, gr, gte, gtr = gathers[0].wait()
        torch.cuda.synchronize()
        assert not gathers[0].timed_out()
        assert torch.equal(go, o) and torch.equal(gr, r) and torch.equal(gte, te) and torch.equal(gtr, tr), t


def test_numpy_api_head_only_transfer_mode():
    """host_obs='head': the NumPy vector API moves only the kinematic head of every observation (the action-history part is
    what the caller itself supplied); it equals the first 12 columns of the full observation, flags and terminal
    observations are unchanged."""
    from gym_pybullet_drones_b200.envs import MultiHoverAviary
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    E, D = 256, 2
    kw = dict(num_drones=D, physics=Physics.DYN, act=ActionType.RPM, num_envs=E, autoreset="same_step")
    e1, e2 = MultiHoverAviary(**kw), MultiHoverAviary(host_obs="head", **kw)
    e1.reset(); e2.reset()
    rng = np.random.default_rng(4)
    seen = 0
    for t in range(60):
        a = rng.uniform(-1, 1, (E, D, 4)).astype(np.float32)
        o1, r1, te1, tr1, i1 = e1.step(a)
        o2, r2, te2, tr2, i2 = e2.step(a)
        assert o2.shape == (E, D, 12) and np.array_equal(o2, o1[..., :12]) and np.array_equal(r1, r2)
        assert np.array_equal(te1, te2) and np.array_equal(tr1, tr2)
        if "final_obs" in i1:
            seen += 1
            assert np.array_equal(i1["final_obs"], i2["final_obs"]) and np.array_equal(i1["final_obs_env"], i2["final_obs_env"])
    assert seen > 5
