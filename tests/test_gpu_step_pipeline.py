"""The pipelined fast step kernel (step_pipe_kernel, DESIGN.md 4.1): 4 consecutive 32-drone tiles per warp, two shared-memory
stages, per-tile readiness.  Every test runs the same sequence with the default kernel, with the classic one-tile-per-warp
kernel (QS_FAST_PIPE=0) and with the general kernel (QS_FAST=0), and compares the bits of everything a step writes; the
readiness words agree and the readiness error word stays zero."""
import contextlib
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MODES = {"pipe": {}, "classic": {"QS_FAST_PIPE": "0"}, "general": {"QS_FAST": "0"}}


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


def _make(E, D, task=True, autoreset="same_step", final_obs=True, rpy_f32=True, phys=False, track=None):
    from gym_pybullet_drones_b200 import _native as N
    from gym_pybullet_drones_b200.envs import MultiHoverAviary
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics

    class NoTask(MultiHoverAviary):
        def _task(self):
            return N.TASK_NONE

    cls = MultiHoverAviary if task else NoTask
    env = cls(num_drones=D, physics=Physics.DYN, act=ActionType.RPM, num_envs=E, autoreset=autoreset, rpy_f32=rpy_f32,
              track_last_action=track)
    if not final_obs:
        env._io.final_obs = None
    if phys:
        gen = torch.Generator(device="cuda").manual_seed(E * 7 + D)
        m = 0.027 * (0.9 + 0.2 * torch.rand(E, device="cuda", dtype=torch.float64, generator=gen))
        env.set_physical_params(m=m)
        assert env._st.phys
    env.reset()
    return env


def _actions(env, T, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.rand((env._E, env._D, env._A), device="cuda", generator=gen) * 2 - 1 for _ in range(T)]


def _outputs(env, final_obs=True):
    out = {"planes": env._planes, "step_counter": env._step_counter, "obs": env._obs_buf[env._cur], "reward": env._reward,
           "terminated": env._terminated, "truncated": env._truncated, "done": env._done, "warp_ticket": env._warp_ticket,
           "warp_done": env._warp_done, "ready_err": env._ready_err}
    if final_obs and env._final_obs is not None:
        out["final_obs"] = env._final_obs
    if env._last_rpm is not None and env._track_last_action:
        out["last_rpm"] = env._last_rpm
    return {k: v.clone() for k, v in out.items()}


def _run_modes(make_envs, body, modes=("pipe", "classic", "general")):
    """body(envs) once per kernel; returns {mode: envs}."""
    res = {}
    for m in modes:
        with _env_vars(MODES[m]):
            envs = make_envs()
            body(envs)
            torch.cuda.synchronize()
        res[m] = envs
    return res


def _assert_same(res, final_obs=True):
    ref = [_outputs(e, final_obs) for e in res["pipe"]]
    for m, envs in res.items():
        for k, e in enumerate(envs):
            got = _outputs(e, final_obs)
            assert int(got["ready_err"].item()) == 0, "%s env %d: a warp waited more than ~1 s for its turn" % (m, k)
            for name in ref[k]:
                if m == "general" and name in ("warp_ticket", "warp_done"):
                    continue                                       # the general kernel takes no tickets
                assert torch.equal(got[name], ref[k][name]), "%s vs pipe, env %d: %s differs" % (m, name, k)


def _stepper(T, seed, dones):
    acts = {}

    def body(envs):
        a = acts.setdefault("a", [_actions(e, T, seed + k) for k, e in enumerate(envs)])
        torch.cuda.synchronize()
        for t in range(T):
            for k, e in enumerate(envs):
                e.step(a[k][t])
                dones.append(e._done.sum())
    return body


def test_bench_pattern_eight_envs_rotating():
    """65 536 drones as 32 768 two-drone aviaries, 8 envs rotating on one stream: the benchmark's launch pattern."""
    dones = []
    res = _run_modes(lambda: [_make(32768, 2) for _ in range(8)], _stepper(12, 100, dones))
    _assert_same(res)
    assert int(torch.stack(dones).sum()) > 0                       # same-step resets happened


# 33, 34 or 35 tiles per env, so the last warp holds 1, 2 or 3 of its 4 tiles; a ragged last tile of 12 drones for D < 32;
# every aviary size
@pytest.mark.parametrize("tiles", [33, 34, 35])
@pytest.mark.parametrize("D", [1, 2, 4, 32])
def test_ragged_batches_every_aviary_size(D, tiles):
    E = tiles if D == 32 else (32 * (tiles - 1) + 12) // D
    dones = []
    res = _run_modes(lambda: [_make(E, D), _make(E, D)], _stepper(48, 200 + D, dones))
    _assert_same(res)
    assert int(torch.stack(dones).sum()) > 0


@pytest.mark.parametrize("rpy_f32", [True, False])
@pytest.mark.parametrize("task,autoreset,final_obs", [(True, "same_step", True), (True, "same_step", False), (True, None, False),
                                                      (False, "same_step", True), (False, None, False)])
def test_kernel_modes(task, autoreset, final_obs, rpy_f32):
    dones = []
    res = _run_modes(lambda: [_make(550, 2, task=task, autoreset=autoreset, final_obs=final_obs, rpy_f32=rpy_f32)],
                     _stepper(40, 300, dones))
    _assert_same(res, final_obs=final_obs)


def test_per_aviary_constants_table_and_last_rpm():
    dones = []
    res = _run_modes(lambda: [_make(2000, 2, phys=True, track=True), _make(550, 2, phys=True)], _stepper(40, 400, dones))
    assert "last_rpm" in _outputs(res["pipe"][0])
    _assert_same(res)
    assert int(torch.stack(dones).sum()) > 0


@pytest.mark.parametrize("chunks", ["1", "3", "4"])
def test_host_api_chunks(chunks, monkeypatch):
    """qs_step_host launches the fast kernel over tile ranges, one launch per chunk."""
    monkeypatch.setenv("QS_HOST_CHUNKS", chunks)
    E, D, T = 4100, 2, 30
    rng = np.random.default_rng(41)
    acts = [rng.uniform(-1, 1, (E, D, 4)).astype(np.float32) for _ in range(T)]
    got = {}

    def body(envs):
        (env,) = envs
        got[len(got)] = [tuple(np.array(x, copy=True) for x in env.step(acts[t])[:4]) for t in range(T)]

    res = _run_modes(lambda: [_make(E, D)], body)
    for m in (1, 2):
        for t in range(T):
            for x, y in zip(got[0][t], got[m][t]):
                assert np.array_equal(x, y), (m, t)
    _assert_same(res)


def test_cuda_graph_replay():
    """Two consecutive steps of one env captured in a CUDA graph and replayed 10 times == 22 eager steps of the classic kernel."""
    E, D = 8200, 2
    g_env = _make(E, D)
    a = _actions(g_env, 2, 31)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        g_env.step(a[0]); g_env.step(a[1])
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        g_env.step(a[0]); g_env.step(a[1])
    for _ in range(10):
        g.replay()
    torch.cuda.synchronize()
    with _env_vars(MODES["classic"]):
        e_env = _make(E, D)
        for _ in range(11):
            e_env.step(a[0]); e_env.step(a[1])
        torch.cuda.synchronize()
    _assert_same({"pipe": [g_env], "classic": [e_env]})
    assert int(g_env._warp_ticket[0].item()) == 22


def test_interleaved_with_reset_rollout_general_step_and_torch_writer():
    """Pipelined steps directly after qs_reset (masked and full), qs_rollout, a general-kernel step of another env, and a
    torch kernel that writes the step's actions."""
    E, D, T = 4100, 2, 12
    src = {}

    def body(envs):
        env, other = envs
        a = src.setdefault("a", _actions(env, T, 51))
        mask = np.zeros(E, bool)
        mask[::3] = True
        act = torch.empty_like(a[0])
        for t in range(T):
            env.step(a[t])
            if t == 2:
                env.reset(options={"reset_mask": mask})
            if t == 5:
                env.reset()
            if t == 7:
                env.rollout(num_steps=3, seed=9)
            with _env_vars(MODES["general"]):
                other.step(a[T - 1 - t])
            torch.mul(a[t], -0.5, out=act)
            env.step(act)

    res = _run_modes(lambda: [_make(E, D), _make(E, D)], body, modes=("pipe", "classic"))
    _assert_same(res)
