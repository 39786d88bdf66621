"""Per-warp readiness of the fast step kernel (DESIGN.md 4.1): consecutive fast steps skip the whole-grid dependency wait and
each warp waits only for the previous step's warp of the same 32 drones.  Every test runs a sequence once on the fast kernel
and once on the general kernel (QS_FAST=0, which always waits for the whole previous grid and takes no tickets) and compares
the bits of everything a step writes; every test ends with the readiness error word still zero."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _make(E, D, act="RPM"):
    from gym_pybullet_drones_b200.envs import MultiHoverAviary
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    env = MultiHoverAviary(num_drones=D, physics=Physics.DYN, act=getattr(ActionType, act), num_envs=E, autoreset="same_step")
    env.reset()
    return env


def _actions(env, T, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.rand((env._E, env._D, env._A), device="cuda", generator=gen) * 2 - 1 for _ in range(T)]


def _outputs(env):
    out = {"planes": env._planes, "step_counter": env._step_counter, "obs": env._obs_buf[env._cur], "reward": env._reward,
           "terminated": env._terminated, "truncated": env._truncated, "done": env._done, "final_obs": env._final_obs}
    if env._last_rpm is not None and env._track_last_action:
        out["last_rpm"] = env._last_rpm
    return {k: v.clone() for k, v in out.items() if v is not None}


def _assert_same(fast, ref, what):
    assert fast.keys() == ref.keys()
    for k in fast:
        assert torch.equal(fast[k], ref[k]), "%s: %s differs" % (what, k)


def _assert_clean(*envs):
    for e in envs:
        assert int(e._ready_err.item()) == 0, "a warp waited more than ~1 s for its turn"


class _General:
    """QS_FAST=0 inside the block: the steps launched there take the general kernel."""

    def __enter__(self):
        self.old = os.environ.get("QS_FAST")
        os.environ["QS_FAST"] = "0"

    def __exit__(self, *a):
        if self.old is None:
            del os.environ["QS_FAST"]
        else:
            os.environ["QS_FAST"] = self.old


def _run_both(make_envs, body):
    """body(envs) once on fast kernels and once on general kernels; returns (fast envs, reference envs)."""
    fast = make_envs()
    body(fast)
    torch.cuda.synchronize()
    with _General():
        ref = make_envs()
        body(ref)
        torch.cuda.synchronize()
    return fast, ref


# E, D, act: the bench size (65 536 drones, 2048 warps) and a ragged ONE_D_RPM size (1000 drones: a last warp of 8 rows,
# 8 x 27 floats = a 16-byte multiple, so the fast kernel takes it)
@pytest.mark.parametrize("E,D,act", [(32768, 2, "RPM"), (1000, 1, "ONE_D_RPM")])
def test_back_to_back_steps_of_one_env(E, D, act):
    T = 200
    acts = {}

    def body(envs):
        (env,) = envs
        a = acts.setdefault("a", _actions(env, T, 11))       # generated before the first step: nothing runs between the steps
        torch.cuda.synchronize()
        for t in range(T):
            env.step(a[t])

    fast, ref = _run_both(lambda: [_make(E, D, act)], body)
    _assert_same(_outputs(fast[0]), _outputs(ref[0]), "fast vs general")
    warps = (E * D + 31) // 32
    assert torch.equal(fast[0]._warp_ticket, torch.full((warps,), T, dtype=torch.int32, device="cuda"))      # every warp, every step
    assert torch.equal(fast[0]._warp_done, fast[0]._warp_ticket)
    assert int(ref[0]._warp_ticket.abs().sum()) == 0                                                          # general kernel: no tickets
    _assert_clean(*fast, *ref)


@pytest.mark.parametrize("n_envs", [2, 8])
def test_envs_alternating_on_one_stream(n_envs):
    E, D, T = 4096, 2, 60
    acts = {}

    def body(envs):
        a = acts.setdefault("a", [_actions(e, T, 21 + k) for k, e in enumerate(envs)])
        torch.cuda.synchronize()
        for t in range(T):
            for k, e in enumerate(envs):
                e.step(a[k][t])

    fast, ref = _run_both(lambda: [_make(E, D) for _ in range(n_envs)], body)
    for k in range(n_envs):
        _assert_same(_outputs(fast[k]), _outputs(ref[k]), "env %d" % k)
    _assert_clean(*fast, *ref)


def test_cuda_graph_replay_of_consecutive_steps():
    """Two consecutive steps of one env captured in a CUDA graph and replayed 10 times == 20 eager steps: the expected ticket
    lives in device memory, not in the captured launch arguments."""
    E, D = 8192, 2
    g_env, e_env = _make(E, D), _make(E, D)
    a = _actions(g_env, 2, 31)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                   # warm-up outside the capture (2 steps: the double buffers end where they started)
        g_env.step(a[0]); g_env.step(a[1])
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        g_env.step(a[0]); g_env.step(a[1])
    for _ in range(10):
        g.replay()
    for _ in range(11):
        e_env.step(a[0]); e_env.step(a[1])
    torch.cuda.synchronize()
    _assert_same(_outputs(g_env), _outputs(e_env), "graph vs eager")
    assert int(g_env._warp_ticket[0].item()) == 22 and torch.equal(g_env._warp_done, g_env._warp_ticket)
    _assert_clean(g_env, e_env)


@pytest.mark.parametrize("chunks", ["1", "3", "4"])
def test_host_api_chunks(chunks, monkeypatch):
    """qs_step_host launches the fast kernel over warp ranges (one launch per chunk, each behind its H2D copy)."""
    monkeypatch.setenv("QS_HOST_CHUNKS", chunks)
    E, D, T = 4096, 2, 30
    rng = np.random.default_rng(41)
    acts = [rng.uniform(-1, 1, (E, D, 4)).astype(np.float32) for _ in range(T)]
    res = {}

    def body(envs):
        (env,) = envs
        res[len(res)] = [tuple(np.array(x, copy=True) for x in env.step(acts[t])[:4]) for t in range(T)]

    fast, ref = _run_both(lambda: [_make(E, D)], body)
    for t in range(T):
        for x, y in zip(res[0][t], res[1][t]):
            assert np.array_equal(x, y), t
    _assert_same(_outputs(fast[0]), _outputs(ref[0]), "host API")
    assert int(fast[0]._warp_ticket[0].item()) == T
    _assert_clean(*fast, *ref)


def test_fast_step_after_reset_rollout_general_step_and_torch_writer():
    """A fast step directly after: qs_reset (masked and full), qs_rollout, a general-kernel step of another env (and that
    general step directly after a fast step of its neighbour), and a torch kernel that writes the step's actions."""
    E, D, T = 4096, 2, 12
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
                env.reset(options={"reset_mask": mask})          # masked reset kernel, then a fast step
            if t == 5:
                env.reset()
            if t == 7:
                env.rollout(num_steps=3, seed=9)                 # rollout kernel, then a fast step
            old = os.environ.get("QS_FAST")
            os.environ["QS_FAST"] = "0"
            try:
                other.step(a[T - 1 - t])                         # general kernel of another env between two fast steps
            finally:
                if old is None:
                    del os.environ["QS_FAST"]
                else:
                    os.environ["QS_FAST"] = old
            torch.mul(a[t], -0.5, out=act)                       # torch kernel writing the next step's actions
            env.step(act)

    fast, ref = _run_both(lambda: [_make(E, D), _make(E, D)], body)
    for k in range(2):
        _assert_same(_outputs(fast[k]), _outputs(ref[k]), "env %d" % k)
    _assert_clean(*fast, *ref)
