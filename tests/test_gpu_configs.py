"""The step and rollout kernels away from the 240 Hz / CF2X defaults (-m gpu): drone models, physics and control rates, initial
attitudes, per-aviary pose tables with same-step autoreset, out-of-range actions, the float64 rpy path, the task-less kernel
instantiations and the launch variants of the environment knobs, each against the float64 oracle or the reference's golden
vectors (tests/golden/rl_configs.npz).

The rate sets the substep count S = pyb_freq / ctrl_freq and the action-buffer length B = ctrl_freq // 2, hence the
observation width od = 12 + B*A.  Which step kernel takes a configuration depends on od (step_fast_eligible in step_fast.cu):
every row of the matrix states the kernel it expects, and the test fails when another one ran, so a change of the eligibility
rule cannot silently drop coverage.  The fast kernel takes per-warp tickets, the general kernel takes none: after a step,
env._warp_ticket is non-zero exactly when the fast kernel ran.

Run as a script (python tests/test_gpu_configs.py OUT.npz) it plays the fixed sequence of the launch-variant test and writes
every output to OUT.npz: the launch knobs are read once per process, so each setting needs a process of its own."""
import contextlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from qs_testlib import FIELDS, ROOT, RTOL, TIGHT, quat_err, relerr
from test_gpu_parity import OBS_FIELDS, OBS_TOL, _borderline, _report_borderline, check_fields, state_of

pytestmark = pytest.mark.gpu

MODELS = {"cf2x": "CF2X", "cf2p": "CF2P", "racer": "RACE"}
PID_TF_TOL = 1e-7       # teacher-forced embedded PID: the controller reads the state through float32 targets (test_gpu_parity)


def _imports():
    from gym_pybullet_drones_b200 import _native as N
    from gym_pybullet_drones_b200.envs import HoverAviary, MultiHoverAviary
    from gym_pybullet_drones_b200.utils.enums import ActionType, DroneModel, Physics
    from oracle import dyn_oracle as O
    return N, HoverAviary, MultiHoverAviary, ActionType, DroneModel, Physics, O


def make_env(kind, D, model, pyb, ctrl, act, E, physics="DYN", **kw):
    _, HoverAviary, MultiHoverAviary, ActionType, DroneModel, Physics, _ = _imports()
    args = dict(drone_model=DroneModel[MODELS[model]], physics=Physics[physics], pyb_freq=pyb, ctrl_freq=ctrl,
                act=ActionType[act.upper()], num_envs=E, **kw)
    return HoverAviary(**args) if kind == "hover" else MultiHoverAviary(num_drones=D, **args)


def make_oracle(kind, D, model, pyb, ctrl, act, E, **kw):
    O = _imports()[-1]
    return O.OracleAviary(kind, E, D, drone_model=model, pyb_freq=pyb, ctrl_freq=ctrl, act=act, **kw)


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


def _ran_fast(env):
    return bool(env._warp_ticket.any())


def _tmax(env):
    return int(env._lib.qs_rollout_max_ticks(env._act_type(), env._B, env._D))


def _report(*fields):
    print("CFG", *fields)


def _state_ratio(st, ora, tol):
    """Worst error / tolerance of one tick over the kinematic state, by the method of test_gpu_parity._compare_with_oracle:
    quaternions up to sign, the Euler angles scaled by cos(pitch), rpy / ang_v (read back from the float32 observation)
    against max(tol, OBS_TOL)."""
    cosp = np.maximum(np.abs(np.cos(ora.rpy[..., 1:2])), 0.02)
    worst = 0.0
    for f in FIELDS:
        ref = getattr(ora, f)
        if f == "quat":
            e = quat_err(st[f], ref)
        elif f == "rpy":
            e = float(np.max(np.abs(st[f] - ref) * cosp / np.maximum(np.abs(ref), 1.0)))
        else:
            e = relerr(st[f], ref)
        worst = max(worst, e / (max(tol, OBS_TOL) if f in OBS_FIELDS else tol))
    return worst


def _outputs(env, obs, rew, te, tr):
    return dict(obs=obs.clone(), rew=rew.clone(), te=te.clone(), tr=tr.clone(), planes=env._planes.clone(),
                sc=env._step_counter.clone())


def _snapshot(ora):
    return dict(pos=ora.pos.copy(), quat=ora.quat.copy(), vel=ora.vel.copy(), rpy_rates=ora.rpy_rates.copy(),
                sc=ora.step_counter.copy(), pid=[a.copy() for a in (ora.ctrl.integral_pos_e, ora.ctrl.last_rpy, ora.ctrl.integral_rpy_e)])


def _force_from_snapshot(env, s):
    env.set_state(pos=s["pos"], quat=s["quat"], vel=s["vel"], rpy_rates=s["rpy_rates"], step_counter=s["sc"])
    for k, a in enumerate(s["pid"]):
        env._pid[3 * k:3 * k + 3] = torch.from_numpy(a.T.copy()).cuda()


# ---------------------------------------------------------------------------------------------------------------
# (a) the reference's golden vectors of rl_configs.npz on the device, E = 3 identical aviaries
# ---------------------------------------------------------------------------------------------------------------
def _rl_config_cases(golden):
    g = golden("rl_configs")
    return g, {c["key"]: c for c in json.loads(str(g["cases"]))}


RL_CONFIG_KEYS = ["race_500_50_rpm", "cf2p_240_16_one_d_rpm", "multi3_race_240_80_rpm_rpys", "cf2x_1000_50_one_d_rpm_timeout",
                  "cf2x_240_1_one_d_rpm_b0", "cf2p_240_60_pid", "cf2x_240_30_rpm_x30"]


@pytest.mark.parametrize("key", RL_CONFIG_KEYS)
def test_rl_configs_golden_on_device(golden, key):
    """Planes within TIGHT of the reference, observations within OBS_TOL, reward and flags on every tick, in aviaries 0 and 2.
    The 60 Hz PID case is teacher-forced (its loop amplifies a 1e-12 perturbation 300-fold in 60 ticks) at 1e-7."""
    g, cases = _rl_config_cases(golden)
    c = cases[key]
    E, D = 3, c.get("nd", 1)
    kw = {"initial_rpys": np.array(c["rpys"])} if "rpys" in c else {}
    env = make_env(c["kind"], D, c["model"], c["pyb"], c["ctrl"], c["act"], E, **kw)
    if c["kind"] == "multihover":
        assert relerr(env.TARGET_POS, g[key + "_TARGET_POS"]) == 0
    obs, _ = env.reset()
    assert relerr(obs[0].cpu().numpy(), g[key + "_obs0"]) < 1e-6
    acts = g[key + "_actions"]
    pid = c["act"] == "pid"
    S = c["pyb"] // c["ctrl"]
    tol = PID_TF_TOL if pid else TIGHT
    worst = 0.0
    for t in range(acts.shape[0]):
        if pid and t > 0:
            env.set_state(pos=np.broadcast_to(g[key + "_pos"][t - 1], (E, D, 3)), quat=np.broadcast_to(g[key + "_quat"][t - 1], (E, D, 4)),
                          vel=np.broadcast_to(g[key + "_vel"][t - 1], (E, D, 3)),
                          rpy_rates=np.broadcast_to(g[key + "_rpy_rates"][t - 1], (E, D, 3)), step_counter=t * S)
            for k, name in enumerate(("pid_integral_pos_e", "pid_last_rpy", "pid_integral_rpy_e")):
                env._pid[3 * k:3 * k + 3] = torch.from_numpy(np.repeat(g[key + "_" + name][t - 1].T, E, axis=1).copy()).cuda()
        a = torch.from_numpy(np.broadcast_to(acts[t], (E,) + acts[t].shape).copy()).cuda()
        obs, rew, term, trunc, _ = env.step(a)
        st = state_of(env)
        for e in (0, 2):
            check_fields(st, g, key, t, tol, e)
            worst = max(worst, max((quat_err(st[f][e], g[key + "_" + f][t]) if f == "quat" else relerr(st[f][e], g[key + "_" + f][t]))
                                   / (max(tol, OBS_TOL) if f in OBS_FIELDS else tol) for f in FIELDS))
            ref_r = g[key + "_reward"][t]
            assert abs(float(rew[e]) - ref_r) <= OBS_TOL * max(1.0, abs(ref_r)), (t, float(rew[e]), ref_r)
            assert bool(term[e]) == bool(g[key + "_terminated"][t]) and bool(trunc[e]) == bool(g[key + "_truncated"][t]), (e, t)
        if t % c["obs_every"] == 0:
            ref_o = g[key + "_obs"][t // c["obs_every"]]
            assert obs.shape[-1] == ref_o.shape[-1]
            for e in (0, 2):
                assert relerr(obs[e].cpu().numpy(), ref_o) < OBS_TOL, t
    assert int(env._ready_err.item()) == 0
    _report("golden", key, "kernel", "fast" if _ran_fast(env) else "general", "worst/tol %.3f" % worst)


# ---------------------------------------------------------------------------------------------------------------
# (b) configuration matrix against the oracle
# ---------------------------------------------------------------------------------------------------------------
_STACK4 = np.array([[0.0, 0.0, 0.06], [0.05, 0.02, 1.6], [0.1, -0.03, 3.1], [-0.05, 0.05, 4.6]])
_RPYS3 = np.array([[0.1, -0.05, 0.3], [-0.08, 0.12, -0.7], [0.03, 0.02, 1.9]])

# row, env kind, D, model, pyb, ctrl, act, E, expected kernel, ticks, extras
MATRIX = [
    ("1", "hover", 1, "racer", 500, 50, "rpm", 1000, "fast", 100, {}),                      # S 10  B 25  od 112
    ("2", "hover", 1, "cf2p", 240, 16, "one_d_rpm", 1000, "fast", 80, {}),                  # S 15  B 8   od 20
    ("3a", "hover", 1, "cf2x", 1000, 50, "one_d_rpm", 1004, "fast", 100, {}),               # S 20  B 25  od 37, N%32 = 12
    ("3b", "hover", 1, "cf2x", 1000, 50, "one_d_rpm", 1001, "general", 100, {}),            # N%32 = 9: 9*37 % 4 != 0
    ("4", "hover", 1, "cf2x", 240, 15, "one_d_rpm", 996, "fast", 100, {}),                  # S 16  B 7   od 19
    ("5", "hover", 1, "cf2x", 240, 240, "one_d_rpm", 500, "fast", 150, {}),                 # S 1   B 120 od 132
    ("6", "hover", 1, "cf2x", 480, 480, "one_d_rpm", 64, "fast", 150, {}),                  # S 1   B 240 od 252: A=1 window > 48 KB
    ("7", "multihover", 16, "cf2x", 240, 120, "rpm", 40, "fast", 100, {}),                  # S 2   B 60  od 252, D = 16
    ("8", "multihover", 2, "cf2x", 480, 160, "rpm", 300, "general", 100, {}),               # S 3   B 80  od 332: stage limit
    ("9", "multihover", 8, "cf2p", 240, 48, "one_d_rpm", 125, "fast", 100, {}),             # S 5   B 24  od 36
    ("10", "multihover", 3, "racer", 240, 80, "rpm", 200, "general", 100, {"rpys": _RPYS3}),   # S 3 B 40 od 172, D = 3
    ("11r", "hover", 1, "cf2x", 240, 2, "rpm", 333, "fast", 10, {}),                        # S 120 B 1   od 16
    ("11o", "hover", 1, "cf2x", 240, 2, "one_d_rpm", 332, "fast", 10, {}),                  # S 120 B 1   od 13
    ("12", "hover", 1, "cf2x", 240, 1, "one_d_rpm", 64, "general", 12, {}),                 # S 240 B 0   od 12
    ("13", "hover", 1, "cf2p", 240, 60, "pid", 256, "general", 40, {"teacher": True}),      # S 4   B 30  od 102
    ("14", "multihover", 2, "cf2p", 240, 48, "vel", 128, "general", 60, {"teacher": True}),  # S 5   B 24  od 108
    ("15", "hover", 1, "cf2x", 480, 60, "one_d_pid", 256, "general", 60, {}),               # S 8   B 30  od 42
    ("16", "multihover", 4, "racer", 240, 60, "rpm", 64, "general", 60,                     # S 4   B 30  od 132, DYN+ effects
     {"physics": "PYB_GND_DRAG_DW", "effects": 7, "xyzs": _STACK4, "scale": 0.3}),
    ("17", "hover", 1, "cf2x", 480, 32, "rpm", 1000, "fast", 150, {}),                      # S 15  B 16  od 76: rollout split at 127
]


def _row_actions(kind, D, act, E, T, extra, seed):
    A = {"rpm": 4, "one_d_rpm": 1, "pid": 3, "vel": 4, "one_d_pid": 1}[act]
    rng = np.random.default_rng(seed)
    if act == "pid":      # one set-point per aviary inside the truncation box
        sp = (np.array([0, 0, 1.0]) + 0.5 * rng.uniform(-1, 1, (E, D, 3))).astype(np.float32)
        return np.broadcast_to(sp, (T, E, D, 3)).copy()
    return (np.float32(extra.get("scale", 1.0)) * rng.uniform(-1, 1, (T, E, D, A)).astype(np.float32)).astype(np.float32)


def _row_tol(act, extra):
    if act == "vel":
        # the VEL command is formed in float32 (norm, unit vector, SPEED_LIMIT * |a3| * unit: BaseRLAviary.py:208-221), which
        # the kernel and NumPy may round an ulp apart: 6e-8 on the target velocity, 1.1e-7 on the state after one teacher-
        # forced tick (measured on the H100), so the row is held to the north-star RTOL rather than PID_TF_TOL
        return RTOL
    if extra.get("teacher"):
        return PID_TF_TOL
    if act in ("pid", "vel", "one_d_pid"):
        return RTOL           # free-running embedded PID (contractive at 480/60: a 1e-12 perturbation stays 1e-12)
    return 1e-7 if extra.get("effects") else TIGHT


@pytest.mark.parametrize("row", MATRIX, ids=[r[0] for r in MATRIX])
def test_config_matrix(row):
    name, kind, D, model, pyb, ctrl, act, E, kernel, T, extra = row
    kw = {}
    if "rpys" in extra:
        kw["initial_rpys"] = extra["rpys"]
    if "xyzs" in extra:
        kw["initial_xyzs"] = extra["xyzs"]
    teacher = extra.get("teacher", False)
    tol = _row_tol(act, extra)
    acts = _row_actions(kind, D, act, E, T, extra, seed=1000 + MATRIX.index(row))
    acts_d = torch.from_numpy(acts).cuda()
    env = make_env(kind, D, model, pyb, ctrl, act, E, physics=extra.get("physics", "DYN"), **kw)
    ora = make_oracle(kind, D, model, pyb, ctrl, act, E, effects=extra.get("effects", 0), **kw)
    S, B = pyb // ctrl, ctrl // 2
    assert env.PYB_STEPS_PER_CTRL == S and env._B == B and env._obs_dim == 12 + B * env._A
    obs, _ = env.reset()
    assert relerr(obs.cpu().numpy(), ora.reset()) < 1e-6
    rec, forced, worst = [], [], 0.0
    for t in range(T):
        if teacher and t > 0:
            forced.append(_snapshot(ora))
            _force_from_snapshot(env, forced[-1])
        obs, rew, term, trunc, _ = env.step(acts_d[t])
        o_obs, o_rew, o_term, o_trunc = ora.step(acts[t])
        if t == 0:
            assert _ran_fast(env) == (kernel == "fast"), "row %s: expected the %s kernel" % (name, kernel)
        rec.append(_outputs(env, obs, rew, term, trunc))
        st = state_of(env)
        r = _state_ratio(st, ora, tol)
        r = max(r, relerr(rew.cpu().numpy(), o_rew) / max(tol, OBS_TOL))
        if t % 5 == 0 or t == T - 1:
            r = max(r, relerr(obs.cpu().numpy(), o_obs) / max(tol, OBS_TOL))
        assert r <= 1.0, (name, t, r)
        worst = max(worst, r)
        assert np.array_equal(term.cpu().numpy(), o_term), t
        clear = ~_borderline(ora, tol)
        assert np.array_equal(trunc.cpu().numpy()[clear], o_trunc[clear]), t
    _report_borderline(name)
    torch.cuda.synchronize()
    assert int(env._ready_err.item()) == 0
    # fast against general: the same sequence on a twin env forced onto the general kernel gives the same bits
    if kernel == "fast":
        twin = make_env(kind, D, model, pyb, ctrl, act, E, physics=extra.get("physics", "DYN"), **kw)
        with _General():
            twin.reset()
            for t in range(T):
                out = _outputs(twin, *twin.step(acts_d[t])[:4])
                for k, v in out.items():
                    assert torch.equal(v, rec[t][k]), (name, "fast vs general", k, t)
        assert not _ran_fast(twin) and int(twin._ready_err.item()) == 0
    # rollout: T ticks in qs_rollout launches == T x step(), bit for bit
    tm = _tmax(env)
    if tm > 0 and not teacher:
        ro = make_env(kind, D, model, pyb, ctrl, act, E, physics=extra.get("physics", "DYN"), **kw)
        ro.reset()
        out = ro.rollout(acts_d)
        assert torch.equal(out["obs"], torch.stack([x["obs"] for x in rec]))
        assert torch.equal(out["rewards"], torch.stack([x["rew"] for x in rec]))
        assert torch.equal(out["terminated"], torch.stack([x["te"] for x in rec]))
        assert torch.equal(out["truncated"], torch.stack([x["tr"] for x in rec]))
        assert torch.equal(ro._planes, rec[-1]["planes"]) and torch.equal(ro._step_counter, rec[-1]["sc"])
        if name == "17":
            assert T > tm      # the rollout crossed a launch split
    else:
        with pytest.raises(ValueError) as ei:
            env.rollout(acts_d)
        if B == 0:
            assert "ACTION_BUFFER_SIZE = 0" in str(ei.value)
    _report("matrix", name, "kernel", kernel, "S %d B %d od %d" % (S, B, env._obs_dim), "tol %.0e" % tol, "worst/tol %.3f" % worst,
            "rollout tmax %d" % tm)


# ---------------------------------------------------------------------------------------------------------------
# (c) the time-out tick at other physics rates
# ---------------------------------------------------------------------------------------------------------------
def _first_truncation_oracle(pyb, ctrl, episode_len_sec=8):
    ora = make_oracle("hover", 1, "cf2x", pyb, ctrl, "one_d_rpm", 1)
    ora.EPISODE_LEN_SEC = episode_len_sec
    ora.reset()
    z = np.zeros((1, 1, 1), np.float32)
    for t in range(100000):
        _, _, _, tr = ora.step(z)
        if tr[0]:
            return t + 1
    raise AssertionError("no time-out")


def _first_truncation_env(env, ticks):
    env.reset()
    z = torch.zeros((env._E, 1, 1), device="cuda")
    first = None
    for t in range(ticks):
        _, _, _, tr, _ = env.step(z)
        if bool(tr.any()):
            assert bool(tr.all())
            first = t + 1
            break
    return first


@pytest.mark.parametrize("pyb,ctrl", [(240, 30), (1000, 50), (500, 50), (333, 111), (240, 240), (240, 1)])
def test_time_out_tick(pyb, ctrl):
    """Zero-action ONE_D_RPM hover episodes end by time-out on the oracle's tick (step_counter / PYB_FREQ > EPISODE_LEN_SEC),
    through step() on both kernels and through rollout() where it is available."""
    expect = _first_truncation_oracle(pyb, ctrl)
    E = 64
    env = make_env("hover", 1, "cf2x", pyb, ctrl, "one_d_rpm", E)
    assert _first_truncation_env(env, expect + 2) == expect
    with _General():
        gen = make_env("hover", 1, "cf2x", pyb, ctrl, "one_d_rpm", E)
        assert _first_truncation_env(gen, expect + 2) == expect
    ro = make_env("hover", 1, "cf2x", pyb, ctrl, "one_d_rpm", E)
    ro.reset()
    z = torch.zeros((expect + 2, E, 1, 1), device="cuda")
    if _tmax(ro) > 0:
        tr = ro.rollout(z)["truncated"]
        first = int(torch.nonzero(tr.all(dim=1))[0, 0]) + 1
        assert first == expect and not bool(tr[:first - 1].any())
    else:
        with pytest.raises(ValueError):
            ro.rollout(z)
    assert int(env._ready_err.item()) == 0
    _report("timeout", "%d/%d" % (pyb, ctrl), "tick", expect, "kernel", "fast" if _ran_fast(env) else "general")


# ---------------------------------------------------------------------------------------------------------------
# (d) per-aviary pose tables with same-step autoreset on the fast kernel
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rpy_f32", [True, False])
def test_per_aviary_tables_same_step_autoreset(rpy_f32):
    """[E, 2, 3] initial_xyzs / initial_rpys (the tables_per_env rows of init_drone and reset_head); every 7th aviary starts
    with |roll| = 0.5 > 0.4, so it is truncated and reset on every tick.  Terminal and reset observations against the oracle's
    masked reset loop."""
    E, D, T = 256, 2, 60
    rng = np.random.default_rng(61)
    xyz = np.zeros((E, D, 3))
    xyz[..., 0:2] = rng.uniform(-0.5, 0.5, (E, D, 2))
    xyz[..., 2] = rng.uniform(0.5, 1.5, (E, D))
    rpy = rng.uniform(-0.2, 0.2, (E, D, 3))
    tilted = np.arange(E) % 7 == 0
    rpy[tilted, 0, 0] = 0.5
    acts = rng.uniform(-1, 1, (T, E, D, 4)).astype(np.float32)
    env = make_env("multihover", D, "cf2x", 240, 30, "rpm", E, initial_xyzs=xyz, initial_rpys=rpy, autoreset="same_step", rpy_f32=rpy_f32)
    ora = make_oracle("multihover", D, "cf2x", 240, 30, "rpm", E, initial_xyzs=xyz, initial_rpys=rpy)
    assert env._tables_per_env and relerr(env.TARGET_POS, ora.TARGET_POS) == 0
    obs, _ = env.reset()
    assert relerr(obs.cpu().numpy(), ora.reset()) < OBS_TOL
    n_done, worst = 0, 0.0
    for t in range(T):
        obs, rew, term, trunc, info = env.step(torch.from_numpy(acts[t]).cuda())
        if t == 0:
            assert _ran_fast(env)
        o_obs, o_rew, o_term, o_trunc = ora.step(acts[t])
        done = o_term | o_trunc
        assert np.array_equal((term | trunc).cpu().numpy(), done), t
        assert done[tilted].all(), t
        assert np.array_equal(info["_final_obs"].cpu().numpy(), done)
        n_done += int(done.sum())
        worst = max(worst, relerr(info["final_obs"].cpu().numpy()[done], o_obs[done]) / OBS_TOL)
        o_obs = ora.reset(mask=done)
        worst = max(worst, relerr(obs.cpu().numpy(), o_obs) / OBS_TOL, relerr(rew.cpu().numpy(), o_rew) / OBS_TOL)
        assert worst <= 1.0, (t, worst)
        assert np.array_equal(env.step_counter.cpu().numpy(), ora.step_counter), t
    assert n_done > T * tilted.sum()          # the tilted aviaries every tick, and others as they fly out
    assert int(env._ready_err.item()) == 0
    _report("tables+autoreset", "rpy_f32=%s" % rpy_f32, "resets", n_done, "worst/tol %.3f" % worst)


# ---------------------------------------------------------------------------------------------------------------
# (e) actions outside [-1, 1]: RPM and ONE_D_RPM are not clipped (BaseRLAviary.py:192,225)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act", ["rpm", "one_d_rpm"])
@pytest.mark.parametrize("kernel", ["fast", "general"])
def test_out_of_range_actions(act, kernel):
    """Actions uniform in [-40, 40]; every 4th aviary sends exactly -20, which is rpm = HOVER_RPM * (1 - 1.0) = 0.  The RPM
    drones tumble at up to ~700 rad/s, where float64 rounding differences grow ~2x per tick: 16 ticks (TIGHT is reached
    after ~22)."""
    E, T = 256, 16
    A = 4 if act == "rpm" else 1
    rng = np.random.default_rng(71)
    acts = (40.0 * rng.uniform(-1, 1, (T, E, 1, A))).astype(np.float32)
    acts[:, ::4] = -20.0
    ctx = _General() if kernel == "general" else contextlib.nullcontext()
    with ctx:
        env = make_env("hover", 1, "cf2x", 240, 30, act, E, track_last_action=True)
        ora = make_oracle("hover", 1, "cf2x", 240, 30, act, E)
        env.reset(); ora.reset()
        worst = 0.0
        for t in range(T):
            obs, rew, term, trunc, _ = env.step(torch.from_numpy(acts[t]).cuda())
            o_obs, o_rew, o_term, o_trunc = ora.step(acts[t])
            if t == 0:
                assert _ran_fast(env) == (kernel == "fast")
            r = max(_state_ratio(state_of(env), ora, TIGHT), relerr(obs.cpu().numpy(), o_obs) / OBS_TOL,
                    relerr(rew.cpu().numpy(), o_rew) / OBS_TOL)
            assert r <= 1.0, (t, r)
            worst = max(worst, r)
            assert np.array_equal(term.cpu().numpy(), o_term)
            clear = ~_borderline(ora, TIGHT)
            assert np.array_equal(trunc.cpu().numpy()[clear], o_trunc[clear]), t
            assert relerr(env.last_clipped_action.cpu().numpy(), ora.last_clipped_action) <= 1e-15    # the decoded RPMs
            assert float(env.last_clipped_action[::4].abs().max()) == 0.0                           # -20 -> exactly 0
    assert int(env._ready_err.item()) == 0
    _report_borderline("out-of-range %s %s" % (act, kernel))
    _report("out-of-range", act, kernel, "worst/tol %.3f" % worst)


# ---------------------------------------------------------------------------------------------------------------
# (f) rpy_f32=False: the reported rpy is the float32 cast of the float64 angles
# ---------------------------------------------------------------------------------------------------------------
def _rpy_bound(ref64):
    """Bound on |obs rpy - float32(oracle rpy)| for a kernel evaluating rpy in float64 on its own quaternion.
    The kernel's quaternion is within TIGHT (absolute: unit quaternion) of the oracle's, which the loop asserts first.  Each
    rotation-matrix entry R[i][j] the angles are made from is quadratic in q with |dR| <= 4 |dq|_inf; roll and yaw are
    atan2(a, b) with a^2 + b^2 = cos^2(pitch), so |d(roll)| <= (|a| + |b|) 4 |dq| / cos^2 p <= 4 sqrt(2) |dq| / cos p, and
    pitch = asin(s) gives |d(pitch)| <= 4 |dq| / cos p: delta = 6 TIGHT / cos(pitch) bounds the float64 difference (libm's
    atan2 / asin add ~1e-16).  Both sides are then rounded to float32, half an ulp each: |f32(x) - f32(y)| <= |x - y| + ulp."""
    cosp = np.maximum(np.abs(np.cos(ref64[..., 1:2])), 0.02)
    delta = 6.0 * TIGHT / cosp
    return np.spacing(np.float32(np.abs(ref64) + delta)).astype(np.float64) + delta


def _rpy_ratio(rpy_f32, T=60, E=512):
    rng = np.random.default_rng(81)
    acts = rng.uniform(-1, 1, (T, E, 1, 4)).astype(np.float32)
    env = make_env("hover", 1, "cf2x", 240, 30, "rpm", E, rpy_f32=rpy_f32)
    ora = make_oracle("hover", 1, "cf2x", 240, 30, "rpm", E)
    env.reset(); ora.reset()
    worst = 0.0
    for t in range(T):
        obs, *_ = env.step(torch.from_numpy(acts[t]).cuda())
        ora.step(acts[t])
        st = state_of(env)
        assert quat_err(st["quat"], ora.quat) <= TIGHT, t
        mine = obs.cpu().numpy()[..., 3:6].astype(np.float64)
        ref = ora.rpy.astype(np.float32).astype(np.float64)
        worst = max(worst, float(np.max(np.abs(mine - ref) / _rpy_bound(ora.rpy))))
    assert _ran_fast(env)
    return worst


def test_rpy_float64_path_is_the_float32_cast():
    worst = _rpy_ratio(False)
    _report("rpy_f32=False", "worst/bound %.3f" % worst)
    assert worst <= 1.0


# ---------------------------------------------------------------------------------------------------------------
# (g) the TASK=false instantiations of the fast kernel on RL observations
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act", ["rpm", "one_d_rpm"])
@pytest.mark.parametrize("autoreset", [None, "same_step"])
def test_task_none_fast_kernel(act, autoreset):
    """An env whose _task() is TASK_NONE runs step_fast_kernel<A, TASK=false, ...>: observations and state planes equal the Hover
    env's bits while nothing finishes, the reward is -1 and both flags are 0."""
    N, HoverAviary, _, ActionType, _, Physics, _ = _imports()

    class NoTaskHover(HoverAviary):
        def _task(self):
            return N.TASK_NONE

    E, T = 320, 20
    kw = dict(physics=Physics.DYN, act=ActionType[act.upper()], num_envs=E, autoreset=autoreset)
    ref, env = HoverAviary(**kw), NoTaskHover(**kw)
    rng = np.random.default_rng(91)
    acts = torch.from_numpy((0.02 * rng.uniform(-1, 1, (T, E, 1, ref._A))).astype(np.float32)).cuda()
    ref.reset(); env.reset()
    for t in range(T):
        o1, r1, te1, tr1, _ = ref.step(acts[t])
        o2, r2, te2, tr2, _ = env.step(acts[t])
        assert not bool((te1 | tr1).any()), "the hover task finished: shorten the sequence"
        assert torch.equal(o1, o2) and torch.equal(ref._planes, env._planes) and torch.equal(ref._step_counter, env._step_counter), t
        assert bool((r2 == -1).all()) and not bool(te2.any()) and not bool(tr2.any()), t
        if autoreset:
            assert not bool(env._done.any())
    assert _ran_fast(env) and _ran_fast(ref) and int(env._ready_err.item()) == 0


def test_kin_rows_twenty_wide_report_their_own_ang_v():
    """ONE_D_RPM at ctrl_freq 16 gives KIN rows of 12 + 8 = 20 floats, the width of a CtrlAviary state vector: the drone state
    vectors and the device Logger ring take ang_v from columns 9-11 of such a row (they used to take 13-15, action history)."""
    from gym_pybullet_drones_b200.utils.Logger import Logger
    E, T = 4, 6
    env = make_env("hover", 1, "cf2p", 240, 16, "one_d_rpm", E)
    ora = make_oracle("hover", 1, "cf2p", 240, 16, "one_d_rpm", E)
    assert env._obs_dim == 20 and not env._state20_obs()
    with tempfile.TemporaryDirectory() as d:
        lg = Logger(logging_freq_hz=16, output_folder=d, num_drones=1).attach(env, aviary=1)
        env.reset(); ora.reset()
        rng = np.random.default_rng(3)
        for t in range(T):
            a = rng.uniform(-1, 1, (E, 1, 1)).astype(np.float32)
            obs, *_ = env.step(torch.from_numpy(a).cuda())
            ora.step(a)
            sv = env._getDroneStateVectors()
            assert relerr(sv[..., 13:16], ora.ang_v) < OBS_TOL, t
            assert np.array_equal(lg._ring[t, 0, 9:12].cpu().numpy(), obs[1, 0, 9:12].double().cpu().numpy()), t
        lg.detach()


# ---------------------------------------------------------------------------------------------------------------
# (h) negative controls: each check above fails on a kernel that is subtly wrong
# ---------------------------------------------------------------------------------------------------------------
def test_negative_control_race_yaw_torque_sign():
    """RACE with its z-torque signs flipped to the CF2X pattern (QsParams.sz) misses the oracle by far more than TIGHT."""
    E, T = 64, 30
    acts = _row_actions("hover", 1, "rpm", E, T, {}, seed=5)
    env = make_env("hover", 1, "racer", 500, 50, "rpm", E)
    for k in range(4):
        env._P.sz[k] = -env._P.sz[k]
    ora = make_oracle("hover", 1, "racer", 500, 50, "rpm", E)
    env.reset(); ora.reset()
    worst = 0.0
    for t in range(T):
        env.step(torch.from_numpy(acts[t]).cuda())
        ora.step(acts[t])
        worst = max(worst, _state_ratio(state_of(env), ora, TIGHT))
    _report("negative", "RACE sz negated", "worst/tol %.3g" % worst)
    assert worst > 1.0


def test_negative_control_rpy_f32_misses_the_float64_bound():
    worst = _rpy_ratio(True)
    _report("negative", "rpy_f32=True", "worst/bound %.3g" % worst)
    assert worst > 1.0


def test_negative_control_episode_length_moves_the_time_out():
    """EPISODE_LEN_SEC raised by one physics step moves the time-out by one tick at 240/240 (S = 1), on both kernels."""
    pyb = ctrl = 240
    base = _first_truncation_oracle(pyb, ctrl)
    longer = 8 + 1 / pyb
    moved = _first_truncation_oracle(pyb, ctrl, longer)
    assert moved == base + 1
    for general in (False, True):
        with (_General() if general else contextlib.nullcontext()):
            env = make_env("hover", 1, "cf2x", pyb, ctrl, "one_d_rpm", 64)
            env._P.episode_len_sec = longer
            got = _first_truncation_env(env, moved + 2)
        _report("negative", "episode_len_sec + 1/240", "general" if general else "fast", "time-out tick", got, "(was %d)" % base)
        assert got == moved


# ---------------------------------------------------------------------------------------------------------------
# 3. launch variants of the environment knobs (read once per process: one subprocess per setting)
# ---------------------------------------------------------------------------------------------------------------
VARIANT_ROWS = ["1", "5", "7", "9"]
VARIANTS = [{}, {"QS_FAST_PIPE": "0"}, {"QS_PDL": "0"}, {"QS_CTA_CAP": "64", "QS_FAST": "0"}, {"QS_CTA_CAP": "128", "QS_FAST": "0"}]
_KNOBS = ("QS_FAST", "QS_FAST_PIPE", "QS_PDL", "QS_CTA_CAP", "QS_HOST_CHUNKS")


def play_variant_sequence(path):
    """Rows 1, 5, 7 and 9 of the matrix with SAME_STEP autoreset, a fixed 50-tick sequence (actions x3, and a 0.05 s episode so
    that every row times out and resets every few ticks); every output of every tick, the final state and, where qs_rollout
    takes the row, a rollout of the same actions -> path (.npz)."""
    T = 50
    out = {}
    for row in MATRIX:
        name, kind, D, model, pyb, ctrl, act, E, kernel, _, extra = row
        if name not in VARIANT_ROWS:
            continue
        acts = torch.from_numpy(_row_actions(kind, D, act, E, T, dict(extra, scale=3.0), seed=2000 + int(name))).cuda()
        env = make_env(kind, D, model, pyb, ctrl, act, E, autoreset="same_step", track_last_action=True)
        env._P.episode_len_sec = 0.05
        env.reset()
        rec = {k: [] for k in ("obs", "rew", "te", "tr", "done", "final_obs")}
        for t in range(T):
            o, r, te, tr, info = env.step(acts[t])
            for k, v in (("obs", o), ("rew", r), ("te", te), ("tr", tr), ("done", info["_final_obs"]), ("final_obs", info["final_obs"])):
                rec[k].append(v.cpu().numpy().copy())
        torch.cuda.synchronize()
        for k, v in rec.items():
            out[name + "_" + k] = np.stack(v)
        out[name + "_planes"] = env._planes.cpu().numpy()
        out[name + "_step_counter"] = env._step_counter.cpu().numpy()
        out[name + "_last_rpm"] = env._last_rpm.cpu().numpy()
        out[name + "_ready_err"] = env._ready_err.cpu().numpy()
        out[name + "_fast"] = np.array(_ran_fast(env))
        if _tmax(env) > 0:
            ro = make_env(kind, D, model, pyb, ctrl, act, E, autoreset="same_step", track_last_action=True)
            ro._P.episode_len_sec = 0.05
            ro.reset()
            res = ro.rollout(acts)
            for k in ("obs", "rewards", "terminated", "truncated"):
                out[name + "_rollout_" + k] = res[k].cpu().numpy()
            out[name + "_rollout_planes"] = ro._planes.cpu().numpy()
    np.savez(path, **out)


def test_launch_variants_give_the_same_bytes():
    """Each knob setting in its own process: the same bytes as the default, and the readiness error word stays zero.  The
    general kernel under QS_CTA_CAP=64 / 128 has to give the fast kernel's bytes as well."""
    with tempfile.TemporaryDirectory() as d:
        results = []
        for k, var in enumerate(VARIANTS):
            path = os.path.join(d, "v%d.npz" % k)
            env = {n: v for n, v in os.environ.items() if n not in _KNOBS}
            env.update(var)
            cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), path]
            p = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
            assert p.returncode == 0, (var, p.stdout[-2000:], p.stderr[-4000:])
            results.append(dict(np.load(path)))
    ref = results[0]
    for name in VARIANT_ROWS:
        assert bool(ref[name + "_fast"]), name
        assert int(ref[name + "_done"].sum()) > 0, name        # autoresets happened inside the sequence
    for var, res in zip(VARIANTS, results):
        assert res.keys() == ref.keys(), var
        for k in ref:
            if k.endswith("_fast"):
                assert bool(res[k]) == ("QS_FAST" not in var), (var, k)
                continue
            assert ref[k].dtype == res[k].dtype and ref[k].tobytes() == res[k].tobytes(), (var, k)
        for name in VARIANT_ROWS:
            assert int(res[name + "_ready_err"].max()) == 0, (var, name)
        _report("variant", var or "default", "same bytes")


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    play_variant_sequence(sys.argv[1])
