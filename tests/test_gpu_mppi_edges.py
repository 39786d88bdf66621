"""-m gpu: the MPPI kernels (mppi_sample_kernel, mppi_update_kernel, mppi_commit_kernel; DESIGN.md 4.5.2) at every decision of
the sample, the update and the commit, against the float64 restatement tests/mppi_ref.py.

Covered: the noise at iterations past 2^30; every sample's J with downwash against mppi_ref.rollout_cost_dw at each aviary size that gives the downwash CTA another
layout (D = 1, 3, 5, 32, 33, 127, 128: idle lanes, one group per CTA, a partial last CTA), with negative controls; the downwash
pair predicate at dx*dx + dy*dy = 100 - 2 ulp, 100 - 1 ulp and 100 through step(), rollout(), CtrlAviary.rollout() and mppi()'s
sample and commit; the update at K = 2 .. 1024 (the 64 KB shared-memory branch), unit counts 1, 2, 3 mod 4 and downwash units of
T D below and above 32; teacher-forced J rows for every rule of the update and the commit, with negative controls; a degenerate
box; one iteration at 65 536 drones, with and without downwash."""
import math
import time

import numpy as np
import pytest
import torch

import diff_ref as DR
import mppi_ref as MR
from test_gpu_mppi import DEV, F64, KEYS, _candidate_J, _env, _mppi, _phys, _targets, _vec

pytestmark = pytest.mark.gpu

ULP100 = 2.0 ** -46                    # the spacing of the doubles just below 100


def _rep(x, K):
    """[n, ...] -> [K n, ...]: sample s of drone i at row s n + i"""
    return x.unsqueeze(0).expand(K, *x.shape).reshape(K * x.shape[0], *x.shape[1:])


def _repT(x, K):
    """[T, n, ...] -> [T, K n, ...]"""
    return x.unsqueeze(1).expand(x.shape[0], K, *x.shape[1:]).reshape(x.shape[0], K * x.shape[1], *x.shape[2:])


def _inputs(m):
    """per drone: rows [n, 16], sig [n], the box lo / hi [T, n, 4] (None without), W [T, n, 13] and Rt [n, 4] of Mppi m"""
    E, D = m.env_shape
    T, n = m.T, m.n
    rows = m.rows.repeat_interleave(D, 0)
    sig = m.sigma.repeat_interleave(D) * rows[:, 12]
    lo = hi = None
    if m.box is not None:
        lo, hi, per_tick = m.box
        lo, hi = (lo, hi) if per_tick else (lo.expand(T, n, 4), hi.expand(T, n, 4))
    w = m.weights.repeat_interleave(D, 0)
    W = torch.stack([w[:, :13]] * (T - 1) + [w[:, 13:26]])
    Rt = w[:, 26:30] / rows[:, 12:13] ** 2
    return rows, sig, lo, hi, W, Rt


def _commands(m, e):
    """the commands v [K, T, n, 4] of the nominal m.rpm with the noise e [K, T, n, 4], clamped into the box"""
    rows, sig, lo, hi, _, _ = _inputs(m)
    v = m.rpm[None] + sig[None, None, :, None] * e
    if lo is not None:
        v = torch.where(v < lo, lo, torch.where(v > hi, hi, v))
    return v


def _ref_J(m, v, dw, **kw):
    """the float64 J [K, n] of the commands v [K, T, n, 4] from the start of Mppi m (dw: mppi_ref.rollout_cost_dw per (sample,
    aviary) group, else mppi_ref.rollout_cost), and with downwash the states [T, K n, 13]"""
    E, D = m.env_shape
    K, T, n = v.shape[0], m.T, m.n
    P, _, _, S, eff = m.cfg
    rows, _, _, _, W, Rt = _inputs(m)
    args = (_rep(rows, K), _rep(_vec(m.planes0, n), K), _rep(m.last_rpm, K), v.permute(1, 0, 2, 3).reshape(T, K * n, 4),
            _repT(_vec(m.targets, n), K), _repT(W, K), _rep(Rt, K), _rep(m.rpm_ref, K), S, eff)
    Kd = DR.model_constants(P, DEV)
    if dw:
        J, x = MR.rollout_cost_dw(Kd, P, args[0], *args[1:], kw.pop("group", D), **kw)
        return J.reshape(K, n), x
    return MR.rollout_cost(Kd, *args).reshape(K, n), None


def _relmax(got, want):
    return ((got - want).abs() / want.abs()).max().item()


def _moving_state(env, seed):
    """the env's start state with velocities of up to 1 m/s, so that drag at the first substep sees the previous rpm"""
    rng = np.random.default_rng(seed)
    E, D = env._E, env._D
    return {"pos": env.pos.clone(), "quat": env.quat.clone(), "vel": torch.tensor(rng.uniform(-1, 1, (E, D, 3)), device=DEV),
            "rpy_rates": torch.tensor(rng.uniform(-1, 1, (E, D, 3)), device=DEV)}


# ---- 0: the noise counter past 2^30 iterations ------------------------------------------------------------------------------

def test_noise_at_iterations_past_2_to_the_30():
    """the counter word 2 it + h in unsigned arithmetic: the device noise at it = 2^30 - 1, 2^30 and 2^31 - 1 against the
    vectorised Philox, each iteration its own noise"""
    env = _env(2, 3, "DYN", seed=81)
    m = _mppi(env, _targets(env, 82), 3, samples=4, seed=0xdeadbeefcafe)
    got = {}
    for it in (2 ** 30 - 1, 2 ** 30, 2 ** 31 - 1):
        e = m.noise(it).cpu().numpy()
        K, T, n = e.shape[:3]
        want = MR.eps_vec(m.seed, np.arange(T)[None, :, None], np.arange(K)[:, None, None], np.arange(n)[None, None, :], it)
        assert np.abs(e - want).max() <= 1e-14, it
        got[it] = e[1:].tobytes()
    assert len(set(got.values())) == 3


# ---- 1: sample J with downwash --------------------------------------------------------------------------------------------

DW_CASES = [
    # id, D, E, K, physics, model, (pyb, ctrl), bounds, rich (per-aviary weights, targets with a time axis, a phys table)
    ("d1", 1, 9, 16, "PYB_DW", "CF2X", (240, 48), None, False),                      # 128 groups per CTA: 144 = 128 + 16
    ("d3", 3, 5, 24, "PYB_GND_DRAG_DW", "CF2P", (240, 240), "per_tick", True),        # 42 per CTA: 120 = 42 + 42 + 36
    ("d5", 5, 3, 16, "PYB_GND_DRAG_DW", "CF2X", (240, 48), "const", False),           # 25 per CTA (125 lanes): 48 = 25 + 23
    ("d32", 32, 3, 5, "PYB_DW", "CF2P", (240, 48), None, True),                       # 4 per CTA: 15 = 4 + 4 + 4 + 3
    ("d33", 33, 2, 7, "PYB_GND_DRAG_DW", "CF2X", (240, 240), "per_tick", True),       # 3 per CTA (99 lanes): 14 = 4 x 3 + 2
    ("d127", 127, 2, 3, "PYB_DW", "CF2X", (240, 240), None, False),                   # one group per CTA, lane 127 idle
    ("d128", 128, 1, 3, "PYB_GND_DRAG_DW", "CF2P", (240, 48), None, True),            # one group per CTA, every lane
]


def _lattice_xyz(D, seed):
    """[D, 3]: columns of four drones 1 m apart in z (a 3 cm jitter in xy), the columns 1.5 m apart on a 6 x 6 grid: every pair in a
    column pushes by about a sixth of the weight, no two drones are close (a pair's force grows as 1/dz^2), some pairs of the
    128-drone aviary are beyond 10 m"""
    rng = np.random.default_rng(seed)
    q = np.arange(D)
    col, lev = q // 4, q % 4
    xyz = np.stack([1.5 * (col % 6), 1.5 * (col // 6), 0.3 + 1.0 * lev], 1).astype(np.float64)
    xyz[:, :2] += rng.uniform(-0.03, 0.03, (D, 2))
    return xyz


def _dw_case(D, E, K, physics, model, rates, bounds, rich, T=6, seed=21):
    env = _env(E, D, physics, model=model, pyb=rates[0], ctrl=rates[1], seed=seed, xyz=_lattice_xyz(D, seed), rpy=0.1)
    h = env.HOVER_RPM
    rng = np.random.default_rng(seed + 1)
    kw = dict(state=_moving_state(env, seed + 4))
    if rich:
        kw.update(Q=torch.tensor(rng.uniform(0.5, 2.0, (E, 13)), device=DEV), R=torch.tensor(rng.uniform(1e-3, 1e-1, (E, 4)), device=DEV),
                  phys=_phys(env, seed + 2))
    if bounds == "const":
        kw["rpm_bounds"] = (torch.full((4,), 0.97 * h, dtype=F64, device=DEV), torch.full((E, D, 4), 1.03 * h, dtype=F64, device=DEV))
    elif bounds == "per_tick":
        kw["rpm_bounds"] = (torch.tensor(h * rng.uniform(0.95, 0.99, (T, E, D, 4)), device=DEV),
                            torch.tensor(h * rng.uniform(1.01, 1.05, (T, E, D, 4)), device=DEV))
    return env, _mppi(env, _targets(env, seed + 3, T=T if rich else None), T, samples=K, sigma=0.05, seed=seed, **kw)


@pytest.mark.parametrize("case", DW_CASES, ids=[c[0] for c in DW_CASES])
def test_downwash_sample_costs_against_reference(case):
    """every sample's J against the float64 downwash rollout of its commands; negative controls: a reference blind to the pairs
    (groups of one drone) and, with drag, one whose substep 0 reads the current rpm instead of the previous tick's"""
    _, D, E, K, physics, model, rates, bounds, rich = case
    env, m = _dw_case(D, E, K, physics, model, rates, bounds, rich)
    m.sample(1)
    v = _commands(m, m.noise(1))
    J, _ = _ref_J(m, v, True)
    rel = _relmax(m.J, J)
    blind = _relmax(m.J, _ref_J(m, v, True, group=1)[0])
    print("%s: sample J max rel err %.2e; blind to the pairs %.2e" % (case[0], rel, blind))
    assert rel <= 1e-10
    assert D == 1 or blind > 1e-8                                            # one drone per aviary: no pair to miss
    if env._effects & DR.EFFECT_DRAG:
        nodrag = _relmax(m.J, _ref_J(m, v, True, drag_up0=False)[0])
        print("%s: substep 0 drag on the current rpm %.2e" % (case[0], nodrag))
        assert nodrag > 1e-8
    if bounds is not None:
        lo, hi = _inputs(m)[2:4]
        assert ((v == lo) | (v == hi)).any()


# ---- 2: the downwash predicate at its boundary -----------------------------------------------------------------------------

BOUNDARY = (100.0 - 2 * ULP100, 100.0 - ULP100, 100.0)      # only the first acts: sqrt(100 - 1 ulp) rounds to 10


def _boundary_xyz():
    """[6, 3]: three pairs 30 m apart in x (no pair across them), the upper drone of pair j 50 m above the lower one and placed so
    that dx*dx + dy*dy (dx, dy the differences of the stored coordinates) is BOUNDARY[j] exactly"""
    rng = np.random.default_rng(5)
    xyz = []
    for j, want in enumerate(BOUNDARY):
        x0, y0 = 30.0 * j - 0.5226219439146438, 1.9087258258254627
        found = None
        while found is None:
            th = rng.uniform(0, 2 * np.pi)
            x1, y1 = x0 + 10.0 * math.cos(th), y0 + 10.0 * math.sin(th)
            for a in range(-6, 7):
                for b in range(-6, 7):
                    xx, yy = x1 + a * math.ulp(x1), y1 + b * math.ulp(y1)
                    dx, dy = xx - x0, yy - y0
                    if dx * dx + dy * dy == want:
                        found = (xx, yy)
        xyz += [(x0, y0, 1.0), (found[0], found[1], 51.0)]
    return np.array(xyz)


def _boundary_ref(P, hover, xyz, lt100=False):
    """the float64 state [6, 13] after one tick of one substep at hover with downwash only (P's time step), and the pair forces"""
    from gym_pybullet_drones_b200.params import nominal_properties, physical_rows
    from gym_pybullet_drones_b200.utils.enums import DroneModel
    nom = nominal_properties(DroneModel.CF2X)
    rows = physical_rows(DroneModel.CF2X, {k: torch.full((6,), v, dtype=F64) for k, v in nom.items()})
    x0 = torch.zeros((6, 13), dtype=F64)
    x0[:, 0:3] = torch.tensor(xyz)
    x0[:, 6] = 1.0
    v = torch.full((1, 6, 4), hover, dtype=F64)
    x = MR.rollout_dw(DR.model_constants(P), P, rows, x0, torch.zeros((6, 4), dtype=F64), v, 1, 4, 6, lt100=lt100)
    fz = MR.dw_fz(P, x0[None, :, 0:3], lt100=lt100)[0]
    return x[0], fz


def _state_err(got, want):
    return float(((got.cpu() - want).abs() / want.abs().clamp(min=1.0)).max())


def test_downwash_predicate_at_its_boundary_in_every_kernel():
    """one tick of one substep (hover rpm, PYB_DW) of three pairs at dx*dx + dy*dy = 100 - 2 ulp, 100 - 1 ulp and 100 through the
    general step kernel, the CtrlAviary rollout kernel and mppi()'s commit and sample kernels (240/240 Hz), and the fused rollout
    kernel (30/30 Hz: at 240 Hz control its action buffer does not fit): every drone's state, and the sample's J, against the
    float64 reference with the oracle's sqrt(dxy2) < 10 (the pair acts on the lower drone of the first pair only); the reference
    with dxy2 < 100 also keeps the 100 - 1 ulp pair and misses every kernel"""
    from gym_pybullet_drones_b200.envs import CtrlAviary, MultiHoverAviary
    from gym_pybullet_drones_b200.utils.enums import ActionType, DroneModel, Physics
    xyz = _boundary_xyz()
    common = dict(drone_model=DroneModel.CF2X, num_drones=6, physics=Physics.PYB_DW, initial_xyzs=xyz, initial_rpys=np.zeros((6, 3)),
                  num_envs=1)

    def ctrl():
        env = CtrlAviary(pyb_freq=240, ctrl_freq=240, **common)
        env.reset()
        assert torch.equal(env.pos[0].cpu(), torch.tensor(xyz))
        return env

    class Unbounded(MultiHoverAviary):
        def _task_params(self):
            return dict(xy_bound=1e3, z_bound=1e3, tilt_bound=0.4, term_dist=1e-4)

    state = lambda e: torch.cat([getattr(e, k)[0] for k in KEYS], -1)
    env = ctrl()
    hover = float(env.HOVER_RPM)
    refs = {}
    for name, P in (("240", env._P), ("30", None)):
        if P is None:
            rl = Unbounded(pyb_freq=30, ctrl_freq=30, act=ActionType.RPM, **common)
            rl.reset()
            assert torch.equal(rl.pos[0].cpu(), torch.tensor(xyz))
            P = rl._P
        (want, fz), (miss, fz100) = _boundary_ref(P, hover, xyz), _boundary_ref(P, hover, xyz, lt100=True)
        assert fz[0] < 0 and fz[1:].eq(0).all()                              # only the 100 - 2 ulp pair acts
        assert fz100[2] < 0 and fz100[4] == 0 and abs(float(miss[2, 9] - want[2, 9])) > 1e-6   # dxy2 < 100 keeps the next
        refs[name] = want, miss
    states = {}
    env.step(torch.full((1, 6, 4), hover, dtype=F64, device=DEV))
    states["step"] = state(env), "240"
    env = ctrl()
    env.rollout(actions=torch.full((1, 1, 6, 4), hover, dtype=F64, device=DEV))
    states["CtrlAviary.rollout"] = state(env), "240"
    rl.rollout(actions=torch.zeros((1, 1, 6, 4), dtype=torch.float32, device=DEV))      # RPM action 0: HOVER_RPM exactly
    states["rollout"] = state(rl), "30"
    env = ctrl()
    tgt = {"pos": env.pos.clone(), "vel": torch.tensor([0.0, 0.0, 1.0], dtype=F64, device=DEV)}
    m = _mppi(env, tgt, 1, rpm=torch.full((1, 1, 6, 4), hover, dtype=F64, device=DEV), samples=2)
    cost = torch.empty((6,), dtype=F64, device=DEV)
    m.nominal(cost)
    states["mppi commit"] = _vec(m.states[0], 6), "240"
    m.sample(0)
    Jref, x = _ref_J(m, m.rpm[None], True)
    Jmiss, _ = _ref_J(m, m.rpm[None], True, lt100=True)
    assert _state_err(x[0], refs["240"][0]) <= 1e-13                         # the same reference through Mppi's inputs
    bad = []
    for name, (got, rate) in states.items():
        want, miss = refs[rate]
        err, err100 = _state_err(got, want), _state_err(got, miss)
        print("%s: max state err %.2e, against dxy2 < 100 %.2e" % (name, err, err100))
        if not (err <= 1e-10 and err100 > 1e-7):
            bad.append(name)
    rel, rel100 = _relmax(m.J[0], Jref[0]), _relmax(m.J[0], Jmiss[0])
    print("mppi sample: J max rel err %.2e, against dxy2 < 100 %.2e" % (rel, rel100))
    if not (rel <= 1e-10 and rel100 > 1e-8):
        bad.append("mppi sample")
    assert not bad, bad
    assert torch.equal(m.J[0], cost)


# ---- 3: the update at its shapes ---------------------------------------------------------------------------------------------

def _check_candidate(m, it, units=None):
    """the device's candidate against mppi_ref.candidate from the device's J and noise, for every unit (or those given); returns
    the worst error, normwise per unit"""
    E, D = m.env_shape
    dw = bool(m.cfg[4] & 4)
    rows, sig, lo, hi, _, _ = _inputs(m)
    J = m.J.cpu().numpy()
    Ju = MR.unit_sum(J, D) if dw else J
    u0, cand = m.rpm.cpu().numpy(), m.cand.cpu().numpy()
    e = m.noise(it).cpu().numpy()
    lo, hi = (None, None) if lo is None else (lo.cpu().numpy(), hi.cpu().numpy())
    _, delta = MR.samples(u0, sig.cpu().numpy(), e, lo, hi)
    worst = 0.0
    for u in (range(Ju.shape[1]) if units is None else units):
        w, _ = MR.weights(Ju[:, u], m.temperature)
        drones = slice(u * D, u * D + D) if dw else slice(u, u + 1)
        ref = MR.candidate(u0[:, drones], delta[:, :, drones], w)
        worst = max(worst, np.abs(cand[:, drones] - ref).max() / np.abs(ref).max())
    return worst


UPDATE_SHAPES = [
    # K, E, D, T, physics: units (E with downwash, else E D) = 1, 2, 3 mod 4
    (2, 5, 1, 8, "DYN"), (31, 3, 2, 8, "DYN"), (32, 7, 1, 8, "DYN"), (33, 9, 1, 8, "PYB_DRAG"),
    (769, 3, 2, 8, "DYN"), (1024, 3, 1, 8, "PYB_GND"),
    (33, 5, 3, 6, "PYB_DW"), (1024, 2, 4, 10, "PYB_DW"), (64, 3, 16, 4, "PYB_GND_DRAG_DW"),
]


@pytest.mark.parametrize("K, E, D, T, physics", UPDATE_SHAPES, ids=["K%d-E%d-D%d-T%d-%s" % s for s in UPDATE_SHAPES])
def test_update_at_its_shapes(K, E, D, T, physics):
    env = _env(E, D, physics, seed=K + D)
    m = _mppi(env, _targets(env, 31), T, samples=K, sigma=0.05, seed=K)
    m.sample(3)
    m.update(3)
    worst = _check_candidate(m, 3)
    print("K %d, %d units: candidate max err %.2e" % (K, m.pick.shape[0], worst))
    assert worst <= 1e-12


# ---- 4: teacher-forced decisions ---------------------------------------------------------------------------------------------

INF, NAN = float("inf"), float("nan")
K_TF = 8
UPDATE_ROWS = [
    [5.0] * K_TF,                                                      # lambda = 0: every weight 1
    [3.0, 1.0, 1.0, 4.0, 1.0, 2.0, 9.0, 1.5],                          # ties at the minimum
    [NAN, 2.0, INF, -INF, 1.0, NAN, 3.0, INF],                         # non-finite costs weigh 0
    [NAN, INF, -INF, NAN, INF, INF, NAN, -INF],                        # none finite: the nominal
    [1e308, 0.5, 1e308, 2.0, 1e308, 7.0, 3.0, 1.0],                    # the finite sum overflows: lambda = inf, weights 1
    [2.0, 1.0, 3.0, 4.0, 5.0, 6.0, 7.0, 8.0],
]


def test_update_teacher_forced_rows():
    """J rows crafted for every rule of the update, one per drone in one launch: the candidate against the reference"""
    env = _env(len(UPDATE_ROWS), 1, "DYN", seed=41)
    m = _mppi(env, _targets(env, 42), 6, samples=K_TF, sigma=0.05, seed=43)
    m.sample(0)
    m.J.copy_(torch.tensor(UPDATE_ROWS, dtype=F64, device=DEV).T)
    m.update(0)
    assert _check_candidate(m, 0) <= 1e-12
    assert torch.equal(m.cand[:, 3], m.rpm[:, 3])                                      # no finite J: the nominal's bits
    w, best = MR.weights(UPDATE_ROWS[4], m.temperature)
    assert best == 1 and np.array_equal(w, [1.0] * K_TF)
    assert MR.weights(UPDATE_ROWS[1], m.temperature)[1] == 1


def test_tiny_temperature_keeps_the_best_sample_bit_for_bit():
    """with a temperature so small that every weight but the best underflows to 0 the candidate is the best sample's commands
    bit for bit, so its J equals J[best] and the commit keeps it (jc <= J[best] at equality)"""
    env = _env(6, 4, "PYB_DRAG", seed=44)
    m = _mppi(env, _targets(env, 45), 8, samples=16, sigma=0.05, seed=46, temperature=1e-200)
    cost = torch.empty((2, m.n), dtype=F64, device=DEV)
    m.nominal(cost[0])
    m.sample(0)
    m.update(0)
    J = m.J.clone()
    best = torch.argmin(J, 0)
    v = _commands(m, m.noise(0))
    assert (best > 0).sum() > 0
    assert torch.equal(m.cand, v[best, :, torch.arange(m.n, device=DEV)].permute(1, 0, 2))
    m.commit(0, cost[1])
    assert (m.pick == -1).all()
    assert torch.equal(cost[1], J[best, torch.arange(m.n, device=DEV)])


def _craft_commit_rows(jcu, rng, sides):
    """per unit u a J row [K_TF] whose lowest entry (at s = 2, tied at s = 5) is jcu[u] moved by sides[u] ulps (-1, 0, +1)"""
    rows = []
    for u, jc in enumerate(jcu):
        t = {-1: math.nextafter(jc, -INF), 0: jc, 1: math.nextafter(jc, INF)}[sides[u]]
        row = list(t + np.abs(t) * rng.uniform(0.1, 1.0, K_TF) + 1.0)
        row[2] = row[5] = t
        rows.append(row)
    return np.array(rows).T                                       # [K, U]


def _split_in_drone_order(Ju, D, rng):
    """per-drone J [K, U D] whose drone-order sum from 0.0 is exactly Ju [K, U] (-c + c + t), and whose reverse-order sum is not
    the same bits wherever a c can be found for it"""
    K, U = Ju.shape
    J = np.zeros((K, U * D))
    for s in range(K):
        for u in range(U):
            t = Ju[s, u]
            part = [0.0] * D
            part[D - 1] = t
            if math.isfinite(t) and D >= 3:
                for c in t * 3.0 ** np.arange(3, 40) * rng.uniform(1, 2):
                    if ((t + c) - c) != t:
                        part[0], part[1] = -c, c
                        break
            J[s, u * D:u * D + D] = part
    assert np.array_equal(MR.unit_sum(J, D), Ju)
    return J


@pytest.mark.parametrize("dw", [False, True], ids=["drone", "aviary"])
def test_commit_teacher_forced_at_equality_and_one_ulp_either_side(dw):
    """J[best] at the candidate's J and one ulp either side, per drone and per aviary (the crafted drone J sum to the target bits in
    drone order): pick exactly, cost_out from the rollout of the chosen commands; negative controls: the highest s of a tie,
    `<` instead of `<=`, and with downwash the unit sum in reverse drone order"""
    env = _env(12, 3, "PYB_DW" if dw else "DYN", seed=51)
    m = _mppi(env, _targets(env, 52), 6, samples=K_TF, sigma=0.05, seed=53)
    E, D = m.env_shape
    U = E if dw else m.n
    cost = torch.empty((m.n,), dtype=F64, device=DEV)
    m.nominal(cost)
    m.sample(0)
    m.update(0)
    J_real = m.J.cpu().numpy()
    jc = _candidate_J(m, m.cand).cpu().numpy()
    jcu = MR.unit_sum(jc[None], D)[0] if dw else jc
    rng = np.random.default_rng(54)
    sides = [(-1, 0, 1)[u % 3] for u in range(U)]
    Ju = _craft_commit_rows(jcu, rng, sides)
    Jc = _split_in_drone_order(Ju, D, rng) if dw else Ju
    m.J.copy_(torch.tensor(Jc, device=DEV))
    m.commit(0, cost)
    pick, got = m.pick.cpu().numpy(), cost.cpu().numpy()
    want = [MR.pick(jcu[u], Ju[:, u]) for u in range(U)]
    assert list(pick) == want and set(want) == {-1, 2}
    assert [p == -1 for p in pick] == [sd >= 0 for sd in sides]
    for u in range(U):
        for i in (range(u * D, u * D + D) if dw else [u]):
            assert got[i] == (jc[i] if pick[u] < 0 else J_real[pick[u], i]), (u, i)
    ties = [MR.pick(jcu[u], Ju[:, u], tie="last") for u in range(U)]
    strict = [MR.pick(jcu[u], Ju[:, u], strict=True) for u in range(U)]
    assert ties != want and strict != want
    if dw:
        rev = MR.unit_sum(Jc, D, reverse=True)
        assert [MR.pick(jcu[u], rev[:, u]) for u in range(U)] != want


# ---- 5: a degenerate box -----------------------------------------------------------------------------------------------------

def test_degenerate_box():
    """lo == hi on some ticks and nominal entries exactly on a bound on others: delta is 0 where lo == hi, so the candidate keeps
    the nominal's bits there; the sample J and the candidate match the reference everywhere"""
    E, D, T, K = 6, 3, 8, 32
    env = _env(E, D, "PYB_GND_DRAG_DW", seed=61)
    env._effects = 3
    h = env.HOVER_RPM
    rng = np.random.default_rng(62)
    lo = h * rng.uniform(0.96, 0.99, (T, E, D, 4))
    hi = h * rng.uniform(1.01, 1.04, (T, E, D, 4))
    lo[2] = hi[2] = h * 1.005                                           # a point box on ticks 2 and 5
    lo[5] = hi[5] = h * rng.uniform(0.98, 1.02, (E, D, 4))
    guess = h * (1 + 0.01 * rng.uniform(-1, 1, (T, E, D, 4)))
    guess[3] = hi[3]                                                     # the nominal on the upper bound on tick 3
    guess[4] = lo[4]                                                     # and on the lower bound on tick 4
    m = _mppi(env, _targets(env, 63), T, rpm=torch.tensor(guess, device=DEV), samples=K, sigma=0.05, seed=64,
              rpm_bounds=(torch.tensor(lo, device=DEV), torch.tensor(hi, device=DEV)))
    assert torch.equal(m.rpm[3], torch.tensor(hi[3], device=DEV).reshape(-1, 4))
    m.sample(0)
    v = _commands(m, m.noise(0))
    J, _ = _ref_J(m, v, False)
    assert _relmax(m.J, J) <= 1e-10
    m.update(0)
    for k in (2, 5):
        assert torch.equal(m.cand[k], m.rpm[k]), k
    assert (m.cand[3] <= m.rpm[3]).all() and (m.cand[4] >= m.rpm[4]).all()
    assert _check_candidate(m, 0) <= 1e-12


# ---- 6: scale ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("physics", ["DYN", "PYB_DW"])
def test_one_iteration_at_scale(physics):
    """one iteration at 65 536 drones (16 384 aviaries of 4), K = 64: every pick against mppi_ref.pick from the device's J and the
    candidate's J, and the candidate on a strided subset of units against the reference with the noise from the vectorised
    Philox"""
    t0 = time.perf_counter()
    E, D, T, K, it = 16384, 4, 8, 64, 2
    env = _env(E, D, physics, seed=71)
    m = _mppi(env, _targets(env, 72), T, samples=K, sigma=0.05, seed=0x5eed5eed5eed)
    dw = physics == "PYB_DW"
    cost = torch.empty((2, m.n), dtype=F64, device=DEV)
    m.nominal(cost[0])
    m.sample(it)
    m.update(it)
    jc = _candidate_J(m, m.cand)
    u_all = m.rpm.cpu().numpy()                                                  # the nominal, before the commit replaces it
    m.commit(it, cost[1])
    J, jc, pick = m.J.cpu().numpy(), jc.cpu().numpy(), m.pick.cpu().numpy()
    Ju, jcu = (MR.unit_sum(J, D), MR.unit_sum(jc[None], D)[0]) if dw else (J, jc)
    U = Ju.shape[1]
    want = np.array([MR.pick(jcu[u], Ju[:, u]) for u in range(U)])
    assert np.array_equal(pick, want)
    # the candidate of every 331st unit, its noise from the vectorised Philox
    units = np.arange(0, U, 331)
    drones = (units[:, None] * D + np.arange(D)).reshape(-1) if dw else units
    _, sig, _, _, _, _ = _inputs(m)
    k, s = np.arange(T)[None, :, None], np.arange(K)[:, None, None]
    e = MR.eps_vec(m.seed, k, s, drones[None, None, :], it)                     # [K, T, len(drones), 4]
    u0 = u_all[:, drones]
    _, delta = MR.samples(u0, sig.cpu().numpy()[drones], e)
    cand = m.cand.cpu().numpy()[:, drones]
    worst = 0.0
    for j, u in enumerate(units):
        w, _ = MR.weights(Ju[:, u], m.temperature)
        sl = slice(j * D, j * D + D) if dw else slice(j, j + 1)
        ref = MR.candidate(u0[:, sl], delta[:, :, sl], w)
        worst = max(worst, np.abs(cand[:, sl] - ref).max() / np.abs(ref).max())
    print("%s at %d drones: picks %d kept / %d sample; candidate max err %.2e on %d units; %.1f s" %
          (physics, m.n, int((pick == -1).sum()), int((pick >= 0).sum()), worst, len(units), time.perf_counter() - t0))
    assert worst <= 1e-12
    assert (pick == -1).any() and (pick >= 0).any()
