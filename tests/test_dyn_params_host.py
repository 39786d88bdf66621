"""Per-aviary physical constants without a GPU: the row builder shared with fill_params, its input checks, and the oracle flying a
different drone per aviary."""
import ctypes as C

import numpy as np
import pytest
import torch

from dyn_params_lib import PerAviaryOracle, random_properties, set_oracle_properties
from gym_pybullet_drones_b200 import _native as N
from gym_pybullet_drones_b200.params import (PHYS_KEYS, AviaryConstants, coerce_physical_args, fill_params, nominal_properties,
                                             physical_rows)
from gym_pybullet_drones_b200.utils.enums import DroneModel
from oracle import dyn_oracle as O

MODELS = [DroneModel.CF2X, DroneModel.CF2P, DroneModel.RACE]


def _rows(model, props):
    return physical_rows(model, {k: torch.as_tensor(np.asarray(props[k], np.float64)).reshape(-1) for k in PHYS_KEYS}).numpy()


def _param_row(P):
    return np.array([P.inv_m, P.gravity, P.kf, P.km, P.kx, P.ky, *P.j, *P.j_inv, P.hover_rpm, P.max_rpm])


_KX_SIGN = {DroneModel.CF2X: -1.0, DroneModel.CF2P: 1.0, DroneModel.RACE: 1.0}


def _reference_row(c):
    """The 14 columns straight from an AviaryConstants' fields, the way the reference's _dynamics / _preprocessAction read
    them: 1/M, GRAVITY, KF, KM, the torque arms (L/sqrt(2) for the X models, BaseAviary.py:846-851; L for CF2P, :852-854),
    diag(J), diag(J_INV) (np.linalg.inv), HOVER_RPM, MAX_RPM.  Independent of physical_rows and of fill_params."""
    arm = float(c.L / np.sqrt(2)) if c.DRONE_MODEL != DroneModel.CF2P else c.L
    return np.array([1.0 / c.M, c.GRAVITY, c.KF, c.KM, _KX_SIGN[c.DRONE_MODEL] * arm, arm, *np.diag(c.J), *np.diag(c.J_INV),
                     float(c.HOVER_RPM), float(c.MAX_RPM)])


def _with_properties(model, p):
    """AviaryConstants whose properties are `p`, every derived field recomputed with BaseAviary.__init__'s formulas (:117-119)."""
    c = AviaryConstants(model, 240, 30)
    c.M, c.KF, c.KM, c.L, c.THRUST2WEIGHT_RATIO = p["m"], p["kf"], p["km"], p["arm"], p["thrust2weight"]
    c.J = np.diag([p["ixx"], p["iyy"], p["izz"]])
    c.J_INV = np.linalg.inv(c.J)
    c.GRAVITY = c.G * c.M
    c.HOVER_RPM = np.sqrt(c.GRAVITY / (4 * c.KF))
    c.MAX_RPM = np.sqrt((c.THRUST2WEIGHT_RATIO * c.GRAVITY) / (4 * c.KF))
    return c


@pytest.mark.parametrize("model", MODELS)
def test_nominal_row_is_the_aviary_constants_bit_for_bit(model):
    """The nominal row, and the QsParams fields fill_params packs, equal the constructor's AviaryConstants fields."""
    c = AviaryConstants(model, 240, 30)
    ref = _reference_row(c)
    row = _rows(model, nominal_properties(model))[0]
    assert row.shape == (N.PHYS_WIDTH,) and np.all(row[14:] == 0)
    assert row[:14].tobytes() == ref.tobytes()
    for pyb, ctrl in ((240, 30), (240, 240), (1000, 50), (240, 48)):
        assert _param_row(fill_params(AviaryConstants(model, pyb, ctrl))).tobytes() == ref.tobytes(), (pyb, ctrl)


@pytest.mark.parametrize("model", MODELS)
def test_derived_columns_follow_aviary_constants(model):
    """Random properties: every column equals the AviaryConstants field derived by BaseAviary.__init__'s formulas."""
    props = random_properties(model, 2000, seed=3)
    rows = _rows(model, props)
    for e in range(2000):
        ref = _reference_row(_with_properties(model, {k: props[k][e] for k in PHYS_KEYS}))
        assert rows[e, :14].tobytes() == ref.tobytes(), (e, rows[e, :14] - ref)


def test_ctypes_mirror_has_the_table_pointer():
    assert N.ABI_VERSION == 4
    names = [f[0] for f in N.QsState._fields_]
    assert names[-1] == "phys" and C.sizeof(N.QsState) == 96


def test_coerce_accepts_scalars_arrays_and_tensors():
    E = 5
    v = coerce_physical_args(E, "cpu", dict(m=0.03, kf=np.full(E, 3e-10), km=torch.full((E,), 8e-12, dtype=torch.float64), arm=None))
    assert set(v) == {"m", "kf", "km"}
    for t in v.values():
        assert t.dtype == torch.float64 and tuple(t.shape) == (E,)
    assert float(v["m"][3]) == 0.03


@pytest.mark.parametrize("bad", [dict(m=np.full(4, 0.03)), dict(m=np.full((5, 1), 0.03)), dict(kf=-1.0), dict(km=0.0),
                                 dict(ixx=float("nan")), dict(izz=np.array([1e-5, 1e-5, np.inf, 1e-5, 1e-5])),
                                 dict(arm="long"), dict(mass=0.03), dict(m=torch.zeros((4,), dtype=torch.float64))])
def test_coerce_refuses_bad_input(bad):
    with pytest.raises(ValueError):
        coerce_physical_args(5, "cpu", bad)


def test_single_env_takes_scalars_only():
    coerce_physical_args(1, "cpu", dict(m=0.03), single=True)
    with pytest.raises(ValueError):
        coerce_physical_args(1, "cpu", dict(m=np.array([0.03])), single=True)


@pytest.mark.parametrize("model", ["cf2x", "cf2p", "racer"])
def test_oracle_with_nominal_per_aviary_arrays_is_unchanged(model):
    """The oracle's per-aviary constants, all nominal, give the scalar oracle's bits (so any difference the GPU tests see comes
    from the constants, not from the broadcasting)."""
    dm = {"cf2x": DroneModel.CF2X, "cf2p": DroneModel.CF2P, "racer": DroneModel.RACE}[model]
    E, D = 3, 2
    a, b = O.OracleAviary("multihover", E, D, drone_model=model, act="rpm"), PerAviaryOracle("multihover", E, D, drone_model=model, act="rpm")
    nom = nominal_properties(dm)
    set_oracle_properties(b, {k: np.full(E, nom[k]) for k in PHYS_KEYS})
    rng = np.random.default_rng(0)
    a.reset(); b.reset()
    for _ in range(20):
        act = rng.uniform(-1, 1, (E, D, 4)).astype(np.float32)
        oa, ob = a.step(act), b.step(act)
        for x, y in zip(oa, ob):
            assert np.array_equal(x, y)


def test_oracle_flies_a_different_drone_per_aviary():
    """Aviary e of a randomised oracle equals a one-aviary oracle built with aviary e's constants."""
    E = 3
    props = random_properties(DroneModel.CF2X, E, seed=5)
    big = PerAviaryOracle("ctrl", E, 1, drone_model="cf2x", effects=O.EFFECT_GND)
    set_oracle_properties(big, props)
    small = []
    for e in range(E):
        o = PerAviaryOracle("ctrl", 1, 1, drone_model="cf2x", effects=O.EFFECT_GND)
        set_oracle_properties(o, {k: props[k][e:e + 1] for k in PHYS_KEYS})
        small.append(o)
    rng = np.random.default_rng(1)
    big.reset(); [o.reset() for o in small]
    for _ in range(30):
        rpm = rng.uniform(10000, 30000, (E, 1, 4))
        ob = big.step(rpm)[0]
        for e in range(E):
            assert np.array_equal(ob[e], small[e].step(rpm[e:e + 1])[0][0])
