"""Helpers of the per-aviary physical-constants tests (test infrastructure): random properties and the float64 oracle flying a
different drone in every aviary.  tests/test_dyn_params_golden.py pins PerAviaryOracle against the unmodified reference with
overwritten constants (tests/golden/dyn_params.npz)."""
import numpy as np

from gym_pybullet_drones_b200.params import PHYS_KEYS, nominal_properties
from oracle import dyn_oracle as O

# the randomisation of the tests and of tools/dyn_params_bench.py: factor ranges per property
SCALES = dict(m=(0.7, 1.3), ixx=(0.7, 1.3), iyy=(0.7, 1.3), izz=(0.7, 1.3), kf=(0.8, 1.2), km=(0.8, 1.2), arm=(0.9, 1.1),
              thrust2weight=(0.9, 1.1))


def random_properties(drone_model, E, seed):
    """{key: [E] float64 ndarray}: the model's nominal properties times seeded uniform factors (SCALES)."""
    rng = np.random.default_rng(seed)
    nom = nominal_properties(drone_model)
    return {k: nom[k] * rng.uniform(*SCALES[k], E) for k in PHYS_KEYS}


class PerAviaryOracle(O.OracleAviary):
    """OracleAviary whose aviary e flies a drone of its own (`set_properties`): the constants the reference reads from the env
    at call time -- M, L, J, J_INV, KF, KM, GRAVITY (_dynamics), HOVER_RPM (_preprocessAction), MAX_RPM (CtrlAviary clip) --
    become per-aviary arrays shaped to broadcast over the drones where the oracle uses them, derived with BaseAviary.__init__'s
    formulas (BaseAviary.py:117-119).  GND_EFF_H_CLIP and the other construction-time constants, and the embedded controller,
    stay as constructed.  Until the first set_properties() it is the plain OracleAviary."""

    PER_AVIARY = ("M", "L", "J", "J_INV", "KF", "KM", "GRAVITY", "HOVER_RPM", "MAX_RPM")

    def __init__(self, *args, props=None, **kw):
        super().__init__(*args, **kw)
        self.props = None
        if props is not None:
            self.set_properties(props)

    def set_properties(self, props, mask=None):
        """props: {PHYS_KEYS: [E] values}; mask: [E] bool of the aviaries to change (None = all)."""
        if self.props is None:
            nom = {"m": self.P.M, "ixx": self.P.J[0], "iyy": self.P.J[1], "izz": self.P.J[2], "kf": self.P.KF, "km": self.P.KM,
                   "arm": self.P.L, "thrust2weight": self.P.T2W}
            self.props = {k: np.full(self.E, float(nom[k])) for k in PHYS_KEYS}
        new = {k: np.broadcast_to(np.asarray(props[k], np.float64), (self.E,)) for k in PHYS_KEYS}
        m_ = np.ones(self.E, bool) if mask is None else np.asarray(mask, bool)
        self.props = {k: np.where(m_, new[k], self.props[k]) for k in PHYS_KEYS}
        P, p = self.P, self.props
        m, kf, km, L, t2w = p["m"], p["kf"], p["km"], p["arm"], p["thrust2weight"]
        J = np.stack([p["ixx"], p["iyy"], p["izz"]], axis=1)
        grav = P.G * m
        P.M, P.KF, P.KM = m[:, None, None], kf[:, None, None], km[:, None, None]      # with rpm [E, D, 4] / forces [E, D, 3]
        P.GRAVITY, P.L = grav[:, None], L[:, None]                                     # with [E, D] force / torque components
        P.J, P.J_INV = J[:, None, :], 1.0 / J[:, None, :]                             # with rpy_rates [E, D, 3]
        P.HOVER_RPM = np.sqrt(grav / (4 * kf))[:, None, None]
        P.MAX_RPM = np.sqrt((t2w * grav) / (4 * kf))[:, None, None]

    def _preprocess(self, action):
        """OracleAviary._preprocess for RPM / ONE_D_RPM with a per-aviary HOVER_RPM (BaseRLAviary.py:187,192,225): the base class
        converts HOVER_RPM with np.float64(), which is meant for a scalar; the arithmetic is the same (float32 `1 + 0.05 a`,
        then the float64 product).  Everything else is the base class's."""
        if self.props is None or self.kind in ("ctrl", "velocity") or self.act not in ("rpm", "one_d_rpm"):
            return super()._preprocess(action)
        action = np.asarray(action)
        if self.B > 0:
            self.action_buffer.pop(0)
            self.action_buffer.append(action.copy())
        rpm = self.P.HOVER_RPM * (1 + 0.05 * action)
        return rpm if self.act == "rpm" else np.repeat(rpm, 4, axis=-1)


def set_oracle_properties(ora, props, mask=None):
    """ora.set_properties(props, mask) for a PerAviaryOracle."""
    assert isinstance(ora, PerAviaryOracle), "use PerAviaryOracle"
    ora.set_properties(props, mask)


def merge(old, new, mask):
    """props `old` with the aviaries of `mask` taken from `new`."""
    return {k: np.where(mask, new[k], old[k]) for k in old}
