"""Tier-2 oracle of the MRAC controller: a batched float64 NumPy restatement of control/MRAC.py.

ORACLE / TEST INFRASTRUCTURE.  It follows MRAC.computeControl (MRAC.py:109-155) with n controllers at once, written from the
reference's formulas in NumPy's own operation order, and needs neither the reference nor the package.  The gains come from
`gains()` (MRAC._compute_K with psi = 0, python-control's `place` taken as scipy's YT pole placement: see
oracle/standins/control) or from a golden fixture."""
import numpy as np

from .dyn_oracle import _URDF, quat_to_euler, quat_to_matrix

MIXERS = {"cf2x": np.array([[-.5, -.5, -1], [-.5, .5, 1], [.5, .5, -1], [.5, -.5, 1]]),        # MRAC.py:37-50
          "cf2p": np.array([[0, -1, -1], [1, 0, 1], [0, 1, -1], [-1, 0, 1]], dtype=float)}
MIXERS["race"] = MIXERS["cf2x"]
_KEY = {"race": "racer"}                                   # the oracle's constants name the RACE model "racer"
PWM2RPM_SCALE, PWM2RPM_CONST, MIN_PWM, MAX_PWM = 0.2685, 4070.3, 20000, 65535


def gains(model="cf2x", g=9.8):
    """dict(A, B, K, Am, Bm, P, Kr_ref_gain, Kx, Kr) of MRAC._compute_K (MRAC.py:56-104)."""
    from scipy.linalg import solve_continuous_lyapunov
    from scipy.signal import place_poles
    u = _URDF[_KEY.get(model, model)]
    psi = 0.0
    a_sub = np.vstack((np.array([[0, 0, 0, g * np.sin(psi), g * np.cos(psi), 0],
                                 [0, 0, 0, -g * np.cos(psi), g * np.sin(psi), 0]]), np.zeros((4, 6))))
    A = np.block([[np.zeros((6, 6)), np.eye(6)], [a_sub, np.zeros((6, 6))]])
    b_sub = np.diag([1 / u["m"], 1 / u["ixx"], 1 / u["iyy"], 1 / u["izz"]])
    B = np.vstack((np.zeros((8, 4)), b_sub))
    K = np.asarray(place_poles(A, B, -np.linspace(1, 12, 12), method="YT").gain_matrix)
    Am = A - B @ K
    return dict(A=A, B=B, K=K, Am=Am, Bm=B.copy(), P=solve_continuous_lyapunov(Am.T, -np.eye(12) * 600),
                Kr_ref_gain=np.linalg.pinv(B) @ Am, Kx=-K.T, Kr=np.eye(4))


def body_rates(rpy, w):
    """Rotation.from_euler('XYZ', rpy).inv().apply(w) (MRAC.py:121), batched: R = Rx(r) Ry(p) Rz(y), returns R^T w."""
    def rot(axis, a):
        c, s = np.cos(a), np.sin(a)
        R = np.zeros(a.shape + (3, 3))
        i, j = [(1, 2), (2, 0), (0, 1)][axis]
        R[..., axis, axis] = 1.0
        R[..., i, i], R[..., i, j], R[..., j, i], R[..., j, j] = c, -s, s, c
        return R
    R = rot(0, rpy[..., 0]) @ rot(1, rpy[..., 1]) @ rot(2, rpy[..., 2])
    return np.einsum("...ji,...j->...i", R, w)


def ang_v_from_state(quat, w):
    """The state vector's ang_v rebuilt from the float64 state: getMatrixFromQuaternion(q) w."""
    return np.einsum("...ij,...j->...i", quat_to_matrix(quat), w)


class OracleMRAC:
    """n reference MRAC controllers: Kx [n, 12, 4], Kr [n, 4, 4], Xm [n, 12], control_counter (one for all, as the batched
    controller's)."""

    def __init__(self, n, model="cf2x", g=9.8, gains_=None):
        G = gains(model, g) if gains_ is None else gains_
        self.n, self.model = n, model
        self.Am, self.Bm, self.P, self.Kr_ref_gain = (np.asarray(G[k], dtype=np.float64) for k in ("Am", "Bm", "P", "Kr_ref_gain"))
        self.Kx = np.broadcast_to(np.asarray(G["Kx"], dtype=np.float64), (n, 12, 4)).copy()
        self.Kr = np.broadcast_to(np.asarray(G["Kr"], dtype=np.float64), (n, 4, 4)).copy()
        self.Xm = np.zeros((n, 12))
        self.Gamma_x, self.Gamma_r = np.eye(12) * 5e-3, np.eye(4) * 5e-3
        self.KF = _URDF[_KEY.get(model, model)]["kf"]
        self.MIX = MIXERS[model]
        self.control_counter = 0

    def reset(self):
        self.control_counter = 0

    def compute(self, dt, pos, quat, vel, ang_vel, target_pos, target_rpy=None, target_vel=None, target_rpy_rates=None):
        """-> rpm [n, 4], pos_e [n, 3], rpy_e [n, 3]; all inputs float64 [n, 3] / [n, 4]."""
        n = self.n
        z = np.zeros((n, 3))
        f = lambda x: z if x is None else np.broadcast_to(np.asarray(x, dtype=np.float64), (n, 3))   # noqa: E731
        pos, vel, ang_vel, quat = f(pos), f(vel), f(ang_vel), np.asarray(quat, dtype=np.float64).reshape(n, 4)
        tpos, trpy, tvel, trr = f(target_pos), f(target_rpy), f(target_vel), f(target_rpy_rates)
        rpy = quat_to_euler(quat)                                                          # :120
        wb = body_rates(rpy, ang_vel)                                                      # :121
        X = np.concatenate([pos, rpy, vel, wb], axis=1)[:, :, None]                        # [n, 12, 1]
        if self.control_counter == 0:
            self.Xm = X[:, :, 0].copy()                                                    # :123-124
        self.control_counter += 1
        r = np.concatenate([tpos, trpy, tvel, trr], axis=1)[:, :, None]
        rt = -self.Kr_ref_gain @ r                                                         # :127-128
        Kx_t, Kr_t = np.swapaxes(self.Kx, 1, 2), np.swapaxes(self.Kr, 1, 2)
        u = Kx_t @ X + Kr_t @ rt                                                           # :131
        e = X - self.Xm[:, :, None]                                                        # :132
        Kx_dot = -self.Gamma_x @ X @ np.swapaxes(e, 1, 2) @ self.P @ self.Bm               # :133
        Kr_dot = -self.Gamma_r @ rt @ np.swapaxes(e, 1, 2) @ self.P @ self.Bm              # :134
        self.Kx = self.Kx + Kx_dot * dt                                                    # :136-137
        self.Kr = self.Kr + Kr_dot * dt
        u = u[:, :, 0]
        thrust = np.maximum(0, u[:, 0])                                                    # :139-142
        tau = np.clip(u[:, 1:4], -3200, 3200)
        thrust = (np.sqrt(thrust / (4 * self.KF)) - PWM2RPM_CONST) / PWM2RPM_SCALE         # :144
        pwm = np.clip(thrust[:, None] + tau @ self.MIX.T, MIN_PWM, MAX_PWM)                # :145-146
        rpm = PWM2RPM_SCALE * pwm + PWM2RPM_CONST                                          # :147
        pos_e, rpy_e = tpos - pos, trpy - rpy                                              # :149-150
        Xm_dot = (self.Am @ self.Xm[:, :, None] + self.Bm @ rt)[:, :, 0]                   # :152-153
        self.Xm = self.Xm + Xm_dot * dt
        return rpm, pos_e, rpy_e
