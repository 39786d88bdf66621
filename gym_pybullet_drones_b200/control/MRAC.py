"""Model reference adaptive controller on the GPU (reference: gym_pybullet_drones/control/MRAC.py)."""
import ctypes as C

import numpy as np
import torch

from .. import _native as N
from ..utils.enums import DroneModel
from .BaseControl import BaseControl

_MIXERS = {DroneModel.CF2X: [[-.5, -.5, -1], [-.5, .5, 1], [.5, .5, -1], [.5, -.5, 1]],         # MRAC.py:37-50
           DroneModel.CF2P: [[0, -1, -1], [+1, 0, 1], [0, 1, -1], [-1, 0, 1]]}
_MIXERS[DroneModel.RACE] = _MIXERS[DroneModel.CF2X]


def mrac_gains(drone_model: DroneModel, g: float = 9.8):
    """MRAC._compute_K (MRAC.py:56-104) with psi = 0, in float64 on the host: a dict of A, B, K, Am, Bm, P, Kr_ref_gain and the
    initial Kx = -K^T, Kr = I.  K is scipy's pole placement (`place_poles(method="YT")`, what python-control's `place` calls)
    at the poles -1 .. -12; P solves Am^T P + P Am = -600 I."""
    from scipy.linalg import solve_continuous_lyapunov
    from scipy.signal import place_poles
    u = BaseControl(drone_model, g)
    m, ixx, iyy, izz = (u._getURDFParameter(k) for k in ("m", "ixx", "iyy", "izz"))
    A = np.zeros((12, 12))
    A[0:6, 6:12] = np.eye(6)
    A[6, 4], A[7, 3] = g, -g                       # g sin(0) = 0, g cos(0) = g
    B = np.zeros((12, 4))
    B[8:12, :] = np.diag([1 / m, 1 / ixx, 1 / iyy, 1 / izz])
    K = np.asarray(place_poles(A, B, -np.linspace(1, 12, 12), method="YT").gain_matrix)
    Am = A - B @ K
    P = solve_continuous_lyapunov(Am.T, -np.eye(12) * 600)
    return dict(A=A, B=B, K=K, Am=Am, Bm=B.copy(), P=P, Kr_ref_gain=np.linalg.pinv(B) @ Am, Kx=-K.T, Kr=np.eye(4))


def mrac_params(drone_model: DroneModel, g: float = 9.8, gains=None):
    """The QsMracParams of a model (include/quadsim.h): the gains of `mrac_gains`, the mixer, KF, the PWM constants and the
    model's MAX_RPM (BaseAviary.py:119)."""
    G = mrac_gains(drone_model, g) if gains is None else gains
    u = BaseControl(drone_model, g)
    p = N.QsMracParams()
    p.Am = ((N._d * 12) * 12)(*[(N._d * 12)(*r) for r in G["Am"]])
    p.bm = (N._d * 4)(*np.diag(G["Bm"][8:12]))
    p.PBm = ((N._d * 4) * 12)(*[(N._d * 4)(*r) for r in G["P"] @ G["Bm"]])
    p.Kr_ref = ((N._d * 12) * 4)(*[(N._d * 12)(*r) for r in G["Kr_ref_gain"]])
    p.gamma_x, p.gamma_r = 5e-3, 5e-3                                                   # MRAC.py:99-100
    p.mixer = ((N._d * 3) * 4)(*[(N._d * 3)(*r) for r in _MIXERS[drone_model]])
    p.kf, p.pwm2rpm_scale, p.pwm2rpm_const, p.min_pwm, p.max_pwm = u.KF, 0.2685, 4070.3, 20000, 65535   # MRAC.py:30-33
    p.max_rpm = float(np.sqrt((u._getURDFParameter("thrust2weight") * u.GRAVITY) / (4 * u.KF)))
    return p


class MRAC(BaseControl):
    """Model reference adaptive controller for Crazyflies (MRAC.py:12), batched: one instance holds the adaptive state (Kx, Kr,
    Xm) of `num_drones` controllers in a float64 CUDA tensor [76, n] and `computeControl` is one launch of qs_mrac_control.

    With `num_drones=1` and NumPy inputs it behaves like one reference controller:
    `computeControl(...) -> (rpm[4], pos_e[3], rpy_e[3])`.  With [n, .] inputs (NumPy or CUDA tensors) the outputs are batched
    the same way.  `reset()` only zeroes `control_counter`, as in the reference: Kx and Kr keep what they adapted and the next
    call re-initialises Xm to the state it is given."""

    def __init__(self, drone_model: DroneModel, g: float = 9.8, *, num_drones: int = 1, device=None):
        if drone_model not in (DroneModel.CF2X, DroneModel.CF2P, DroneModel.RACE):
            raise ValueError("[ERROR] MRAC requires DroneModel.CF2X or DroneModel.CF2P or DroneModel.RACE")     # MRAC.py:20-22
        if not torch.cuda.is_available():
            raise RuntimeError("gym_pybullet_drones_b200 needs a CUDA device: the controller has no CPU path")
        super().__init__(drone_model=drone_model, g=g)
        self._lib = N.lib()
        self.num_drones = n = int(num_drones)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.PWM2RPM_SCALE, self.PWM2RPM_CONST, self.MIN_PWM, self.MAX_PWM = 0.2685, 4070.3, 20000, 65535
        self.MIXER_MATRIX = np.array(_MIXERS[drone_model], dtype=np.float64)
        gains = mrac_gains(drone_model, g)
        self.Am, self.Bm, self.P, self.Kr_ref_gain = gains["Am"], gains["Bm"], gains["P"], gains["Kr_ref_gain"]
        self.Gamma_x, self.Gamma_r = np.eye(12) * 5e-3, np.eye(4) * 5e-3
        self._P = mrac_params(drone_model, g, gains)
        self._state = torch.zeros((N.MRAC_STATE, n), dtype=torch.float64, device=self.device)
        self.set_state(Kx=np.broadcast_to(gains["Kx"], (n, 12, 4)), Kr=np.broadcast_to(gains["Kr"], (n, 4, 4)))
        f32 = dict(dtype=torch.float32, device=self.device)
        self._rpm = torch.zeros((n, 4), dtype=torch.float64, device=self.device)
        self._pos_e, self._rpy_e = torch.zeros((n, 3), **f32), torch.zeros((n, 3), **f32)

    #### adaptive state (names of MRAC.py) ####
    @property
    def Kx(self):
        """[n, 12, 4] float64 (NumPy)."""
        return self._state[0:48].t().cpu().numpy().reshape(self.num_drones, 12, 4)

    @property
    def Kr(self):
        """[n, 4, 4] float64 (NumPy)."""
        return self._state[48:64].t().cpu().numpy().reshape(self.num_drones, 4, 4)

    @property
    def Xm(self):
        """[n, 12] float64 (NumPy)."""
        return self._state[64:76].t().cpu().numpy().reshape(self.num_drones, 12)

    def set_state(self, Kx=None, Kr=None, Xm=None):
        """Overwrites any of Kx [n, 12, 4], Kr [n, 4, 4], Xm [n, 12] (e.g. to feed a reference controller's state)."""
        n = self.num_drones
        for lo, hi, a in ((0, 48, Kx), (48, 64, Kr), (64, 76, Xm)):
            if a is not None:
                v = np.asarray(a.cpu().numpy() if isinstance(a, torch.Tensor) else a, dtype=np.float64)
                if v.size != n * (hi - lo):
                    raise ValueError("expected %d values per drone, got shape %s" % (hi - lo, v.shape))
                self._state[lo:hi] = torch.as_tensor(np.array(v.reshape(n, hi - lo).T, order="C"), device=self.device)

    def _dev(self, x, width):
        """-> contiguous float64 device tensor [n, width], or None."""
        if x is None:
            return None
        t = x if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x, dtype=np.float64))
        t = t.to(device=self.device, dtype=torch.float64)
        if t.numel() != self.num_drones * width:
            raise ValueError("expected shape (%d, %d), got %s" % (self.num_drones, width, tuple(t.shape)))
        return t.reshape(self.num_drones, width).contiguous()

    def _init_flag(self):
        init = 1 if self.control_counter == 0 else 0                            # MRAC.py:123-125
        self.control_counter += 1
        return init

    def computeControlFromEnv(self, env, target_pos, target_rpy=None, target_vel=None, target_rpy_rates=None, control_timestep=None):
        """computeControl for every drone of `env` (num_drones == env's drone count), reading pos / quat / vel / ang_v from the env's
        float64 state on the device (qs_mrac_control_state) and returning float64 RPMs [n, 4] in the env's float64 command buffer:
        `env.step(rpm)` with that tensor applies them without a copy -- the mrac.py loop in float64 end to end.  Targets: [n, 3]
        arrays / tensors (float64).  The position and rpy errors of the call are in `last_pos_e` / `last_rpy_e`."""
        n = env._N
        if n != self.num_drones:
            raise ValueError("controller for %d drones used with an env of %d" % (self.num_drones, n))
        if env._rpm_cmd is None:
            raise ValueError("computeControlFromEnv needs an env with raw RPM actions (CtrlAviary)")
        if torch.device(env.device) != self.device:
            raise ValueError("the controller's state is on %s, the env's on %s" % (self.device, env.device))
        tp, tr, tv, trr = (self._dev(x, 3) for x in (target_pos, target_rpy, target_vel, target_rpy_rates))
        ptr = lambda t: None if t is None else t.data_ptr()      # noqa: E731
        dt = float(env.CTRL_TIMESTEP if control_timestep is None else control_timestep)
        init = self._init_flag()
        with torch.cuda.device(self.device):
            rc = self._lib.qs_mrac_control_state(C.byref(self._P), self._state.data_ptr(), init, dt, C.byref(env._st), n,
                                                 ptr(tp), ptr(tr), ptr(tv), ptr(trr), env._rpm_cmd.data_ptr(),
                                                 self._pos_e.data_ptr(), self._rpy_e.data_ptr(), torch.cuda.current_stream(self.device).cuda_stream)
        N.check(rc, "qs_mrac_control_state")
        return env._rpm_cmd.view(env._E, env._D, 4) if env.VECTORIZED else env._rpm_cmd

    @property
    def last_pos_e(self):
        return self._pos_e

    @property
    def last_rpy_e(self):
        return self._rpy_e

    def computeControl(self, control_timestep, cur_pos, cur_quat, cur_vel, cur_ang_vel, target_pos,
                       target_rpy=None, target_vel=None, target_rpy_rates=None):
        """Computes the MRAC control action (as RPMs) (MRAC.py:109-155): float64 RPMs [n, 4], float32 pos_e / rpy_e [n, 3]."""
        numpy_in = not isinstance(cur_pos, torch.Tensor)
        pos, quat, vel, angv = self._dev(cur_pos, 3), self._dev(cur_quat, 4), self._dev(cur_vel, 3), self._dev(cur_ang_vel, 3)
        tp, tr, tv, trr = (self._dev(x, 3) for x in (target_pos, target_rpy, target_vel, target_rpy_rates))
        ptr = lambda t: None if t is None else t.data_ptr()      # noqa: E731
        init = self._init_flag()
        with torch.cuda.device(self.device):
            rc = self._lib.qs_mrac_control(C.byref(self._P), self._state.data_ptr(), init, float(control_timestep),
                                           pos.data_ptr(), quat.data_ptr(), vel.data_ptr(), angv.data_ptr(),
                                           tp.data_ptr(), ptr(tr), ptr(tv), ptr(trr), self.num_drones, self._rpm.data_ptr(),
                                           self._pos_e.data_ptr(), self._rpy_e.data_ptr(), torch.cuda.current_stream(self.device).cuda_stream)
        N.check(rc, "qs_mrac_control")
        if not numpy_in:
            return self._rpm, self._pos_e, self._rpy_e
        rpm, pe, re = self._rpm.cpu().numpy(), self._pos_e.cpu().numpy().astype(np.float64), self._rpy_e.cpu().numpy().astype(np.float64)
        if self.num_drones == 1 and np.ndim(cur_pos) == 1:
            return rpm[0], pe[0], re[0]
        return rpm, pe, re
