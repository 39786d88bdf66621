"""Crazyflie cascaded PID on the GPU (reference: gym_pybullet_drones/control/DSLPIDControl.py)."""
import ctypes as C

import numpy as np
import torch

from .. import _native as N
from ..params import AviaryConstants, PIDCoefficients, fill_params
from ..utils.enums import DroneModel
from .BaseControl import BaseControl


class DSLPIDControl(BaseControl):
    """PID control class for Crazyflies (DSLPIDControl.py:9), batched: one instance holds the integral and
    last-rpy state of `num_drones` controllers in a float64 CUDA tensor [9, n] and `computeControl` is one
    launch of qs_pid_control.

    With `num_drones=1` and NumPy inputs it behaves like one reference controller:
    `computeControl(...) -> (rpm[4], pos_e[3], yaw_e)`.  With [n, .] inputs (NumPy or CUDA tensors) the
    outputs are batched the same way."""

    def __init__(self, drone_model: DroneModel, g: float = 9.8, *, num_drones: int = 1, device=None):
        if drone_model != DroneModel.CF2X and drone_model != DroneModel.CF2P:
            raise ValueError("[ERROR] in DSLPIDControl.__init__(), DSLPIDControl requires DroneModel.CF2X or DroneModel.CF2P")   # :33-35
        if not torch.cuda.is_available():
            raise RuntimeError("gym_pybullet_drones_b200 needs a CUDA device: the controller has no CPU path")
        self._lib = N.lib()
        self.num_drones = int(num_drones)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self._g = g
        co = PIDCoefficients.default()
        self.P_COEFF_FOR, self.I_COEFF_FOR, self.D_COEFF_FOR = co.P_COEFF_FOR, co.I_COEFF_FOR, co.D_COEFF_FOR
        self.P_COEFF_TOR, self.I_COEFF_TOR, self.D_COEFF_TOR = co.P_COEFF_TOR, co.I_COEFF_TOR, co.D_COEFF_TOR
        self.PWM2RPM_SCALE, self.PWM2RPM_CONST, self.MIN_PWM, self.MAX_PWM = 0.2685, 4070.3, 20000, 65535
        self._state = torch.zeros((9, self.num_drones), dtype=torch.float64, device=self.device)
        n = self.num_drones
        f32 = dict(dtype=torch.float32, device=self.device)
        self._rpm, self._pos_e, self._yaw_e = torch.zeros((n, 4), **f32), torch.zeros((n, 3), **f32), torch.zeros((n,), **f32)
        super().__init__(drone_model=drone_model, g=g)
        self._coefficients_changed()

    def _coefficients_changed(self):
        c = AviaryConstants(self.DRONE_MODEL)
        co = PIDCoefficients(*(np.asarray(getattr(self, a), dtype=np.float64) for a in
                               ('P_COEFF_FOR', 'I_COEFF_FOR', 'D_COEFF_FOR', 'P_COEFF_TOR', 'I_COEFF_TOR', 'D_COEFF_TOR')))
        self._P = fill_params(c, pid_model=self.DRONE_MODEL, pid_coeffs=co, pid_g=self._g)

    def reset(self):
        """Zeroes counters, last rpy and the integral errors (DSLPIDControl.py:65-78)."""
        super().reset()
        if hasattr(self, "_state"):
            self._state.zero_()

    #### state accessors (names of DSLPIDControl.py:73-78) ####
    @property
    def integral_pos_e(self):
        return self._state[0:3].t().double().cpu().numpy().reshape(-1, 3).squeeze()

    @property
    def last_rpy(self):
        return self._state[3:6].t().double().cpu().numpy().reshape(-1, 3).squeeze()

    @property
    def integral_rpy_e(self):
        return self._state[6:9].t().double().cpu().numpy().reshape(-1, 3).squeeze()

    def set_state(self, integral_pos_e=None, last_rpy=None, integral_rpy_e=None):
        for k, a in ((0, integral_pos_e), (3, last_rpy), (6, integral_rpy_e)):
            if a is not None:
                self._state[k:k + 3] = torch.as_tensor(np.asarray(a, dtype=np.float64).reshape(self.num_drones, 3).T.copy(), device=self.device)

    def _dev(self, x, width, allow_none=False):
        """-> (contiguous float32 device tensor [n, width] or strided view, row stride in floats)."""
        if x is None:
            return None, 0
        if isinstance(x, torch.Tensor):
            t = x if (x.device == self.device and x.dtype == torch.float32) else x.to(device=self.device, dtype=torch.float32)
        else:
            t = torch.as_tensor(np.asarray(x, dtype=np.float32), device=self.device)
        t = t.reshape(self.num_drones, width) if t.numel() == self.num_drones * width and t.dim() != 2 else t
        if t.dim() != 2 or t.shape != (self.num_drones, width):
            raise ValueError("expected shape (%d, %d), got %s" % (self.num_drones, width, tuple(t.shape)))
        if t.stride(1) != 1:
            t = t.contiguous()
        return t, t.stride(0)

    def computeControlFromEnv(self, env, target_pos, target_rpy=None, target_vel=None, target_rpy_rates=None, control_timestep=None):
        """computeControl for every drone of `env` (num_drones == env's drone count), reading pos / quat / vel from the env's
        float64 state on the device (qs_pid_control_state) and returning float64 RPMs [n, 4] in the env's float64
        command buffer: `env.step(rpm)` with that tensor applies them without a copy or a float32 rounding
        -- the pid.py loop (examples/pid.py:131-150) in float64 end to end.  Targets: [n, 3] arrays / tensors (float64).
        Targets, RPMs and the controller state are indexed by drone id, also after `env.reorder_by_morton()`."""
        n = env._N
        if n != self.num_drones:
            raise ValueError("controller for %d drones used with an env of %d" % (self.num_drones, n))
        self.control_counter += 1
        dev = self.device
        order = env._order                       # reorder_by_morton(): the kernel pairs env storage slot i with row / column i

        def t64(x):
            if x is None:
                return None
            t = x if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x, dtype=np.float64))
            t = t.to(device=dev, dtype=torch.float64).reshape(n, 3)
            return t.contiguous() if order is None else t[order]
        tp, tr, tv, trr = t64(target_pos), t64(target_rpy), t64(target_vel), t64(target_rpy_rates)
        ptr = lambda t: None if t is None else t.data_ptr()      # noqa: E731
        dt = float(env.CTRL_TIMESTEP if control_timestep is None else control_timestep)
        with torch.cuda.device(dev):
            if order is None:
                state, rpm, pos_e, yaw_e = self._state, env._rpm_cmd, self._pos_e, self._yaw_e
            else:                                # run in storage order, then scatter back to drone ids
                state, rpm = self._state[:, order], torch.empty_like(env._rpm_cmd)
                pos_e, yaw_e = torch.empty_like(self._pos_e), torch.empty_like(self._yaw_e)
            rc = self._lib.qs_pid_control_state(C.byref(self._P), state.data_ptr(), dt, C.byref(env._st), n,
                                                ptr(tp), ptr(tr), ptr(tv), ptr(trr), rpm.data_ptr(),
                                                pos_e.data_ptr(), yaw_e.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
            N.check(rc, "qs_pid_control_state")
            if order is not None:
                self._state[:, order] = state
                env._rpm_cmd[order] = rpm
                self._pos_e[order], self._yaw_e[order] = pos_e, yaw_e
        return env._rpm_cmd.view(env._E, env._D, 4) if env.VECTORIZED else env._rpm_cmd

    def computeControl(self, control_timestep, cur_pos, cur_quat, cur_vel, cur_ang_vel, target_pos,
                       target_rpy=None, target_vel=None, target_rpy_rates=None):
        """Computes the PID control action (as RPMs) (DSLPIDControl.py:82-145).  `cur_ang_vel` is unused (:96)."""
        self.control_counter += 1
        numpy_in = not isinstance(cur_pos, torch.Tensor)
        pos, ps = self._dev(cur_pos, 3)
        quat, qs_ = self._dev(cur_quat, 4)
        vel, vs = self._dev(cur_vel, 3)
        tpos, _ = self._dev(target_pos, 3)
        trpy, _ = self._dev(target_rpy, 3)
        tvel, _ = self._dev(target_vel, 3)
        trr, _ = self._dev(target_rpy_rates, 3)
        tpos = tpos.contiguous()
        ptr = lambda t: None if t is None else t.contiguous().data_ptr()   # noqa: E731
        with torch.cuda.device(self.device):
            rc = self._lib.qs_pid_control(C.byref(self._P), self._state.data_ptr(), float(control_timestep),
                                          pos.data_ptr(), ps, quat.data_ptr(), qs_, vel.data_ptr(), vs,
                                          tpos.data_ptr(), ptr(trpy), ptr(tvel), ptr(trr),
                                          self.num_drones, self._rpm.data_ptr(), self._pos_e.data_ptr(), self._yaw_e.data_ptr(),
                                          torch.cuda.current_stream(self.device).cuda_stream)
        N.check(rc, "qs_pid_control")
        if not numpy_in:
            return self._rpm, self._pos_e, self._yaw_e
        rpm, pe, ye = self._rpm.cpu().numpy().astype(np.float64), self._pos_e.cpu().numpy().astype(np.float64), self._yaw_e.cpu().numpy().astype(np.float64)
        if self.num_drones == 1 and np.ndim(cur_pos) == 1:
            return rpm[0], pe[0], float(ye[0])
        return rpm, pe, ye
