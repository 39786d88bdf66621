"""High-level velocity-command aviary on the GPU simulator (reference: gym_pybullet_drones/envs/VelocityAviary.py)."""
import numpy as np

from .. import _native as N
from .._compat import spaces
from ..utils.enums import DroneModel, Physics
from .BaseAviary import BaseAviary


class VelocityAviary(BaseAviary):
    """Multi-drone environment class for high-level planning (VelocityAviary.py:9): action = (vx, vy, vz, fraction of
    SPEED_LIMIT) per drone, turned into RPMs by the embedded DSLPIDControl with target_pos = current position, target
    yaw = current yaw and target_vel = SPEED_LIMIT*|a3|*unit(a0:3) (VelocityAviary.py:129-168); observation = the 20-float
    state vectors, reward -1, never done (same dummy task as CtrlAviary).  One fused launch: qs_step(act=VEL, OBS_STATE20)."""

    def __init__(self,
                 drone_model: DroneModel = DroneModel.CF2X,
                 num_drones: int = 1,
                 neighbourhood_radius: float = np.inf,
                 initial_xyzs=None,
                 initial_rpys=None,
                 physics: Physics = Physics.PYB,
                 pyb_freq: int = 240,
                 ctrl_freq: int = 240,
                 gui=False,
                 record=False,
                 obstacles=False,
                 user_debug_gui=True,
                 output_folder='results',
                 **vec_kwargs):
        if drone_model not in [DroneModel.CF2X, DroneModel.CF2P]:
            raise ValueError("VelocityAviary needs a DSLPIDControl-capable drone model (CF2X/CF2P)")   # VelocityAviary.py:61-62
        super().__init__(drone_model=drone_model, num_drones=num_drones, neighbourhood_radius=neighbourhood_radius,
                         initial_xyzs=initial_xyzs, initial_rpys=initial_rpys, physics=physics,
                         pyb_freq=pyb_freq, ctrl_freq=ctrl_freq, gui=gui, record=record, obstacles=obstacles,
                         user_debug_gui=user_debug_gui, output_folder=output_folder, **vec_kwargs)
        self.SPEED_LIMIT = 0.03 * self.MAX_SPEED_KMH * (1000 / 3600)      # VelocityAviary.py:78

    def _act_type(self):
        return N.ACT_VEL

    def _state20_obs(self):
        return True

    def _actionSpace(self):
        lo = np.array([[-1, -1, -1, 0] for i in range(self.NUM_DRONES)])
        hi = np.array([[1, 1, 1, 1] for i in range(self.NUM_DRONES)])
        return spaces.Box(low=lo, high=hi, dtype=np.float32)

    def _observationSpace(self):
        m = self.MAX_RPM
        lo = np.array([[-np.inf, -np.inf, 0., -1., -1., -1., -1., -np.pi, -np.pi, -np.pi, -np.inf, -np.inf, -np.inf, -np.inf, -np.inf, -np.inf, 0., 0., 0., 0.] for i in range(self.NUM_DRONES)])
        hi = np.array([[np.inf, np.inf, np.inf, 1., 1., 1., 1., np.pi, np.pi, np.pi, np.inf, np.inf, np.inf, np.inf, np.inf, np.inf, m, m, m, m] for i in range(self.NUM_DRONES)])
        return spaces.Box(low=lo, high=hi, dtype=np.float32)

    def rollout(self, actions, record=True, out=None):
        """T control ticks in ONE kernel launch (qs_ctrl_rollout): exactly T calls of `step(actions[k])`, bit for bit, with the
        drone and embedded-controller state in registers between ticks.  Vector API only; `actions` [T, E, D, 4] float32.
        Returns a dict of CUDA tensors: `obs` [T, E, D, 20] (absent with `record=False`) and `rpm` [T, E, D, 4] float64 (the RPMs
        the controller produced); `out` reuses the buffers of a previous result.  The env ends where T step() calls leave it
        (state, controller state, step counters, current observation, an attached Logger).  See CtrlAviary.rollout."""
        return self._ctrl_rollout(N.CTRL_VEL, actions=actions, record=record, out=out)

    def _computeObs(self):
        obs = self._obs_buf[self._cur]
        return self._shape_obs(obs) if self.VECTORIZED else self._obs_to_host_single(obs)
