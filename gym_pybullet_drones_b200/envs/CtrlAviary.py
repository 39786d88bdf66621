"""Raw-RPM control aviary on the GPU simulator (reference: gym_pybullet_drones/envs/CtrlAviary.py)."""
import numpy as np

from .. import _native as N
from .._compat import spaces
from ..utils.enums import DroneModel, Physics
from .BaseAviary import BaseAviary


class CtrlAviary(BaseAviary):
    """Multi-drone environment class for control applications (CtrlAviary.py:7): action = RPMs clipped to
    [0, MAX_RPM] (CtrlAviary.py:121-140), observation = the 20-float state vector of every drone
    (CtrlAviary.py:106-117), reward -1, never terminated/truncated (CtrlAviary.py:144-185)."""

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
        super().__init__(drone_model=drone_model, num_drones=num_drones, neighbourhood_radius=neighbourhood_radius,
                         initial_xyzs=initial_xyzs, initial_rpys=initial_rpys, physics=physics,
                         pyb_freq=pyb_freq, ctrl_freq=ctrl_freq, gui=gui, record=record, obstacles=obstacles,
                         user_debug_gui=user_debug_gui, output_folder=output_folder, **vec_kwargs)

    def _act_type(self):
        return N.ACT_RAW_RPM

    def _actionSpace(self):
        lo = np.array([[0., 0., 0., 0.] for i in range(self.NUM_DRONES)])
        hi = np.array([[self.MAX_RPM] * 4 for i in range(self.NUM_DRONES)])
        return spaces.Box(low=lo, high=hi, dtype=np.float32)

    def _observationSpace(self):
        m = self.MAX_RPM
        lo = np.array([[-np.inf, -np.inf, 0., -1., -1., -1., -1., -np.pi, -np.pi, -np.pi, -np.inf, -np.inf, -np.inf, -np.inf, -np.inf, -np.inf, 0., 0., 0., 0.] for i in range(self.NUM_DRONES)])
        hi = np.array([[np.inf, np.inf, np.inf, 1., 1., 1., 1., np.pi, np.pi, np.pi, np.inf, np.inf, np.inf, np.inf, np.inf, np.inf, m, m, m, m] for i in range(self.NUM_DRONES)])
        return spaces.Box(low=lo, high=hi, dtype=np.float32)

    def rollout(self, actions=None, controller=None, waypoints=None, start=None, offset=None, target_rpy=None, target_vel=None,
                target_rpy_rates=None, control_timestep=None, record=True, errors=False, out=None, *, num_steps=None, log_targets=False):
        """T control ticks in ONE kernel launch (qs_ctrl_rollout): the drone state, the controller state and the previous RPMs stay
        in registers between ticks.  Vector API only; every `Physics` mode (downwash up to 128 drones per aviary) and a per-aviary
        `set_physical_params` table.  Pass exactly one of:

        * `actions` [T, E, D, 4]: RPMs, float32 or float64 (the reference's float64 RPMs, no float32 rounding) -- T calls of
          `step(actions[k])`, bit for bit.
        * `controller`: a `DSLPIDControl(num_drones=E*D)` on the env's device.  Tick k runs, for every drone i,
          `rpm = controller.computeControlFromEnv(env, target_pos, target_rpy, target_vel, target_rpy_rates, control_timestep)`
          followed by `step(rpm)`, bit for bit, with
              target_pos(k, i) = waypoints[(start[i] + k) % W][i if per-drone else 0] + offset[i]
          `waypoints` [W, 3] (one path shared by all drones) or [W, E, D, 3] (one per drone); `start` [E, D] int (default 0: the
          phase of each drone on the path); `offset` [E, D, 3] (e.g. INIT_XYZS' z, as in pid.py); `target_rpy` / `target_vel` /
          `target_rpy_rates` [E, D, 3] or [3], constant over the rollout (default 0).  `num_steps` = T (default W, one pass);
          `control_timestep` defaults to CTRL_TIMESTEP.  The schedule index k counts from 0 in every call: to continue a
          rollout, advance `start` by the ticks already run.  `controller.control_counter` advances by T.

        Returns a dict of CUDA tensors: `obs` [T, E, D, 20] (the state vector after each tick; absent with `record=False`: at many
        drones and ticks the full buffer is large, and the env's current observation is updated either way), `rpm` [T, E, D, 4]
        float64 (the applied, clipped RPMs) and with `errors=True` (controller only) `pos_e` [T, E, D, 3] / `yaw_e` [T, E, D]
        (float32, as computeControlFromEnv returns them).  `out` reuses the buffers of a previous result.
        Afterwards the env is exactly where T step() calls leave it: state, last_clipped_action, step counters, current
        observation, reward -1 and an attached Logger (one entry per tick; `log_targets=True` logs the tick's targets as the
        controls, pid.py's layout, instead of the Logger's current controls).
        What the kernel refuses (downwash with more than 128 drones per aviary, a controller of the wrong size or device, both
        actions and a controller, the single-env API) raises ValueError."""
        if controller is not None or actions is None:
            return self._ctrl_rollout(N.CTRL_TRACK, actions=actions, controller=controller, num_steps=num_steps, waypoints=waypoints,
                                      start=start, offset=offset, target_rpy=target_rpy, target_vel=target_vel,
                                      target_rpy_rates=target_rpy_rates, control_timestep=control_timestep, record=record,
                                      errors=errors, out=out, log_targets=log_targets)
        return self._ctrl_rollout(N.CTRL_RAW, actions=actions, record=record, errors=errors, out=out)

    @staticmethod
    def schedule_targets(waypoints, start, offset, num_steps):
        """NumPy restatement of the controller rollout's target rule (for tests / reproducibility): [T, n, 3] float64 with
        targets[k, i] = waypoints[(start[i] + k) % W][i if per-drone else 0] + offset[i]; `waypoints` [W, 3] or [W, n, 3]
        (or [W, E, D, 3]), `start` [n] ints, `offset` [n, 3] or None."""
        wp = np.asarray(waypoints, dtype=np.float64)
        st = np.asarray(start, dtype=np.int64).reshape(-1)
        n, W = st.shape[0], wp.shape[0]
        wp = wp.reshape(W, 1, 3) if wp.ndim == 2 else wp.reshape(W, n, 3)
        rows = (st[None, :] + np.arange(int(num_steps))[:, None]) % W                      # [T, n], Python's mod: never negative
        cols = np.zeros(n, dtype=np.int64) if wp.shape[1] == 1 else np.arange(n)
        tp = wp[rows, cols[None, :]]
        return tp if offset is None else tp + np.asarray(offset, dtype=np.float64).reshape(1, n, 3)

    def _computeObs(self):
        obs = self._obs_buf[self._cur]
        return self._shape_obs(obs) if self.VECTORIZED else self._obs_to_host_single(obs)
