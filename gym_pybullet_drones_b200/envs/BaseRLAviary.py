"""RL plumbing of the GPU aviaries: action types, action buffer, KIN observations.

Mirrors `BaseRLAviary` (gym_pybullet_drones/envs/BaseRLAviary.py:13-322).  The per-drone
Python loops of `_preprocessAction` / `_computeObs` live inside the fused CUDA step
(qs_step): this class only declares the spaces and the kernel configuration.
"""
import ctypes as C

import numpy as np
import torch

from .. import _native as N
from .._compat import spaces
from ..utils.enums import ActionType, DroneModel, ObservationType, Physics
from .BaseAviary import BaseAviary

_ACT = {ActionType.RPM: (N.ACT_RPM, 4), ActionType.VEL: (N.ACT_VEL, 4), ActionType.PID: (N.ACT_PID, 3),
        ActionType.ONE_D_RPM: (N.ACT_ONE_D_RPM, 1), ActionType.ONE_D_PID: (N.ACT_ONE_D_PID, 1)}


class BaseRLAviary(BaseAviary):
    """Base single and multi-agent environment class for reinforcement learning (BaseRLAviary.py:10)."""

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
                 obs: ObservationType = ObservationType.KIN,
                 act: ActionType = ActionType.RPM,
                 **vec_kwargs):
        #### Create a buffer for the last .5 sec of actions (BaseRLAviary.py:66) ####
        self.ACTION_BUFFER_SIZE = int(ctrl_freq // 2)
        if obs != ObservationType.KIN:
            raise NotImplementedError("ObservationType.RGB needs PyBullet's renderer; the GPU simulator provides KIN")
        if act not in _ACT:
            print("[ERROR] in BaseRLAviary._actionSpace()")
            raise ValueError("unknown ActionType %r" % (act,))
        self.OBS_TYPE = obs
        self.ACT_TYPE = act
        if act in [ActionType.PID, ActionType.VEL, ActionType.ONE_D_PID] and drone_model not in [DroneModel.CF2X, DroneModel.CF2P]:
            raise ValueError("[ERROR] in BaseRLAviary.__init()__, no controller is available for the specified drone_model")   # :77-78
        super().__init__(drone_model=drone_model, num_drones=num_drones, neighbourhood_radius=neighbourhood_radius,
                         initial_xyzs=initial_xyzs, initial_rpys=initial_rpys, physics=physics,
                         pyb_freq=pyb_freq, ctrl_freq=ctrl_freq, gui=gui, record=record,
                         obstacles=True, user_debug_gui=False, vision_attributes=False, **vec_kwargs)
        if act == ActionType.VEL:
            self.SPEED_LIMIT = 0.03 * self.MAX_SPEED_KMH * (1000 / 3600)       # BaseRLAviary.py:95

    #### kernel configuration ####################################################
    def _act_type(self):
        return _ACT[self.ACT_TYPE][0]

    def _act_width(self):
        return _ACT[self.ACT_TYPE][1]

    def _act_buffer_size(self):
        return self.ACTION_BUFFER_SIZE

    ################################################################################

    def _actionSpace(self):
        """Box(-1, 1, (NUM_DRONES, A)) (BaseRLAviary.py:132-156)."""
        size = _ACT[self.ACT_TYPE][1]
        act_lower_bound = np.array([-1 * np.ones(size) for i in range(self.NUM_DRONES)])
        act_upper_bound = np.array([+1 * np.ones(size) for i in range(self.NUM_DRONES)])
        return spaces.Box(low=act_lower_bound, high=act_upper_bound, dtype=np.float32)

    def _observationSpace(self):
        """Box of shape (NUM_DRONES, 12 + ACTION_BUFFER_SIZE*A) (BaseRLAviary.py:243-277)."""
        lo, hi = -np.inf, np.inf
        size = _ACT[self.ACT_TYPE][1]
        kin_lo = np.array([[lo, lo, 0, lo, lo, lo, lo, lo, lo, lo, lo, lo] for i in range(self.NUM_DRONES)])
        kin_hi = np.array([[hi] * 12 for i in range(self.NUM_DRONES)])
        buf = self.ACTION_BUFFER_SIZE * size
        obs_lower_bound = np.hstack([kin_lo, -np.ones((self.NUM_DRONES, buf))])
        obs_upper_bound = np.hstack([kin_hi, +np.ones((self.NUM_DRONES, buf))])
        return spaces.Box(low=obs_lower_bound, high=obs_upper_bound, dtype=np.float32)

    def _computeObs(self):
        """Current observation (BaseRLAviary.py:284-322): [D, 12+B*A] ndarray, or the [E, D, .] tensor."""
        obs = self._obs_buf[self._cur]
        return self._shape_obs(obs) if self.VECTORIZED else self._obs_to_host_single(obs)

    ################################################################################

    def rollout(self, actions=None, num_steps=None, seed=0, out=None, policy=None, noise=None, final_obs=False, final_values=False):
        """T control ticks in one kernel launch (qs_rollout): exactly `num_steps` calls of `step()` with the same
        actions, but the drone state stays in registers and the action history in shared memory between ticks.

        Vector API only.  `actions`: float32 CUDA tensor [T, E, D, A], or None for uniform[-1, 1) actions generated on the
        device from (`seed`, tick, drone) -- the synthetic random-action workload.  Every autoreset mode of the env is
        honoured.  Returns a dict of CUDA tensors in rollout-buffer layout:
        obs [T, E, D, obs_dim] (observation AFTER each tick), actions [T, E, D, A], rewards / terminated / truncated [T, E].
        `out` may pass a previous result dict to reuse its buffers.

        With autoreset="next_step" (gymnasium >= 1.0, CleanRL-style loops) an aviary that finishes at tick k is reset by tick
        k+1, which ignores its action: obs[k+1] is the reset observation, rewards[k+1] = 0, terminated / truncated[k+1] = False.
        The result then also holds `autoreset` [T, E] bool, the ticks that only reset an aviary (a learner masks these
        transitions out): autoreset[0] is the env's pending reset from before the call, autoreset[k] = terminated[k-1] |
        truncated[k-1] after it.  obs[k] is then the terminal observation, so no final_obs is needed, and with a critic the
        time-out bootstrap value V(obs[k]) is values[k+1] where autoreset[k+1]; for the last tick it is the next rollout's
        values[0].

        `final_obs=True` (same-step autoreset only) adds `final_obs` [T, E, D, obs_dim]: the terminal observation of every
        aviary that finished at tick k, bit for bit `step()`'s `info["final_obs"]`; `final_values=True` (with a policy that has
        a critic) adds `final_values` [T, E]: the critic on those terminal observations.  Both are valid where
        `terminated | truncated` and unspecified elsewhere.  SB3's `collect_rollouts` bootstraps a time-out with them:
        `rewards[k] += gamma * final_values[k]` where `truncated[k]`.

        `policy` (a `gym_pybullet_drones_b200.policy.MlpPolicy`): the actions of every tick come from the policy evaluated
        INSIDE the kernel on the current observation -- SB3 `collect_rollouts` (examples/learn.py:93) without a policy launch
        or an action tensor per tick.  `noise` [T, E, D*A] standard-normal draws (None = act deterministically).  The result
        then also holds `log_probs` [T, E] and, with a critic, `values` [T, E]; `actions` are the UNCLIPPED samples (what PPO
        stores), the env applied them clipped to [-1, 1].  Every action type (RPM, ONE_D_RPM, and PID, VEL, ONE_D_PID through the
        embedded DSLPID controller), every `Physics` mode (DYN and the ground effect, drag and downwash variants) and a per-aviary
        `set_physical_params` table are supported; the physics is bit for bit that of `rollout(actions)` fed the clipped actions.
        Up to 64 drones per aviary and 32 action outputs (D * A) per aviary; what the kernel refuses raises ValueError with the
        reason."""
        if not self.VECTORIZED:
            raise ValueError("rollout() needs the vector API (num_envs=...)")
        if self._dw_fz is not None:
            raise ValueError("rollout() needs drones_per_env <= 128")
        if (final_obs or final_values) and not (self._flags & N.FLAG_AUTORESET_SAME_STEP):
            raise ValueError("rollout(final_obs=..., final_values=...) needs autoreset='same_step'")
        if final_values and (policy is None or policy.critic is None):
            raise ValueError("rollout(final_values=True) needs a policy with a critic")
        E, D, A, od, dev = self._E, self._D, self._A, self._obs_dim, self.device
        if policy is not None:
            if actions is not None:
                raise ValueError("pass either actions or a policy")
            if policy.in_dim != D * od or policy.out_dim != D * A:
                raise ValueError("policy must map %d inputs to %d outputs" % (D * od, D * A))
            if noise is not None:
                noise = noise.to(device=dev, dtype=torch.float32).contiguous()
                if noise.numel() % (E * D * A) or (num_steps is not None and noise.numel() != int(num_steps) * E * D * A):
                    raise ValueError("noise must be [T, %d, %d]" % (E, D * A))
                num_steps = noise.numel() // (E * D * A)
        if actions is not None:
            actions = actions.to(device=dev, dtype=torch.float32).contiguous()
            T = actions.shape[0]
            if tuple(actions.shape[1:]) not in ((E, D, A), (E * D, A)):
                raise ValueError("actions must be [T, %d, %d, %d]" % (E, D, A))
        else:
            T = int(num_steps)
        if out is None or out["obs"].shape[0] != T:
            out = dict(obs=torch.empty((T, E, D, od), dtype=torch.float32, device=dev),
                       actions=actions if actions is not None else torch.empty((T, E, D, A), dtype=torch.float32, device=dev),
                       rewards=torch.empty((T, E), dtype=torch.float32, device=dev),
                       terminated=torch.empty((T, E), dtype=torch.bool, device=dev),
                       truncated=torch.empty((T, E), dtype=torch.bool, device=dev))
        elif actions is not None:
            out["actions"] = actions
        if policy is not None:
            if "log_probs" not in out:
                out["log_probs"] = torch.empty((T, E), dtype=torch.float32, device=dev)
            if policy.critic is not None and "values" not in out:
                out["values"] = torch.empty((T, E), dtype=torch.float32, device=dev)
        if final_obs and "final_obs" not in out:
            out["final_obs"] = torch.empty((T, E, D, od), dtype=torch.float32, device=dev)
        if final_values and "final_values" not in out:
            out["final_values"] = torch.empty((T, E), dtype=torch.float32, device=dev)
        next_step = bool(self._flags & N.FLAG_AUTORESET_NEXT_STEP)
        if next_step and "autoreset" not in out:
            out["autoreset"] = torch.empty((T, E), dtype=torch.bool, device=dev)
        tmax = self._lib.qs_rollout_max_ticks(self._act_type(), self._B, D)
        if tmax <= 0:
            if self._B == 0:
                raise ValueError("rollout() needs an action buffer: ctrl_freq=%d gives ACTION_BUFFER_SIZE = 0" % self.CTRL_FREQ)
            raise ValueError("rollout() is not available for this observation width (action buffer too long for shared memory)")
        io = N.QsRolloutIO()
        io.seed, io.act_buffer_size = int(seed) & 0xFFFFFFFFFFFFFFFF, self._B
        n = self._N
        with self._on_device():
            stream = self._stream()
            if next_step:
                out["autoreset"][0].copy_(self._pending)             # the latch the first tick starts from (kernel-owned state)
            k0 = 0
            while k0 < T:
                tt = min(tmax, T - k0)
                cur = self._cur
                io.actions = out["actions"][k0].data_ptr() if actions is not None else None
                io.actions_out = out["actions"][k0].data_ptr() if actions is None else None
                io.obs_init = self._obs_ptr[cur]
                io.obs = out["obs"][k0].data_ptr()
                io.obs_last = self._obs_ptr[1 - cur]
                io.reward, io.terminated, io.truncated = out["rewards"][k0].data_ptr(), out["terminated"][k0].data_ptr(), out["truncated"][k0].data_ptr()
                io.done = None
                io.final_obs = out["final_obs"][k0].data_ptr() if final_obs else None
                io.final_values = out["final_values"][k0].data_ptr() if final_values else None
                io.tick0, io.T = int(getattr(self, "_rollout_tick", 0)) + k0, tt
                if policy is not None:
                    qp = policy.c_struct(None if noise is None else noise.view(T, -1)[k0], out["log_probs"][k0],
                                         out["values"][k0] if policy.critic is not None else None)
                    io.policy = C.addressof(qp)
                    io.actions, io.actions_out = None, out["actions"][k0].data_ptr()
                rc = self._lib.qs_rollout(C.byref(self._P), C.byref(self._st), C.byref(io), self._act_type(), self._task(),
                                          E, D, self.PYB_STEPS_PER_CTRL, self._effects, self._flags, stream)
                N.check(rc, "qs_rollout")
                self._cur = 1 - cur
                k0 += tt
            if next_step:
                torch.logical_or(out["terminated"][:-1], out["truncated"][:-1], out=out["autoreset"][1:])
        self._rollout_tick = int(getattr(self, "_rollout_tick", 0)) + T
        # keep the per-step outputs of the env consistent with the last tick
        self._reward.copy_(out["rewards"][-1]); self._terminated.copy_(out["terminated"][-1]); self._truncated.copy_(out["truncated"][-1])
        return out

    @staticmethod
    def rollout_actions_reference(seed, tick0, num_steps, n_drones, width):
        """NumPy restatement of the device action generator (for tests / reproducibility):
        splitmix64(seed + 2*((tick0+k)*N + i) + {0,1}) -> four uint32 -> (u >> 8) * 2^-23 - 1."""
        M = np.uint64(0xFFFFFFFFFFFFFFFF)

        def sm64(x):
            with np.errstate(over="ignore"):
                x = (x + np.uint64(0x9E3779B97F4A7C15)) & M
                z = x
                z = ((z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)) & M
                z = ((z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)) & M
                return z ^ (z >> np.uint64(31))
        k = np.arange(num_steps, dtype=np.uint64)[:, None]
        i = np.arange(n_drones, dtype=np.uint64)[None, :]
        with np.errstate(over="ignore"):
            key = np.uint64(seed) + np.uint64(2) * ((np.uint64(tick0) + k) * np.uint64(n_drones) + i)
        r0, r1 = sm64(key), sm64(key + np.uint64(1))
        u = np.stack([r0 & np.uint64(0xFFFFFFFF), r0 >> np.uint64(32), r1 & np.uint64(0xFFFFFFFF), r1 >> np.uint64(32)], axis=-1)
        f = ((u >> np.uint64(8)).astype(np.float32) * np.float32(1.0 / 8388608.0) - np.float32(1.0)).astype(np.float32)
        return f[..., :width]
