"""H100-native base aviary: E independent aviaries of D drones stepped in lockstep on one GPU.

Keeps the constructor, attribute names, template-method hooks and reset/step
surface of the reference's `BaseAviary` (gym_pybullet_drones/envs/BaseAviary.py:25-383)
but owns no PyBullet client: the per-drone state is a structure of arrays of
float64 CUDA tensors and `step()` is one call into the C-ABI CUDA library
(include/quadsim.h).  Every `Physics` member runs the explicit `Physics.DYN`
model (BaseAviary.py:815-892); the PYB_* members switch on the corresponding
DYN+ aerodynamic terms.

Two calling conventions, chosen by `num_envs`:
  * `num_envs=None` (default): a single aviary with the reference's gymnasium `Env`
    API -- `reset() -> (obs[D, ...] ndarray, info)`, `step(action[D, A]) -> (obs, float,
    bool, bool, info)` -- so `examples/learn.py`, `pid.py` style code runs unchanged.
  * `num_envs=E`: gymnasium `VectorEnv`-style API over E aviaries -- `reset() ->
    (obs[E, D, ...], infos)`, `step(actions[E, D, A]) -> (obs, rewards[E],
    terminations[E], truncations[E], infos)` with torch CUDA tensors in/out (zero
    copy) or NumPy arrays in/out (pinned staging buffers).
"""
import ctypes as C
import warnings

import numpy as np
import torch

from .. import _native as N
from .._compat import (AUTORESET_DISABLED, AUTORESET_NEXT_STEP, AUTORESET_SAME_STEP, Env, batch_box, spaces)
from ..params import (PHYS_KEYS, AviaryConstants, coerce_physical_args, fill_params, nominal_properties, physical_rows,
                      euler_from_quaternion, quaternion_from_euler)
from ..utils.enums import DroneModel, Physics

_PHYSICS_EFFECTS = {
    Physics.PYB: 0, Physics.DYN: 0,
    Physics.PYB_GND: N.EFFECT_GND, Physics.PYB_DRAG: N.EFFECT_DRAG, Physics.PYB_DW: N.EFFECT_DW,
    Physics.PYB_GND_DRAG_DW: N.EFFECT_GND | N.EFFECT_DRAG | N.EFFECT_DW,
}

_AUTORESET = {None: 0, "disabled": 0, AUTORESET_DISABLED: 0,
              "next_step": N.FLAG_AUTORESET_NEXT_STEP, AUTORESET_NEXT_STEP: N.FLAG_AUTORESET_NEXT_STEP,
              "same_step": N.FLAG_AUTORESET_SAME_STEP, AUTORESET_SAME_STEP: N.FLAG_AUTORESET_SAME_STEP}


_TASK_HOOKS = ("_computeReward", "_computeTerminated", "_computeTruncated")


class BaseAviary(Env):
    """Base class for the GPU aviaries (reference: envs/BaseAviary.py:19).

    Template-method seam (BaseAviary.py:1021-1104): the built-in envs evaluate `_preprocessAction`, `_computeObs`,
    `_computeReward`, `_computeTerminated`, `_computeTruncated` inside the fused kernel.  A USER subclass that overrides
    one of them is honoured: the kernel then only advances the physics (and writes the built-in observation), and the
    overridden hooks run in Python after every tick on the device state (`pos`, `quat`, `vel`, `rpy_rates`,
    `_getDroneStateVector(i)`, the built-in `super()._compute*()` values).  Single-env API: the hooks return what the
    reference's hooks return.  Vector API: `_computeReward/_computeTerminated/_computeTruncated` return [E] arrays or
    tensors; same-step autoreset is then carried out by the host side of the env."""

    metadata = {"render_modes": []}
    _EXTERNAL_DOWNWASH = False      # True: the downwash force always comes from `_downwash_stage` (sharded formations)

    ################################################################################

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
                 vision_attributes=False,
                 output_folder='results',
                 *,
                 num_envs=None,
                 device=None,
                 autoreset=None,
                 autoreset_clears_controllers=False,
                 autoreset_clears_action_buffer=False,
                 rpy_f32=True,
                 host_copy=True,
                 track_last_action=None,
                 host_obs="full",
                 ):
        """Same positional/keyword parameters as the reference (BaseAviary.py:25-40).

        Keyword-only extensions
        -----------------------
        num_envs : int | None
            None = single aviary with the reference's Env API; E = vectorised API over E aviaries.
        device : torch.device | str | int | None
            CUDA device holding the state (default: the current CUDA device).
        autoreset : None | "next_step" | "same_step" | "disabled"
            Vector-env autoreset mode (gymnasium's AutoresetMode members are accepted too).
        autoreset_clears_controllers, autoreset_clears_action_buffer : bool
            The reference's reset() clears neither the embedded PID controllers nor the action
            buffer (quirk kept by default); set to clear them when an env auto-resets.
        rpy_f32 : bool
            Evaluate the reported roll/pitch/yaw with float32 atan2f/asinf on float64 arguments (default; error ~2e-7 rad,
            far inside the 1e-5 parity bound); False = float64 atan2/asin.  Only the reported angles change: the tilt
            truncation is decided on float64 angles, and the observation of a freshly reset drone carries float64 angles,
            in both modes.
        track_last_action : bool | None
            Keep `last_clipped_action` (BaseAviary.py:372, 32 bytes written per drone and tick).  None = only where the model
            needs it (drag, CtrlAviary/VelocityAviary state vectors, formations) or for the single-env API.
        host_obs : "full" | "head"
            NumPy vector API only.  "head": step() returns only the kinematic head of every observation, [E, D, 12]
            (pos3 rpy3 vel3 ang_v3): the rest of a KIN observation is the buffer of the last actions, which a caller that
            supplies the actions already holds -- 3 MB instead of 19 MB cross PCIe per step of 65 536 drones.
        host_copy : bool
            NumPy mode only: return fresh arrays (True) or views of the pinned staging buffers
            that stay valid until the next-but-one step (False).
        """
        if not torch.cuda.is_available():
            raise RuntimeError("gym_pybullet_drones_b200 needs a CUDA device: the simulator has no CPU path")
        self._lib = N.lib()
        if gui or record:
            warnings.warn("gui/record are not available on the GPU simulator (no renderer); ignored")
        if physics != Physics.DYN:
            # the reference's PYB* members run Bullet's solver (ground plane, collisions); here every member runs the
            # explicit DYN integrator (BaseAviary.py:815-892), PYB_* adding the matching aerodynamic terms
            warnings.warn("Physics.%s runs the explicit Physics.DYN model on the GPU simulator%s: there is no Bullet solver, "
                          "no ground plane and no collisions (a drone below z=0 keeps falling); pass physics=Physics.DYN "
                          "to silence this warning" % (physics.name, "" if physics == Physics.PYB else " plus the %s force terms" % physics.value),
                          stacklevel=3)
        if vision_attributes:
            raise NotImplementedError("RGB observations need PyBullet's renderer; only ObservationType.KIN is supported")
        #### Constants (BaseAviary.py:74-128) ######################
        c = AviaryConstants(drone_model, pyb_freq, ctrl_freq)
        self.__dict__.update(vars(c))
        self._consts = c
        #### Parameters / options ##################################
        self.NUM_DRONES = int(num_drones)
        self.NEIGHBOURHOOD_RADIUS = neighbourhood_radius
        self.GUI, self.RECORD, self.PHYSICS = False, False, physics
        self.OBSTACLES, self.USER_DEBUG, self.OUTPUT_FOLDER = obstacles, user_debug_gui, output_folder
        self.VISION_ATTR = False
        self.VECTORIZED = num_envs is not None
        self.num_envs = int(num_envs) if self.VECTORIZED else 1
        if self.num_envs <= 0 or self.NUM_DRONES <= 0:
            raise ValueError("num_envs and num_drones must be positive")
        self._E, self._D = self.num_envs, self.NUM_DRONES
        self._N = self._E * self._D
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.type != "cuda":
            raise ValueError("device must be a CUDA device")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self._effects = _PHYSICS_EFFECTS[physics]
        if autoreset not in _AUTORESET:
            raise ValueError("autoreset must be None, 'next_step', 'same_step' or 'disabled'")
        self._flags = _AUTORESET[autoreset]
        if autoreset_clears_controllers:
            self._flags |= N.FLAG_AUTORESET_CLEARS_PID
        if autoreset_clears_action_buffer:
            self._flags |= N.FLAG_AUTORESET_CLEARS_HISTORY
        if rpy_f32:
            self._flags |= N.FLAG_RPY_F32
        self.autoreset_mode = {0: AUTORESET_DISABLED, N.FLAG_AUTORESET_NEXT_STEP: AUTORESET_NEXT_STEP,
                               N.FLAG_AUTORESET_SAME_STEP: AUTORESET_SAME_STEP}[_AUTORESET[autoreset]]
        #### hooks overridden by a user subclass (the built-in envs leave them to the kernel) ####
        self._hook_task = [h for h in _TASK_HOOKS if self._user_override(h)]
        self._hook_obs = self._user_override("_computeObs")
        self._hook_pre = self._user_override("_preprocessAction")
        self._py_hooks = bool(self._hook_task or self._hook_obs or self._hook_pre)
        self._py_autoreset = False
        if self._py_hooks:
            if self._hook_pre and self._act_type() != N.ACT_RAW_RPM:
                raise NotImplementedError("_preprocessAction can only be overridden on raw-RPM envs (CtrlAviary): the RL action "
                                          "types are decoded inside the kernel, which also keeps the action buffer of the observation")
            if self._flags & N.FLAG_AUTORESET_NEXT_STEP:
                raise NotImplementedError("autoreset='next_step' is not available with Python task hooks; use 'same_step' or reset(options={'reset_mask': ...})")
            if self._hook_task:      # the kernel must not reset on its own verdict: the host does it after the hooks ran
                self._py_autoreset = bool(self._flags & N.FLAG_AUTORESET_SAME_STEP)
                self._flags &= ~(N.FLAG_AUTORESET_SAME_STEP | N.FLAG_AUTORESET_NEXT_STEP)
        self.metadata = dict(self.metadata, autoreset_mode=self.autoreset_mode)
        self._host_copy = host_copy
        self._track_last_action = track_last_action
        if host_obs not in ("full", "head"):
            raise ValueError("host_obs must be 'full' or 'head'")
        self._host_obs_head = host_obs == "head"
        self._log = None                     # (QsLogRing, controls tensor) while a utils.Logger is attached
        self._gather = None                  # sharding.ObsGather: the tick also writes its rows into the learner's tensor
        self._order = self._inv = None       # reorder_by_morton(): storage index -> drone id and back
        self._phys = None                    # [E, 16] QsState.phys rows, allocated by the first set_physical_params()
        self._phys_props = None              # [E, 8] the PHYS_KEYS values behind them
        #### Initial poses (BaseAviary.py:194-207); [D,3] shared by all aviaries or [E,D,3] per aviary ####
        self._tables_per_env = False
        if initial_xyzs is None:
            self.INIT_XYZS = c.default_init_xyzs(self.NUM_DRONES)
        else:
            self.INIT_XYZS = self._check_init(initial_xyzs, "initial_xyzs")
        if initial_rpys is None:
            self.INIT_RPYS = np.zeros((self.NUM_DRONES, 3))
        else:
            self.INIT_RPYS = self._check_init(initial_rpys, "initial_rpys")
        #### Action/observation spaces (hooks of the subclasses) ####
        self.action_space = self._actionSpace()
        self.observation_space = self._observationSpace()
        if self.VECTORIZED:
            self.single_action_space, self.single_observation_space = self.action_space, self.observation_space
            self.action_space = batch_box(self.single_action_space, self._E)
            self.observation_space = batch_box(self.single_observation_space, self._E)
        #### Device state ##########################################
        self._allocate()
        self._housekeeping()

    ################################################################################
    # configuration supplied by subclasses

    def _user_override(self, name):
        """True if the hook `name` is defined by a class outside this package, i.e. by a user subclass."""
        for klass in type(self).__mro__:
            if name in vars(klass):
                return not klass.__module__.startswith(__name__.split(".envs.")[0] + ".")
        return False

    def _act_type(self):
        """QS_ACT_* of this env (RAW_RPM for CtrlAviary-style envs)."""
        raise NotImplementedError

    def _task(self):
        return N.TASK_NONE

    def _act_width(self):
        return 4

    def _act_buffer_size(self):
        return 0

    def _task_params(self):
        """dict(xy_bound=..., episode_len_sec=...) overrides for QsParams."""
        return {}

    def _state20_obs(self):
        """True: observations are the [D, 20] state vectors of _getDroneStateVector (CtrlAviary, VelocityAviary)."""
        return self._act_type() == N.ACT_RAW_RPM

    def _target_table(self):
        """[D,3] / [E,D,3] TARGET_POS or None."""
        return None

    ################################################################################

    def _check_init(self, arr, name):
        a = np.asarray(arr, dtype=np.float64)
        if a.shape == (self.NUM_DRONES, 3):
            return a
        if a.shape == (self._E, self.NUM_DRONES, 3) and self.VECTORIZED:
            self._tables_per_env = True
            return a
        raise ValueError("[ERROR] invalid %s in BaseAviary.__init__(), try %s.reshape(NUM_DRONES,3)" % (name, name))

    def _table(self, arr, width=3):
        """[D,w] or [E,D,w] float64 -> float64 device table [rows,4] (32-byte rows)."""
        a = np.asarray(arr, dtype=np.float64)
        if self._tables_per_env:
            a = np.broadcast_to(a, (self._E, self._D, a.shape[-1])).reshape(self._N, a.shape[-1])
        else:
            a = a.reshape(self._D, a.shape[-1])
        out = np.zeros((a.shape[0], 4), np.float64)
        out[:, :a.shape[1]] = a
        return torch.from_numpy(out).to(self.device)

    def _allocate(self):
        dev, E, D, n = self.device, self._E, self._D, self._N
        self._A = self._act_width()
        self._B = self._act_buffer_size()
        raw = self._state20_obs()
        self._obs_dim = 20 if raw else 12 + self._B * self._A
        if raw and self._act_type() != N.ACT_RAW_RPM:
            self._flags |= N.FLAG_OBS_STATE20
        f32 = dict(dtype=torch.float32, device=dev)
        f64 = dict(dtype=torch.float64, device=dev)
        #### persistent state, float64 (include/quadsim.h: QsState): [pos|w.x] [quat] [vel|w.y] planes of [n,4] + w.z [n] ####
        self._planes = torch.zeros((13 * n,), **f64)
        self._plane = self._planes[:12 * n].view(3, n, 4)
        self._wz = self._planes[12 * n:]
        self._last_rpm = torch.zeros((n, 4), **f64)
        self._step_counter = torch.zeros((E,), dtype=torch.int32, device=dev)
        self._pending = torch.zeros((E,), dtype=torch.uint8, device=dev)
        needs_pid = self._act_type() in (N.ACT_PID, N.ACT_VEL, N.ACT_ONE_D_PID)
        self._pid = torch.zeros((9, n), **f64) if needs_pid else None
        self._obs_buf = [torch.zeros((n, self._obs_dim), **f32), torch.zeros((n, self._obs_dim), **f32)]
        self._cur = 0
        self._reward = torch.zeros((E,), **f32)
        self._terminated = torch.zeros((E,), dtype=torch.bool, device=dev)
        self._truncated = torch.zeros((E,), dtype=torch.bool, device=dev)
        self._done = torch.zeros((E,), dtype=torch.bool, device=dev)
        self._final_obs = torch.zeros((n, self._obs_dim), **f32) if (self._flags & N.FLAG_AUTORESET_SAME_STEP) else None
        big_dw = (self._effects & N.EFFECT_DW) and (D > 128 or self._EXTERNAL_DOWNWASH)
        self._dw_fz = torch.zeros((n,), **f32) if big_dw else None
        self._pos_f32 = torch.zeros((n, 4), **f32) if big_dw else None                       # float32 position mirror (pair kernels)
        self._dw_boxes = torch.zeros((E, (D + 31) // 32, 8), **f32) if big_dw else None     # chunk boxes (qs_downwash_boxed)
        self._action_dev = torch.zeros((n, self._A), **f32)
        self._rpm_cmd = torch.zeros((n, 4), **f64) if raw and self._act_type() == N.ACT_RAW_RPM else None      # float64 RPM commands
        #### tables ####
        if np.asarray(self.INIT_XYZS).ndim != np.asarray(self.INIT_RPYS).ndim and self._tables_per_env:
            pass  # _table() broadcasts the [D,3] one
        self._init_pos = self._table(self.INIT_XYZS)
        self._init_quat = self._table(quaternion_from_euler(self.INIT_RPYS), 4)
        tt = self._target_table()
        self._target = self._table(tt) if tt is not None else None
        #### C structs (pointers are stable: tensors are never reallocated) ####
        tp = dict(episode_len_sec=float(getattr(self, "EPISODE_LEN_SEC", 8)))
        tp.update(self._task_params())
        self._P = fill_params(self._consts, **tp)
        st = N.QsState()
        track = self._track_last_action
        if track is None:
            track = (not self.VECTORIZED) or raw or bool(self._effects & N.EFFECT_DRAG) or big_dw
        self._track_last_action = bool(track)
        st.planes, st.last_rpm = self._planes.data_ptr(), (self._last_rpm.data_ptr() if track else None)
        st.step_counter, st.pending_reset = self._step_counter.data_ptr(), self._pending.data_ptr()
        st.pid = self._pid.data_ptr() if self._pid is not None else None
        st.init_pos, st.init_quat = self._init_pos.data_ptr(), self._init_quat.data_ptr()
        st.target_pos = self._target.data_ptr() if self._target is not None else None
        st.pos_f32 = self._pos_f32.data_ptr() if self._pos_f32 is not None else None
        st.tables_per_env = 1 if self._tables_per_env else 0
        self._st = st
        #### observation head of a freshly reset drone, tabulated once on the device (SAME_STEP autoreset) ####
        self._reset_head = torch.zeros((self._init_pos.shape[0], 12), **f32)
        with self._on_device():
            N.check(self._lib.qs_reset_heads(C.byref(st), self._init_pos.shape[0], self._flags, self._reset_head.data_ptr(),
                                             self._stream()), "qs_reset_heads")
        st.reset_head = self._reset_head.data_ptr()
        io = N.QsStepIO()
        io.reward, io.terminated, io.truncated = self._reward.data_ptr(), self._terminated.data_ptr(), self._truncated.data_ptr()
        io.final_obs = self._final_obs.data_ptr() if self._final_obs is not None else None
        io.done = self._done.data_ptr()
        io.dw_fz = self._dw_fz.data_ptr() if self._dw_fz is not None else None
        io.act_buffer_size = self._B
        io.tick_substeps = 0
        # per-warp readiness of the fast step kernel (include/quadsim.h): consecutive steps of this env overlap warp by warp
        self._warp_ticket = torch.zeros(((n + 31) // 32,), dtype=torch.int32, device=dev)
        self._warp_done = torch.zeros(((n + 31) // 32,), dtype=torch.int32, device=dev)
        self._ready_err = torch.zeros((1,), dtype=torch.int32, device=dev)
        io.warp_ticket, io.warp_done, io.ready_err = self._warp_ticket.data_ptr(), self._warp_done.data_ptr(), self._ready_err.data_ptr()
        self._io = io
        #### pre-resolved handles for the per-step fast path ####
        self._obs_ptr = [b.data_ptr() for b in self._obs_buf]
        self._obs_view = [b.view(E, D, self._obs_dim) for b in self._obs_buf]
        self._final_view = self._final_obs.view(E, D, self._obs_dim) if self._final_obs is not None else None
        self._simple_launch = self._dw_fz is None and not raw and not self._state20_obs() and not self._py_hooks
        self._qs_step = self._lib.qs_step
        self._step_head = (C.byref(self._P), C.byref(self._st), C.byref(io), self._act_type(), self._task(),
                           E, D, self.PYB_STEPS_PER_CTRL, self._effects, self._flags)
        self._dev_index = self.device.index
        call = N.QsStepCall()
        call.p, call.st, call.io = C.addressof(self._P), C.addressof(self._st), C.addressof(io)
        call.act_type, call.task, call.n_envs, call.drones_per_env = self._act_type(), self._task(), E, D
        call.substeps, call.effects, call.flags = self.PYB_STEPS_PER_CTRL, self._effects, self._flags
        self._call, self._call_ptr, self._qs_step_call = call, C.addressof(call), self._lib.qs_step_call
        self._raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)
        #### pinned host staging for the NumPy API (double buffered: views stay valid until the next-but-one step) ####
        self._h_action = torch.zeros((n, self._A), dtype=torch.float32).pin_memory()
        self._h_obs = [torch.zeros((n, self._obs_dim), dtype=torch.float32).pin_memory() for _ in range(2)]
        self._h_reward = [torch.zeros((E,), dtype=torch.float32).pin_memory() for _ in range(2)]
        self._h_term = [torch.zeros((E,), dtype=torch.bool).pin_memory() for _ in range(2)]
        self._h_trunc = [torch.zeros((E,), dtype=torch.bool).pin_memory() for _ in range(2)]
        self._hcur = 0
        self._h_done = [torch.zeros((E,), dtype=torch.bool).pin_memory() for _ in range(2)]
        self._h_nfinal = [torch.zeros((1,), dtype=torch.int32).pin_memory() for _ in range(2)]
        self._h_idx = [torch.zeros((E,), dtype=torch.int64).pin_memory() for _ in range(2)]
        self._idx_dev = torch.zeros((E,), dtype=torch.int64, device=dev)
        self._nfinal_dev = torch.zeros((1,), dtype=torch.int32, device=dev)
        self._h_head = [torch.zeros((n, 12), dtype=torch.float32).pin_memory() for _ in range(2)] if (self._host_obs_head and not raw) else None
        self._h_final = None
        if self._final_obs is not None:
            self._h_final = [torch.zeros((E, D, self._obs_dim), dtype=torch.float32).pin_memory() for _ in range(2)]
        # qs_step_host's second stream: the compaction + gather of the terminal observations run next to the observation copy,
        # and the chunked pipeline brings chunk c's observation rows down while chunk c+1's actions go up and its tick runs
        self._side_stream = torch.cuda.Stream(device=dev)
        self._ev_fork, self._ev_join = torch.cuda.Event(), torch.cuda.Event()
        with self._on_device():
            self._ev_fork.record(); self._ev_join.record()              # materialise the cudaEvent_t handles
        self._h_action_np = self._h_action.numpy()
        self._h_action_view = self._h_action_np.reshape(E, D, self._A) if self.VECTORIZED else self._h_action_np.reshape(D, self._A)
        self._h_action_ptr = self._h_action.data_ptr()
        self._hio, self._h_np, self._h_fin_np = [], [], []
        for k in range(2):
            h = N.QsHostIO()
            h.action_host, h.obs_host = self._h_action.data_ptr(), self._h_obs[k].data_ptr()
            h.reward_host, h.terminated_host = self._h_reward[k].data_ptr(), self._h_term[k].data_ptr()
            h.truncated_host, h.done_host = self._h_trunc[k].data_ptr(), self._h_done[k].data_ptr()
            h.final_env_host, h.n_final_host = self._h_idx[k].data_ptr(), self._h_nfinal[k].data_ptr()
            h.action_dev, h.final_env_dev, h.n_final_dev = self._action_dev.data_ptr(), self._idx_dev.data_ptr(), self._nfinal_dev.data_ptr()
            if self._host_obs_head and not raw:
                h.obs_head_host = self._h_head[k].data_ptr()
            if self._final_obs is not None:
                h.final_obs_host = self._h_final[k].data_ptr()
            h.side_stream, h.ev_fork, h.ev_join = self._side_stream.cuda_stream, self._ev_fork.cuda_event, self._ev_join.cuda_event
            self._hio.append(h)
            self._h_np.append((self._h_obs[k].numpy().reshape(E, D, self._obs_dim), self._h_reward[k].numpy(),
                               self._h_term[k].numpy(), self._h_trunc[k].numpy()))
            self._h_fin_np.append((self._h_nfinal[k].numpy(), self._h_idx[k].numpy(),
                                   self._h_final[k].numpy() if self._h_final is not None else None))

    def pinned_actions(self):
        """float32 ndarray view ([E, D, A], or [D, A] for the single-env API) of the env's page-locked action buffer: fill it
        and pass it to step() -- the H2D copy then starts from it directly, without the staging memcpy that an ordinary
        ndarray needs.  Any other page-locked array (torch.empty(...).pin_memory().numpy()) is recognised as well."""
        return self._h_action_view

    ################################################################################
    # state views (float64 CUDA tensors; names follow BaseAviary.py:470-476).  Vector API: views of the state planes, except
    # after reorder_by_morton(), where they are copies gathered into drone-id order.

    def _by_id(self, t):
        """Per-drone rows [N, ...] of the storage order in drone-id order: `t` itself unless reorder_by_morton() has permuted
        the storage (then a gathered copy)."""
        return t if self._inv is None else t[self._inv]

    @property
    def pos(self):
        p = self._by_id(self._plane[0, :, 0:3])
        return p.view(self._E, self._D, 3) if self.VECTORIZED else self._host(p)

    @property
    def quat(self):
        q = self._by_id(self._plane[1])
        return q.view(self._E, self._D, 4) if self.VECTORIZED else self._host(q)

    @property
    def vel(self):
        v = self._by_id(self._plane[2, :, 0:3])
        return v.view(self._E, self._D, 3) if self.VECTORIZED else self._host(v)

    @property
    def rpy_rates(self):
        w = self._by_id(torch.stack([self._plane[0, :, 3], self._plane[2, :, 3], self._wz], dim=1))
        return w.view(self._E, self._D, 3) if self.VECTORIZED else w.cpu().numpy()

    @property
    def step_counter(self):
        return self._step_counter if self.VECTORIZED else int(self._step_counter[0].item())

    @property
    def last_clipped_action(self):
        if not self._track_last_action:
            raise AttributeError("last_clipped_action is not tracked by this env (pass track_last_action=True)")
        r = self._by_id(self._last_rpm)
        return r.view(self._E, self._D, 4) if self.VECTORIZED else self._host(r)

    @staticmethod
    def _host(t):
        return t.detach().cpu().numpy().astype(np.float64)

    @property
    def pid_state(self):
        """[9, E*D] float64 CUDA tensor of the embedded controllers (integral_pos_e, last_rpy, integral_rpy_e) or None.  The
        controllers' own state, columns in drone-id order; after reorder_by_morton() a gathered copy."""
        if self._pid is None or self._inv is None:
            return self._pid
        return self._pid[:, self._inv]

    def set_state(self, pos=None, quat=None, vel=None, rpy_rates=None, step_counter=None):
        """Overwrites (parts of) the kinematic state; arrays are [E,D,k] / [D,k] in drone-id order (stored as float64)."""
        def dev(a, k):
            if isinstance(a, torch.Tensor):
                t = a.to(device=self.device, dtype=torch.float64).reshape(self._N, k)
            else:
                t = torch.as_tensor(np.asarray(a, dtype=np.float64).reshape(self._N, k), device=self.device)
            return t if self._order is None else t[self._order]          # storage slot i holds drone _order[i]
        if pos is not None:
            self._plane[0, :, 0:3] = dev(pos, 3)
            if self._pos_f32 is not None:
                self._pos_f32[:, 0:3] = self._plane[0, :, 0:3].float()
        if quat is not None:
            self._plane[1] = dev(quat, 4)
        if vel is not None:
            self._plane[2, :, 0:3] = dev(vel, 3)
        if rpy_rates is not None:
            w = dev(rpy_rates, 3)
            self._plane[0, :, 3], self._plane[2, :, 3] = w[:, 0], w[:, 1]
            self._wz[:] = w[:, 2]
        if step_counter is not None:
            self._step_counter[:] = torch.as_tensor(np.broadcast_to(np.asarray(step_counter), (self._E,)).astype(np.int32), device=self.device)

    ################################################################################
    # per-aviary physical constants (domain randomisation; include/quadsim.h, QsState.phys)

    def set_physical_params(self, m=None, ixx=None, iyy=None, izz=None, kf=None, km=None, arm=None, thrust2weight=None, envs=None,
                            check=False):
        """Gives every aviary its own drone: mass, inertia, motor constants, arm and thrust-to-weight ratio (the DRONE_PROPERTIES
        keys).  The reference reads M, J, J_INV, KF, KM, L, GRAVITY (_dynamics), HOVER_RPM (action decode) and MAX_RPM (CtrlAviary
        clip) from the env at every call, so a user can change them between episodes; here they live in a per-aviary table that
        the step and rollout kernels read.  GRAVITY = G*M, HOVER_RPM, MAX_RPM, J^-1 and the torque arms are derived as
        BaseAviary.__init__ does (params.physical_rows).  The drone model (mixing signs), propeller offsets, ground-effect, drag
        and downwash coefficients, SPEED_LIMIT, the task and the embedded DSLPIDControl (a nominal CF2X, as in the reference) stay
        env-wide.

        Each value: a scalar, an [E] NumPy array or an [E] CUDA tensor; None keeps the current value.  `envs`: [E] bool mask
        (NumPy or CUDA) of the aviaries to change, None = all.  Wrong shapes, and non-finite or non-positive scalars / NumPy
        values, raise ValueError.  By default CUDA tensors are not read back (no host synchronisation, so the call can sit between
        the steps of a training loop): an aviary whose new values are not all finite and positive keeps its previous row, and
        `physical_params_rejected` (an int64 CUDA tensor) counts such aviaries.  `check=True` reads them back first (one
        synchronisation) and raises ValueError like the host inputs, changing nothing.  The single-env API takes scalars.

        A change takes effect at the next step() or rollout(); a rollout keeps each aviary's row for all its ticks.  With
        same-step autoreset, `set_physical_params(..., envs=done)` after a step re-randomises exactly the aviaries that start a
        new episode.  The first call allocates the table; it is never reallocated.  The M, KF, ... attributes keep describing
        the constructor's model.  Not available for aviaries larger than one CTA with downwash or for FormationShard."""
        if self._dw_fz is not None:
            raise ValueError("set_physical_params() is not available with external downwash (num_drones > 128 with downwash, "
                             "formations): the split-substep and formation kernels take the constants of QsParams only")
        vals = coerce_physical_args(self._E, self.device, dict(m=m, ixx=ixx, iyy=iyy, izz=izz, kf=kf, km=km, arm=arm,
                                                               thrust2weight=thrust2weight), single=not self.VECTORIZED)
        if check:
            bad = [k for k, v in vals.items() if not bool((torch.isfinite(v) & (v > 0)).all())]
            if bad:
                raise ValueError("%s must be finite and positive" % ", ".join(bad))
        sel = None
        if envs is not None:
            if not self.VECTORIZED:
                raise ValueError("envs= needs the vector API (num_envs=...)")
            sel = torch.as_tensor(envs, device=self.device)
            if sel.dtype != torch.bool or tuple(sel.shape) != (self._E,):
                raise ValueError("envs must be a [%d] bool mask" % self._E)
        with self._on_device():
            if self._phys is None:
                nom = nominal_properties(self.DRONE_MODEL)
                self._phys_props = torch.tensor([[nom[k] for k in PHYS_KEYS]] * self._E, dtype=torch.float64, device=self.device)
                self._phys_rejected = torch.zeros((), dtype=torch.int64, device=self.device)
                self._phys = physical_rows(self.DRONE_MODEL, {k: self._phys_props[:, j] for j, k in enumerate(PHYS_KEYS)}, self.G)
                self._st.phys = self._phys.data_ptr()
            if not vals:
                return
            new = self._phys_props.clone()
            ok = torch.ones((self._E,), dtype=torch.bool, device=self.device)
            for k, v in vals.items():
                new[:, PHYS_KEYS.index(k)] = v
                ok &= torch.isfinite(v) & (v > 0)
            take = ok if sel is None else ok & sel
            self._phys_rejected += ((~ok) if sel is None else (~ok & sel)).sum()
            rows = physical_rows(self.DRONE_MODEL, {k: new[:, j] for j, k in enumerate(PHYS_KEYS)}, self.G)
            self._phys_props.copy_(torch.where(take[:, None], new, self._phys_props))
            self._phys.copy_(torch.where(take[:, None], rows, self._phys))

    @property
    def physical_params_rejected(self):
        """int64 CUDA tensor: aviaries whose CUDA-tensor values set_physical_params() refused (not finite and positive)."""
        return self._phys_rejected if self._phys is not None else torch.zeros((), dtype=torch.int64, device=self.device)

    def physical_params(self):
        """{key: [E] float64 CUDA tensor} of the eight PHYS_KEYS values every aviary flies with (the constructor's model until
        the first set_physical_params())."""
        if self._phys_props is None:
            nom = nominal_properties(self.DRONE_MODEL)
            return {k: torch.full((self._E,), nom[k], dtype=torch.float64, device=self.device) for k in PHYS_KEYS}
        return {k: self._phys_props[:, j].clone() for j, k in enumerate(PHYS_KEYS)}

    ################################################################################

    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def _on_device(self):
        return torch.cuda.device(self.device)

    def _housekeeping(self, mask=None):
        """BaseAviary._housekeeping (BaseAviary.py:451-505): counters, poses, velocities, rates, last action."""
        with self._on_device():
            raw = self._state20_obs()
            m = None if mask is None else mask.data_ptr()
            rc = self._lib.qs_reset(C.byref(self._P), C.byref(self._st), m, self._E, self._D, 0,
                                    self._obs_buf[self._cur].data_ptr(), self._obs_dim, 1 if raw else 0, self._stream())
        N.check(rc, "qs_reset")

    def reset(self, seed: int = None, options: dict = None):
        """Resets the environment(s) (BaseAviary.py:220-255).  Deterministic like the reference: `seed` only
        seeds `np_random`.  options: {"reset_mask": bool[E]} restricts the reset to some aviaries (vector API);
        {"reset_controllers": True} / {"reset_action_buffer": True} also clear what the reference leaves alone."""
        super().reset(seed=seed)
        options = options or {}
        mask = options.get("reset_mask")
        mask_t = None
        if mask is not None:
            mask_t = torch.as_tensor(mask, device=self.device).to(torch.uint8).contiguous()
            if mask_t.shape != (self._E,):
                raise ValueError("reset_mask must have shape (num_envs,)")
        self._housekeeping(mask_t)
        if options.get("reset_controllers") and self._pid is not None:
            if mask_t is None:
                self._pid.zero_()
            else:
                self._pid.view(9, self._E, self._D)[:, mask_t.bool()] = 0
        if options.get("reset_action_buffer") and self._B > 0:
            o = self._obs_buf[self._cur].view(self._E, self._D, self._obs_dim)
            if mask_t is None:
                o[:, :, 12:] = 0
            else:
                o[mask_t.bool(), :, 12:] = 0
        obs = self._obs_buf[self._cur]
        if self.VECTORIZED:
            return self._shape_obs(obs), {}
        return self._obs_to_host_single(obs), self._computeInfo()

    ################################################################################

    def _launch(self, action_dev, f64=False):
        """One control tick on the device (BaseAviary.step, BaseAviary.py:259-383)."""
        io, cur = self._io, self._cur
        if self._order is not None:                      # the caller speaks drone ids, the buffers are in Morton order
            action_dev = action_dev.reshape(self._N, -1)[self._order].contiguous()
        io.action = action_dev.data_ptr()
        f64_flag = N.FLAG_ACTION_F64 if f64 else 0
        io.obs_prev = self._obs_buf[cur].data_ptr()
        io.obs = self._obs_buf[1 - cur].data_ptr()
        S = self.PYB_STEPS_PER_CTRL
        stream = self._stream()
        raw = self._act_type() == N.ACT_RAW_RPM
        L = self._lib
        if self._state20_obs():
            self._reward.fill_(-1.0)                       # dummy task (CtrlAviary.py:144-185, VelocityAviary.py:172-228)
        if self._dw_fz is None:
            if raw:
                rc = L.qs_dyn_substeps(C.byref(self._P), C.byref(self._st), io.action, io.obs, None,
                                       self._E, self._D, S, self._effects, self._flags | f64_flag, stream)
            else:
                rc = L.qs_step(C.byref(self._P), C.byref(self._st), C.byref(io), self._act_type(), self._task(),
                               self._E, self._D, S, self._effects, self._flags, stream)
            N.check(rc, "qs_step")
        else:
            # aviary larger than one CTA with downwash: positions couple the drones every substep
            for s in range(S):
                self._downwash_stage(stream)
                if raw:
                    last = s == S - 1
                    fl = self._flags | (N.FLAG_RPM_FROM_LAST if s > 0 else f64_flag)      # substeps 1.. re-read the clipped rpm of substep 0
                    rc = self._dyn_substep(io.action if s == 0 else None, io.obs if last else None, fl, stream)
                else:
                    fl = self._flags | (N.FLAG_RPM_FROM_LAST if s > 0 else 0) | (N.FLAG_SKIP_EPILOGUE if s < S - 1 else 0)
                    io.tick_substeps = S
                    rc = L.qs_step(C.byref(self._P), C.byref(self._st), C.byref(io), self._act_type(), self._task(),
                                   self._E, self._D, 1, self._effects, fl, stream)
                N.check(rc, "qs_step(split)")
        self._cur = 1 - cur
        if self._log is not None:
            self._log_append()
        return self._obs_buf[self._cur]

    def _ctrl_rollout(self, mode, actions=None, controller=None, num_steps=None, waypoints=None, start=None, offset=None,
                      target_rpy=None, target_vel=None, target_rpy_rates=None, control_timestep=None, record=True, errors=False,
                      out=None, log_targets=False):
        """rollout() of the state-vector envs (CtrlAviary, VelocityAviary): one qs_ctrl_rollout launch of T ticks in `mode`
        (N.CTRL_RAW / CTRL_VEL / CTRL_TRACK), or of qs_ctrl_rollout_mrac (N.CTRL_MRAC); see CtrlAviary.rollout."""
        if not self.VECTORIZED:
            raise ValueError("rollout() needs the vector API (num_envs=...)")
        if self._py_hooks:
            raise ValueError("rollout() evaluates the built-in hooks inside the kernel: not available when a subclass overrides them")
        if self._EXTERNAL_DOWNWASH:
            raise ValueError("rollout() is not available with external downwash (formations)")
        E, D, n, dev = self._E, self._D, self._N, self.device
        io = N.QsCtrlRolloutIO()
        flags = self._flags & N.FLAG_RPY_F32
        keep = []                                            # device inputs that must live until the launch is enqueued

        def rows3(x, name):
            if x is None:
                return None
            t = x if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x, dtype=np.float64))
            t = t.to(device=dev, dtype=torch.float64)
            if t.numel() == 3:
                t = t.reshape(1, 3).expand(n, 3)
            elif t.numel() != n * 3:
                raise ValueError("%s must be [3], [%d, %d, 3] or [%d, 3]" % (name, E, D, n))
            t = t.reshape(n, 3).contiguous()
            keep.append(t)
            return t.data_ptr()
        mio = None
        if mode in (N.CTRL_TRACK, N.CTRL_MRAC):
            if actions is not None:
                raise ValueError("pass either actions or a controller")
            if controller is None:
                raise ValueError("rollout() needs actions [T, E, D, 4] or a controller")
            if getattr(controller, "num_drones", None) != n or not hasattr(controller, "_state"):
                raise ValueError("the controller must be a DSLPIDControl or an MRAC for the env's %d drones (num_drones=%d)" % (n, n))
            if torch.device(controller.device) != dev:
                raise ValueError("the controller's state is on %s, the env's on %s" % (controller.device, dev))
            if waypoints is None:
                raise ValueError("a controller rollout needs waypoints [W, 3] or [W, E, D, 3]")
            wp = waypoints if isinstance(waypoints, torch.Tensor) else torch.as_tensor(np.asarray(waypoints, dtype=np.float64))
            wp = wp.to(device=dev, dtype=torch.float64).contiguous()
            if wp.dim() == 2 and wp.shape[1] == 3:
                W, M = wp.shape[0], 1
            elif wp.dim() >= 3 and wp.shape[-1] == 3 and wp[0].numel() == n * 3:
                W, M = wp.shape[0], n
            else:
                raise ValueError("waypoints must be [W, 3] (one path for every drone) or [W, %d, %d, 3] (one per drone)" % (E, D))
            if W == 0:
                raise ValueError("waypoints must hold at least one row")
            T = W if num_steps is None else int(num_steps)
            if start is None:
                st0 = torch.zeros((n,), dtype=torch.int32, device=dev)
            else:
                st0 = start if isinstance(start, torch.Tensor) else torch.as_tensor(np.asarray(start))
                st0 = st0.to(device=dev, dtype=torch.int32)
                st0 = (st0.reshape(1).expand(n) if st0.numel() == 1 else st0.reshape(n)).contiguous()
            keep += [wp, st0]
            if mode == N.CTRL_TRACK:
                io.ctrl_params = C.addressof(controller._P)
                io.pid_state = controller._state.data_ptr()
            else:
                mio = N.QsMracRolloutIO()
                mio.params, mio.state = C.addressof(controller._P), controller._state.data_ptr()
                mio.init = 1 if controller.control_counter == 0 else 0          # MRAC.py:123-124, at tick 0
            io.control_timestep = float(self.CTRL_TIMESTEP if control_timestep is None else control_timestep)
            io.waypoints, io.W, io.M, io.start = wp.data_ptr(), W, M, st0.data_ptr()
            io.offset = rows3(offset, "offset")
            io.target_rpy, io.target_vel = rows3(target_rpy, "target_rpy"), rows3(target_vel, "target_vel")
            io.target_rpy_rates = rows3(target_rpy_rates, "target_rpy_rates")
            io.log_targets = 1 if log_targets else 0
        else:
            if controller is not None:
                raise ValueError("pass either actions or a controller" if actions is not None else "%s.rollout() takes no controller" % type(self).__name__)
            if actions is None:
                raise ValueError("rollout() needs actions [T, %d, %d, 4]" % (E, D))
            if errors:
                raise ValueError("errors=True (pos_e / yaw_e) needs a controller rollout")
            a = actions if isinstance(actions, torch.Tensor) else torch.as_tensor(np.asarray(actions))
            f64 = mode == N.CTRL_RAW and a.dtype == torch.float64
            a = a.to(device=dev, dtype=torch.float64 if f64 else torch.float32).contiguous()
            if a.numel() == 0 or a.numel() % (n * 4) or a.shape[-1] != 4:
                raise ValueError("actions must be [T, %d, %d, 4]" % (E, D))
            if a.data_ptr() % 32:
                a = a.clone()
            keep.append(a)
            T = a.numel() // (n * 4)
            io.actions = a.data_ptr()
            if f64:
                flags |= N.FLAG_ACTION_F64
        if T <= 0:
            raise ValueError("num_steps must be > 0")
        shapes = dict(obs=((T, E, D, 20), torch.float32), rpm=((T, E, D, 4), torch.float64))
        if errors:
            shapes.update(pos_e=((T, E, D, 3), torch.float32))
            if mode == N.CTRL_MRAC:
                shapes.update(rpy_e=((T, E, D, 3), torch.float32))
            else:
                shapes.update(yaw_e=((T, E, D), torch.float32))
        if not record:
            del shapes["obs"]
        res = {}
        for k, (shp, dt) in shapes.items():
            b = out.get(k) if out is not None else None
            if b is None:
                b = torch.empty(shp, dtype=dt, device=dev)
            elif tuple(b.shape) != shp or b.dtype != dt or b.device != dev or not b.is_contiguous():
                raise ValueError("out[%r] must be a contiguous %s tensor of shape %s on %s" % (k, dt, shp, dev))
            res[k] = b
        ptr = lambda k: res[k].data_ptr() if k in res else None      # noqa: E731
        io.T = T
        io.obs, io.rpm, io.pos_e, io.yaw_e = ptr("obs"), ptr("rpm"), ptr("pos_e"), ptr("yaw_e")
        if mio is not None:
            mio.rpy_e = ptr("rpy_e")
        tgt = self._cur ^ (T & 1)                          # the buffer T step() calls would leave current
        io.obs_last = self._obs_ptr[tgt]
        if self._log is not None:
            ring, controls = self._log
            io.log = C.addressof(ring)
            io.log_controls = controls.data_ptr() if controls is not None else None
        with self._on_device():
            self._reward.fill_(-1.0)                       # dummy task (CtrlAviary.py:144-185)
            if mio is not None:
                rc = self._lib.qs_ctrl_rollout_mrac(C.byref(self._P), C.byref(self._st), C.byref(io), C.byref(mio), E, D,
                                                    self.PYB_STEPS_PER_CTRL, self._effects, flags, self._stream())
            else:
                rc = self._lib.qs_ctrl_rollout(C.byref(self._P), C.byref(self._st), C.byref(io), mode, E, D, self.PYB_STEPS_PER_CTRL,
                                               self._effects, flags, self._stream())
        N.check(rc, "qs_ctrl_rollout" if mio is None else "qs_ctrl_rollout_mrac")
        self._cur = tgt
        if controller is not None:
            controller.control_counter += T
        return res

    def _dyn_substep(self, rpm_ptr, state20_ptr, flags, stream):
        """One DYN substep with the downwash force of `_downwash_stage` (raw-RPM envs, split loop); FormationShard fuses its
        position exchange into this launch."""
        return self._lib.qs_dyn_substeps(C.byref(self._P), C.byref(self._st), rpm_ptr, state20_ptr, self._dw_fz.data_ptr(),
                                         self._E, self._D, 1, self._effects, flags, stream)

    def _log_append(self):
        """One entry per logged drone into the attached device ring (utils.Logger.attach, qs_log_append)."""
        ring, controls = self._log
        N.check(self._lib.qs_log_append(C.byref(self._P), C.byref(self._st), self._obs_ptr[self._cur], self._obs_dim,
                                        controls.data_ptr() if controls is not None else None, C.byref(ring), self._E, self._D,
                                        torch.cuda.current_stream(self.device).cuda_stream), "qs_log_append")

    def _downwash_stage(self, stream):
        """Pairwise downwash force of the current positions into `_dw_fz` (BaseAviary.py:785-811), once per substep."""
        N.check(self._lib.qs_downwash_boxed(C.byref(self._P), C.byref(self._st), self._E, self._D, self._dw_boxes.data_ptr(),
                                            self._dw_fz.data_ptr(), stream), "qs_downwash_boxed")

    def _shape_obs(self, obs):
        if self._inv is not None:
            obs = obs[self._inv]
        return obs.view(self._E, self._D, self._obs_dim)

    def _obs_to_host_single(self, obs):
        if self._inv is not None:
            obs = obs[self._inv]
        return obs.detach().cpu().numpy().reshape(self._D, self._obs_dim)

    def reorder_by_morton(self, bits=16):
        """Re-bins a large formation on the device (SURVEY.md 8f rank 3; BaseAviary.py:785-811): the downwash kernels skip
        32-drone chunks whose bounding boxes cannot interact, which only pays while consecutive indices are neighbours in
        space.  This sorts the STORAGE order of the drones along a Z-order curve of their current xy positions (keys, sort and
        the permutation of every per-drone buffer run on the GPU).  Call it every K ticks for formations that mix.
        One aviary per env (num_envs == 1), unsharded.

        Everything a caller passes or receives keeps the caller's drone ids: the actions and float64 RPMs of `step` (NumPy or
        torch, vector or single-env API), its observations and `info["final_obs"]`, `reset`, `set_state`, the state views
        (`pos`, `quat`, `vel`, `rpy_rates`, `last_clipped_action`, `pid_state`: copies gathered into drone-id order rather
        than views once the env is reordered), `_getDroneStateVectors` / `_getDroneStateVector` / `render`, `adjacency` /
        `_getAdjacencyMatrix`, and the targets, controller state and RPMs of `DSLPIDControl` / `MRAC.computeControlFromEnv`.
        The device-side Logger ring records storage slots, so a Logger cannot be attached to a reordered env and a reorder
        is refused while one is attached (ValueError); `Logger.detach()` first.  Returns the permutation (storage slot i
        holds drone `order[i]`)."""
        if self._E != 1 or self._dw_fz is None:
            raise ValueError("reorder_by_morton() is for one large aviary with external downwash (num_drones > 128, num_envs == 1)")
        if getattr(self, "shard", None) is not None and self.shard.world > 1:
            raise ValueError("reorder_by_morton() does not move drones between GPUs")
        if self._log is not None:
            raise ValueError("reorder_by_morton() with a Logger attached: the device ring records storage slots, which the "
                             "reorder would mix between two entries; detach() the Logger first")
        n = self._N
        with self._on_device():
            xy = self._plane[0, :, 0:2]
            lo, hi = xy.min(dim=0).values, xy.max(dim=0).values
            q = ((xy - lo) / (hi - lo).clamp_min(1e-12) * float((1 << bits) - 1)).to(torch.int64)

            def spread(v):
                v = v & 0xFFFF
                v = (v | (v << 8)) & 0x00FF00FF
                v = (v | (v << 4)) & 0x0F0F0F0F
                v = (v | (v << 2)) & 0x33333333
                v = (v | (v << 1)) & 0x55555555
                return v
            perm = torch.argsort(spread(q[:, 0]) | (spread(q[:, 1]) << 1), stable=True)      # new slot i <- old slot perm[i]
            self._plane.copy_(self._plane[:, perm].clone())
            self._wz.copy_(self._wz[perm].clone())
            # (_rpm_cmd and _action_dev are not permuted: they hold the caller's commands in drone-id order)
            for t in (self._last_rpm, self._pos_f32, self._obs_buf[0], self._obs_buf[1], self._dw_fz):
                if t is not None:
                    t.copy_(t[perm].clone())
            if self._pid is not None:
                self._pid.copy_(self._pid[:, perm].clone())
            for t in (self._init_pos, self._init_quat, self._target, self._reset_head):      # per-drone rows (E == 1: D == N)
                if t is not None and t.shape[0] == n:
                    t.copy_(t[perm].clone())
            self._order = perm if self._order is None else self._order[perm]
            self._inv = torch.empty_like(self._order)
            self._inv[self._order] = torch.arange(n, device=self.device)
        return self._order

    def step(self, action):
        """Advances every aviary by one control tick.

        Vector API: `action` is a float32 CUDA tensor [E, D, A] (used in place) or an ndarray (copied through a
        pinned buffer); returns tensors or ndarrays accordingly.  Single-env API: ndarray [D, A] in, the
        reference's 5-tuple out (BaseAviary.py:262-290)."""
        if self._py_hooks:
            return self._step_hooked(action)
        if type(action) is torch.Tensor and self.VECTORIZED and self._simple_launch:
            #### fast path: device tensor in, device tensors out, one kernel launch, no other device work ####
            a = action
            if a.numel() != self._N * self._A:
                raise ValueError("action must have %d x %d x %d elements, got shape %s" % (self._E, self._D, self._A, tuple(a.shape)))
            if a.dtype is not torch.float32 or a.device != self.device or not a.is_contiguous() or (a.data_ptr() & 15):
                self._action_dev.copy_(a.reshape(self._N, self._A))
                a = self._action_dev
            if torch.cuda.current_device() != self._dev_index:
                with self._on_device():
                    return self.step(action)
            io, cur = self._io, self._cur
            io.action = a.data_ptr()
            io.obs_prev = self._obs_ptr[cur]
            io.obs = self._obs_ptr[1 - cur]
            if self._gather is not None:
                self._gather.arm(io)
            stream = self._raw_stream(self._dev_index) if self._raw_stream else torch.cuda.current_stream().cuda_stream
            rc = self._qs_step_call(self._call_ptr, stream)
            if rc:
                N.check(rc, "qs_step")
            self._cur = cur = 1 - cur
            if self._log is not None:
                self._log_append()
            if self._final_view is None:
                return self._obs_view[cur], self._reward, self._terminated, self._truncated, {}
            return (self._obs_view[cur], self._reward, self._terminated, self._truncated,
                    {"final_obs": self._final_view, "_final_obs": self._done})
        with self._on_device():
            if isinstance(action, torch.Tensor) and action.dtype == torch.float64 and self._act_type() == N.ACT_RAW_RPM:
                #### float64 RPMs (e.g. DSLPIDControl.computeControlFromEnv): no float32 rounding on the way in ####
                if action.data_ptr() != self._rpm_cmd.data_ptr():
                    self._rpm_cmd.copy_(action.to(self.device).reshape(self._N, 4))
                obs = self._launch(self._rpm_cmd, f64=True)
                if not self.VECTORIZED:
                    return self._single_result(obs)
                return self._shape_obs(obs), self._reward, self._terminated, self._truncated, {}
            if isinstance(action, torch.Tensor):
                a = action
                if a.device != self.device or a.dtype != torch.float32:
                    a = a.to(device=self.device, dtype=torch.float32)
                a = a.reshape(self._N, self._A)
                if not a.is_contiguous() or (a.data_ptr() & 15):
                    self._action_dev.copy_(a)
                    a = self._action_dev
                obs = self._launch(a)
                if not self.VECTORIZED:
                    return self._single_result(obs)
                info = {}
                if self._final_obs is not None:
                    info = {"final_obs": self._by_id(self._final_obs).view(self._E, self._D, self._obs_dim), "_final_obs": self._done}
                return self._shape_obs(obs), self._reward, self._terminated, self._truncated, info
            #### NumPy path: pinned H2D of the action, D2H of the results, all inside this call ####
            if self._rpm_cmd is not None and isinstance(action, np.ndarray) and action.dtype == np.float64:
                # CtrlAviary with the reference's float64 RPM arrays (examples/pid.py:143): no float32 rounding on the way in
                self._rpm_cmd.copy_(torch.from_numpy(np.ascontiguousarray(action).reshape(self._N, 4)))
                return self.step(self._rpm_cmd)
            a_np = np.asarray(action, dtype=np.float32).reshape(self._N, self._A)
            if self._simple_launch:
                o, rew, term, trunc, info = self._step_host(a_np)
                if self.VECTORIZED:
                    return o, rew, term, trunc, info
                # single-env API of the reference: (obs[D, .], float, bool, bool, info)  (BaseAviary.py:376-383)
                return o[0], float(rew[0]), bool(term[0]), bool(trunc[0]), self._computeInfo()
            self._h_action.numpy()[...] = a_np
            self._action_dev.copy_(self._h_action, non_blocking=True)
            obs = self._launch(self._action_dev)
            if not self.VECTORIZED:
                return self._single_result(obs)
            k = self._hcur
            self._hcur = 1 - k
            h_obs, h_rew, h_te, h_tr = self._h_obs[k], self._h_reward[k], self._h_term[k], self._h_trunc[k]
            h_obs.copy_(self._by_id(obs), non_blocking=True)
            h_rew.copy_(self._reward, non_blocking=True)
            h_te.copy_(self._terminated, non_blocking=True)
            h_tr.copy_(self._truncated, non_blocking=True)
            torch.cuda.current_stream(self.device).synchronize()
            o = h_obs.numpy().reshape(self._E, self._D, self._obs_dim)
            rew, term, trunc = h_rew.numpy(), h_te.numpy(), h_tr.numpy()
            if self._host_copy:
                o, rew, term, trunc = o.copy(), rew.copy(), term.copy(), trunc.copy()
            return o, rew, term, trunc, {}

    def _step_host(self, a_np):
        """One qs_step_host call: every host<->device copy of the tick happens inside the C library."""
        k = self._hcur
        self._hcur = 1 - k
        io, cur, h = self._io, self._cur, self._hio[k]
        ptr = a_np.ctypes.data
        if ptr != self._h_action_ptr:
            if a_np.flags.c_contiguous and self._lib.qs_host_is_pinned(ptr):
                h.action_host = ptr                              # caller-owned page-locked array: no staging copy
            else:
                self._h_action_np[...] = a_np
                h.action_host = self._h_action_ptr
        else:
            h.action_host = ptr
        io.obs_prev = self._obs_ptr[cur]
        io.obs = self._obs_ptr[1 - cur]
        rc = self._lib.qs_step_host(*self._step_head[:3], C.byref(h), *self._step_head[3:], torch.cuda.current_stream().cuda_stream)
        if rc:
            N.check(rc, "qs_step_host")
        self._cur = 1 - cur
        if self._log is not None:
            self._log_append()
        o, rew, term, trunc = self._h_np[k]
        if self._h_head is not None:
            o = self._h_head[k].numpy().reshape(self._E, self._D, 12)
        info = {}
        if self._final_obs is not None:
            nf, idx, fin = self._h_fin_np[k]
            nd = int(nf[0])
            info = {"_final_obs": term | trunc}
            if nd:
                info["final_obs_env"] = idx[:nd]                                 # indices of the finished aviaries (ascending)
                info["final_obs"] = fin[:nd]                                     # their terminal observations [k, D, obs_dim]
        if self._host_copy:
            o, rew, term, trunc = o.copy(), rew.copy(), term.copy(), trunc.copy()
            if "final_obs" in info:
                info["final_obs"], info["final_obs_env"] = info["final_obs"].copy(), info["final_obs_env"].copy()
        return o, rew, term, trunc, info

    def _step_hooked(self, action):
        """step() when a user subclass overrides template-method hooks (BaseAviary.py:1021-1104): kernel tick, then the hooks."""
        numpy_in = not isinstance(action, torch.Tensor)
        with self._on_device():
            if self._hook_pre:                                 # raw-RPM envs: action -> RPMs (CtrlAviary.py:121-140)
                action = self._preprocessAction(action)
            f64 = self._rpm_cmd is not None and getattr(action, "dtype", None) in (np.float64, torch.float64)
            if f64:                                            # raw-RPM envs keep the reference's float64 RPMs
                a = action if isinstance(action, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(action))
                self._rpm_cmd.copy_(a.to(self.device).reshape(self._N, 4))
                self._launch(self._rpm_cmd, f64=True)
            else:
                a = action if isinstance(action, torch.Tensor) else torch.as_tensor(np.asarray(action, dtype=np.float32))
                self._action_dev.copy_(a.to(device=self.device, dtype=torch.float32).reshape(self._N, self._A))
                self._launch(self._action_dev)
            obs = self._computeObs()
            rew, term, trunc = self._computeReward(), self._computeTerminated(), self._computeTruncated()
            if not self.VECTORIZED:
                if isinstance(obs, torch.Tensor):
                    obs = obs.detach().cpu().numpy()
                to_f = lambda x: float(x.item()) if isinstance(x, torch.Tensor) else float(x)      # noqa: E731
                to_b = lambda x: bool(x.item()) if isinstance(x, torch.Tensor) else bool(x)        # noqa: E731
                return obs, to_f(rew), to_b(term), to_b(trunc), self._computeInfo()
            dev = self.device
            rew = torch.as_tensor(rew, device=dev).to(torch.float32).reshape(self._E)
            term = torch.as_tensor(term, device=dev).to(torch.bool).reshape(self._E)
            trunc = torch.as_tensor(trunc, device=dev).to(torch.bool).reshape(self._E)
            info = {}
            if self._py_autoreset:
                done = term | trunc
                info = {"final_obs": obs.clone() if isinstance(obs, torch.Tensor) else np.array(obs), "_final_obs": done}
                if bool(done.any()):
                    self._housekeeping(done.to(torch.uint8).contiguous())
                    obs = self._computeObs()
            if numpy_in:
                cv = lambda x: x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else x     # noqa: E731
                return cv(obs), cv(rew), cv(term), cv(trunc), {k: cv(v) for k, v in info.items()}
            return obs, rew, term, trunc, info

    def _single_result(self, obs):
        o = self._obs_to_host_single(obs)
        return (o, float(self._reward[0].item()), bool(self._terminated[0].item()), bool(self._truncated[0].item()),
                self._computeInfo())

    ################################################################################

    def render(self, mode='human', close=False):
        """Text printout of the first aviary (BaseAviary.py:387-412); there is no renderer."""
        st = self._getDroneStateVectors()[0]
        sc = int(self._step_counter[0].item())
        print("\n[INFO] BaseAviary.render() ——— it {:04d}".format(sc), "——— simulation time {:.1f}s".format(sc * self.PYB_TIMESTEP))
        for i in range(self.NUM_DRONES):
            s = st[i]
            print("[INFO] BaseAviary.render() ——— drone {:d}".format(i),
                  "——— x {:+06.2f}, y {:+06.2f}, z {:+06.2f}".format(s[0], s[1], s[2]),
                  "——— velocity {:+06.2f}, {:+06.2f}, {:+06.2f}".format(s[10], s[11], s[12]),
                  "——— roll {:+06.2f}, pitch {:+06.2f}, yaw {:+06.2f}".format(s[7] * self.RAD2DEG, s[8] * self.RAD2DEG, s[9] * self.RAD2DEG),
                  "——— angular velocity {:+06.4f}, {:+06.4f}, {:+06.4f} ——— ".format(s[13], s[14], s[15]))

    def close(self):
        """Nothing to disconnect (BaseAviary.py:416-421)."""

    def getPyBulletClient(self):
        """There is no PyBullet client; kept for API compatibility (BaseAviary.py:425-433)."""
        return -1

    def getDroneIds(self):
        return np.arange(self.NUM_DRONES)

    ################################################################################

    def _getDroneStateVectors(self):
        """[E, D, 20] float64 ndarray of _getDroneStateVector (BaseAviary.py:541-561), computed from the state planes."""
        pos, quat, vel = self._plane[0, :, 0:3], self._plane[1], self._plane[2, :, 0:3]
        rpy = euler_from_quaternion(quat)
        obs = self._obs_buf[self._cur]
        ang_v = obs[:, 13:16].double() if self._state20_obs() else obs[:, 9:12].double()      # (a KIN row can be 20 wide)
        sv = self._by_id(torch.cat([pos, quat, rpy, vel, ang_v, self._last_rpm], dim=1))
        return sv.view(self._E, self._D, 20).cpu().numpy()

    def _getDroneStateVector(self, nth_drone):
        return self._getDroneStateVectors()[0, nth_drone]

    def adjacency(self, out=None):
        """Neighbourhood query for every aviary: uint8 tensor [E, D, D], 1 where i == j or the drones are closer
        than NEIGHBOURHOOD_RADIUS (BaseAviary._getAdjacencyMatrix, BaseAviary.py:658-675).  Rows and columns are drone ids."""
        if out is None:
            out = torch.empty((self._E, self._D, self._D), dtype=torch.uint8, device=self.device)
        with self._on_device():
            N.check(self._lib.qs_adjacency(C.byref(self._st), self._E, self._D, float(self.NEIGHBOURHOOD_RADIUS),
                                           out.data_ptr(), self._stream()), "qs_adjacency")
            if self._inv is not None:                      # the kernel indexes storage slots (E == 1 after reorder_by_morton)
                out[0] = out[0][self._inv][:, self._inv]
        return out

    def _getAdjacencyMatrix(self):
        """BaseAviary._getAdjacencyMatrix (BaseAviary.py:658-675) for the first aviary: float64 ndarray [D, D]."""
        return self.adjacency()[0].cpu().numpy().astype(np.float64)

    ################################################################################
    # hooks (BaseAviary.py:1021-1104)

    def _actionSpace(self):
        raise NotImplementedError

    def _observationSpace(self):
        raise NotImplementedError

    def _computeObs(self):
        """Current observation, as the kernel wrote it (BaseAviary.py:1048-1056)."""
        obs = self._obs_buf[self._cur]
        return self._shape_obs(obs) if self.VECTORIZED else self._obs_to_host_single(obs)

    def _computeReward(self):
        """The kernel's reward of the last tick: [E] tensor, or a float for the single-env API (BaseAviary.py:1060-1068)."""
        return self._reward if self.VECTORIZED else float(self._reward[0].item())

    def _computeTerminated(self):
        return self._terminated if self.VECTORIZED else bool(self._terminated[0].item())

    def _computeTruncated(self):
        return self._truncated if self.VECTORIZED else bool(self._truncated[0].item())

    def _computeInfo(self):
        return {"answer": 42}


_ = spaces
