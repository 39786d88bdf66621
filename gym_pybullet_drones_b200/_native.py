"""ctypes binding of libquadsim.so (C ABI: include/quadsim.h).

The CUDA library is the product: if it is missing or does not load this module
raises -- there is no CPU or PyTorch fallback anywhere in the package.
"""
import ctypes as C
import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
LIB_PATH = os.environ.get("QS_LIBQUADSIM", os.path.join(_HERE, "libquadsim.so"))    # override: A/B builds in tools/
_CSRC = os.path.join(_HERE, "csrc")
SOURCES = [os.path.join(_CSRC, f) for f in ("quadsim.cu", "step_fast.cu", "step_general.cu", "rollout.cu", "rollout_next.cu", "rollout_mlp.cu", "rollout_ctrl.cu",
                                             "formation.cu", "mrac.cu", "dyn_traj.cu", "dyn_ctrl_traj.cu", "dyn_policy_traj.cu", "dyn_jvp.cu",
                                             "dyn_ctrl_jvp.cu", "dyn_policy_jvp.cu", "ilqr.cu")]
HEADERS = [os.path.join(_CSRC, "quad_core.cuh"), os.path.join(_CSRC, "mrac_core.cuh"), os.path.join(_CSRC, "dyn_adjoint.cuh"), os.path.join(_CSRC, "dyn_tangent.cuh"), os.path.join(_CSRC, "pid_adjoint.cuh"), os.path.join(_CSRC, "pid_tangent.cuh"), os.path.join(_CSRC, "ctrl_io.cuh"), os.path.join(_CSRC, "mlp_adjoint.cuh"), os.path.join(_CSRC, "mlp_tangent.cuh"), os.path.join(_CSRC, "policy_actor.cuh"), os.path.join(_CSRC, "traj_io.cuh"), os.path.join(_CSRC, "riccati.cuh"), os.path.join(_CSRC, "lqr_law.cuh"), os.path.join(_CSRC, "qs_common.cuh"), os.path.join(_CSRC, "rollout_kernel.cuh"),
           os.path.join(_ROOT, "include", "quadsim.h")]
OBJ_DIR = os.path.join(_ROOT, "build", "obj")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]      # H100 (Hopper)
# -fmad=false: every kernel that advances the state rounds each operation as written (fused only where the source says
# __fma_rn), so qs_rollout(T), T x qs_step and the fast and general step kernels give the same float64 bits; with contraction
# the compiler fuses differently per kernel (on sm_90a the PID step and rollout kernels drifted apart in the last bits)
NVCC_FLAGS = ARCH + ["-O3", "-lineinfo", "-std=c++17", "-fmad=false", "-Xcompiler", "-fPIC"]

# enums of include/quadsim.h
MODEL_CF2X, MODEL_CF2P, MODEL_RACE = 0, 1, 2
ACT_RPM, ACT_PID, ACT_VEL, ACT_ONE_D_RPM, ACT_ONE_D_PID, ACT_RAW_RPM = 0, 1, 2, 3, 4, 5
TASK_NONE, TASK_HOVER = 0, 1
EFFECT_GND, EFFECT_DRAG, EFFECT_DW = 1, 2, 4
FLAG_AUTORESET_SAME_STEP, FLAG_AUTORESET_NEXT_STEP, FLAG_RPY_F32 = 1, 2, 4
FLAG_AUTORESET_CLEARS_PID, FLAG_AUTORESET_CLEARS_HISTORY = 8, 16
FLAG_OBS_STATE20 = 32
FLAG_SKIP_EPILOGUE, FLAG_RPM_FROM_LAST, FLAG_ACTION_F64 = 0x100, 0x200, 0x400
CTRL_RAW, CTRL_VEL, CTRL_TRACK = 0, 1, 2          # qs_ctrl_rollout modes
CTRL_MRAC = 3                                     # qs_ctrl_rollout_mrac
CTRL_LQR = 4                                      # qs_ctrl_rollout_lqr
MRAC_STATE = 76                                   # doubles of one MRAC's adaptive state (Kx 48, Kr 16, Xm 12)
ABI_VERSION = 4
MLP_TANH, MLP_RELU = 0, 1                         # QsMlpPolicy.activation
MLP_MAX_HIDDEN, MLP_MAX_WIDTH = 4, 256
PHYS_WIDTH = 16          # float64 columns of one QsState.phys row

_d = C.c_double


class QsParams(C.Structure):
    _fields_ = [
        ("dt", _d), ("ctrl_dt", _d), ("pyb_freq", _d), ("m", _d), ("inv_m", _d), ("gravity", _d), ("kf", _d), ("km", _d),
        ("j", _d * 3), ("j_inv", _d * 3), ("hover_rpm", _d), ("max_rpm", _d),
        ("sx", _d * 4), ("sy", _d * 4), ("sz", _d * 4), ("kx", _d), ("ky", _d),
        ("gnd_eff_coeff", _d), ("prop_radius", _d), ("gnd_eff_h_clip", _d), ("prop_xyz", (_d * 3) * 4),
        ("drag_coeff", _d * 3), ("dw_coeff", _d * 3),
        ("episode_len_sec", _d), ("xy_bound", _d), ("z_bound", _d), ("tilt_bound", _d), ("term_dist", _d),
        ("speed_limit", _d),
        ("pid_p_for", _d * 3), ("pid_i_for", _d * 3), ("pid_d_for", _d * 3),
        ("pid_p_tor", _d * 3), ("pid_i_tor", _d * 3), ("pid_d_tor", _d * 3),
        ("pid_mixer", (_d * 3) * 4),
        ("pid_pwm2rpm_scale", _d), ("pid_pwm2rpm_const", _d), ("pid_min_pwm", _d), ("pid_max_pwm", _d),
        ("pid_gravity", _d), ("pid_kf", _d),
        ("drone_model", C.c_int), ("pad_", C.c_int),
    ]


class QsState(C.Structure):
    _fields_ = [
        ("planes", C.c_void_p), ("last_rpm", C.c_void_p), ("step_counter", C.c_void_p), ("pending_reset", C.c_void_p),
        ("pid", C.c_void_p), ("init_pos", C.c_void_p), ("init_quat", C.c_void_p), ("target_pos", C.c_void_p),
        ("reset_head", C.c_void_p), ("pos_f32", C.c_void_p), ("tables_per_env", C.c_int), ("pad_", C.c_int),
        ("phys", C.c_void_p),
    ]


class QsStepIO(C.Structure):
    _fields_ = [
        ("action", C.c_void_p), ("obs_prev", C.c_void_p), ("obs", C.c_void_p), ("reward", C.c_void_p),
        ("terminated", C.c_void_p), ("truncated", C.c_void_p), ("final_obs", C.c_void_p), ("done", C.c_void_p), ("dw_fz", C.c_void_p),
        ("act_buffer_size", C.c_int), ("tick_substeps", C.c_int),
        ("obs_gather", C.c_void_p), ("reward_gather", C.c_void_p), ("terminated_gather", C.c_void_p), ("truncated_gather", C.c_void_p),
        ("gather_flag", C.c_void_p), ("gather_counter", C.c_void_p), ("gather_seq", C.c_uint), ("pad_", C.c_uint),
        ("warp_ticket", C.c_void_p), ("warp_done", C.c_void_p), ("ready_err", C.c_void_p),
    ]


class QsRolloutIO(C.Structure):
    _fields_ = [
        ("actions", C.c_void_p), ("actions_out", C.c_void_p), ("obs_init", C.c_void_p), ("obs", C.c_void_p), ("obs_last", C.c_void_p),
        ("reward", C.c_void_p), ("terminated", C.c_void_p), ("truncated", C.c_void_p), ("done", C.c_void_p),
        ("seed", C.c_ulonglong), ("tick0", C.c_longlong), ("T", C.c_int), ("act_buffer_size", C.c_int), ("policy", C.c_void_p),
        ("final_obs", C.c_void_p), ("final_values", C.c_void_p),
    ]


class QsPolicy(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("w1", "b1", "w2", "b2", "w3", "b3", "log_std", "vw1", "vb1", "vw2", "vb2", "vw3", "vb3",
                                          "noise", "logprob", "values")] + [("in_dim", C.c_int), ("out_dim", C.c_int), ("nt3", C.c_int), ("pad_", C.c_int)]


class QsMlpNet(C.Structure):
    _fields_ = [("w", C.c_void_p * (MLP_MAX_HIDDEN + 1)), ("b", C.c_void_p * (MLP_MAX_HIDDEN + 1)), ("depth", C.c_int),
                ("width", C.c_int * MLP_MAX_HIDDEN), ("out_tiles", C.c_int)]


class QsMlpPolicy(C.Structure):
    _fields_ = [("actor", QsMlpNet), ("critic", QsMlpNet), ("activation", C.c_int), ("in_dim", C.c_int), ("out_dim", C.c_int),
                ("pad_", C.c_int), ("log_std", C.c_void_p), ("noise", C.c_void_p), ("logprob", C.c_void_p), ("values", C.c_void_p)]


class QsDwPublish(C.Structure):
    _fields_ = [("gathered", C.POINTER(C.c_void_p)), ("flags", C.POINTER(C.c_void_p)), ("counter", C.c_void_p),
                ("n_total", C.c_int), ("world", C.c_int), ("rank", C.c_int), ("offset", C.c_int), ("seq", C.c_uint), ("pad_", C.c_int)]


class QsHostIO(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("action_host", "obs_host", "reward_host", "terminated_host", "truncated_host", "done_host",
                                          "final_obs_host", "final_env_host", "n_final_host", "action_dev", "final_env_dev", "n_final_dev",
                                          "obs_head_host", "side_stream", "ev_fork", "ev_join")]


class QsLogRing(C.Structure):
    _fields_ = [("ring", C.c_void_p), ("head", C.c_void_p), ("capacity", C.c_int), ("first_drone", C.c_int), ("n_drones", C.c_int), ("kin_rows", C.c_int)]


class QsCtrlRolloutIO(C.Structure):
    _fields_ = [("T", C.c_int), ("log_targets", C.c_int), ("actions", C.c_void_p),
                ("ctrl_params", C.c_void_p), ("pid_state", C.c_void_p), ("control_timestep", C.c_double),
                ("waypoints", C.c_void_p), ("W", C.c_int), ("M", C.c_int), ("start", C.c_void_p), ("offset", C.c_void_p),
                ("target_rpy", C.c_void_p), ("target_vel", C.c_void_p), ("target_rpy_rates", C.c_void_p),
                ("obs", C.c_void_p), ("rpm", C.c_void_p), ("pos_e", C.c_void_p), ("yaw_e", C.c_void_p), ("obs_last", C.c_void_p),
                ("log", C.c_void_p), ("log_controls", C.c_void_p)]


class QsMracParams(C.Structure):
    _fields_ = [("Am", (_d * 12) * 12), ("bm", _d * 4), ("PBm", (_d * 4) * 12), ("Kr_ref", (_d * 12) * 4),
                ("gamma_x", _d), ("gamma_r", _d), ("mixer", (_d * 3) * 4),
                ("kf", _d), ("pwm2rpm_scale", _d), ("pwm2rpm_const", _d), ("min_pwm", _d), ("max_pwm", _d), ("max_rpm", _d)]


class QsMracRolloutIO(C.Structure):
    _fields_ = [("params", C.c_void_p), ("state", C.c_void_p), ("init", C.c_int), ("pad_", C.c_int), ("rpy_e", C.c_void_p)]


class QsLqrRolloutIO(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("K", "z_nom", "rpm_nom", "lo", "hi")] + [
        ("per_tick", C.c_int), ("n_z", C.c_int), ("T_plan", C.c_int), ("tick0", C.c_int)]


class QsDynTrajIO(C.Structure):
    _fields_ = [("T", C.c_int), ("pad_", C.c_int)] + [(n, C.c_void_p) for n in (
        "state0", "rpm", "last_rpm", "phys", "states", "g_states", "g_rpm", "g_state0", "g_last_rpm", "g_phys", "scratch")]


class QsDynTrajJvpIO(C.Structure):
    _fields_ = [("T", C.c_int), ("pad_", C.c_int)] + [(n, C.c_void_p) for n in (
        "state0", "rpm", "last_rpm", "phys", "states", "t_state0", "t_rpm", "t_last_rpm", "t_phys", "t_states", "jac")]


class QsDynCtrlTrajIO(C.Structure):
    _fields_ = [("T", C.c_int), ("pad_", C.c_int), ("control_timestep", C.c_double)] + [(n, C.c_void_p) for n in (
        "state0", "pid0", "target_pos", "target_vel", "target_rpy", "target_rpy_rates", "last_rpm", "phys", "gains",
        "states", "rpm", "pid_states", "g_states", "g_rpm_out", "g_state0", "g_pid0", "g_target_pos", "g_target_vel",
        "g_target_rpy", "g_target_rpy_rates", "g_last_rpm", "g_phys", "g_gains", "scratch")]


class QsDynCtrlTrajJvpIO(C.Structure):
    _fields_ = [("T", C.c_int), ("pad_", C.c_int), ("control_timestep", C.c_double)] + [(n, C.c_void_p) for n in (
        "state0", "pid0", "target_pos", "target_vel", "target_rpy", "target_rpy_rates", "last_rpm", "phys", "gains",
        "states", "rpm", "pid_states", "t_state0", "t_pid0", "t_target_pos", "t_target_vel", "t_target_rpy", "t_target_rpy_rates",
        "t_last_rpm", "t_phys", "t_gains", "t_states", "t_rpm", "jac")]


class QsDynPolicyTrajIO(C.Structure):
    _fields_ = [("T", C.c_int), ("act_buffer_size", C.c_int), ("activation", C.c_int), ("depth", C.c_int),
                ("width", C.c_int * MLP_MAX_HIDDEN), ("in_dim", C.c_int), ("out_dim", C.c_int),
                ("w", C.c_void_p * (MLP_MAX_HIDDEN + 1)), ("b", C.c_void_p * (MLP_MAX_HIDDEN + 1))] + [(n, C.c_void_p) for n in (
        "log_std", "noise", "state0", "last_rpm", "phys", "action_buffer", "states", "actions", "obs", "g_states", "g_actions",
        "g_raw", "g_state0", "g_last_rpm", "g_phys", "g_action_buffer", "scratch")]


class QsDynPolicyTrajJvpIO(C.Structure):
    _fields_ = [("T", C.c_int), ("act_buffer_size", C.c_int), ("activation", C.c_int), ("depth", C.c_int),
                ("width", C.c_int * MLP_MAX_HIDDEN), ("in_dim", C.c_int), ("out_dim", C.c_int),
                ("w", C.c_void_p * (MLP_MAX_HIDDEN + 1)), ("b", C.c_void_p * (MLP_MAX_HIDDEN + 1))] + [(n, C.c_void_p) for n in (
        "log_std", "noise", "state0", "last_rpm", "phys", "action_buffer", "states", "actions", "obs", "t_state0", "t_last_rpm",
        "t_phys", "t_action_buffer", "t_raw_in", "t_states", "t_actions", "jac")]


class QsIlqrIO(C.Structure):
    _fields_ = [("T", C.c_int), ("n_alpha", C.c_int)] + [(n, C.c_void_p) for n in (
        "jac", "state0", "last_rpm", "phys", "targets", "weights", "rpm_ref", "alpha", "states", "rpm", "mu", "K", "k", "dV", "J",
        "status", "converged", "cost_in", "cost_out")]


class QsIlqrBoxIO(C.Structure):
    _fields_ = [("base", QsIlqrIO), ("rpm_lo", C.c_void_p), ("rpm_hi", C.c_void_p), ("per_tick", C.c_int), ("pad_", C.c_int),
                ("active", C.c_void_p)]


class QsStepCall(C.Structure):
    _fields_ = [("p", C.c_void_p), ("st", C.c_void_p), ("io", C.c_void_p),
                ("act_type", C.c_int), ("task", C.c_int), ("n_envs", C.c_int), ("drones_per_env", C.c_int), ("substeps", C.c_int),
                ("effects", C.c_uint), ("flags", C.c_uint), ("pad_", C.c_int)]


EXPORTS = ["qs_abi_version", "qs_last_error", "qs_sizeof_params", "qs_sizeof_state", "qs_sizeof_step_io",
           "qs_sizeof_rollout_io", "qs_sizeof_host_io", "qs_step", "qs_step_call", "qs_step_host", "qs_rollout", "qs_rollout_max_ticks", "qs_dyn_substeps", "qs_dyn_substeps_pub", "qs_pid_control",
           "qs_downwash", "qs_downwash_boxed", "qs_dw_gathered_floats", "qs_dw_boxes", "qs_downwash_rows", "qs_dw_publish", "qs_enable_peer_access", "qs_ipc_export", "qs_ipc_import", "qs_adjacency", "qs_reset", "qs_reset_heads", "qs_host_is_pinned", "qs_log_append", "qs_sizeof_log_ring", "qs_wait_flags", "qs_pid_control_state",
           "qs_ctrl_rollout", "qs_sizeof_ctrl_rollout_io", "qs_rollout_mlp", "qs_rollout_mlp_max_ticks", "qs_sizeof_mlp_policy",
           "qs_mrac_control", "qs_mrac_control_state", "qs_ctrl_rollout_mrac", "qs_sizeof_mrac_params", "qs_sizeof_mrac_rollout_io",
           "qs_dyn_traj", "qs_dyn_traj_vjp", "qs_sizeof_dyn_traj_io", "qs_dyn_ctrl_traj", "qs_dyn_ctrl_traj_vjp",
           "qs_sizeof_dyn_ctrl_traj_io", "qs_dyn_policy_traj", "qs_dyn_policy_traj_vjp", "qs_sizeof_dyn_policy_traj_io",
           "qs_dyn_traj_jvp", "qs_dyn_tick_jac", "qs_sizeof_dyn_traj_jvp_io", "qs_dyn_ctrl_traj_jvp", "qs_dyn_ctrl_tick_jac",
           "qs_sizeof_dyn_ctrl_traj_jvp_io", "qs_dyn_policy_traj_jvp", "qs_dyn_policy_tick_jac", "qs_sizeof_dyn_policy_traj_jvp_io",
           "qs_ilqr_backward", "qs_ilqr_line_search", "qs_ilqr_commit", "qs_sizeof_ilqr_io", "qs_ilqr_box_backward",
           "qs_ilqr_box_line_search", "qs_ilqr_box_commit", "qs_sizeof_ilqr_box_io", "qs_ctrl_rollout_lqr",
           "qs_sizeof_lqr_rollout_io"]
MAX_PEERS = 16


def build(force=False, verbose=False):
    """Compile libquadsim.so in-tree for sm_90a with nvcc (no torch headers): one object per translation unit, compiled
    in parallel and only when its source or a header changed, then linked into the shared library."""
    from concurrent.futures import ThreadPoolExecutor
    newest_hdr = max(os.path.getmtime(p) for p in HEADERS)
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.isfile(nvcc):
        if not force and os.path.isfile(LIB_PATH):
            return LIB_PATH
        raise RuntimeError("nvcc not found: cannot build libquadsim.so")
    os.makedirs(OBJ_DIR, exist_ok=True)
    objs, jobs = [], []
    for src in SOURCES:
        obj = os.path.join(OBJ_DIR, os.path.splitext(os.path.basename(src))[0] + ".o")
        objs.append(obj)
        if force or not os.path.isfile(obj) or os.path.getmtime(obj) < max(newest_hdr, os.path.getmtime(src)):
            jobs.append([nvcc] + NVCC_FLAGS + ["-c", "-o", obj, src])
    if not jobs and os.path.isfile(LIB_PATH) and os.path.getmtime(LIB_PATH) >= max(os.path.getmtime(o) for o in objs):
        return LIB_PATH

    def run(cmd):
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("nvcc failed:\n%s\n%s" % (" ".join(cmd), res.stderr))
        return res.stderr

    with ThreadPoolExecutor(max_workers=max(1, min(len(jobs), os.cpu_count() or 1))) as ex:
        logs = list(ex.map(run, jobs))
    logs.append(run([nvcc, "-shared"] + ARCH + ["-o", LIB_PATH] + objs))
    if verbose:
        print("\n".join(l for l in logs if l))
    return LIB_PATH


_lib = None


def lib():
    """Loads (once) and returns the CUDA library.  Raises if it is not built: no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise ImportError("libquadsim.so is not built (%s).  Run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "or gym_pybullet_drones_b200._native.build().  There is no CPU fallback." % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    L.qs_abi_version.restype = C.c_int
    L.qs_last_error.restype = C.c_char_p
    for n in ("qs_sizeof_params", "qs_sizeof_state", "qs_sizeof_step_io", "qs_sizeof_rollout_io"):
        getattr(L, n).restype = C.c_int
    L.qs_step.restype = C.c_int
    L.qs_step.argtypes = [C.POINTER(QsParams), C.POINTER(QsState), C.POINTER(QsStepIO), C.c_int, C.c_int,
                          C.c_int, C.c_int, C.c_int, C.c_uint, C.c_uint, C.c_void_p]
    L.qs_step_call.restype = C.c_int
    L.qs_step_call.argtypes = [C.c_void_p, C.c_void_p]
    L.qs_step_host.restype = C.c_int
    L.qs_step_host.argtypes = [C.POINTER(QsParams), C.POINTER(QsState), C.POINTER(QsStepIO), C.POINTER(QsHostIO), C.c_int, C.c_int,
                               C.c_int, C.c_int, C.c_int, C.c_uint, C.c_uint, C.c_void_p]
    L.qs_sizeof_host_io.restype = C.c_int
    L.qs_host_is_pinned.restype = C.c_int
    L.qs_host_is_pinned.argtypes = [C.c_void_p]
    L.qs_rollout.restype = C.c_int
    L.qs_rollout.argtypes = [C.POINTER(QsParams), C.POINTER(QsState), C.POINTER(QsRolloutIO), C.c_int, C.c_int,
                             C.c_int, C.c_int, C.c_int, C.c_uint, C.c_uint, C.c_void_p]
    L.qs_rollout_max_ticks.restype = C.c_int
    L.qs_rollout_max_ticks.argtypes = [C.c_int, C.c_int, C.c_int]
    L.qs_rollout_mlp.restype = C.c_int
    L.qs_rollout_mlp.argtypes = [C.POINTER(QsParams), C.POINTER(QsState), C.POINTER(QsRolloutIO), C.POINTER(QsMlpPolicy), C.c_int, C.c_int,
                                 C.c_int, C.c_int, C.c_int, C.c_uint, C.c_uint, C.c_void_p]
    L.qs_rollout_mlp_max_ticks.restype = C.c_int
    L.qs_rollout_mlp_max_ticks.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int]
    L.qs_sizeof_mlp_policy.restype = C.c_int
    L.qs_ctrl_rollout.restype = C.c_int
    L.qs_ctrl_rollout.argtypes = [C.POINTER(QsParams), C.POINTER(QsState), C.POINTER(QsCtrlRolloutIO), C.c_int, C.c_int, C.c_int,
                                  C.c_int, C.c_uint, C.c_uint, C.c_void_p]
    L.qs_sizeof_ctrl_rollout_io.restype = C.c_int
    L.qs_ctrl_rollout_mrac.restype = C.c_int
    L.qs_ctrl_rollout_mrac.argtypes = [C.POINTER(QsParams), C.POINTER(QsState), C.POINTER(QsCtrlRolloutIO), C.POINTER(QsMracRolloutIO),
                                       C.c_int, C.c_int, C.c_int, C.c_uint, C.c_uint, C.c_void_p]
    L.qs_mrac_control.restype = C.c_int
    L.qs_mrac_control.argtypes = [C.POINTER(QsMracParams), C.c_void_p, C.c_int, C.c_double] + [C.c_void_p] * 8 + \
        [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.qs_mrac_control_state.restype = C.c_int
    L.qs_mrac_control_state.argtypes = [C.POINTER(QsMracParams), C.c_void_p, C.c_int, C.c_double, C.POINTER(QsState), C.c_int] + \
        [C.c_void_p] * 8
    L.qs_sizeof_mrac_params.restype = C.c_int
    L.qs_sizeof_mrac_rollout_io.restype = C.c_int
    L.qs_ctrl_rollout_lqr.restype = C.c_int
    L.qs_ctrl_rollout_lqr.argtypes = [C.POINTER(QsParams), C.POINTER(QsState), C.POINTER(QsCtrlRolloutIO), C.POINTER(QsLqrRolloutIO),
                                      C.c_int, C.c_int, C.c_int, C.c_uint, C.c_uint, C.c_void_p]
    L.qs_sizeof_lqr_rollout_io.restype = C.c_int
    for n in ("qs_dyn_traj", "qs_dyn_traj_vjp"):
        getattr(L, n).restype = C.c_int
        getattr(L, n).argtypes = [C.POINTER(QsParams), C.POINTER(QsDynTrajIO), C.c_int, C.c_int, C.c_int, C.c_uint, C.c_void_p]
    L.qs_sizeof_dyn_traj_io.restype = C.c_int
    for n in ("qs_dyn_traj_jvp", "qs_dyn_tick_jac"):
        getattr(L, n).restype = C.c_int
        getattr(L, n).argtypes = [C.POINTER(QsParams), C.POINTER(QsDynTrajJvpIO), C.c_int, C.c_int, C.c_int, C.c_uint, C.c_void_p]
    L.qs_sizeof_dyn_traj_jvp_io.restype = C.c_int
    for n in ("qs_dyn_ctrl_traj", "qs_dyn_ctrl_traj_vjp"):
        getattr(L, n).restype = C.c_int
        getattr(L, n).argtypes = [C.POINTER(QsParams), C.POINTER(QsParams), C.POINTER(QsDynCtrlTrajIO), C.c_int, C.c_int, C.c_int,
                                  C.c_uint, C.c_void_p]
    L.qs_sizeof_dyn_ctrl_traj_io.restype = C.c_int
    for n in ("qs_dyn_ctrl_traj_jvp", "qs_dyn_ctrl_tick_jac"):
        getattr(L, n).restype = C.c_int
        getattr(L, n).argtypes = [C.POINTER(QsParams), C.POINTER(QsParams), C.POINTER(QsDynCtrlTrajJvpIO), C.c_int, C.c_int, C.c_int,
                                  C.c_uint, C.c_void_p]
    L.qs_sizeof_dyn_ctrl_traj_jvp_io.restype = C.c_int
    for n in ("qs_dyn_policy_traj", "qs_dyn_policy_traj_vjp"):
        getattr(L, n).restype = C.c_int
        getattr(L, n).argtypes = [C.POINTER(QsParams), C.POINTER(QsDynPolicyTrajIO), C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint,
                                  C.c_void_p]
    L.qs_sizeof_dyn_policy_traj_io.restype = C.c_int
    for n in ("qs_dyn_policy_traj_jvp", "qs_dyn_policy_tick_jac"):
        getattr(L, n).restype = C.c_int
        getattr(L, n).argtypes = [C.POINTER(QsParams), C.POINTER(QsDynPolicyTrajJvpIO), C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint,
                                  C.c_void_p]
    L.qs_sizeof_dyn_policy_traj_jvp_io.restype = C.c_int
    for n in ("qs_ilqr_backward", "qs_ilqr_line_search", "qs_ilqr_commit"):
        getattr(L, n).restype = C.c_int
        getattr(L, n).argtypes = [C.POINTER(QsParams), C.POINTER(QsIlqrIO), C.c_int, C.c_int, C.c_int, C.c_uint, C.c_void_p]
    L.qs_sizeof_ilqr_io.restype = C.c_int
    for n in ("qs_ilqr_box_backward", "qs_ilqr_box_line_search", "qs_ilqr_box_commit"):
        getattr(L, n).restype = C.c_int
        getattr(L, n).argtypes = [C.POINTER(QsParams), C.POINTER(QsIlqrBoxIO), C.c_int, C.c_int, C.c_int, C.c_uint, C.c_void_p]
    L.qs_sizeof_ilqr_box_io.restype = C.c_int
    L.qs_dyn_substeps.restype = C.c_int
    L.qs_dyn_substeps.argtypes = [C.POINTER(QsParams), C.POINTER(QsState), C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_int, C.c_int, C.c_int, C.c_uint, C.c_uint, C.c_void_p]
    L.qs_dyn_substeps_pub.restype = C.c_int
    L.qs_dyn_substeps_pub.argtypes = [C.POINTER(QsParams), C.POINTER(QsState), C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_int, C.c_int, C.c_int, C.c_uint, C.c_uint, C.POINTER(QsDwPublish), C.c_void_p]
    L.qs_pid_control.restype = C.c_int
    L.qs_pid_control.argtypes = [C.POINTER(QsParams), C.c_void_p, C.c_double,
                                 C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.qs_pid_control_state.restype = C.c_int
    L.qs_pid_control_state.argtypes = [C.POINTER(QsParams), C.c_void_p, C.c_double, C.POINTER(QsState), C.c_int,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.qs_downwash.restype = C.c_int
    L.qs_downwash.argtypes = [C.POINTER(QsParams), C.POINTER(QsState), C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.qs_downwash_boxed.restype = C.c_int
    L.qs_downwash_boxed.argtypes = [C.POINTER(QsParams), C.POINTER(QsState), C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.qs_dw_gathered_floats.restype = C.c_longlong
    L.qs_dw_gathered_floats.argtypes = [C.c_int]
    L.qs_dw_boxes.restype = C.c_int
    L.qs_dw_boxes.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.qs_downwash_rows.restype = C.c_int
    L.qs_downwash_rows.argtypes = [C.POINTER(QsParams), C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_uint, C.c_int,
                                   C.c_void_p, C.c_void_p, C.c_void_p]
    L.qs_dw_publish.restype = C.c_int
    L.qs_dw_publish.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.c_int, C.POINTER(C.c_void_p), C.c_int, C.c_int,
                                C.c_uint, C.c_void_p, C.c_void_p]
    L.qs_enable_peer_access.restype = C.c_int
    L.qs_enable_peer_access.argtypes = [C.c_int]
    L.qs_ipc_export.restype = C.c_int
    L.qs_ipc_export.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_ulonglong)]
    L.qs_ipc_import.restype = C.c_int
    L.qs_ipc_import.argtypes = [C.c_void_p, C.c_ulonglong, C.POINTER(C.c_void_p)]
    L.qs_adjacency.restype = C.c_int
    L.qs_adjacency.argtypes = [C.POINTER(QsState), C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p]
    L.qs_reset_heads.restype = C.c_int
    L.qs_reset_heads.argtypes = [C.POINTER(QsState), C.c_int, C.c_uint, C.c_void_p, C.c_void_p]
    L.qs_wait_flags.restype = C.c_int
    L.qs_wait_flags.argtypes = [C.c_void_p, C.c_uint, C.c_int, C.c_void_p, C.c_void_p]
    L.qs_log_append.restype = C.c_int
    L.qs_log_append.argtypes = [C.POINTER(QsParams), C.POINTER(QsState), C.c_void_p, C.c_int, C.c_void_p, C.POINTER(QsLogRing),
                                C.c_int, C.c_int, C.c_void_p]
    L.qs_sizeof_log_ring.restype = C.c_int
    L.qs_reset.restype = C.c_int
    L.qs_reset.argtypes = [C.POINTER(QsParams), C.POINTER(QsState), C.c_void_p, C.c_int, C.c_int,
                           C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    if L.qs_abi_version() != ABI_VERSION:
        raise ImportError("libquadsim.so ABI %d != binding ABI %d: rebuild" % (L.qs_abi_version(), ABI_VERSION))
    if (L.qs_sizeof_params(), L.qs_sizeof_state(), L.qs_sizeof_step_io(), L.qs_sizeof_rollout_io()) != \
            (C.sizeof(QsParams), C.sizeof(QsState), C.sizeof(QsStepIO), C.sizeof(QsRolloutIO)):
        raise ImportError("libquadsim.so struct layout differs from the ctypes mirror: rebuild")
    if L.qs_sizeof_log_ring() != C.sizeof(QsLogRing) or L.qs_sizeof_host_io() != C.sizeof(QsHostIO) or \
            L.qs_sizeof_ctrl_rollout_io() != C.sizeof(QsCtrlRolloutIO) or L.qs_sizeof_mlp_policy() != C.sizeof(QsMlpPolicy) or \
            L.qs_sizeof_mrac_params() != C.sizeof(QsMracParams) or L.qs_sizeof_mrac_rollout_io() != C.sizeof(QsMracRolloutIO) or \
            L.qs_sizeof_dyn_traj_io() != C.sizeof(QsDynTrajIO) or L.qs_sizeof_dyn_ctrl_traj_io() != C.sizeof(QsDynCtrlTrajIO) or \
            L.qs_sizeof_dyn_policy_traj_io() != C.sizeof(QsDynPolicyTrajIO) or L.qs_sizeof_dyn_traj_jvp_io() != C.sizeof(QsDynTrajJvpIO) or \
            L.qs_sizeof_dyn_ctrl_traj_jvp_io() != C.sizeof(QsDynCtrlTrajJvpIO) or \
            L.qs_sizeof_dyn_policy_traj_jvp_io() != C.sizeof(QsDynPolicyTrajJvpIO):
        raise ImportError("libquadsim.so struct layout differs from the ctypes mirror (log ring / host io / ctrl rollout io / mlp policy / mrac / "
                          "dyn traj io / dyn ctrl traj io / dyn policy traj io / dyn traj jvp io / dyn ctrl traj jvp io / "
                          "dyn policy traj jvp io): rebuild")
    if L.qs_sizeof_ilqr_io() != C.sizeof(QsIlqrIO) or L.qs_sizeof_ilqr_box_io() != C.sizeof(QsIlqrBoxIO):
        raise ImportError("libquadsim.so struct layout differs from the ctypes mirror (ilqr io / ilqr box io): rebuild")
    if L.qs_sizeof_lqr_rollout_io() != C.sizeof(QsLqrRolloutIO):
        raise ImportError("libquadsim.so struct layout differs from the ctypes mirror (lqr rollout io): rebuild")
    _lib = L
    return L


def check(rc, what):
    """Maps the C-ABI error convention to exceptions (the reference prints '[ERROR]' and exit()s)."""
    if rc == 0:
        return
    msg = lib().qs_last_error().decode()
    if rc < 0:
        raise ValueError("%s: %s (QS_ERR %d)" % (what, msg, rc))
    raise RuntimeError("%s: CUDA error %d: %s" % (what, rc, msg))
