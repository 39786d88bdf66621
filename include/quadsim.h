/*
 * quadsim.h -- C ABI of the H100-native vectorised quadrotor simulator (libquadsim.so).
 *
 * The reference (utiasDSL/gym-pybullet-drones) is pure Python and has no FFI; this ABI is the
 * drop-in boundary for its Physics.DYN hot path.  Each entry point names the reference
 * interface it replaces (paths relative to gym_pybullet_drones/ in the reference tree):
 *
 *   qs_step          <- BaseAviary.step (envs/BaseAviary.py:259-383) for BaseRLAviary envs:
 *                       _preprocessAction (envs/BaseRLAviary.py:160-239), S x _dynamics
 *                       (envs/BaseAviary.py:815-892), _computeObs KIN (envs/BaseRLAviary.py:307-319),
 *                       Hover/MultiHover reward/terminated/truncated (envs/HoverAviary.py:68-117,
 *                       envs/MultiHoverAviary.py:75-130)
 *   qs_dyn_substeps  <- CtrlAviary step: clip (envs/CtrlAviary.py:121-140) + S x _dynamics +
 *                       _getDroneStateVector (envs/BaseAviary.py:541-561)
 *   qs_pid_control   <- DSLPIDControl.computeControl (control/DSLPIDControl.py:82-259) and
 *                       BaseControl.computeControlFromState (control/BaseControl.py:55-93)
 *   qs_downwash      <- BaseAviary._downwash (envs/BaseAviary.py:785-811), pairwise term
 *   qs_downwash_rows / qs_dw_publish <- the same loop for one formation sharded over GPUs (rows = local drones)
 *   qs_adjacency     <- BaseAviary._getAdjacencyMatrix (envs/BaseAviary.py:658-675)
 *   qs_reset         <- BaseAviary.reset/_housekeeping (envs/BaseAviary.py:220-255,451-505)
 *   qs_log_append    <- Logger.log (utils/Logger.py:83-119): one entry per logged drone and tick, kept on the device
 *   qs_ctrl_rollout  <- T ticks of the CtrlAviary / VelocityAviary loops (examples/pid.py:131-150, pid_velocity.py, downwash.py)
 *
 * Conventions
 *   - plain C, no CUDA/torch types: device buffers are raw pointers owned by the caller; the
 *     library allocates nothing persistent and keeps no global state but a thread-local error
 *     string.  "planes" pointers must be 16-byte aligned.
 *   - every call is asynchronous: it enqueues on `stream` (a cudaStream_t passed as void*) and
 *     returns; safe under CUDA-graph capture.
 *   - return value: 0 = ok; <0 = argument error (QS_ERR_*); >0 = cudaError_t of the launch.
 *     qs_last_error() gives a message for the last non-zero return on the calling thread.
 *   - arithmetic: the persistent state is float64 in HBM and is advanced in float64 registers, like the
 *     reference (numpy float64 + Bullet doubles); actions and observations are float32 (the reference casts its
 *     observations to float32, BaseRLAviary.py:315).  See DESIGN.md.
 */
#ifndef QUADSIM_H_
#define QUADSIM_H_

#ifdef __cplusplus
extern "C" {
#endif

#define QS_ABI_VERSION 4     /* 2: the persistent state (planes, last_rpm, pid, init/target tables) is float64;
                                3: QsStepIO.pdl_hint replaced by the per-warp readiness words;
                                4: QsState.phys, per-aviary physical constants */

/* drone models (utils/enums.py:3-9) */
enum { QS_MODEL_CF2X = 0, QS_MODEL_CF2P = 1, QS_MODEL_RACE = 2 };

/* action types (utils/enums.py:33-39); QS_ACT_RAW_RPM is CtrlAviary's clipped raw RPM */
enum { QS_ACT_RPM = 0, QS_ACT_PID = 1, QS_ACT_VEL = 2, QS_ACT_ONE_D_RPM = 3, QS_ACT_ONE_D_PID = 4, QS_ACT_RAW_RPM = 5 };

/* task (reward / termination rule) */
enum { QS_TASK_NONE = 0,        /* CtrlAviary: reward -1, never done (envs/CtrlAviary.py:144-200) */
       QS_TASK_HOVER = 1 };     /* Hover/MultiHover: sum_d max(0, 2-|e_d|^4), sum_d |e_d| < 1e-4, bounds/tilt/time-out */

/* DYN+ aerodynamic terms: the reference's PYB_* force models restated as explicit forces (DESIGN.md) */
enum { QS_EFFECT_GND = 1, QS_EFFECT_DRAG = 2, QS_EFFECT_DW = 4 };

/* qs_step flags */
enum { QS_FLAG_AUTORESET_SAME_STEP = 1,   /* SB3 VecEnv semantics: done envs are reset inside the step; the
                                             terminal observation goes to QsStepIO.final_obs */
       QS_FLAG_AUTORESET_NEXT_STEP = 2,   /* gymnasium>=1.0 default: a done env is reset by the NEXT step call,
                                             which ignores that env's action */
       QS_FLAG_RPY_F32 = 4,               /* evaluate the output roll/pitch/yaw with float32 atan2/asin; decisions (tilt
                                             truncation) and reset observations still use float64 angles */
       /* The reference's reset() clears neither the embedded PID controllers nor the action buffer
          (SURVEY.md 3.3); autoreset keeps that behaviour unless asked otherwise: */
       QS_FLAG_AUTORESET_CLEARS_PID = 8,
       QS_FLAG_AUTORESET_CLEARS_HISTORY = 16,
       QS_FLAG_OBS_STATE20 = 32,          /* qs_step writes [N][20] _getDroneStateVector rows instead of KIN observations (no action
                                             buffer, task must be QS_TASK_NONE): VelocityAviary = act VEL + this flag */
       /* Split-substep protocol for aviaries larger than one CTA with downwash (positions couple the drones
          every substep, so each substep is its own launch: qs_downwash, then qs_step(substeps=1)):
          all but the last launch of a tick pass SKIP_EPILOGUE (no obs/reward/flags/counter); all but the first
          pass RPM_FROM_LAST (the rpm decoded by the first launch is re-read from QsState.last_rpm). */
       QS_FLAG_SKIP_EPILOGUE = 0x100,
       QS_FLAG_RPM_FROM_LAST = 0x200,
       QS_FLAG_ACTION_F64 = 0x400 };      /* qs_dyn_substeps: `rpm` points to float64 [N][4] (32-byte aligned), e.g. the output of
                                             qs_pid_control_state: the reference's float64 RPMs without a float32 rounding */

enum { QS_ERR_NULL = -1, QS_ERR_ALIGN = -2, QS_ERR_SIZE = -3, QS_ERR_ENUM = -4, QS_ERR_UNSUPPORTED = -5 };

/* Physical + task constants.  All double: filled by the host exactly as BaseAviary.__init__ does
 * (envs/BaseAviary.py:74-128) and passed by value into the launch (kernel constant bank). */
typedef struct QsParams {
    double dt;             /* PYB_TIMESTEP = 1/pyb_freq                      BaseAviary.py:83 */
    double ctrl_dt;        /* CTRL_TIMESTEP = 1/ctrl_freq                    BaseAviary.py:82 */
    double pyb_freq;       /* PYB_FREQ (for the time-out test)               HoverAviary.py:113 */
    double m;              /* M                                              cf2x.urdf:11 */
    double inv_m;          /* 1/M (host-computed; the kernels multiply instead of dividing, BaseAviary.py:858) */
    double gravity;        /* GRAVITY = G*M                                  BaseAviary.py:117 */
    double kf, km;         /* KF, KM                                         cf2x.urdf:5 */
    double j[3];           /* diag(J)                                        cf2x.urdf:12 */
    double j_inv[3];       /* diag(J^-1)                                     BaseAviary.py:1000 */
    double hover_rpm;      /* HOVER_RPM                                      BaseAviary.py:118 */
    double max_rpm;        /* MAX_RPM                                        BaseAviary.py:119 */
    /* torque mixing of _dynamics (BaseAviary.py:842-854): tau_x = kx * sum_i sx[i] f_i etc.; sz carries RACE's sign flip */
    double sx[4], sy[4], sz[4];
    double kx, ky;
    /* ground effect (BaseAviary.py:715-750) */
    double gnd_eff_coeff, prop_radius, gnd_eff_h_clip;
    double prop_xyz[4][3]; /* propeller link COM offsets                      cf2x.urdf:42,54,66,78 */
    /* drag (BaseAviary.py:754-781), downwash (BaseAviary.py:785-811) */
    double drag_coeff[3];
    double dw_coeff[3];
    /* task constants (HoverAviary.py:51-52,109-115; MultiHoverAviary.py:123-129) */
    double episode_len_sec, xy_bound, z_bound, tilt_bound, term_dist;
    /* BaseRLAviary VEL action (BaseRLAviary.py:95) */
    double speed_limit;
    /* DSLPIDControl gains/constants (control/DSLPIDControl.py:37-60); pid_gravity/pid_kf are the CONTROLLER's
     * model constants (BaseControl.py:35-40; BaseRLAviary always embeds CF2X, BaseRLAviary.py:76) */
    double pid_p_for[3], pid_i_for[3], pid_d_for[3];
    double pid_p_tor[3], pid_i_tor[3], pid_d_tor[3];
    double pid_mixer[4][3];
    double pid_pwm2rpm_scale, pid_pwm2rpm_const, pid_min_pwm, pid_max_pwm;
    double pid_gravity, pid_kf;
    int drone_model;       /* QS_MODEL_* (informational; mixing is in sx/sy/sz/kx/ky) */
    int pad_;
} QsParams;

/* Per-drone persistent state, structure of arrays of float64, N = n_envs * drones_per_env drones.
 * planes: double[13*N], 32-byte aligned (every thread moves its 104 bytes with three 32-byte and one 8-byte access):
 *   plane 0 = [N][4] {pos.x, pos.y, pos.z, w.x}   plane 1 = [N][4] {q.x, q.y, q.z, q.w}  (Bullet order x,y,z,w)
 *   plane 2 = [N][4] {vel.x, vel.y, vel.z, w.y}   plane 3 = [N]    {w.z}                 (at planes + 12*N)
 * w = body rates (`rpy_rates`, BaseAviary.py:877).  Round 1 stored float32 planes: the rounding of the stored
 * quaternion alone cost 1e-5 of parity on tumbling drones (DESIGN.md, "precision"); float64 storage costs 40 more
 * bytes per drone and direction and puts the kernels within 1e-12 of the float64 reference. */
typedef struct QsState {
    double* planes;                 /* [13*N], see above */
    double* last_rpm;               /* [N][4] last_clipped_action (BaseAviary.py:372); nullable unless DRAG / RAW_RPM / split substeps */
    int* step_counter;              /* [E] physics steps since reset (BaseAviary.py:382) */
    unsigned char* pending_reset;   /* [E] NEXT_STEP autoreset latch; nullable otherwise */
    double* pid;                    /* [9][N]: integral_pos_e xyz, last_rpy xyz, integral_rpy_e xyz
                                       (DSLPIDControl.py:73-78); nullable unless a PID action type */
    const double* init_pos;         /* [D or N][4] INIT_XYZS (xyz, pad)             BaseAviary.py:194-201 */
    const double* init_quat;        /* [D or N][4] getQuaternionFromEuler(INIT_RPYS) BaseAviary.py:488 */
    const double* target_pos;       /* [D or N][4] TARGET_POS (HoverAviary.py:51, MultiHoverAviary.py:71); nullable for QS_TASK_NONE */
    const float* reset_head;        /* optional [D or N][12] float32: the kinematic head (pos3 rpy3 vel3 ang_v3) of the observation of a
                                       freshly reset drone, filled once by qs_reset_heads; lets SAME_STEP autoreset take the leaner
                                       kernels (without it the head is recomputed inside the tick: same values) */
    float* pos_f32;                 /* optional [N][4] float32 mirror of the positions {x, y, z, 0}, refreshed by every kernel that
                                       stores the state: the input of the float32 pairwise downwash kernels (qs_downwash*,
                                       qs_dw_publish); nullable otherwise */
    int tables_per_env;             /* 0: the three tables have D rows shared by all envs; 1: N rows */
    int pad_;
    const double* phys;             /* optional [E][16] float64, 32-byte aligned: per-aviary physical constants (domain randomisation),
                                       see "Per-aviary physical constants" below; NULL = every aviary flies the drone of QsParams */
} QsState;

/* Per-aviary physical constants (QsState.phys).  Row e, shared by the D drones of aviary e, holds the constants the reference
 * reads from the env object at call time (envs/BaseAviary.py:838-858 _dynamics, BaseRLAviary.py:192,225 HOVER_RPM,
 * CtrlAviary.py:140 MAX_RPM), derived as BaseAviary.__init__ does (BaseAviary.py:117-119):
 *     [0] inv_m = 1/M   [1] gravity = G*M   [2] kf   [3] km   [4] kx   [5] ky   [6..8] diag(J)   [9..11] diag(J^-1)
 *     [12] hover_rpm   [13] max_rpm   [14..15] pad
 * kx / ky carry the arm and the model's torque-mixing sign exactly as in QsParams.  Everything else stays in QsParams: the
 * mixing signs, the propeller offsets, GND_EFF_COEFF / PROP_RADIUS / GND_EFF_H_CLIP, DRAG_COEFF, DW_COEFF, SPEED_LIMIT, the
 * task and the embedded controller's constants (the reference's embedded DSLPIDControl reads its own CF2X URDF).
 * With the table, qs_step (both kernel families, qs_step_host), qs_rollout (with and without a policy) and qs_dyn_substeps
 * (including the MAX_RPM clip) read row e in place of the QsParams fields; with NULL they run unchanged, same bits.
 * qs_pid_control / qs_pid_control_state and the formation paths do not take it: a non-NULL table with external downwash
 * (QsStepIO.dw_fz, the split-substep protocol of aviaries larger than one CTA) or with qs_dyn_substeps_pub is refused with
 * QS_ERR_UNSUPPORTED.
 * Ordering: the kernels only READ the table.  The caller writes it between launches with ordinary stream-ordered work (torch
 * kernels, copies): such work never lets its successor start early, so it is complete before the next step, rollout or
 * substep starts, whether or not that kernel is a programmatic dependent -- the argument made for the action tensor at qs_step.
 * A change therefore takes effect at the next launch; a rollout keeps each aviary's row for all its T ticks. */

/* Inputs/outputs of one control tick. */
typedef struct QsStepIO {
    const float* action;        /* [N][A] float32; A = 4 (RPM, VEL, RAW_RPM), 3 (PID), 1 (ONE_D_*) */
    const float* obs_prev;      /* [N][12+B*A] previous observation: source of the action history (BaseRLAviary.py:316-319) */
    float* obs;                 /* out: RL: [N][12+B*A] = pos3 rpy3 vel3 ang_v3 + B buffered actions oldest->newest
                                        RAW_RPM: [N][20] _getDroneStateVector; nullable (state-only step) */
    float* reward;              /* out [E] */
    unsigned char* terminated;  /* out [E] */
    unsigned char* truncated;   /* out [E] */
    float* final_obs;           /* out [N][obs_dim] rows of envs that finished, SAME_STEP autoreset only; nullable */
    unsigned char* done;        /* out [E] terminated | truncated (the `_final_obs` mask of gymnasium's vector API); nullable */
    const float* dw_fz;         /* [N] downwash force along body z from qs_downwash; required iff QS_EFFECT_DW */
    int act_buffer_size;        /* B = ctrl_freq//2 (BaseRLAviary.py:66); 0 for RAW_RPM */
    int tick_substeps;          /* physics steps the step counter advances by in the epilogue; 0 = `substeps`
                                   (only the split-substep protocol passes PYB_STEPS_PER_CTRL here) */
    /* Fused observation gather (SURVEY.md 8e: "optional all-gather of observations where the learner wants a single tensor"):
     * a second destination for this tick's rows, normally the LEARNER GPU's [E_total][D][obs_dim] tensor at this rank's
     * row offset, mapped into this process by CUDA IPC / peer access.  The kernel's bulk store writes the finished rows
     * straight over NVLink (no separate collective), per-aviary reward/flags likewise, and the last warp to finish raises
     * *gather_flag to gather_seq with release semantics at system scope (the learner waits with qs_wait_flags).  All NULL =
     * off.  Supported by the RL configurations of step_fast.cu (QS_ERR_UNSUPPORTED otherwise). */
    float* obs_gather;                  /* [N][obs_dim] rows of THIS rank inside the gathered tensor */
    float* reward_gather;               /* [E] nullable */
    unsigned char* terminated_gather;   /* [E] nullable */
    unsigned char* truncated_gather;    /* [E] nullable */
    unsigned* gather_flag;              /* one word on the learner, nullable */
    unsigned* gather_counter;           /* one zeroed device word owned by the caller (arrival count); required with gather_flag */
    unsigned gather_seq;
    unsigned pad_;
    /* Per-tile readiness of the fast step kernels (DESIGN.md 4.1), one word each per tile of 32 consecutive drones: device words
     * owned by the caller, zero-initialised once, and passed with EVERY qs_step / qs_step_host call on the same state and
     * observation buffers (or never).  With them a tile waits only for the same tile of the previous step on these buffers,
     * instead of for the whole previous kernel of the stream, so consecutive steps overlap.  All NULL = the whole-grid wait.
     * ready_err becomes non-zero if a tile ever waited longer than ~1 s for its turn (the step then went ahead unordered). */
    unsigned* warp_ticket;              /* [ceil(N / 32)] */
    unsigned* warp_done;                /* [ceil(N / 32)] */
    unsigned* ready_err;                /* one word */
} QsStepIO;

/* Spins (bounded, ~2 s, then *err_flag = 1) until flags[r] - seq >= 0 for every r < world: the learner side of obs_gather. */
int qs_wait_flags(const unsigned* flags, unsigned seq, int world, unsigned* err_flag, void* stream);

/* On-device policy for qs_rollout (SURVEY.md 8f rank 1; the caller is SB3's collect_rollouts, examples/learn.py:67-95): an
 * SB3-MlpPolicy-shaped actor -- flatten(the aviary's [D][obs_dim] observation) -> 64 tanh -> 64 tanh -> linear mean, state
 * independent log_std, Gaussian sample, clip to [-1, 1] for the env -- and optionally the critic (same shape, 1 output),
 * evaluated inside the rollout kernel from the observation window in shared memory on the tensor cores (mma m16n8k16 F16) with
 * a two-term split of both operands (fp32-level accuracy: x w ~ x_hi w_hi + 2^-11 (x_hi w_lo' + x_lo' w_hi), fp32 accumulation;
 * w_hi = fp16(w), w_lo' = fp16(2048 (w - w_hi))).  Observations saturate at +-(65504 + 65504 / 2048) = +-65535.984375: both
 * fp16 conversions clamp to 65504, so x_hi + x_lo' / 2048 stops growing there (not at fp16's 65504).
 * Every weight matrix W[in][out] is given in FRAGMENT ORDER: rows padded with zeros to a multiple of 16, columns to a multiple
 * of 8 (the last layer's to 8 * nt3, the critic's to 8), then [k-step ks][n-tile n][lane l] x 4 words, lane l = 4 g + t:
 *     word 0 = {w_hi[16 ks + ka][8 n + g], w_hi[16 ks + ka + 1][8 n + g]}   (low half, high half)
 *     word 1 = {w_hi[16 ks + kb][8 n + g], w_hi[16 ks + kb + 1][8 n + g]}
 *     word 2, 3 = the same two pairs of w_lo'
 * with (ka, kb) = (2 t, 2 t + 8) for layers 2 and 3 -- the B fragment of mma.m16n8k16 -- and (ka, kb) = (4 t, 4 t + 2) for
 * layer 1 (its A operand is read as 4 consecutive observation elements per lane; any permutation of k inside a k-step is
 * allowed as long as A and B agree).  gym_pybullet_drones_b200/policy.py prepares the arrays (16-byte aligned).
 * in_dim = drones_per_env * obs_dim and out_dim = drones_per_env * A for any action type (A = 4, 3 or 1), out_dim <= 32.
 * QsPolicy is SB3's default shape only; QsMlpPolicy (qs_rollout_mlp, below) describes every other supported net_arch. */
typedef struct QsPolicy {
    const unsigned* w1; const float* b1;      /* [ceil(in_dim / 16)][8][32][4], [64]   in_dim = D * obs_dim */
    const unsigned* w2; const float* b2;      /* [4][8][32][4], [64] */
    const unsigned* w3; const float* b3;      /* [4][nt3][32][4], [8 nt3]   out_dim = D * A real columns */
    const float* log_std;                     /* [out_dim] */
    const unsigned* vw1; const float* vb1;    /* critic, same arrangement ([..][8], [4][8], [4][1] tiles); all NULL = no critic */
    const unsigned* vw2; const float* vb2;
    const unsigned* vw3; const float* vb3;
    const float* noise;        /* [T][E][out_dim] standard-normal draws (e.g. torch.randn), or NULL: action = mean */
    float* logprob;            /* out [T][E] log-probability of the sampled (unclipped) action; nullable */
    float* values;             /* out [T][E] critic output; nullable (required NULL without a critic) */
    int in_dim, out_dim;
    int nt3, pad_;             /* padded action outputs = 8 * nt3 (nt3 = 1, 2 or 4) */
} QsPolicy;

/* Multi-tick rollout: T control ticks in ONE launch (SURVEY.md 8f rank 1; the caller is SB3's collect_rollouts,
 * examples/learn.py:93).  Exactly T calls of qs_step with the same flags -- SAME_STEP, NEXT_STEP or no autoreset -- but the
 * drone state stays in registers and the action history in shared memory between ticks: per tick only the action is read and
 * the observation row, reward and flags are written.
 * NEXT_STEP autoreset: an aviary whose QsState.pending_reset latch is set at the start of a tick is only reset by it, as by
 * qs_step: its action is ignored (no decode, no controller, no physics; actions_out and, with a policy, logprob / values are
 * still written), its observation is the reset pose with the action history unshifted (zeroed with CLEARS_HISTORY), reward 0,
 * terminated / truncated 0.  The latch is carried from tick to tick (a tick's done sets it for the next) and stored at the end,
 * so it crosses launches and mixes with qs_step.  obs[k] of an aviary that finished at k is its terminal observation, and the
 * policy's values[k+1] the critic on it.
 * Terminal observations (SAME_STEP autoreset): at tick k the kernel writes final_obs[k][i] for every drone i of an aviary that
 * finished at k, bit for bit the row qs_step writes to QsStepIO.final_obs, and with a policy critic final_values[k][e] = the
 * critic on that aviary's terminal rows (the value SB3 bootstraps a truncated episode with).  Entries of the aviaries that did
 * not finish at k are not written.  The critic pass runs only in CTAs that hold a finished aviary at that tick. */
typedef struct QsRolloutIO {
    const float* actions;       /* [T][N][A] float32, or NULL: uniform[-1,1) actions generated on the device from (seed, tick, drone) */
    float* actions_out;         /* out [T][N][A] the actions that were applied; nullable */
    const float* obs_init;      /* [N][12+B*A] observation before the first tick (source of the initial action history) */
    float* obs;                 /* out [T][N][12+B*A] (PPO rollout-buffer layout) */
    float* obs_last;            /* out [N][12+B*A] copy of the last tick's observation (the env's current observation); nullable */
    float* reward;              /* out [T][E] */
    unsigned char* terminated;  /* out [T][E] */
    unsigned char* truncated;   /* out [T][E] */
    unsigned char* done;        /* out [T][E]; nullable */
    unsigned long long seed;    /* device action generator: splitmix64(seed + 2*((tick0+k)*N + drone) + {0,1}) */
    long long tick0;            /* global index of the first tick of this launch (continues the generator's stream) */
    int T;                      /* ticks in this launch; qs_rollout_max_ticks() bounds it (shared-memory window) */
    int act_buffer_size;        /* B */
    const QsPolicy* policy;     /* optional (HOST pointer): the actions come from this policy evaluated on the current observation;
                                   `actions` must then be NULL, actions_out receives the sampled, UNCLIPPED actions (what PPO
                                   stores), the env applies them clipped to [-1, 1], through the embedded DSLPID controller
                                   for PID / VEL / ONE_D_PID: the physics is bit for bit that of `actions` = the clipped
                                   samples.  Every action type; effects none, GND, DRAG, DW or all three (GND|DRAG, GND|DW and
                                   DRAG|DW return QS_ERR_UNSUPPORTED); drones_per_env <= 64; QsPolicy is the 64 tanh -> 64 tanh
                                   network only: other shapes go through qs_rollout_mlp (QsMlpPolicy) with policy = NULL here. */
    float* final_obs;           /* out [T][N][12+B*A] terminal observations (see above); nullable.  Needs QS_FLAG_AUTORESET_SAME_STEP
                                   (QS_ERR_UNSUPPORTED otherwise; under NEXT_STEP obs[k] already is the terminal observation) */
    float* final_values;        /* out [T][E] critic on the terminal observations; nullable.  Needs SAME_STEP autoreset
                                   (QS_ERR_UNSUPPORTED) and a policy with a critic (QS_ERR_NULL) */
} QsRolloutIO;

/* Host-buffer variant of one control tick (what a CPU-side caller such as SB3's DummyVecEnv loop sees): pinned host
 * arrays in, pinned host arrays out, every host<->device copy inside the call.  The terminal observations of the
 * aviaries that finished (SAME_STEP autoreset) are compacted on the device (ascending aviary index) and written by the
 * gather kernel straight into the pinned host arrays (mapped memory), so nothing waits for the host in the middle of
 * the tick; with side_stream/ev_fork/ev_join they move concurrently with the copy of the observations. */
typedef struct QsHostIO {
    const float* action_host;        /* [N][A]  (pinned) */
    float* obs_host;                 /* out [N][obs_dim] */
    float* reward_host;              /* out [E] */
    unsigned char* terminated_host;  /* out [E] */
    unsigned char* truncated_host;   /* out [E] */
    unsigned char* done_host;        /* out [E] */
    float* final_obs_host;           /* out: rows [k][D][obs_dim] of the k aviaries that finished (SAME_STEP autoreset); nullable.
                                        Pinned AND mapped (cudaHostAlloc / cudaHostRegister): written by a kernel */
    long long* final_env_host;       /* out [E]: their aviary indices, ascending (pinned, mapped) */
    int* n_final_host;               /* out: k (pinned, mapped) */
    float* action_dev;               /* caller-owned device scratch [N][A] */
    long long* final_env_dev;        /* caller-owned device scratch [E] */
    int* n_final_dev;                /* caller-owned device scratch [1] */
    float* obs_head_host;            /* optional [N][12] (pinned, mapped): when set, only the kinematic head (pos3 rpy3 vel3 ang_v3) of every
                                        observation row travels -- packed by a kernel into this array -- and obs_host is NOT written: a caller
                                        that supplied the actions already holds the action-history part of the rows (5/6 of the bytes) */
    void* side_stream;               /* optional second cudaStream_t: the compaction + gather of the terminal observations run on it next to
                                        the observation copy; with the chunked pipeline (fast-kernel configurations, >= 16 384 drones or
                                        QS_HOST_CHUNKS=n) it carries the per-chunk observation copies instead, each behind its chunk's tick */
    void* ev_fork;                   /* optional cudaEvent_t pair (timing disabled) used to fork/join side_stream; both or neither */
    void* ev_join;
} QsHostIO;

/* 1 if `p` points into page-locked host memory known to the CUDA driver (cudaHostAlloc / cudaHostRegister), else 0. */
int qs_host_is_pinned(const void* p);

int qs_abi_version(void);
const char* qs_last_error(void);
int qs_sizeof_params(void);
int qs_sizeof_state(void);
int qs_sizeof_step_io(void);
int qs_sizeof_rollout_io(void);
int qs_sizeof_host_io(void);

/* One control tick for n_envs aviaries of drones_per_env drones: action decode -> `substeps` x DYN ->
 * obs / reward / terminated / truncated (+ autoreset).  RL action types; task = QS_TASK_HOVER or NONE.
 *
 * Ordering with the work before it on `stream`: the step kernels are launched as programmatic dependents (they may start
 * before the previous kernel of the stream has finished).  With QsStepIO.warp_ticket / warp_done a fast step kernel does
 * not wait for the whole previous kernel when that kernel is a fast step of this library: it then waits per warp for the
 * previous step on its own buffers only.  Kernels and copies that do not trigger their successor early (torch kernels,
 * qs_reset, qs_rollout, memcpy) are complete before the step starts, and the library's other early-triggering kernels are
 * always waited for.  The caller's side of the contract: a kernel of the caller's own that triggers programmatic launch
 * early (griddepcontrol.launch_dependents / cudaTriggerProgrammaticLaunchCompletion) must not directly precede qs_step
 * on the stream when it writes that step's action or state. */
int qs_step(const QsParams* p, const QsState* st, const QsStepIO* io, int act_type, int task,
            int n_envs, int drones_per_env, int substeps, unsigned effects, unsigned flags, void* stream);

/* qs_step with all arguments in one caller-owned struct (a hot loop then passes two pointers per tick). */
typedef struct QsStepCall {
    const QsParams* p; const QsState* st; const QsStepIO* io;
    int act_type, task, n_envs, drones_per_env, substeps;
    unsigned effects, flags;
    int pad_;
} QsStepCall;
int qs_step_call(const QsStepCall* c, void* stream);

/* qs_step with host buffers: H2D(action) -> fused tick -> D2H(reward, flags) -> D2H(obs) (+ a compact D2H of the terminal
 * observations of finished aviaries).  `io` carries the device buffers exactly as for qs_step (io->action is ignored).
 * Large batches are pipelined in chunks of whole warps (chunk c's observation rows travel while chunk c+1's actions go up and
 * its tick runs); the results are the same bits as one qs_step over the whole batch.
 * Unlike every other entry point this one SYNCHRONISES `stream` before returning (the host arrays are valid on return). */
int qs_step_host(const QsParams* p, const QsState* st, const QsStepIO* io, const QsHostIO* h, int act_type, int task,
                 int n_envs, int drones_per_env, int substeps, unsigned effects, unsigned flags, void* stream);

/* T fused control ticks (see QsRolloutIO).  RL action types, KIN observations, drones_per_env <= 128, autoreset SAME_STEP,
 * NEXT_STEP or none (flags as qs_step: both modes together return QS_ERR_ENUM, NEXT_STEP needs QsState.pending_reset
 * (QS_ERR_NULL) and the init tables; under SAME_STEP the terminal observations go to QsRolloutIO.final_obs, their critic values
 * to final_values).
 * qs_rollout_max_ticks gives the largest T for an observation width. */
int qs_rollout(const QsParams* p, const QsState* st, const QsRolloutIO* io, int act_type, int task,
               int n_envs, int drones_per_env, int substeps, unsigned effects, unsigned flags, void* stream);
int qs_rollout_max_ticks(int act_type, int act_buffer_size, int drones_per_env);

/* On-device policy of any SB3 MlpPolicy net_arch in scope, for qs_rollout_mlp: per network 1 to QS_MLP_MAX_HIDDEN hidden layers
 * of 1 to QS_MLP_MAX_WIDTH units, one activation for the whole policy after every hidden layer, linear output layers, and
 * independent actor and critic shapes (SB3's net_arch = dict(pi = [...], vf = [...])).  The arithmetic is QsPolicy's (two-term
 * fp16 split of both operands, fp32 accumulation, the same saturation of the observation); a [64, 64] tanh network gives the
 * bits of qs_rollout with the QsPolicy of the same weights.
 * Layer l = 0 .. depth maps K_l inputs to N_l outputs: K_0 = in_dim padded to a multiple of 16, K_l = N_(l-1); the hidden
 * widths N_0 .. N_(depth-1) are padded with zero columns (and zero biases) to a multiple of 64, the output layer to
 * N_depth = 8 out_tiles.  w[l] is W_l[K_l][N_l] in QsPolicy's FRAGMENT ORDER, [K_l / 16][N_l / 8][32][4] words, with the
 * (4 t, 4 t + 2) permutation of k for layer 0 and the mma B fragment's (2 t, 2 t + 8) for the others; b[l] is [N_l]. */
#define QS_MLP_MAX_HIDDEN 4
#define QS_MLP_MAX_WIDTH 256
enum { QS_MLP_TANH = 0, QS_MLP_RELU = 1 };
typedef struct QsMlpNet {
    const unsigned* w[QS_MLP_MAX_HIDDEN + 1];   /* device, 16-byte aligned */
    const float* b[QS_MLP_MAX_HIDDEN + 1];
    int depth;                                  /* hidden layers, 1 .. QS_MLP_MAX_HIDDEN; 0 = no network (critic only) */
    int width[QS_MLP_MAX_HIDDEN];               /* padded hidden widths N_0 .. N_(depth-1): multiples of 64, <= QS_MLP_MAX_WIDTH */
    int out_tiles;                              /* N_depth / 8: 1, 2 or 4 for the actor (out_dim real columns), 1 for the critic */
} QsMlpNet;
typedef struct QsMlpPolicy {
    QsMlpNet actor;
    QsMlpNet critic;           /* depth 0 = no critic */
    int activation;            /* QS_MLP_TANH or QS_MLP_RELU */
    int in_dim, out_dim;       /* as QsPolicy: D * obs_dim and D * A (<= 32) */
    int pad_;
    const float* log_std;      /* [out_dim] */
    const float* noise;        /* as QsPolicy */
    float* logprob;
    float* values;             /* nullable; requires a critic */
} QsMlpPolicy;
int qs_sizeof_mlp_policy(void);

/* qs_rollout with the actions of a QsMlpPolicy (io->policy must be NULL, io->actions too): the same outputs, autoreset modes,
 * action types, effects and per-aviary table as qs_rollout with a QsPolicy.  Every warp stages the split activations of the
 * hidden layers in shared memory, 2 x 16 rows x max width x 4 bytes, which the per-launch tick limit accounts for:
 * qs_rollout_mlp_max_ticks(act_type, act_buffer_size, drones_per_env, max padded hidden width of the two networks). */
int qs_rollout_mlp(const QsParams* p, const QsState* st, const QsRolloutIO* io, const QsMlpPolicy* policy, int act_type, int task,
                   int n_envs, int drones_per_env, int substeps, unsigned effects, unsigned flags, void* stream);
int qs_rollout_mlp_max_ticks(int act_type, int act_buffer_size, int drones_per_env, int max_width);

/* CtrlAviary semantics: rpm[N][4] (float32) clipped to [0, MAX_RPM], `substeps` x DYN, optional [N][20] state vectors.
 * With QS_FLAG_RPM_FROM_LAST `rpm` is ignored and the rpm of the previous call is re-read from QsState.last_rpm. */
int qs_dyn_substeps(const QsParams* p, const QsState* st, const float* rpm, float* state20_out, const float* dw_fz,
                    int n_envs, int drones_per_env, int substeps, unsigned effects, unsigned flags, void* stream);

/* DSLPIDControl.computeControl for n drones.  cur_pos/cur_quat/cur_vel are read with a row stride (in floats),
 * so they can point into [n][20] state vectors (strides 20; BaseControl.computeControlFromState) or packed arrays.
 * target_rpy/target_vel/target_rpy_rates may be NULL (= zeros, the reference defaults).  pid_state: double[9][n]. */
int qs_pid_control(const QsParams* p, double* pid_state, double control_timestep,
                   const float* cur_pos, int pos_stride, const float* cur_quat, int quat_stride,
                   const float* cur_vel, int vel_stride,
                   const float* target_pos, const float* target_rpy, const float* target_vel, const float* target_rpy_rates,
                   int n, float* rpm_out, float* pos_e_out, float* yaw_e_out, void* stream);

/* The same controller for the n = n_envs * drones_per_env drones of a simulator state: pos / quat / vel are read from the
 * float64 planes (three coalesced 32-byte accesses per drone instead of strided float32 state vectors), the targets are
 * float64 [n][3] (target_rpy / target_vel / target_rpy_rates nullable = zeros), and the RPMs are written as float64 [n][4],
 * clipped to [0, MAX_RPM] like CtrlAviary._preprocessAction (envs/CtrlAviary.py:121-140) -- e.g. straight into
 * QsState.last_rpm, from where qs_dyn_substeps(QS_FLAG_RPM_FROM_LAST, rpm = NULL) applies them: the pid.py control loop
 * (examples/pid.py:131-150) in float64 end to end, with nothing leaving the device. */
int qs_pid_control_state(const QsParams* p, double* pid_state, double control_timestep, const QsState* st, int n,
                         const double* target_pos, const double* target_rpy, const double* target_vel, const double* target_rpy_rates,
                         double* rpm_out, float* pos_e_out, float* yaw_e_out, void* stream);

/* Pairwise downwash within each aviary: fz_out[n] = sum over drones i of the same aviary with dz>0, dxy<10 of
 * -alpha*exp(-.5 (dxy/beta)^2) (force along n's body z).  Reads the float32 position mirror QsState.pos_f32. */
int qs_downwash(const QsParams* p, const QsState* st, int n_envs, int drones_per_env, float* fz_out, void* stream);

/* Downwash with a workspace: like qs_downwash, but first tabulates the bounding boxes of every 32 consecutive drones
 * (boxes_ws: float [n_envs][ceil(D/32)][8], 16-byte aligned) and then evaluates, per group of 32 rows, only the chunks
 * whose box can contribute (exact: a skipped pair fails the reference's predicate or its Gaussian is 0.0f). */
int qs_downwash_boxed(const QsParams* p, const QsState* st, int n_envs, int drones_per_env, float* boxes_ws, float* fz_out, void* stream);

/* Downwash for ONE formation sharded across GPUs (SURVEY.md 8e/8f-3: one exchange of positions per substep).
 * "gathered array": the [n_total][4] positions of the WHOLE formation immediately followed by its chunk boxes
 * [ceil(n_total/32)][8]; qs_dw_gathered_floats(n_total) floats, 16-byte aligned.  It is filled either by
 * qs_dw_publish from every rank (positions + boxes pushed into every rank's array, own and NVLink peers), or by an
 * all-gather of the positions followed by qs_dw_boxes.
 * qs_downwash_rows: rows_pos = the [n_rows][4] positions this GPU owns (plane 0 of its state).  If ready_flags != NULL
 * the kernel first waits (bounded, ~2 s, then *err_flag = 1) until ready_flags[r] - seq >= 0 for r < world. */
#define QS_MAX_PEERS 16
long long qs_dw_gathered_floats(int n_total);
int qs_dw_boxes(float* gathered, int n_total, void* stream);
int qs_downwash_rows(const QsParams* p, const float* rows_pos, int n_rows, const float* gathered, int n_total,
                     const unsigned* ready_flags, unsigned seq, int world, unsigned* err_flag, float* fz_out, void* stream);

/* Pushes pos[0..n) (+ the boxes of its chunks; offset % 32 == 0) into gathered[r] at drone offset `offset` for every
 * rank r < world (device pointers in a HOST array), then stores seq to flags[r][rank] with release semantics.
 * counter: one zeroed device word owned by the caller (inter-CTA arrival count, reset by the kernel). */
int qs_dw_publish(const float* pos, int n, int offset, float* const* gathered, int n_total, unsigned* const* flags, int world, int rank,
                  unsigned seq, unsigned* counter, void* stream);

/* The same push fused into the dynamics kernel: qs_dyn_substeps (one formation = one aviary, n_envs == 1, this rank's slice of
 * drones_per_env drones) whose epilogue publishes the NEW positions -- exactly what qs_dw_publish would push from QsState.pos_f32
 * after the call -- under sequence number pub->seq.  The exchange for the next substep's qs_downwash_rows then costs no launch
 * of its own (SURVEY.md 8f rank 3).  pub == NULL: plain qs_dyn_substeps. */
typedef struct QsDwPublish {
    float* const* gathered;     /* [world] device pointers (HOST array), as for qs_dw_publish */
    unsigned* const* flags;     /* [world] */
    unsigned* counter;          /* one zeroed device word (arrival count; may be shared with qs_dw_publish calls of the same stream) */
    int n_total, world, rank, offset;
    unsigned seq;
    int pad_;
} QsDwPublish;
int qs_dyn_substeps_pub(const QsParams* p, const QsState* st, const float* rpm, float* state20_out, const float* dw_fz,
                        int n_envs, int drones_per_env, int substeps, unsigned effects, unsigned flags, const QsDwPublish* pub, void* stream);

/* CUDA IPC for the exchange buffers of one-process-per-GPU runs: export the 64-byte handle of the allocation that
 * contains ptr plus ptr's byte offset in it; import maps a peer's handle into this process (peer access enabled
 * lazily) and returns the peer's ptr.  Import a given handle once per process. */
int qs_ipc_export(const void* ptr, void* handle64, unsigned long long* offset);
int qs_ipc_import(const void* handle64, unsigned long long offset, void** ptr_out);

/* cudaDeviceEnablePeerAccess(peer_device) for the current device; already-enabled is not an error. */
int qs_enable_peer_access(int peer_device);

/* BaseAviary._getAdjacencyMatrix (envs/BaseAviary.py:658-675) for every aviary: out[e][i][j] = 1 if i == j or
 * |pos_i - pos_j| < radius else 0 (unsigned char [E][D][D]). */
int qs_adjacency(const QsState* st, int n_envs, int drones_per_env, double radius, unsigned char* out, void* stream);

/* Fills `out` ([rows][12] float32, 16-byte aligned; rows = D or N like the init tables) with the observation head of a freshly
 * reset drone: (float)INIT_XYZS, float32 casts of the float64 rpy of the initial quaternion, zeros -- exactly what qs_reset and
 * the tick write for an aviary they reset, with or without QS_FLAG_RPY_F32 (`flags` is accepted and ignored).  Point
 * QsState.reset_head at it afterwards. */
int qs_reset_heads(const QsState* st, int rows, unsigned flags, float* out, void* stream);

/* Device-side trajectory ring in the reference Logger's layout (utils/Logger.py:83-127).  One call appends ONE entry for
 * each of the drones [first_drone, first_drone + n_drones): the 16 logged states in Logger.py:117 order (pos3, vel3, rpy3,
 * ang_v3, rpm4), the 12 control targets, the simulation time of the entry and 3 pad doubles -- 32 float64 per drone and
 * entry, ring[(head % capacity)][drone][32]; the kernel then advances *head.  pos/vel/rpm come from the float64 state
 * (planes, last_rpm), rpy is re-evaluated from the quaternion in float64, ang_v is taken from the observation rows
 * (float32: columns 9-11 of a KIN row, 13-15 of a [20] state vector).  kin_rows = 1: the rows are KIN observations whatever
 * obs_dim (a KIN row is 20 floats wide too, e.g. ONE_D_RPM at ctrl_freq 16); 0: state vectors iff obs_dim == 20.  controls: [n_drones][12] float32 device array or NULL (zeros).
 * Nothing crosses PCIe until the caller copies the ring (Logger.save). */
typedef struct QsLogRing {
    double* ring;            /* [capacity][n_drones][32] */
    long long* head;         /* device counter: entries appended so far */
    int capacity, first_drone, n_drones, kin_rows;
} QsLogRing;
int qs_sizeof_log_ring(void);
int qs_log_append(const QsParams* p, const QsState* st, const float* obs, int obs_dim, const float* controls,
                  const QsLogRing* ring, int n_envs, int drones_per_env, void* stream);

/* Control-env rollout: T control ticks of CtrlAviary / VelocityAviary in ONE launch, the drone state, the controller state and
 * the previous RPMs in registers between ticks.  Modes:
 *   QS_CTRL_RAW    CtrlAviary with given RPMs: T x qs_dyn_substeps (float32 actions, or float64 with QS_FLAG_ACTION_F64)
 *   QS_CTRL_VEL    VelocityAviary: T x qs_step(QS_ACT_VEL, QS_FLAG_OBS_STATE20), the embedded controller on QsState.pid
 *   QS_CTRL_TRACK  CtrlAviary driven by a DSLPIDControl (examples/pid.py:131-150): per tick qs_pid_control_state with the
 *                  controller's own QsParams on its [9][N] state and the tick's targets (RPMs clipped to the controller's max_rpm),
 *                  then qs_dyn_substeps(QS_FLAG_ACTION_F64) on those RPMs.  Target position of drone i at tick k of the launch:
 *                      waypoints[(start[i] + k) mod W][M == 1 ? 0 : i] + offset[i]      (mod as Python's %, never negative)
 *                  one shared path with per-drone phases (pid.py), per-drone paths (M = N), a full schedule (W = T, M = N).
 * Each tick gives the bits of the per-tick calls it replaces.  DYN+ effects: none, GND, DRAG, DW (in-CTA, drones_per_env <= 128)
 * or all three; flags: QS_FLAG_RPY_F32, QS_FLAG_ACTION_F64 (RAW).  The per-tick outputs are nullable: without obs only obs_last
 * (the env's observation buffer) receives the last tick's rows. */
enum { QS_CTRL_RAW = 0, QS_CTRL_VEL = 1, QS_CTRL_TRACK = 2 };
typedef struct QsCtrlRolloutIO {
    int T;                          /* ticks in this launch */
    int log_targets;                /* TRACK with a log ring: 1 = log the tick's targets as the 12 controls (target_pos, target_rpy,
                                       target_vel, target_rpy_rates, as float32: pid.py's layout); 0 = log_controls */
    const void* actions;            /* RAW / VEL: [T][N][4] float32 (16-byte aligned), RAW with QS_FLAG_ACTION_F64: float64 (32-byte aligned) */
    /* TRACK: the controller */
    const QsParams* ctrl_params;    /* HOST pointer: the controller's QsParams (pid_* gains and model constants, max_rpm) */
    double* pid_state;              /* [9][N] the controller's state (read at the start, stored at the end) */
    double control_timestep;        /* the controller's dt (CTRL_TIMESTEP) */
    const double* waypoints;        /* [W][M][3] */
    int W, M;                       /* W > 0; M = 1 or N */
    const int* start;               /* [N] */
    const double* offset;           /* [N][3], nullable = zeros */
    const double* target_rpy;       /* [N][3] constant targets, each nullable = zeros */
    const double* target_vel;
    const double* target_rpy_rates;
    /* per-tick outputs, all nullable */
    float* obs;                     /* out [T][N][20] _getDroneStateVector rows (16-byte aligned) */
    double* rpm;                    /* out [T][N][4] the applied (clipped) RPMs (32-byte aligned) */
    float* pos_e;                   /* out [T][N][3] TRACK: position error, as computeControlFromEnv returns it */
    float* yaw_e;                   /* out [T][N]    TRACK: yaw error */
    float* obs_last;                /* out [N][20] the last tick's rows (16-byte aligned); nullable */
    const QsLogRing* log;           /* HOST pointer, nullable: one entry per logged drone and tick, the bytes of qs_log_append after
                                       every tick of the per-tick loop; the kernel then advances *head by T */
    const float* log_controls;      /* [n_drones][12] controls logged without log_targets; nullable = zeros */
} QsCtrlRolloutIO;
int qs_sizeof_ctrl_rollout_io(void);
int qs_ctrl_rollout(const QsParams* p, const QsState* st, const QsCtrlRolloutIO* io, int mode, int n_envs, int drones_per_env,
                    int substeps, unsigned effects, unsigned flags, void* stream);

/* MRAC (control/MRAC.py): the model reference adaptive controller, float64, one controller per drone.
 * QsMracParams holds the per-model constants the gains were synthesised into (MRAC._compute_K with psi = 0, on the host):
 * Am = A - B K, the diagonal of the nonzero block Bm[8:12][0:4], P Bm with P = solve_lyapunov(Am^T, -600 I), Kr_ref_gain =
 * pinv(B) Am, the adaptation rates Gamma_x = gamma_x I and Gamma_r = gamma_r I, the mixer and the PWM constants.
 * The adaptive state of N controllers is double[QS_MRAC_STATE][N]: rows 0-47 Kx[12][4] (row-major), 48-63 Kr[4][4], 64-75 Xm[12].
 * `init` != 0 is the reference's control_counter == 0: the call first sets Xm to the current state X.
 * One call per drone (MRAC.computeControl, MRAC.py:109-155):
 *   rpy = getEulerFromQuaternion(q); w_b = R_XYZ(rpy)^T cur_ang_vel (scipy's intrinsic 'XYZ' on Bullet's rpy, as the reference);
 *   X = [pos, rpy, vel, w_b]; rt = -Kr_ref_gain [tpos, trpy, tvel, trates]; u = Kx^T X + Kr^T rt; e = X - Xm;
 *   Kx += dt (-gamma_x X e^T P Bm); Kr += dt (-gamma_r rt e^T P Bm); thrust = max(0, u0); tau = clip(u1..3, +-3200);
 *   rpm = 0.2685 clip((sqrt(thrust / 4 KF) - 4070.3) / 0.2685 + MIX tau, 20000, 65535) + 4070.3; pos_e = tpos - pos;
 *   rpy_e = trpy - rpy; Xm += dt (Am Xm + Bm rt). */
#define QS_MRAC_STATE 76
typedef struct QsMracParams {
    double Am[12][12];
    double bm[4];                   /* Bm[8 + j][j]; every other entry of Bm is 0 */
    double PBm[12][4];              /* P Bm */
    double Kr_ref[4][12];           /* Kr_ref_gain */
    double gamma_x, gamma_r;
    double mixer[4][3];
    double kf, pwm2rpm_scale, pwm2rpm_const, min_pwm, max_pwm;
    double max_rpm;                 /* qs_mrac_control_state and the rollout clip the RPMs to [0, max_rpm] (CtrlAviary.py:140) */
} QsMracParams;
int qs_sizeof_mrac_params(void);

/* MRAC.computeControl for n drones: cur_pos / cur_vel / cur_ang_vel / target_* are float64 [n][3], cur_quat float64 [n][4]
 * (target_rpy / target_vel / target_rpy_rates nullable = zeros).  rpm_out: float64 [n][4], the reference's unclipped RPMs;
 * pos_e_out / rpy_e_out: float32 [n][3], nullable. */
int qs_mrac_control(const QsMracParams* p, double* mrac_state, int init, double control_timestep,
                    const double* cur_pos, const double* cur_quat, const double* cur_vel, const double* cur_ang_vel,
                    const double* target_pos, const double* target_rpy, const double* target_vel, const double* target_rpy_rates,
                    int n, double* rpm_out, float* pos_e_out, float* rpy_e_out, void* stream);

/* The same controller for the n drones of a simulator state, as qs_pid_control_state: pos / quat / vel / rates from the float64
 * planes, cur_ang_vel = getMatrixFromQuaternion(q) w (the state vector's ang_v, BaseAviary.py:873, rebuilt in float64: the
 * quaternion increment is body-frame, so R_old w = R_new w), RPMs clipped to [0, max_rpm] into rpm_out (float64 [n][4], 32-byte
 * aligned), e.g. the env's float64 command buffer. */
int qs_mrac_control_state(const QsMracParams* p, double* mrac_state, int init, double control_timestep, const QsState* st, int n,
                          const double* target_pos, const double* target_rpy, const double* target_vel, const double* target_rpy_rates,
                          double* rpm_out, float* pos_e_out, float* rpy_e_out, void* stream);

/* qs_ctrl_rollout with an MRAC in the loop (mode QS_CTRL_MRAC): per tick qs_mrac_control_state on the tick's targets (the TRACK
 * schedule of QsCtrlRolloutIO: waypoints, start, offset, target_rpy, target_vel, target_rpy_rates, control_timestep), then
 * qs_dyn_substeps(QS_FLAG_ACTION_F64) on those RPMs; tick 0 initialises Xm iff mio->init.  QsCtrlRolloutIO.ctrl_params,
 * pid_state and yaw_e are not used; its obs, rpm, pos_e, obs_last and log outputs are written as for QS_CTRL_TRACK.
 * Each thread keeps its controller's 76 doubles in shared memory for the whole launch. */
enum { QS_CTRL_MRAC = 3 };
typedef struct QsMracRolloutIO {
    const QsMracParams* params;     /* HOST pointer */
    double* state;                  /* [QS_MRAC_STATE][N] (read at the start, stored at the end) */
    int init;                       /* 1: tick 0 sets Xm = X (the controller's control_counter is 0) */
    int pad_;
    float* rpy_e;                   /* out [T][N][3], nullable */
} QsMracRolloutIO;
int qs_sizeof_mrac_rollout_io(void);
int qs_ctrl_rollout_mrac(const QsParams* p, const QsState* st, const QsCtrlRolloutIO* io, const QsMracRolloutIO* mio, int n_envs,
                         int drones_per_env, int substeps, unsigned effects, unsigned flags, void* stream);

/* qs_ctrl_rollout with the time-varying LQR tracker of an iLQR plan in the loop (mode QS_CTRL_LQR, DESIGN.md 4.1e): io->T ticks
 * from plan tick tick0.  Tick k of the launch (plan tick p = tick0 + k), drone i:
 *   dz   = (x - z_nom[p][0:13], and with n_z = 17 rpm_prev - z_nom[p][13:17]), x the float64 state in drone_vec's order
 *          (px py pz qx qy qz qw vx vy vz wx wy wz), rpm_prev the applied RPMs of the tick before (QsState.last_rpm at k = 0);
 *   u_j  = rpm_nom[p][i][j] + s_j,  s_j = sum_{q=0}^{n_z-1} K[p][j][q] dz_q summed in that order from 0.0 (qs_ilqr_line_search's
 *          feedback term, without the feed-forward);
 *   with lo / hi: u_j = min(max(u_j, lo_j), hi_j) (qs::clampd); then the env's clip to [0, MAX_RPM of the aviary's row] and the
 *   substeps of qs_dyn_substeps(QS_FLAG_ACTION_F64) for any effect set qs_ctrl_rollout accepts.
 * QsCtrlRolloutIO.actions must be NULL; T, obs, rpm, obs_last, log and log_controls act as for QS_CTRL_RAW, and so do the env
 * state, last_rpm and the step counters.  Non-finite gains are not screened: they reach the RPMs and the clip. */
enum { QS_CTRL_LQR = 4 };
typedef struct QsLqrRolloutIO {
    const double* K;                /* [T_plan][N][4][n_z] (ilqr's layout) */
    const double* z_nom;            /* [T_plan][N][n_z] the nominal loop state before each tick */
    const double* rpm_nom;          /* [T_plan][N][4] the nominal raw commands (32-byte aligned) */
    const double* lo;               /* [N][4], or [T_plan][N][4] with per_tick (32-byte aligned); nullable together with hi */
    const double* hi;
    int per_tick;                   /* 0 or 1 */
    int n_z;                        /* 13, or 17 (the plan's loop state carries the previous clipped RPMs: needs QsState.last_rpm) */
    int T_plan;                     /* ticks of the plan, > 0 */
    int tick0;                      /* the plan tick of this launch's tick 0: 0 <= tick0, tick0 + T <= T_plan */
} QsLqrRolloutIO;
int qs_sizeof_lqr_rollout_io(void);
int qs_ctrl_rollout_lqr(const QsParams* p, const QsState* st, const QsCtrlRolloutIO* io, const QsLqrRolloutIO* lio, int n_envs,
                        int drones_per_env, int substeps, unsigned effects, unsigned flags, void* stream);

/* Differentiable raw-RPM trajectories (DESIGN.md 4.5): T control ticks of Physics.DYN (+ GND and/or DRAG, no downwash) from a
 * given state, and the reverse-mode product (VJP) of that trajectory with cotangents of its T states.  The env is not touched:
 * every input and output is a caller-owned float64 device array.  A "state" is 13 N doubles in QsState.planes' layout
 * ([pos|w.x] [quat] [vel|w.y] as [N][4] each, then w.z [N]).  Tick k applies clip(rpm[k], 0, MAX_RPM) for `substeps` substeps,
 * exactly as qs_dyn_substeps(QS_FLAG_ACTION_F64) does, and drag's first substep reads the previous tick's clipped RPMs (last_rpm
 * for tick 0).  The VJP differentiates the exponential map of _integrateQ everywhere (also where |w| <= 1e-8, where the forward
 * keeps the quaternion) and the quaternion renormalisation on tick entry; the RPM clip passes the gradient for
 * 0 <= rpm <= MAX_RPM and gives it to MAX_RPM above; the ground-effect height clip and the upright switch are differentiated
 * with the forward's predicates.  One thread per drone; deterministic. */
typedef struct QsDynTrajIO {
    int T;                          /* ticks, > 0 */
    int pad_;
    const double* state0;           /* [13 N] the state before tick 0 */
    const double* rpm;              /* [T][N][4] RPM commands (clipped in the kernel) */
    const double* last_rpm;         /* [N][4] the clipped RPMs of the tick before tick 0 (drag); nullable = zeros */
    const double* phys;             /* [n_envs][16] QsState.phys rows; nullable = the constants of QsParams */
    double* states;                 /* qs_dyn_traj out: [T][13 N], entry k = the state after tick k */
    /* qs_dyn_traj_vjp: `states` is read (the forward's output), and */
    const double* g_states;         /* [T][13 N] cotangents of the states */
    double* g_rpm;                  /* out [T][N][4] */
    double* g_state0;               /* out [13 N] */
    double* g_last_rpm;             /* out [N][4], nullable */
    double* g_phys;                 /* out [N][16]: PER DRONE (sum the drones of an aviary for its row); nullable */
    double* scratch;                /* [substeps][13][N] workspace (the substep states of one tick) */
} QsDynTrajIO;
int qs_sizeof_dyn_traj_io(void);
/* effects: 0, QS_EFFECT_GND, QS_EFFECT_DRAG or both (QS_EFFECT_DW: QS_ERR_UNSUPPORTED) */
int qs_dyn_traj(const QsParams* p, const QsDynTrajIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects, void* stream);
int qs_dyn_traj_vjp(const QsParams* p, const QsDynTrajIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                    void* stream);

/* The raw-RPM trajectories of qs_dyn_traj with downwash, and their VJP (DESIGN.md 4.5, downwash adjoint): the same arguments and
 * QsDynTrajIO, effects QS_EFFECT_DW or QS_EFFECT_GND | QS_EFFECT_DRAG | QS_EFFECT_DW only.  Each substep is qs_ctrl_rollout's:
 * the pair force from the aviary's positions at the substep's start, then one substep that renormalises the quaternion on entry;
 * so the forward is qs_ctrl_rollout's (QS_CTRL_RAW) bit for bit.  The VJP differentiates the pair term through both drones of
 * every pair that acts (the forward's predicate, no term at its jump; at dxy2 = 0 the xy derivatives are 0) and each substep's
 * entry renormalisation; the downwash coefficients and the propeller radius are constants.  One CTA of 128 threads holds whole
 * aviaries, so the pair work is O(D^2) per substep.  Refusals in this order: NULL pointers and sizes as qs_dyn_traj, then
 * QS_ERR_UNSUPPORTED for any other effect set and for drones_per_env > 128, QS_ERR_ALIGN for phys.  Deterministic (no atomics). */
int qs_dyn_traj_dw(const QsParams* p, const QsDynTrajIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                   void* stream);
int qs_dyn_traj_dw_vjp(const QsParams* p, const QsDynTrajIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                       void* stream);

/* Forward mode of the raw-RPM trajectories of qs_dyn_traj (DESIGN.md 4.5): the tangent of the T states along given tangents of
 * the inputs (JVP), and the dense Jacobians of every tick.  Both read the forward's `states` and restart each tick from the
 * stored state k-1 (state0 for k = 0), so the trajectory is linearised at the forward's bits, and both take the derivative
 * decisions of qs_dyn_traj_vjp (they are its exact transpose).  Layouts as in QsDynTrajIO.  All indices are 64-bit. */
typedef struct QsDynTrajJvpIO {
    int T;                          /* ticks, > 0 */
    int pad_;
    const double* state0;           /* [13 N] the state before tick 0 */
    const double* rpm;              /* [T][N][4] RPM commands (clipped in the kernel) */
    const double* last_rpm;         /* [N][4] the clipped RPMs of the tick before tick 0 (drag); nullable = zeros */
    const double* phys;             /* [n_envs][16] QsState.phys rows; nullable = the constants of QsParams */
    const double* states;           /* [T][13 N] qs_dyn_traj's output for these inputs */
    /* qs_dyn_traj_jvp: tangents of the inputs, each nullable = zero */
    const double* t_state0;         /* [13 N] */
    const double* t_rpm;            /* [T][N][4] of the raw (unclipped) commands */
    const double* t_last_rpm;       /* [N][4] */
    const double* t_phys;           /* [n_envs][16], 16-byte aligned */
    double* t_states;               /* qs_dyn_traj_jvp out: [T][13 N] the tangents of the states */
    /* qs_dyn_tick_jac out: [T][N][13][C], C = 17 (21 with QS_EFFECT_DRAG); row r = component r of the state after tick k (pos,
     * quat x y z w, vel, rpy_rates); columns 0..12 = the stored state before tick k, 13..16 = the raw rpm[k], and with drag
     * 17..20 = the clipped RPMs of tick k-1 (last_rpm for k = 0) */
    double* jac;
} QsDynTrajJvpIO;
int qs_sizeof_dyn_traj_jvp_io(void);
/* effects as qs_dyn_traj; QS_ERR_SIZE also when T N C / 128 exceeds 2^31-1 CTAs (qs_dyn_tick_jac) */
int qs_dyn_traj_jvp(const QsParams* p, const QsDynTrajJvpIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                    void* stream);
int qs_dyn_tick_jac(const QsParams* p, const QsDynTrajJvpIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                    void* stream);

/* Differentiable closed-loop trajectories (DESIGN.md 4.5): T control ticks of a DSLPIDControl tracking per-tick targets around
 * Physics.DYN (+ GND and/or DRAG, no downwash), and their VJP.  Tick k is the QS_CTRL_TRACK tick of qs_ctrl_rollout, in the same
 * order: pid_control with the controller's QsParams `cp` (its gains, or the aviary's row of `gains`; its model constants), the
 * controller's max_rpm clip, the env's clip (row MAX_RPM), `substeps` substeps.  States as in QsDynTrajIO; a controller state is
 * [9][N] (integral_pos_e, last_rpy, integral_rpy_e).  The VJP follows QsDynTrajIO's decisions for the physics and clips every
 * controller clip as torch.clamp; the target yaw is target_rpy[i][2] (the only component the controller reads).  One thread per
 * drone; deterministic (per-drone gradients of per-aviary rows, no atomics). */
typedef struct QsDynCtrlTrajIO {
    int T;                          /* ticks, > 0 */
    int pad_;
    double control_timestep;        /* the controller's dt, > 0 */
    const double* state0;           /* [13 N] the state before tick 0 */
    const double* pid0;             /* [9][N] the controller state before tick 0 */
    const double* target_pos;       /* [T][N][3] */
    const double* target_vel;       /* [N][3], nullable = zeros */
    const double* target_rpy;       /* [N][3], nullable = zeros */
    const double* target_rpy_rates; /* [N][3], nullable = zeros */
    const double* last_rpm;         /* [N][4] the clipped RPMs of the tick before tick 0 (drag); nullable = zeros */
    const double* phys;             /* [n_envs][16] QsState.phys rows; nullable = the constants of the env's QsParams */
    const double* gains;            /* [n_envs][18] P_FOR, I_FOR, D_FOR, P_TOR, I_TOR, D_TOR; nullable = cp's */
    double* states;                 /* qs_dyn_ctrl_traj out: [T][13 N], entry k = the state after tick k */
    double* rpm;                    /* qs_dyn_ctrl_traj out: [T][N][4] the applied (clipped) RPMs */
    double* pid_states;             /* qs_dyn_ctrl_traj out: [T][9][N] the controller state at the start of tick k */
    /* qs_dyn_ctrl_traj_vjp: states, rpm and pid_states are read (the forward's outputs), and */
    const double* g_states;         /* [T][13 N] cotangents of the states */
    const double* g_rpm_out;        /* [T][N][4] cotangents of rpm, nullable = zeros */
    double* g_state0;               /* out [13 N] */
    double* g_pid0;                 /* out [9][N], nullable */
    double* g_target_pos;           /* out [T][N][3], nullable */
    double* g_target_vel;           /* out [N][3], nullable */
    double* g_target_rpy;           /* out [N][3] (components 0 and 1 are zero), nullable */
    double* g_target_rpy_rates;     /* out [N][3], nullable */
    double* g_last_rpm;             /* out [N][4], nullable */
    double* g_phys;                 /* out [N][16]: PER DRONE (sum the drones of an aviary for its row); nullable */
    double* g_gains;                /* out [N][18]: PER DRONE; nullable */
    double* scratch;                /* [substeps][13][N] workspace */
} QsDynCtrlTrajIO;
int qs_sizeof_dyn_ctrl_traj_io(void);
/* cp: HOST pointer to the controller's QsParams.  effects as qs_dyn_traj. */
int qs_dyn_ctrl_traj(const QsParams* p, const QsParams* cp, const QsDynCtrlTrajIO* io, int n_envs, int drones_per_env, int substeps,
                     unsigned effects, void* stream);
int qs_dyn_ctrl_traj_vjp(const QsParams* p, const QsParams* cp, const QsDynCtrlTrajIO* io, int n_envs, int drones_per_env,
                         int substeps, unsigned effects, void* stream);

/* The closed-loop trajectories of qs_dyn_ctrl_traj with downwash, and their VJP: the same arguments and QsDynCtrlTrajIO, the
 * effects, layout, refusals and derivative of qs_dyn_traj_dw around the controller of qs_dyn_ctrl_traj (called once per drone per
 * tick before the substeps, as qs_ctrl_rollout's QS_CTRL_TRACK tick). */
int qs_dyn_ctrl_traj_dw(const QsParams* p, const QsParams* cp, const QsDynCtrlTrajIO* io, int n_envs, int drones_per_env, int substeps,
                        unsigned effects, void* stream);
int qs_dyn_ctrl_traj_dw_vjp(const QsParams* p, const QsParams* cp, const QsDynCtrlTrajIO* io, int n_envs, int drones_per_env,
                            int substeps, unsigned effects, void* stream);

/* Forward mode of the closed-loop trajectories of qs_dyn_ctrl_traj (DESIGN.md 4.5): the tangents of the T states and applied
 * RPMs along given tangents of the inputs (JVP), and the dense Jacobians of every closed-loop tick.  Both read the forward's
 * states, rpm and pid_states and restart tick k from the stored state k-1 (state0 for k = 0) and controller state pid_states[k],
 * so the loop is linearised at the forward's bits, and both take the derivative decisions of qs_dyn_ctrl_traj_vjp (they are its
 * exact transpose).  The controller reads the stored, unnormalised quaternion, so the closed-loop Jacobian has no quaternion null
 * space.  Layouts as in QsDynCtrlTrajIO.  All indices are 64-bit. */
typedef struct QsDynCtrlTrajJvpIO {
    int T;                          /* ticks, > 0 */
    int pad_;
    double control_timestep;        /* the controller's dt, > 0 */
    const double* state0;           /* [13 N] the state before tick 0 */
    const double* pid0;             /* [9][N] the controller state before tick 0 */
    const double* target_pos;       /* [T][N][3] */
    const double* target_vel;       /* [N][3], nullable = zeros */
    const double* target_rpy;       /* [N][3], nullable = zeros */
    const double* target_rpy_rates; /* [N][3], nullable = zeros */
    const double* last_rpm;         /* [N][4] the clipped RPMs of the tick before tick 0 (drag); nullable = zeros */
    const double* phys;             /* [n_envs][16] QsState.phys rows; nullable = the constants of the env's QsParams */
    const double* gains;            /* [n_envs][18]; nullable = cp's */
    const double* states;           /* [T][13 N] qs_dyn_ctrl_traj's states for these inputs */
    const double* rpm;              /* [T][N][4] qs_dyn_ctrl_traj's applied RPMs */
    const double* pid_states;       /* [T][9][N] qs_dyn_ctrl_traj's controller states */
    /* qs_dyn_ctrl_traj_jvp: tangents of the inputs, each nullable = zero */
    const double* t_state0;         /* [13 N] */
    const double* t_pid0;           /* [9][N] */
    const double* t_target_pos;     /* [T][N][3] */
    const double* t_target_vel;     /* [N][3] */
    const double* t_target_rpy;     /* [N][3] (only component 2, the yaw, is read) */
    const double* t_target_rpy_rates; /* [N][3] */
    const double* t_last_rpm;       /* [N][4] */
    const double* t_phys;           /* [n_envs][16], 16-byte aligned */
    const double* t_gains;          /* [n_envs][18] */
    double* t_states;               /* qs_dyn_ctrl_traj_jvp out: [T][13 N] the tangents of the states */
    double* t_rpm;                  /* qs_dyn_ctrl_traj_jvp out: [T][N][4] the tangents of the applied RPMs */
    /* qs_dyn_ctrl_tick_jac out: [T][N][26][C], C = 25 (29 with QS_EFFECT_DRAG).  Rows: x_{k+1} (13: pos, quat x y z w, vel,
     * rpy_rates), the controller state after tick k's call (9: integral_pos_e, last_rpy, integral_rpy_e), the applied RPMs u_k (4).
     * Columns: the stored x_k (13), the controller state s_k = pid_states[k] (9), with drag u_{k-1} (4, last_rpm for k = 0), then
     * target_pos[k] (3).  With z_k = (x_k, s_k[, u_{k-1}]) of n_z = 22 (26) entries, jac[..., :n_z, :n_z] is dz_{k+1} / dz_k. */
    double* jac;
} QsDynCtrlTrajJvpIO;
int qs_sizeof_dyn_ctrl_traj_jvp_io(void);
/* refusals as qs_dyn_ctrl_traj, and NULL outputs, t_phys not 16-byte aligned, QS_ERR_SIZE when T N C / 128 exceeds 2^31-1 CTAs
 * (qs_dyn_ctrl_tick_jac) */
int qs_dyn_ctrl_traj_jvp(const QsParams* p, const QsParams* cp, const QsDynCtrlTrajJvpIO* io, int n_envs, int drones_per_env,
                         int substeps, unsigned effects, void* stream);
int qs_dyn_ctrl_tick_jac(const QsParams* p, const QsParams* cp, const QsDynCtrlTrajJvpIO* io, int n_envs, int drones_per_env,
                         int substeps, unsigned effects, void* stream);

/* Differentiable policy trajectories (DESIGN.md 4.5): T control ticks of an MLP actor driving Physics.DYN (+ GND and/or DRAG, no
 * downwash) through the RPM or ONE_D_RPM action decode, and their VJP.  Tick k: the aviary's float64 observation
 * [D][12 + B A] (pos, rpy, vel, ang_v = R_last w, then the B buffered clipped actions, oldest first) of the state after tick
 * k - 1 (of state0 for k = 0, with R_last = R(q0 / |q0|)); raw = actor(obs) + exp(log_std) noise[k]; a = clip(raw, -1, 1)
 * enters the buffer; rpm = HOVER_RPM (1 + 0.05 a) (ONE_D_RPM: on all four motors), the env's MAX_RPM clip, `substeps` substeps.
 * The actor is flatten -> `depth` hidden layers (width[l] units, `activation` after each) -> linear, weights float64 row-major
 * [in][out].  A CTA owns whole aviaries for all T ticks.  The VJP follows QsDynTrajIO's decisions for the physics, clips the
 * action as torch.clamp, differentiates ReLU as h > 0 and the Euler angles on the forward's branch of the gimbal guard.  It
 * writes g_raw, the cotangent of every raw action (what the actor's weights, log_std and the noise need: one batched pass over
 * the saved observations); the weights' gradients themselves are not formed here.  Deterministic (no atomics). */
typedef struct QsDynPolicyTrajIO {
    int T;                          /* ticks, > 0 */
    int act_buffer_size;            /* B > 0 */
    int activation;                 /* QS_MLP_TANH or QS_MLP_RELU */
    int depth;                      /* hidden layers, 1 .. QS_MLP_MAX_HIDDEN */
    int width[QS_MLP_MAX_HIDDEN];   /* hidden widths, 1 .. QS_MLP_MAX_WIDTH (unpadded) */
    int in_dim, out_dim;            /* D (12 + B A) and D A <= 32 */
    const double* w[QS_MLP_MAX_HIDDEN + 1];   /* [in][out] row-major per layer */
    const double* b[QS_MLP_MAX_HIDDEN + 1];   /* [out] */
    const double* log_std;          /* [out_dim] */
    const double* noise;            /* [T][n_envs][out_dim], nullable = the mean action */
    const double* state0;           /* [13 N] the state before tick 0 */
    const double* last_rpm;         /* [N][4] the clipped RPMs of the tick before tick 0 (drag); nullable = zeros */
    const double* phys;             /* [n_envs][16] QsState.phys rows; nullable = the constants of QsParams */
    const double* action_buffer;    /* [N][B][A] the buffered actions before tick 0, oldest first */
    double* states;                 /* qs_dyn_policy_traj out: [T][13 N], entry k = the state after tick k */
    double* actions;                /* qs_dyn_policy_traj out: [T][N][A] the raw (unclipped) actions */
    double* obs;                    /* qs_dyn_policy_traj out: [T][n_envs][in_dim] what the actor saw at tick k */
    /* qs_dyn_policy_traj_vjp: states, actions and obs are read (the forward's outputs), and */
    const double* g_states;         /* [T][13 N] cotangents of the states */
    const double* g_actions;        /* [T][N][A] cotangents of the raw actions, nullable = zeros */
    double* g_raw;                  /* out [T][N][A]: the whole cotangent of raw action k (g_actions included) */
    double* g_state0;               /* out [13 N] */
    double* g_last_rpm;             /* out [N][4], nullable */
    double* g_phys;                 /* out [N][16]: PER DRONE (sum the drones of an aviary for its row); nullable */
    double* g_action_buffer;        /* out [N][B][A], nullable */
    double* scratch;                /* [substeps][13][N] workspace */
} QsDynPolicyTrajIO;
int qs_sizeof_dyn_policy_traj_io(void);
/* act_type: QS_ACT_RPM or QS_ACT_ONE_D_RPM (others: QS_ERR_UNSUPPORTED).  effects as qs_dyn_traj.  QS_ERR_UNSUPPORTED also for
 * drones_per_env > 32 or D A > 32, and where the VJP's rows of 8 aviaries (per aviary in_dim + depth * max width + out_dim +
 * 2 max(in_dim, max width) + D B A doubles) exceed the 227 KB of a CTA's shared memory: the forward refuses what its VJP would. */
int qs_dyn_policy_traj(const QsParams* p, const QsDynPolicyTrajIO* io, int act_type, int n_envs, int drones_per_env, int substeps,
                       unsigned effects, void* stream);
int qs_dyn_policy_traj_vjp(const QsParams* p, const QsDynPolicyTrajIO* io, int act_type, int n_envs, int drones_per_env,
                           int substeps, unsigned effects, void* stream);

/* Forward mode of the policy trajectories of qs_dyn_policy_traj (DESIGN.md 4.5): the tangents of the T states and raw actions
 * along given tangents of the inputs (JVP), and the dense Jacobians of every tick of every aviary.  Both read the forward's
 * states, actions and obs and restart tick k from the stored state k-1 (state0 for k = 0), the saved observation obs[k] and the
 * stored raw actions, so the loop is linearised at the forward's bits, and both take the derivative decisions of
 * qs_dyn_policy_traj_vjp (they are its exact transpose).  The actor's parameters and the noise enter through t_raw_in, the tangent
 * they add to each raw action (J_theta t_theta + exp(log_std) (t_log_std noise + t_noise), formed by the caller over the saved
 * observations).  The fields up to obs are QsDynPolicyTrajIO's.  All indices are 64-bit.
 *
 * The loop state z_k of an aviary is drone-major; per drone: pos (3), quat x y z w (4), vel (3), rpy_rates (3), the observation's
 * ang_v (3: R_last w, which is neither an input nor an output of the trajectory), the B buffered clipped actions (B A, oldest
 * first) and with QS_EFFECT_DRAG the applied RPMs of the previous tick (4): n_z = D (16 + B A), or D (20 + B A) with drag. */
typedef struct QsDynPolicyTrajJvpIO {
    int T;                          /* ticks, > 0 */
    int act_buffer_size;            /* B > 0 */
    int activation;                 /* QS_MLP_TANH or QS_MLP_RELU */
    int depth;                      /* hidden layers, 1 .. QS_MLP_MAX_HIDDEN */
    int width[QS_MLP_MAX_HIDDEN];   /* hidden widths, 1 .. QS_MLP_MAX_WIDTH (unpadded) */
    int in_dim, out_dim;            /* D (12 + B A) and D A <= 32 */
    const double* w[QS_MLP_MAX_HIDDEN + 1];   /* [in][out] row-major per layer */
    const double* b[QS_MLP_MAX_HIDDEN + 1];   /* [out] */
    const double* log_std;          /* [out_dim] */
    const double* noise;            /* [T][n_envs][out_dim], nullable */
    const double* state0;           /* [13 N] the state before tick 0 */
    const double* last_rpm;         /* [N][4] (drag); nullable = zeros */
    const double* phys;             /* [n_envs][16]; nullable = the constants of QsParams */
    const double* action_buffer;    /* [N][B][A] */
    const double* states;           /* [T][13 N] qs_dyn_policy_traj's states for these inputs */
    const double* actions;          /* [T][N][A] qs_dyn_policy_traj's raw actions */
    const double* obs;              /* [T][n_envs][in_dim] qs_dyn_policy_traj's observations */
    /* qs_dyn_policy_traj_jvp: tangents of the inputs, each nullable = zero */
    const double* t_state0;         /* [13 N] */
    const double* t_last_rpm;       /* [N][4] */
    const double* t_phys;           /* [n_envs][16], 16-byte aligned (HOVER_RPM enters through the decode, MAX_RPM the clip) */
    const double* t_action_buffer;  /* [N][B][A] */
    const double* t_raw_in;         /* [T][N][A] the tangent the actor's parameters and the noise add to raw action k */
    double* t_states;               /* qs_dyn_policy_traj_jvp out: [T][13 N] the tangents of the states */
    double* t_actions;              /* qs_dyn_policy_traj_jvp out: [T][N][A] the tangents of the raw actions */
    /* qs_dyn_policy_tick_jac out: [T][n_envs][R][R], R = n_z + D A.  Rows: z_{k+1}, then raw_k (D A, drone-major).  Columns: z_k,
     * then delta_k, an additive perturbation of raw_k (the noise's columns are delta's times exp(log_std)); the raw_k x delta_k
     * block is the identity.  The tangents are NULL here. */
    double* jac;
} QsDynPolicyTrajJvpIO;
int qs_sizeof_dyn_policy_traj_jvp_io(void);
/* refusals as qs_dyn_policy_traj, and NULL outputs, t_phys not 16-byte aligned, QS_ERR_SIZE when the grid exceeds 2^31-1 CTAs */
int qs_dyn_policy_traj_jvp(const QsParams* p, const QsDynPolicyTrajJvpIO* io, int act_type, int n_envs, int drones_per_env,
                           int substeps, unsigned effects, void* stream);
int qs_dyn_policy_tick_jac(const QsParams* p, const QsDynPolicyTrajJvpIO* io, int act_type, int n_envs, int drones_per_env,
                           int substeps, unsigned effects, void* stream);

/* Batched iLQR of raw-RPM trajectories (DESIGN.md 4.5.1): Gauss-Newton DDP, one independent problem per drone (no downwash).
 * Drone i minimises J = 1/2 sum_k (x_k - r_k)' W_k (x_k - r_k) + 1/2 sum_k (u_k - u_ref)' Rt (u_k - u_ref) over its raw commands
 * u_k = rpm[k], where x_k is the state after tick k (qs_dyn_traj's states[k]), W_k = diag(Q) for k < T-1 and diag(Q_final) for
 * k = T-1, and Rt = diag(R) / HOVER_RPM^2 with the drone's row constants.  The loop state is z_k = x_{k-1} (state0 for k = 0),
 * n_z = 13, or with drag z_k = (x_{k-1}, the clipped u_{k-1}), n_z = 17.  One iteration is qs_dyn_tick_jac at the nominal,
 * qs_ilqr_backward, qs_ilqr_line_search and qs_ilqr_commit; none of them reads anything back to the host.  The rollouts of the
 * line search and the commit are qs_dyn_traj's ticks, so a committed trajectory is qs_dyn_traj's output for the committed rpm. */
typedef struct QsIlqrIO {
    int T;                          /* ticks, > 0 */
    int n_alpha;                    /* qs_ilqr_line_search / qs_ilqr_commit: step sizes in alpha, 1..16 */
    const double* jac;              /* [T][N][13][C] qs_dyn_tick_jac's output at the nominal (qs_ilqr_backward) */
    const double* state0;           /* [13 N] the state before tick 0 */
    const double* last_rpm;         /* [N][4] the clipped RPMs of the tick before tick 0 (drag); nullable = zeros */
    const double* phys;             /* [n_envs][16] QsState.phys rows; nullable = the constants of QsParams */
    const double* targets;          /* [T][13 N] r_k in the planes layout of the states */
    const double* weights;          /* [n_envs][30]: Q (13), Q_final (13), R (4), all >= 0 and R > 0 (not checked here) */
    const double* rpm_ref;          /* [N][4] u_ref */
    const double* alpha;            /* [n_alpha] step sizes */
    double* states;                 /* [T][13 N] the nominal trajectory; qs_ilqr_commit: in/out */
    double* rpm;                    /* [T][N][4] the nominal raw commands; qs_ilqr_commit: in/out */
    double* mu;                     /* [N] the regularisation; qs_ilqr_backward and qs_ilqr_commit: in/out */
    double* K;                      /* [T][N][4][n_z] feedback gains (qs_ilqr_backward out); line search / commit: nullable = 0 */
    double* k;                      /* [T][N][4] feed-forward gains (qs_ilqr_backward out); line search / commit: nullable = 0 */
    double* dV;                     /* [N][2] sum k'Qu and 1/2 sum k'Quu k of the backward pass (qs_ilqr_backward out) */
    double* J;                      /* [n_alpha][N] J(alpha) (qs_ilqr_line_search out, qs_ilqr_commit in) */
    int* status;                    /* [N] 0, or 1 when Quu stayed indefinite through 8 raised regularisations (qs_ilqr_backward
                                     * out); line search: nullable = 0 */
    unsigned char* converged;       /* [N] 0 / 1 (qs_ilqr_commit in/out); line search: nullable = 0 */
    const double* cost_in;          /* [N] the nominal's J (qs_ilqr_commit) */
    double* cost_out;               /* [N] the committed J (qs_ilqr_commit out) */
} QsIlqrIO;
int qs_sizeof_ilqr_io(void);
/* Backward pass (Riccati recursion) at the nominal, for k = T-1 .. 0: V += the stage cost of x_k; Qx = A'V_x,
 * Qu = Rt (u_k - u_ref) + B'V_x, Qxx = A'V_xx A, Quu = Rt + B'V_xx B, Qux = B'V_xx A; Quu_mu = Quu + mu diag(Quu) by a 4x4
 * Cholesky; k = -Quu_mu^-1 Qu, K = -Quu_mu^-1 Qux; V_x = Qx + K'Quu k + K'Qu + Qux'k, V_xx = Qxx + K'Quu K + K'Qux + Qux'K,
 * symmetrised.  A failed Cholesky sets mu = max(1e-6, 10 mu) and restarts the drone's pass, at most 8 times.  With drag
 * A = [[A_x, B_last], [0, 0]] and B = [[B_x], [diag(clip'(u_k))]].  One warp per drone. */
int qs_ilqr_backward(const QsParams* p, const QsIlqrIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                     void* stream);
/* J(alpha_a) of the rollout u_k = rpm[k] + alpha_a k_k + K_k (z_k - z_nom,k) from z_nom,0, for every drone and step size; no state
 * is stored.  A drone with status != 0 or converged gets +inf. */
int qs_ilqr_line_search(const QsParams* p, const QsIlqrIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                        void* stream);
/* Per drone: the largest alpha with J(alpha) < cost_in and cost_in - J(alpha) >= 1e-4 (-(alpha dV1 + alpha^2 dV2)).  If there is
 * one, its rollout overwrites states and rpm, cost_out = its J (the line search's bits), mu = mu / 10 (0 below 1e-6), and a
 * relative decrease below 1e-9 sets converged; otherwise cost_out = cost_in and mu = max(1e-6, 10 mu).  A converged drone is
 * left as it is. */
int qs_ilqr_commit(const QsParams* p, const QsIlqrIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                   void* stream);

/* Control-limited iLQR (DESIGN.md 4.5.1): the problem of QsIlqrIO with every raw command held to the box
 * rpm_lo <= u_k <= rpm_hi.  The bounds must satisfy 0 <= rpm_lo <= rpm_hi <= MAX_RPM of the drone's row (not checked here), and
 * the nominal rpm must lie in the box: the clip to [0, MAX_RPM] in the dynamics then never binds. */
typedef struct QsIlqrBoxIO {
    QsIlqrIO base;                  /* as for qs_ilqr_backward / qs_ilqr_line_search / qs_ilqr_commit */
    const double* rpm_lo;           /* [N][4] raw RPM, or [T][N][4] with per_tick */
    const double* rpm_hi;           /* [N][4] raw RPM, or [T][N][4] with per_tick */
    int per_tick;                   /* 0: one box per drone; 1: one per tick and drone */
    int pad_;
    signed char* active;            /* [T][N][4] qs_ilqr_box_backward out: -1 where k_k holds a rotor at rpm_lo, +1 at rpm_hi,
                                     * 0 free; nullable */
} QsIlqrBoxIO;
int qs_sizeof_ilqr_box_io(void);
/* qs_ilqr_backward with k_k = argmin 1/2 k'Quu_mu k + Qu'k subject to rpm_lo,k - u_k <= k <= rpm_hi,k - u_k: the unconstrained k
 * when it lies in the box (then K, k and dV are qs_ilqr_backward's bits), otherwise a projected-Newton box QP from clamp(0) on
 * Quu_mu.  Rows of K on held rotors are 0, free rows -(Quu_mu,ff)^-1 Qux,f; dV and the value update take this k and K.  A free
 * block without a Cholesky factor restarts the pass as a failed Quu_mu does.  Refusals as qs_ilqr_backward, and NULL
 * rpm_lo / rpm_hi, per_tick not 0 or 1. */
int qs_ilqr_box_backward(const QsParams* p, const QsIlqrBoxIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                         void* stream);
/* qs_ilqr_line_search with u_k clamped to [rpm_lo,k, rpm_hi,k] before the tick and the stage cost */
int qs_ilqr_box_line_search(const QsParams* p, const QsIlqrBoxIO* io, int n_envs, int drones_per_env, int substeps,
                            unsigned effects, void* stream);
/* qs_ilqr_commit with u_k clamped as in the line search; the clamped u_k is stored.  A drone with status 0 and dV1 = dV2 = 0
 * (k = 0 at every tick, e.g. every rotor held at a bound) is set converged with cost_out = cost_in and mu unchanged. */
int qs_ilqr_box_commit(const QsParams* p, const QsIlqrBoxIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                       void* stream);

/* The derivative of an iLQR solution (DESIGN.md 4.5.1 "Gradients of the solution"): given the cotangents g_X of the solution's
 * states and g_U of its rpm, the adjoint LQR  min_w 1/2 sum dx_k' W_k dx_k + 1/2 sum w_k' Rt w_k - sum g_X,k . dx_k
 * - sum g_U,k . w_k  with dz_0 = 0, dz_{k+1} = F_k [dz_k; w_k] and w = 0 on held rotors, where F_k = [A | B] is the solve's (from
 * qs_dyn_tick_jac at the solution, with drag's rows of the clipped RPMs) and W_k, Rt are QsIlqrIO's.  Its solution
 * w_S = H_SS^-1 G_S (H = J'W J + Rt the Gauss-Newton Hessian, G = g_U + J'g_X, J = dX/dU, S the free rotor-ticks) gives the
 * solution's gradients (ilqr.IlqrSolution).  One warp per drone in both entry points. */
typedef struct QsIlqrAdjointIO {
    int T;                          /* ticks, > 0 */
    int pad_;
    const double* jac;              /* [T][N][13][C] qs_dyn_tick_jac's output at the solution */
    const double* rpm;              /* [T][N][4] the solution's raw commands (drag: the clip's derivative) */
    const double* phys;             /* [n_envs][16] QsState.phys rows (16-byte aligned); nullable = the constants of QsParams */
    const double* weights;          /* [n_envs][30]: Q (13), Q_final (13), R (4), as QsIlqrIO */
    const signed char* active;      /* [T][N][4] the held rotors (nonzero) of the solve's last backward pass; nullable = none held
                                     * (then the unconstrained kernels run) */
    const double* g_states;         /* [T][13 N] g_X in the planes layout of the states (qs_ilqr_adjoint) */
    const double* g_rpm;            /* [T][N][4] g_U; nullable = zeros (qs_ilqr_adjoint) */
    double* K;                      /* [T][N][4][n_z] the adjoint's feedback gains: qs_ilqr_adjoint out, rollout in */
    double* k;                      /* [T][N][4] its feed-forward: qs_ilqr_adjoint out, rollout in */
    int* status;                    /* [N] 0, or 1 when a tick's free block of Quu has no Cholesky factor: qs_ilqr_adjoint out,
                                     * rollout in */
    double* w;                      /* [T][N][4] qs_ilqr_adjoint_rollout out: w_k, 0 on held rotors; NaN where status != 0 */
    double* dx;                     /* [T][13 N] qs_ilqr_adjoint_rollout out: the state part of dz_{k+1}; NaN where status != 0 */
} QsIlqrAdjointIO;
int qs_sizeof_ilqr_adjoint_io(void);
/* The adjoint's Riccati pass, k = T-1 .. 0: qs_ilqr_backward's recursion at mu = 0 with the stage's linear term -g_X,k (V_x),
 * Qu = -g_U,k + B'V_x, and the held rotors of `active` fixed at 0: Quu's free block is factored (held rows and columns replaced
 * by the identity), k = -Quu_ff^-1 Qu_f and K = -Quu_ff^-1 Qux_f on free rotors, 0 on held ones.  Without `active` K is
 * qs_ilqr_backward's K at mu = 0 bit for bit.  No regularisation ladder: a failed factor sets status = 1 and leaves the ticks
 * below it unwritten.  Refusals, in this order: NULL params / io, NULL jac / rpm / weights / K / k / status, NULL g_states,
 * sizes, effects (QS_ERR_UNSUPPORTED for downwash), phys alignment. */
int qs_ilqr_adjoint(const QsParams* p, const QsIlqrAdjointIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                    void* stream);
/* The adjoint's linear forward pass: w_k = k_k + K_k dz_k (0 on held rotors), dz_{k+1} = F_k [dz_k; w_k] from dz_0 = 0, each sum
 * in index order from 0.0.  Refusals as qs_ilqr_adjoint, with NULL w / dx in place of NULL g_states. */
int qs_ilqr_adjoint_rollout(const QsParams* p, const QsIlqrAdjointIO* io, int n_envs, int drones_per_env, int substeps,
                            unsigned effects, void* stream);

/* Differentiable tracker loops (DESIGN.md 4.5): T control ticks of an iLQR plan's time-varying LQR tracker around Physics.DYN
 * (+ GND and/or DRAG, no downwash), and their VJP.  Tick k (plan tick p = tick0 + k) is the QS_CTRL_LQR tick of
 * qs_ctrl_rollout_lqr, in the same order: dz from the state and the RPMs applied at the tick before (last_rpm at k = 0),
 * u = rpm_nom[p] + K[p] dz, the optional box clampd(u, lo, hi), the env's clip to [0, MAX_RPM of the row], `substeps` substeps.
 * States as in QsDynTrajIO, the plan in ilqr's layout as in QsLqrRolloutIO.  The VJP follows QsDynTrajIO's decisions for the
 * physics and the env's clip; the box is torch.clamp with constant bounds (the gradient passes for lo <= u <= hi); the law is
 * linear: g_rpm_nom[p] = lambda, g_K[p] = lambda dz^T, g_z_nom[p] = -K[p]^T lambda, and K[p]^T lambda joins the cotangent of the
 * stored state (its quaternion unnormalised) and, with n_z = 17, of the RPMs applied at the tick before.  One thread per drone;
 * deterministic (per-drone gradients of per-aviary rows, no atomics). */
typedef struct QsDynLqrTrajIO {
    int T;                          /* ticks, > 0 */
    int n_z;                        /* 13, or 17 (dz carries the RPMs applied at the tick before) */
    int T_plan;                     /* ticks of the plan */
    int tick0;                      /* the plan tick of tick 0: 0 <= tick0, tick0 + T <= T_plan */
    int per_tick;                   /* 0: lo / hi are [N][4]; 1: [T_plan][N][4] */
    int pad_;
    const double* state0;           /* [13 N] the state before tick 0 */
    const double* last_rpm;         /* [N][4] the RPMs applied at the tick before tick 0 (drag, n_z = 17); nullable = zeros */
    const double* phys;             /* [n_envs][16] QsState.phys rows (16-byte aligned); nullable = the constants of QsParams */
    const double* K;                /* [T_plan][N][4][n_z] */
    const double* z_nom;            /* [T_plan][N][n_z] */
    const double* rpm_nom;          /* [T_plan][N][4] (32-byte aligned) */
    const double* lo;               /* the box (32-byte aligned); nullable together with hi = no box */
    const double* hi;
    double* states;                 /* qs_dyn_lqr_traj out: [T][13 N], entry k = the state after tick k */
    double* rpm;                    /* qs_dyn_lqr_traj out: [T][N][4] the applied (clipped) RPMs */
    /* qs_dyn_lqr_traj_vjp: states and rpm are read (the forward's outputs), and */
    const double* g_states;         /* [T][13 N] cotangents of the states */
    const double* g_rpm;            /* [T][N][4] cotangents of rpm, nullable = zeros */
    double* g_state0;               /* out [13 N] */
    double* g_last_rpm;             /* out [N][4], nullable */
    double* g_phys;                 /* out [N][16]: PER DRONE (sum the drones of an aviary for its row); nullable */
    double* g_K;                    /* out [T_plan][N][4][n_z]: the flown plan ticks only are written; nullable */
    double* g_z_nom;                /* out [T_plan][N][n_z]: the flown plan ticks only are written; nullable */
    double* g_rpm_nom;              /* out [T_plan][N][4]: the flown plan ticks only are written; nullable */
    double* scratch;                /* [substeps][13][N] workspace */
} QsDynLqrTrajIO;
int qs_sizeof_dyn_lqr_traj_io(void);
/* effects as qs_dyn_traj.  Refusals, in this order: NULL pointers, sizes, effects (QS_ERR_ENUM, QS_ERR_UNSUPPORTED for downwash),
 * n_z not 13 or 17, ticks outside the plan, only one of lo and hi, per_tick not 0 or 1, alignment. */
int qs_dyn_lqr_traj(const QsParams* p, const QsDynLqrTrajIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                    void* stream);
int qs_dyn_lqr_traj_vjp(const QsParams* p, const QsDynLqrTrajIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                        void* stream);

/* MPPI (model predictive path integral) trajectory optimisation (DESIGN.md 4.5.2): the cost J of QsIlqrIO, minimised by
 * importance-weighted averages of random perturbations of the nominal rpm.  The unit of a decision is the drone, or with
 * downwash (effects & QS_EFFECT_DW) the aviary, whose J is the sum of its drones' J in drone order.  One iteration is
 * qs_mppi_sample, qs_mppi_update and qs_mppi_commit; none of them reads anything back to the host.
 * Noise: eps[k][s][i][r] = the normals of Philox4x32-10 with key (seed & 0xffffffff, seed >> 32) and counter
 * (k, s, i, 2 iteration + h), whose words (w0, w1) and (w2, w3) give u = ((w << 32 | w') >> 11 + 0.5) 2^-53 and by Box-Muller
 * rotors 2h and 2h + 1; eps = 0 for sample 0.  Sample s applies v_k = u_k + sig_i eps (sig_i = sigma[e] HOVER_RPM of the row),
 * clamped to [rpm_lo, rpm_hi] with a box; its perturbation is delta = v - u with a box, sig_i eps without.  Nothing of size
 * K T N is stored: the update regenerates eps from the counter. */
typedef struct QsMppiIO {
    int T;                          /* ticks, > 0 */
    int K;                          /* samples, 2..1024; sample 0 is the nominal */
    int iteration;                  /* >= 0: the noise's counter */
    int per_tick;                   /* 0: rpm_lo / rpm_hi are [N][4]; 1: [T][N][4] */
    unsigned long long seed;        /* the noise's key */
    double temperature;             /* finite, > 0 (qs_mppi_update) */
    const double* state0;           /* [13 N] the state before tick 0 */
    const double* last_rpm;         /* [N][4] the clipped RPMs of the tick before tick 0 (drag); nullable = zeros */
    const double* phys;             /* [n_envs][16] QsState.phys rows (16-byte aligned); nullable = the constants of QsParams */
    const double* targets;          /* [T][13 N], as QsIlqrIO */
    const double* weights;          /* [n_envs][30], as QsIlqrIO */
    const double* rpm_ref;          /* [N][4], as QsIlqrIO */
    const double* sigma;            /* [n_envs] the noise scale relative to HOVER_RPM, finite and > 0 (not checked here) */
    const double* rpm_lo;           /* the box, nullable together with rpm_hi = none; as QsIlqrBoxIO, and the nominal lies in it */
    const double* rpm_hi;
    double* rpm;                    /* [T][N][4] the nominal raw commands: qs_mppi_commit in/out, the others in */
    double* states;                 /* [T][13 N] the nominal's trajectory: qs_mppi_commit out */
    double* J;                      /* [K][N] each drone's J of each sample: qs_mppi_sample out, update and commit in */
    double* cand;                   /* [T][N][4] the candidate: qs_mppi_update out, qs_mppi_commit in (NULL: see commit) */
    double* cost_out;               /* [N] each drone's J of the committed nominal: qs_mppi_commit out */
    int* pick;                      /* qs_mppi_commit out, nullable: per unit, [N] by drone or with downwash [n_envs] by aviary;
                                     * -1 the candidate was kept, else the sample taken */
    double* noise;                  /* [K][T][N][4] qs_mppi_noise out */
} QsMppiIO;
int qs_sizeof_mppi_io(void);
/* J[s][i] of every sample's rollout (qs_ilqr_line_search's ticks and stage cost with the sample's commands); no state is
 * stored.  Without downwash one thread per (drone, sample); with downwash whole (aviary, sample) groups per 128-thread CTA, the
 * positions shared every substep as qs_ctrl_rollout does.  Refusals, in this order: NULL params / io, NULL pointers, sizes
 * (T, K in 2..1024, iteration >= 0, the grid), per_tick not 0 or 1, only one of rpm_lo and rpm_hi, effects (QS_ERR_ENUM;
 * QS_ERR_UNSUPPORTED outside 0, GND, DRAG, GND|DRAG, DW, GND|DRAG|DW, or downwash with drones_per_env > 128), phys alignment.
 * qs_mppi_update and qs_mppi_commit refuse the same, and a temperature that is not finite and > 0 (update). */
int qs_mppi_sample(const QsParams* p, const QsMppiIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                   void* stream);
/* One warp per unit: J_min, the mean over the finite J_s, lambda = temperature (mean - J_min), w_s = exp(-(J_s - J_min) /
 * lambda) (1 when lambda = 0, 0 for a non-finite J_s), each sum in s order; cand = u + sum_s w_s delta_s / sum_s w_s with the
 * noise regenerated per entry (the nominal when no J_s is finite). */
int qs_mppi_update(const QsParams* p, const QsMppiIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                   void* stream);
/* Rolls out the candidate (clamped to the box), then per unit keeps it when its J is <= the best sample's J (the lowest s
 * with the least finite J), otherwise takes that sample's commands; writes rpm, states, cost_out and pick.  With cand NULL it
 * rolls out the nominal itself into states and cost_out (J is not read): the trajectory before the first iteration. */
int qs_mppi_commit(const QsParams* p, const QsMppiIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                   void* stream);
/* noise[s][k][i][r] = eps of (T, K, seed, iteration) for every sample, tick, drone and rotor.  Refusals: NULL io / noise, sizes. */
int qs_mppi_noise(const QsMppiIO* io, int n_envs, int drones_per_env, void* stream);

/* Reset envs to their initial pose.  mask: [E] bytes, nullable = all envs.  Zeroes velocities, body rates,
 * last_rpm, step counter; with reset_pid != 0 also the PID state (the reference never does, SURVEY.md 3.3).
 * If obs != NULL also refreshes the kinematic part of the RL observation rows (obs_dim > 0) or the [N][20]
 * state vectors (obs_dim == 20 and act_buffer_size == 0). */
int qs_reset(const QsParams* p, const QsState* st, const unsigned char* mask, int n_envs, int drones_per_env,
             int reset_pid, float* obs, int obs_dim, int raw_state20, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* QUADSIM_H_ */
