// rollout_ctrl.cu -- qs_ctrl_rollout: T control ticks of the control envs per launch (DESIGN.md 4.1e).  CtrlAviary with given RPMs
// (RAW), VelocityAviary (VEL, the embedded controller on QsState.pid) and CtrlAviary driven by a DSLPIDControl that tracks a
// waypoint schedule (TRACK: the pid.py / downwash.py loop, computeControlFromEnv + step, inside the kernel).  Unlike qs_rollout there
// is no action history: the state vector rows are written from registers through a small shared-memory stage, so this is a
// translation unit of its own and leaves every rollout_kernel entry as it was.
#include "qs_common.cuh"

namespace qsi {
namespace {

constexpr int kCtrlTPB = 128;

struct CtrlRolloutArgs {
    QsParams P;          // the env: physics, MAX_RPM clip, the embedded controller of VEL
    QsParams CP;         // TRACK: the DSLPIDControl's own constants (gains, model, g, max_rpm)
    QsState st;
    QsCtrlRolloutIO io;
    QsLogRing rg;        // valid iff has_log
    long long N;
    int n_envs, D, substeps, tpb;
    unsigned flags;
    int has_log;
};

// the state stored back at the end of the rollout: the quaternion is already renormalised (round_to_planes after every tick), so
// it is stored as it is -- store_drone would renormalise a second time and could move the last bit
__device__ __forceinline__ void store_drone_rounded(const QsState& st, long long N, long long i, const qs::Drone& d) {
    st256(st.planes, i, d.px, d.py, d.pz, d.wx);
    st256(st.planes, N + i, d.qx, d.qy, d.qz, d.qw);
    st256(st.planes, 2 * N + i, d.vx, d.vy, d.vz, d.wy);
    st.planes[12 * N + i] = d.wz;
    if (st.pos_f32) st4(st.pos_f32, i, make_float4((float)d.px, (float)d.py, (float)d.pz, 0.f));
}

// what store_drone + load_drone do to the state between two ticks (the rollout kernel's helper): the quaternion is renormalised
__device__ __forceinline__ void round_to_planes(qs::Drone& d) {
    const double inv = rsqrt(qs::quat_norm2(d.qx, d.qy, d.qz, d.qw));
    d.qx = __dmul_rn(d.qx, inv); d.qy = __dmul_rn(d.qy, inv); d.qz = __dmul_rn(d.qz, inv); d.qw = __dmul_rn(d.qw, inv);
}

// TRACK targets of drone i at tick k (include/quadsim.h, QsCtrlRolloutIO): the waypoint row (start[i] + k) mod W, column 0 (M = 1)
// or i (M = N), plus offset[i]
__device__ __forceinline__ void track_target(const QsCtrlRolloutIO& io, long long N, long long i, int k, double& tx, double& ty, double& tz) {
    long long r = ((long long)__ldg(io.start + i) + k) % io.W;
    if (r < 0) r += io.W;
    const double* w = io.waypoints + (r * io.M + (io.M == 1 ? 0 : i)) * 3;
    tx = __ldg(w); ty = __ldg(w + 1); tz = __ldg(w + 2);
    if (io.offset) { tx = tx + __ldg(io.offset + 3 * i); ty = ty + __ldg(io.offset + 3 * i + 1); tz = tz + __ldg(io.offset + 3 * i + 2); }
}
__device__ __forceinline__ void const_target(const double* p, long long i, double& x, double& y, double& z) {
    if (p) { x = __ldg(p + 3 * i); y = __ldg(p + 3 * i + 1); z = __ldg(p + 3 * i + 2); } else { x = y = z = 0.0; }
}

// MODE = QS_CTRL_RAW / VEL / TRACK; EFF = the DYN+ set (0, GND, DRAG, DW, all three); PHYS = the per-aviary constants table.
// One thread per drone for all T ticks: the drone, the controller state and (drag) the previous RPMs stay in registers and are
// stored once at the end.  Per tick and substep the arithmetic is the code of qs_dyn_substeps / qs_step(VEL) / pid_state_kernel,
// in the same order, so the rollout gives their bits.
// 128 registers (4 CTAs of 128 threads per SM): the entries with the controller in the loop spill some of their state at that
// size, but on the H100 the occupancy pays more than the registers (168 or 255 registers were slower, DESIGN.md 4.1e).
template <int EFF, int MODE, bool PHYS>
__global__ void __launch_bounds__(kCtrlTPB, 4) ctrl_rollout_kernel(const __grid_constant__ CtrlRolloutArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const QsParams& P = a.P;
    const QsCtrlRolloutIO& io = a.io;
    const int tpb = a.tpb, D = a.D, T = io.T, t = threadIdx.x;
    const long long N = a.N;
    const long long c0 = (long long)blockIdx.x * tpb;
    const long long i = c0 + t;
    const bool live = (t < tpb) && (i < N);
    const int rows = (int)((N - c0) < tpb ? (N - c0) : tpb);
    float* row_s = reinterpret_cast<float*>(smem_raw);                               // [tpb][20] state vector rows
    double* pos_s = reinterpret_cast<double*>(row_s + (size_t)tpb * 20);              // [tpb][3] in-CTA downwash
    const long long e = live ? i / D : 0;
    const int le = t / D;

    qs::Drone d;
    qs::PidState pst = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    double rpm_prev[4] = {0, 0, 0, 0};
    int sc = 0;
    long long lj = -1, head0 = 0;                // the Logger ring: my entry column, the ring head before the first tick
    if (live) {
        load_drone(a.st.planes, N, i, d);
        if ((EFF & QS_EFFECT_DRAG) && a.st.last_rpm) load_rpm(a.st.last_rpm, i, rpm_prev);
        if (MODE == QS_CTRL_VEL) load_pid(a.st.pid, N, i, pst);
        if (MODE == QS_CTRL_TRACK) load_pid(io.pid_state, N, i, pst);
        sc = a.st.step_counter[e];
        if (a.has_log && i >= a.rg.first_drone && i < (long long)a.rg.first_drone + a.rg.n_drones) {
            lj = i - a.rg.first_drone;
            head0 = *a.rg.head;
        }
    }
    const bool rows_out = io.obs != nullptr;
    double rpm[4] = {0, 0, 0, 0};
    for (int k = 0; k < T; ++k) {
        // ---- this tick's RPMs ----------------------------------------------------------------------------------------
        double R_last[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
        qs::PhysRow ph;
        double pe[3] = {0, 0, 0}, ye = 0.0;
        if (live) {
            if constexpr (MODE == QS_CTRL_RAW) {
                const double mr = PHYS ? load_phys_rpm(a.st.phys, e).max_rpm : P.max_rpm;
                if (a.flags & QS_FLAG_ACTION_F64) {
                    const D4 v = ld256_nc(static_cast<const double*>(io.actions), (long long)k * N + i);
                    rpm[0] = qs::clampd(v.x, 0.0, mr); rpm[1] = qs::clampd(v.y, 0.0, mr);                     // CtrlAviary.py:140
                    rpm[2] = qs::clampd(v.z, 0.0, mr); rpm[3] = qs::clampd(v.w, 0.0, mr);
                } else {
                    const float4 v = ldg4(static_cast<const float*>(io.actions), (long long)k * N + i);
                    rpm[0] = qs::clampd((double)v.x, 0.0, mr); rpm[1] = qs::clampd((double)v.y, 0.0, mr);
                    rpm[2] = qs::clampd((double)v.z, 0.0, mr); rpm[3] = qs::clampd((double)v.w, 0.0, mr);
                }
            } else if constexpr (MODE == QS_CTRL_VEL) {
                const float4 v = ldg4(static_cast<const float*>(io.actions), (long long)k * N + i);
                const float act[4] = {v.x, v.y, v.z, v.w};
                double r_, p_, cur_yaw;
                qs::quat_to_euler<false>(d.qx, d.qy, d.qz, d.qw, r_, p_, cur_yaw);
                if constexpr (PHYS) qs::decode_action_k<true>(P, load_phys_rpm(a.st.phys, e), QS_ACT_VEL, act, d, cur_yaw, pst, rpm);
                else qs::decode_action<true>(P, QS_ACT_VEL, act, d, cur_yaw, pst, rpm);
            } else {
                // computeControlFromEnv (pid_state_kernel): the controller's constants, its max_rpm clip, then the env's clip
                double tx, ty, tz, rx, ry, rz, vx, vy, vz, wx, wy, wz;
                track_target(io, N, i, k, tx, ty, tz);
                const_target(io.target_rpy, i, rx, ry, rz);
                const_target(io.target_vel, i, vx, vy, vz);
                const_target(io.target_rpy_rates, i, wx, wy, wz);
                qs::pid_control(a.CP, pst, io.control_timestep, d.px, d.py, d.pz, d.qx, d.qy, d.qz, d.qw, d.vx, d.vy, d.vz,
                                tx, ty, tz, rz, vx, vy, vz, wx, wy, wz, rpm, pe, ye);
                const double mr = PHYS ? load_phys_rpm(a.st.phys, e).max_rpm : P.max_rpm;
#pragma unroll
                for (int j = 0; j < 4; ++j) rpm[j] = qs::clampd(qs::clampd(rpm[j], 0.0, a.CP.max_rpm), 0.0, mr);
            }
            if constexpr (PHYS && !(EFF & QS_EFFECT_DW)) ph = load_phys(a.st.phys, e);       // after the controller
        }
        // ---- S substeps --------------------------------------------------------------------------------------------
        if (EFF & QS_EFFECT_DW) {
            for (int s = 0; s < a.substeps; ++s) {
                if (live) { pos_s[3 * t] = d.px; pos_s[3 * t + 1] = d.py; pos_s[3 * t + 2] = d.pz; }
                __syncthreads();
                if (live) {
                    double fz = 0.0;
                    const int b = le * D;
                    for (int q = 0; q < D; ++q) {                                 // BaseAviary.py:798-811
                        const double dz = pos_s[3 * (b + q) + 2] - d.pz;
                        const double dx = pos_s[3 * (b + q)] - d.px, dy = pos_s[3 * (b + q) + 1] - d.py;
                        const double dxy2 = dx * dx + dy * dy;
                        if (dz > 0.0 && dxy2 < 100.0) fz += qs::downwash_pair(P, dz, dxy2);
                    }
                    // the previous RPMs selected element by element: a pointer chosen at run time between the two arrays puts
                    // both into local memory inside the substep loop; for the same reason the row of constants is re-read (L1)
                    // every substep rather than held across the barriers
                    double rp[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) rp[j] = s == 0 ? rpm_prev[j] : rpm[j];
                    if constexpr (PHYS) qs::dyn_tick_k<EFF>(P, load_phys(a.st.phys, e), d, rpm, rp, fz, 1, R_last);
                    else qs::dyn_tick<EFF>(P, d, rpm, rp, fz, 1, R_last);
                }
                __syncthreads();
            }
        } else if (live) {
            if constexpr (PHYS) qs::dyn_tick_k<EFF>(P, ph, d, rpm, rpm_prev, 0.0, a.substeps, R_last);
            else qs::dyn_tick<EFF>(P, d, rpm, rpm_prev, 0.0, a.substeps, R_last);
        }
        // ---- state vector, per-tick outputs, Logger entry -------------------------------------------------------------
        const bool last = k == T - 1;
        const bool stage = rows_out || (last && io.obs_last);
        if (live) {
            qs::Derived o;
            if (a.flags & QS_FLAG_RPY_F32) qs::derive<true>(d, R_last, o); else qs::derive<false>(d, R_last, o);
            round_to_planes(d);                                   // what store_drone + load_drone do between two ticks
            sc += a.substeps;                                     // BaseAviary.py:382
            const long long ki = (long long)k * N + i;
            if (io.rpm) st256(io.rpm, ki, rpm[0], rpm[1], rpm[2], rpm[3]);
            if (MODE == QS_CTRL_TRACK) {
                if (io.pos_e) { float* pp = io.pos_e + 3 * ki; pp[0] = (float)pe[0]; pp[1] = (float)pe[1]; pp[2] = (float)pe[2]; }
                if (io.yaw_e) io.yaw_e[ki] = (float)ye;
            }
            // _getDroneStateVector (BaseAviary.py:541-561), the row of qs_dyn_substeps: quaternion normalised, ang_v of the last substep
            float h[20];
            h[0] = (float)d.px; h[1] = (float)d.py; h[2] = (float)d.pz;
            h[3] = (float)d.qx; h[4] = (float)d.qy; h[5] = (float)d.qz; h[6] = (float)d.qw;
            h[7] = (float)o.roll; h[8] = (float)o.pitch; h[9] = (float)o.yaw;
            h[10] = (float)d.vx; h[11] = (float)d.vy; h[12] = (float)d.vz;
            h[13] = (float)o.ax; h[14] = (float)o.ay; h[15] = (float)o.az;
            h[16] = (float)rpm[0]; h[17] = (float)rpm[1]; h[18] = (float)rpm[2]; h[19] = (float)rpm[3];
            if (stage) {
                float4* r4 = reinterpret_cast<float4*>(row_s + (size_t)t * 20);
#pragma unroll
                for (int q = 0; q < 5; ++q) r4[q] = make_float4(h[4 * q], h[4 * q + 1], h[4 * q + 2], h[4 * q + 3]);
            }
            if (lj >= 0) {
                // Logger.log (Logger.py:117) as log_append_kernel writes it after the step: rpy re-evaluated in float64 from the
                // stored quaternion, ang_v from the float32 row, the applied RPMs, the simulation time after the tick
                double roll, pitch, yaw;
                qs::quat_to_euler<false>(d.qx, d.qy, d.qz, d.qw, roll, pitch, yaw);
                double* ow = a.rg.ring + (((head0 + k) % a.rg.capacity) * a.rg.n_drones + lj) * 32;
                ow[0] = d.px; ow[1] = d.py; ow[2] = d.pz; ow[3] = d.vx; ow[4] = d.vy; ow[5] = d.vz;
                ow[6] = roll; ow[7] = pitch; ow[8] = yaw;
                ow[9] = h[13]; ow[10] = h[14]; ow[11] = h[15];
                const bool lr = a.st.last_rpm != nullptr;
                ow[12] = lr ? rpm[0] : 0.0; ow[13] = lr ? rpm[1] : 0.0; ow[14] = lr ? rpm[2] : 0.0; ow[15] = lr ? rpm[3] : 0.0;
                if (MODE == QS_CTRL_TRACK && io.log_targets) {
                    // pid.py's controls: the tick's targets (target_pos, target_rpy, target_vel, target_rpy_rates), as float32
                    double c[12];
                    track_target(io, N, i, k, c[0], c[1], c[2]);
                    const_target(io.target_rpy, i, c[3], c[4], c[5]);
                    const_target(io.target_vel, i, c[6], c[7], c[8]);
                    const_target(io.target_rpy_rates, i, c[9], c[10], c[11]);
                    for (int q = 0; q < 12; ++q) ow[16 + q] = (double)(float)c[q];
                } else {
                    for (int q = 0; q < 12; ++q) ow[16 + q] = io.log_controls ? (double)io.log_controls[12 * lj + q] : 0.0;
                }
                ow[28] = (double)sc * P.dt;
                ow[29] = ow[30] = ow[31] = 0.0;
            }
            rpm_prev[0] = rpm[0]; rpm_prev[1] = rpm[1]; rpm_prev[2] = rpm[2]; rpm_prev[3] = rpm[3];
        }
        if (stage) {                                              // CTA-uniform
            __syncthreads();
            // the CTA's rows [c0, c0 + rows) are one contiguous span of rows * 80 bytes
            const float4* src = reinterpret_cast<const float4*>(row_s);
            float4* out = rows_out ? reinterpret_cast<float4*>(io.obs + ((long long)k * N + c0) * 20) : nullptr;
            float4* lastp = (last && io.obs_last) ? reinterpret_cast<float4*>(io.obs_last + c0 * 20) : nullptr;
            for (int j = t; j < rows * 5; j += blockDim.x) {
                const float4 v = src[j];
                if (out) out[j] = v;
                if (lastp) lastp[j] = v;
            }
            __syncthreads();
        }
    }
    if (live) {
        store_drone_rounded(a.st, N, i, d);
        if (a.st.last_rpm) st256(a.st.last_rpm, i, rpm[0], rpm[1], rpm[2], rpm[3]);
        if (MODE == QS_CTRL_VEL) store_pid(a.st.pid, N, i, pst);
        if (MODE == QS_CTRL_TRACK) store_pid(io.pid_state, N, i, pst);
        if (i - e * D == 0) a.st.step_counter[e] = sc;
    }
}

__global__ void ctrl_log_advance_kernel(long long* head, int T) { *head += T; }      // after every CTA has read it (stream order)

template <int EFF, bool PHYS>
void launch_eff(const CtrlRolloutArgs& a, int mode, int blocks, int threads, size_t sm, cudaStream_t s) {
    if (mode == QS_CTRL_RAW) ctrl_rollout_kernel<EFF, QS_CTRL_RAW, PHYS><<<blocks, threads, sm, s>>>(a);
    else if (mode == QS_CTRL_VEL) ctrl_rollout_kernel<EFF, QS_CTRL_VEL, PHYS><<<blocks, threads, sm, s>>>(a);
    else ctrl_rollout_kernel<EFF, QS_CTRL_TRACK, PHYS><<<blocks, threads, sm, s>>>(a);
}

template <bool PHYS>
void launch_ctrl(const CtrlRolloutArgs& a, int mode, unsigned eff, int blocks, int threads, size_t sm, cudaStream_t s) {
    switch (eff) {
        case 0: launch_eff<0, PHYS>(a, mode, blocks, threads, sm, s); break;
        case QS_EFFECT_GND: launch_eff<QS_EFFECT_GND, PHYS>(a, mode, blocks, threads, sm, s); break;
        case QS_EFFECT_DRAG: launch_eff<QS_EFFECT_DRAG, PHYS>(a, mode, blocks, threads, sm, s); break;
        case QS_EFFECT_DW: launch_eff<QS_EFFECT_DW, PHYS>(a, mode, blocks, threads, sm, s); break;
        default: launch_eff<7, PHYS>(a, mode, blocks, threads, sm, s); break;
    }
}

}  // namespace
}  // namespace qsi

using namespace qsi;

extern "C" {

int qs_sizeof_ctrl_rollout_io(void) { return (int)sizeof(QsCtrlRolloutIO); }

int qs_ctrl_rollout(const QsParams* p, const QsState* st, const QsCtrlRolloutIO* io, int mode, int n_envs, int drones_per_env,
                    int substeps, unsigned effects, unsigned flags, void* stream) {
    if (!p || !io) return fail(QS_ERR_NULL, "qs_ctrl_rollout: NULL params/io");
    if (int rc = check_state(st, 0)) return rc;
    if (n_envs <= 0 || drones_per_env <= 0 || substeps <= 0 || io->T <= 0) return fail(QS_ERR_SIZE, "qs_ctrl_rollout: n_envs, drones_per_env, substeps and T must be > 0");
    if ((long long)n_envs * drones_per_env > 0x7fffffffLL) return fail(QS_ERR_SIZE, "qs_ctrl_rollout: n_envs * drones_per_env exceeds 2^31-1");
    if (mode != QS_CTRL_RAW && mode != QS_CTRL_VEL && mode != QS_CTRL_TRACK) return fail(QS_ERR_ENUM, "qs_ctrl_rollout: bad mode (QS_CTRL_RAW, QS_CTRL_VEL or QS_CTRL_TRACK)");
    if (effects & ~7u) return fail(QS_ERR_ENUM, "qs_ctrl_rollout: bad effects");
    const unsigned eff = effects & 7u;
    if (eff != 0 && eff != QS_EFFECT_GND && eff != QS_EFFECT_DRAG && eff != QS_EFFECT_DW && eff != 7u)
        return fail(QS_ERR_UNSUPPORTED, "qs_ctrl_rollout: supports no DYN+ effect, GND, DRAG, DW or all three; not GND|DRAG, GND|DW or DRAG|DW");
    if ((eff & QS_EFFECT_DW) && drones_per_env > kCtrlTPB)
        return fail(QS_ERR_UNSUPPORTED, "qs_ctrl_rollout: downwash needs drones_per_env <= 128 (larger aviaries take the per-tick qs_downwash + qs_dyn_substeps path)");
    if (flags & ~(unsigned)(QS_FLAG_RPY_F32 | QS_FLAG_ACTION_F64))
        return fail(QS_ERR_UNSUPPORTED, "qs_ctrl_rollout: only QS_FLAG_RPY_F32 and QS_FLAG_ACTION_F64 are supported (no autoreset, no split substeps)");
    const bool f64 = flags & QS_FLAG_ACTION_F64;
    if (f64 && mode != QS_CTRL_RAW) return fail(QS_ERR_UNSUPPORTED, "qs_ctrl_rollout: QS_FLAG_ACTION_F64 is for QS_CTRL_RAW actions");
    if ((eff & QS_EFFECT_DRAG) && !st->last_rpm) return fail(QS_ERR_NULL, "qs_ctrl_rollout: DRAG needs QsState.last_rpm");
    if (mode == QS_CTRL_TRACK) {
        if (io->actions) return fail(QS_ERR_UNSUPPORTED, "qs_ctrl_rollout: QS_CTRL_TRACK takes a controller, not actions");
        if (!io->ctrl_params || !io->pid_state) return fail(QS_ERR_NULL, "qs_ctrl_rollout: QS_CTRL_TRACK needs a controller (ctrl_params, pid_state)");
        if (!io->waypoints || !io->start) return fail(QS_ERR_NULL, "qs_ctrl_rollout: QS_CTRL_TRACK needs waypoints and start");
        if (io->W <= 0) return fail(QS_ERR_SIZE, "qs_ctrl_rollout: W (waypoint rows) must be > 0");
        if (io->M != 1 && (long long)io->M != (long long)n_envs * drones_per_env) return fail(QS_ERR_SIZE, "qs_ctrl_rollout: M (waypoint columns) must be 1 or N");
        if (!(io->control_timestep > 0.0)) return fail(QS_ERR_SIZE, "qs_ctrl_rollout: control_timestep must be > 0");
    } else {
        if (!io->actions) return fail(QS_ERR_NULL, "qs_ctrl_rollout: actions is NULL");
        if (f64 ? !aligned32(io->actions) : !aligned16(io->actions))
            return fail(QS_ERR_ALIGN, "qs_ctrl_rollout: actions must be 16-byte aligned (float32) / 32-byte aligned (float64)");
        if (mode == QS_CTRL_VEL && !st->pid) return fail(QS_ERR_NULL, "qs_ctrl_rollout: QS_CTRL_VEL needs QsState.pid");
    }
    if (io->rpm && !aligned32(io->rpm)) return fail(QS_ERR_ALIGN, "qs_ctrl_rollout: rpm must be 32-byte aligned");
    if ((io->obs && !aligned16(io->obs)) || (io->obs_last && !aligned16(io->obs_last)))
        return fail(QS_ERR_ALIGN, "qs_ctrl_rollout: obs / obs_last must be 16-byte aligned");
    CtrlRolloutArgs a;
    memset(&a, 0, sizeof(a));
    if (io->log) {
        const QsLogRing& r = *io->log;
        if (!r.ring || !r.head) return fail(QS_ERR_NULL, "qs_ctrl_rollout: NULL log ring");
        if (r.capacity <= 0 || r.n_drones <= 0 || r.first_drone < 0 || (long long)r.first_drone + r.n_drones > (long long)n_envs * drones_per_env)
            return fail(QS_ERR_SIZE, "qs_ctrl_rollout: bad log ring geometry");
        a.rg = r;
        a.has_log = 1;
    }
    a.P = *p;
    if (mode == QS_CTRL_TRACK) a.CP = *io->ctrl_params;
    a.st = *st; a.io = *io;
    a.N = (long long)n_envs * drones_per_env;
    a.n_envs = n_envs; a.D = drones_per_env; a.substeps = substeps; a.flags = flags;
    // in-CTA downwash: whole aviaries per CTA; otherwise any 128 consecutive drones (one-warp CTAs for downwash, as the step kernels
    // use up to 32 drones per aviary, measured slower on the H100: DESIGN.md 4.1e)
    a.tpb = (eff & QS_EFFECT_DW) ? block_size_for(drones_per_env, kCtrlTPB) : kCtrlTPB;
    const int blocks = (int)((a.N + a.tpb - 1) / a.tpb);
    const int threads = ((a.tpb + 31) / 32) * 32;
    const size_t sm = (size_t)a.tpb * 20 * 4 + ((eff & QS_EFFECT_DW) ? (size_t)a.tpb * 3 * 8 : 0);
    cudaStream_t s = (cudaStream_t)stream;
    if (st->phys) launch_ctrl<true>(a, mode, eff, blocks, threads, sm, s);
    else launch_ctrl<false>(a, mode, eff, blocks, threads, sm, s);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess && a.has_log) {
        ctrl_log_advance_kernel<<<1, 1, 0, s>>>(a.rg.head, io->T);
        e = cudaGetLastError();
    }
    return e == cudaSuccess ? 0 : cuda_fail(e, "qs_ctrl_rollout launch");
}

}  // extern "C"
