// dyn_dw_traj.cu -- qs_dyn_traj_dw / qs_dyn_traj_dw_vjp and qs_dyn_ctrl_traj_dw / qs_dyn_ctrl_traj_dw_vjp: the differentiable
// raw-RPM and DSLPIDControl trajectories of dyn_traj.cu and dyn_ctrl_traj.cu with downwash (include/quadsim.h, DESIGN.md 4.5,
// downwash adjoint).  Downwash couples the drones of an aviary, so the unit is the aviary: one CTA of 128 threads holds
// 128 / D whole aviaries, D threads each (mppi.cu's layout), and every thread runs every barrier.
//   forward:  each substep is ctrl_rollout_kernel's (positions through shared memory, qs::downwash_fz, one dyn_tick_k substep),
//             round_to_planes after each tick; the closed loop calls the controller once per drone per tick before them.
//   backward: tick by tick in reverse, the tick's substeps recomputed cooperatively (their start states into the scratch
//             record), then per substep in reverse: fz recomputed from the start positions, dw_substep_vjp (drone-local, gives
//             lambda = the cotangent of fz) and, after a barrier, downwash_pos_vjp (the pair terms from the aviary's lambdas).
// The checks and the launch over DwTrajEffects are traj_io.cuh's; the per-drone inputs, clips and stores are the twins'.
#include "qs_common.cuh"
#include "dyn_adjoint.cuh"
#include "ctrl_io.cuh"

namespace qsi {
namespace {

constexpr int kDwTPB = 128;                    // whole aviaries of up to 128 drones per CTA

struct DwTrajArgs {
    QsParams P;
    QsDynTrajIO io;
    long long N;
    int D, substeps;
    int tpb;                                   // the threads of a CTA that hold whole aviaries (D * (128 / D))
};

struct DwCtrlTrajArgs {
    QsParams P;                                // the env: physics, MAX_RPM clip
    QsParams CP;                               // the DSLPIDControl's own constants
    QsDynCtrlTrajIO io;
    long long N;
    int D, substeps, tpb;
};

// The S substeps of one aviary tick from d with clipped rpm u (drag: up in substep 0, u afterwards), each ctrl_rollout_kernel's.
// Every thread of the CTA calls it; `live` ones compute.  `between(s)` follows substep s (the VJP's record).
template <int EFF, class Hook = qs::NoHook>
__device__ __forceinline__ void dw_tick(const QsParams& P, const qs::PhysRow& c, bool live, int t, int b, int D, int S, double* pos_s,
                                        qs::Drone& d, const double u[4], const double up[4], Hook between = Hook()) {
    for (int s = 0; s < S; ++s) {
        if (live) { pos_s[3 * t] = d.px; pos_s[3 * t + 1] = d.py; pos_s[3 * t + 2] = d.pz; }
        __syncthreads();
        if (live) {
            const double fz = qs::downwash_fz(P, pos_s, b, D, d.px, d.py, d.pz);
            double rp[4], R_last[9];
#pragma unroll
            for (int j = 0; j < 4; ++j) rp[j] = s == 0 ? up[j] : u[j];
            qs::dyn_tick_k<EFF>(P, c, d, u, rp, fz, 1, R_last);
            between(s);
        }
        __syncthreads();
    }
}

// The adjoint of dw_tick from the tick-start state d0 (as stored).  L: in, the cotangent of the tick's end state; out, of d0.
// Lu / Lup (drag's previous RPMs) / G accumulate.  pos_s [3 tpb] and lam_s [tpb] are the CTA's shared arrays.
template <int EFF>
__device__ __forceinline__ void dw_tick_vjp(const QsParams& P, const qs::PhysRow& c, bool live, int t, int b, int D, int S, double* pos_s,
                                            double* lam_s, const qs::Drone& d0, const double u[4], const double up[4], ScratchRec& rec,
                                            qs::Drone& L, double Lu[4], double Lup[4], qs::PhysGrad& G) {
    {
        qs::Drone d = d0;
        dw_tick<EFF>(P, c, live, t, b, D, S, pos_s, d, u, up, qs::RecordHook<ScratchRec>{&d, &rec, S - 1});
    }
    const double ds_prev = qs::drag_sum(up), ds_cur = qs::drag_sum(u);
    double Lds_prev = 0.0, Lds_cur = 0.0;
    for (int s = S - 1; s >= 0; --s) {
        qs::Drone x = d0;
        if (live) {
            if (s > 0) rec.load(s - 1, x);
            pos_s[3 * t] = x.px; pos_s[3 * t + 1] = x.py; pos_s[3 * t + 2] = x.pz;
        }
        __syncthreads();
        if (live) {
            const double fz = qs::downwash_fz(P, pos_s, b, D, x.px, x.py, x.pz);
            lam_s[t] = qs::dw_substep_vjp<EFF>(P, c, x, u, s == 0 ? ds_prev : ds_cur, fz, L, Lu, s == 0 ? Lds_prev : Lds_cur, G);
        }
        __syncthreads();
        if (live) qs::downwash_pos_vjp(P, pos_s, lam_s, b, D, t - b, L);
        __syncthreads();                                // before the next substep overwrites pos_s and lam_s
    }
    if (EFF & QS_EFFECT_DRAG) {
        const double kk = 2.0 * 3.14159265358979323846;
#pragma unroll
        for (int j = 0; j < 4; ++j) { Lup[j] += (kk / 60.0) * Lds_prev; Lu[j] += (kk / 60.0) * Lds_cur; }
    }
}

template <int EFF>
__global__ void __launch_bounds__(kDwTPB) dyn_dw_traj_kernel(const __grid_constant__ DwTrajArgs a) {
    __shared__ double pos_s[3 * kDwTPB];
    const QsDynTrajIO& io = a.io;
    const long long N = a.N;
    const DwSlot sl = dw_slot(a, N / a.D);
    const long long i = sl.G * a.D + sl.q;
    qs::PhysRow c;
    qs::Drone d;
    double up[4] = {0, 0, 0, 0};
    if (sl.live) {
        c = row_of(a, i);
        ld_state(io.state0, N, i, d);
        if ((EFF & QS_EFFECT_DRAG) && io.last_rpm) ld4(io.last_rpm, i, up);
    }
    for (int k = 0; k < io.T; ++k) {
        double raw[4], u[4] = {0, 0, 0, 0};
        if (sl.live) {
            ld4(io.rpm, (long long)k * N + i, raw);
            clip_rpm(raw, c.max_rpm, u);
        }
        dw_tick<EFF>(a.P, c, sl.live, threadIdx.x, sl.b, a.D, a.substeps, pos_s, d, u, up);
        if (sl.live) {
            round_to_planes(d);
            st_state(io.states + (long long)k * 13 * N, N, i, d);
#pragma unroll
            for (int j = 0; j < 4; ++j) up[j] = u[j];
        }
    }
}

template <int EFF>
__global__ void __launch_bounds__(kDwTPB) dyn_dw_traj_vjp_kernel(const __grid_constant__ DwTrajArgs a) {
    __shared__ double pos_s[3 * kDwTPB];
    __shared__ double lam_s[kDwTPB];
    const QsDynTrajIO& io = a.io;
    const long long N = a.N;
    const DwSlot sl = dw_slot(a, N / a.D);
    const long long i = sl.G * a.D + sl.q;
    qs::PhysRow c;
    if (sl.live) c = row_of(a, i);
    ScratchRec rec = {io.scratch, N, i};
    qs::PhysGrad G = zero_phys_grad();
    qs::Drone L = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    double Lup_next[4] = {0, 0, 0, 0};          // drag: the cotangent of this tick's clipped RPMs from tick k + 1's first substep
    for (int k = io.T - 1; k >= 0; --k) {
        qs::Drone d0 = {};
        double raw[4], u[4] = {0, 0, 0, 0}, up[4] = {0, 0, 0, 0};
        if (sl.live) {
            add_state(io.g_states + (long long)k * 13 * N, N, i, L);
            tick_inputs<EFF>(a, c.max_rpm, i, k, d0, raw, u, up);
        }
        double Lu[4] = {Lup_next[0], Lup_next[1], Lup_next[2], Lup_next[3]}, Lup[4] = {0, 0, 0, 0};
        dw_tick_vjp<EFF>(a.P, c, sl.live, threadIdx.x, sl.b, a.D, a.substeps, pos_s, lam_s, d0, u, up, rec, L, Lu, Lup, G);
        if (sl.live) {
            double gr[4];
            qs::rpm_clip_vjp(raw, c.max_rpm, Lu, gr, G.g[13]);
            double* o = io.g_rpm + 4 * ((long long)k * N + i);
            o[0] = gr[0]; o[1] = gr[1]; o[2] = gr[2]; o[3] = gr[3];
#pragma unroll
            for (int j = 0; j < 4; ++j) Lup_next[j] = Lup[j];
        }
    }
    if (sl.live) {
        st_state(io.g_state0, N, i, L);
        store_start_grads(io, i, Lup_next, G);
    }
}

template <int EFF>
__global__ void __launch_bounds__(kDwTPB) dyn_dw_ctrl_traj_kernel(const __grid_constant__ DwCtrlTrajArgs a) {
    __shared__ double pos_s[3 * kDwTPB];
    const QsDynCtrlTrajIO& io = a.io;
    const long long N = a.N;
    const DwSlot sl = dw_slot(a, N / a.D);
    const long long i = sl.G * a.D + sl.q;
    qs::PhysRow c;
    qs::PidGains K;
    qs::Drone d;
    qs::PidState st;
    double up[4] = {0, 0, 0, 0};
    if (sl.live) {
        c = row_of(a, i);
        K = gains_of(a, i);
        ld_state(io.state0, N, i, d);
        load_pid(io.pid0, N, i, st);
        if ((EFF & QS_EFFECT_DRAG) && io.last_rpm) ld4(io.last_rpm, i, up);
    }
    for (int k = 0; k < io.T; ++k) {
        double raw[4], u1[4], u[4] = {0, 0, 0, 0};
        if (sl.live) {
            store_pid(io.pid_states + (long long)k * 9 * N, N, i, st);
            control(a, K, st, d, targets_of(io, N, i, k), c.max_rpm, raw, u1, u);
        }
        dw_tick<EFF>(a.P, c, sl.live, threadIdx.x, sl.b, a.D, a.substeps, pos_s, d, u, up);
        if (sl.live) {
            round_to_planes(d);
            st_state(io.states + (long long)k * 13 * N, N, i, d);
            double* o = io.rpm + 4 * ((long long)k * N + i);
#pragma unroll
            for (int j = 0; j < 4; ++j) { o[j] = u[j]; up[j] = u[j]; }
        }
    }
}

template <int EFF>
__global__ void __launch_bounds__(kDwTPB) dyn_dw_ctrl_traj_vjp_kernel(const __grid_constant__ DwCtrlTrajArgs a) {
    __shared__ double pos_s[3 * kDwTPB];
    __shared__ double lam_s[kDwTPB];
    const QsDynCtrlTrajIO& io = a.io;
    const long long N = a.N;
    const DwSlot sl = dw_slot(a, N / a.D);
    const long long i = sl.G * a.D + sl.q;
    qs::PhysRow c;
    qs::PidGains K;
    if (sl.live) {
        c = row_of(a, i);
        K = gains_of(a, i);
    }
    ScratchRec rec = {io.scratch, N, i};
    qs::PhysGrad G = zero_phys_grad();
    double Lg[18];
#pragma unroll
    for (int j = 0; j < 18; ++j) Lg[j] = 0.0;
    qs::PidTargets Lt = {{0, 0, 0}, 0, {0, 0, 0}, {0, 0, 0}};
    qs::Drone L = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    qs::PidState Ls = {0, 0, 0, 0, 0, 0, 0, 0, 0};      // the cotangent of the controller state after tick k
    double Lup_next[4] = {0, 0, 0, 0};                 // drag: the cotangent of this tick's applied RPMs from tick k + 1
    for (int k = io.T - 1; k >= 0; --k) {
        qs::Drone d0 = {};
        qs::PidState st0;
        qs::PidTargets t;
        double raw[4], u1[4], u[4] = {0, 0, 0, 0}, up[4] = {0, 0, 0, 0};
        double Lu[4] = {Lup_next[0], Lup_next[1], Lup_next[2], Lup_next[3]}, Lup[4] = {0, 0, 0, 0};
        if (sl.live) {
            add_state(io.g_states + (long long)k * 13 * N, N, i, L);
            ld_state(k == 0 ? io.state0 : io.states + (long long)(k - 1) * 13 * N, N, i, d0);
            load_pid(io.pid_states + (long long)k * 9 * N, N, i, st0);
            t = targets_of(io, N, i, k);
            qs::PidState st = st0;
            control(a, K, st, d0, t, c.max_rpm, raw, u1, u);
            if (EFF & QS_EFFECT_DRAG) {
                if (k > 0) ld4(io.rpm, (long long)(k - 1) * N + i, up);
                else if (io.last_rpm) ld4(io.last_rpm, i, up);
            }
            if (io.g_rpm_out) {
                double gr[4];
                ld4(io.g_rpm_out, (long long)k * N + i, gr);
#pragma unroll
                for (int j = 0; j < 4; ++j) Lu[j] += gr[j];
            }
        }
        dw_tick_vjp<EFF>(a.P, c, sl.live, threadIdx.x, sl.b, a.D, a.substeps, pos_s, lam_s, d0, u, up, rec, L, Lu, Lup, G);
        if (sl.live) {
            // the env's clip (gradient to the row's MAX_RPM), then the controller's (its max_rpm is a constant of the controller)
            double Lu1[4], Lraw[4], g_cmax = 0.0;
            qs::rpm_clip_vjp(u1, c.max_rpm, Lu, Lu1, G.g[13]);
            qs::rpm_clip_vjp(raw, a.CP.max_rpm, Lu1, Lraw, g_cmax);
            Lt.tp[0] = Lt.tp[1] = Lt.tp[2] = 0.0;         // target_pos is per tick: its cotangent is written, not carried
            qs::pid_control_vjp(a.CP, K, st0, io.control_timestep, d0, t, Lraw, Ls, L, Lt, Lg);
            if (io.g_target_pos) {
                double* o = io.g_target_pos + 3 * ((long long)k * N + i);
                o[0] = Lt.tp[0]; o[1] = Lt.tp[1]; o[2] = Lt.tp[2];
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) Lup_next[j] = Lup[j];
        }
    }
    if (!sl.live) return;
    st_state(io.g_state0, N, i, L);
    if (io.g_pid0) store_pid(io.g_pid0, N, i, Ls);
    auto st3 = [&](double* p, const double v[3]) { if (p) { p[3 * i] = v[0]; p[3 * i + 1] = v[1]; p[3 * i + 2] = v[2]; } };
    st3(io.g_target_vel, Lt.tv);
    st3(io.g_target_rpy_rates, Lt.trr);
    const double ly[3] = {0.0, 0.0, Lt.tyaw};
    st3(io.g_target_rpy, ly);
    store_start_grads(io, i, Lup_next, G);
    if (io.g_gains) {
        double* o = io.g_gains + 18 * i;
#pragma unroll
        for (int j = 0; j < 18; ++j) o[j] = Lg[j];
    }
}

// The checks of the downwash entry points after their twins' NULL and size checks: the effect set, the aviary size, phys alignment
inline int dw_check(const char* what, unsigned effects, int drones_per_env, const double* phys) {
    if (!with_int(DwTrajEffects{}, (int)effects, [](auto) {}))
        return fail(QS_ERR_UNSUPPORTED, what, "supports DW and GND|DRAG|DW only (without downwash: the per-drone entry point)");
    if (drones_per_env > kDwTPB) return fail(QS_ERR_UNSUPPORTED, what, "downwash needs drones_per_env <= 128");
    if (phys && !aligned16(phys)) return fail(QS_ERR_ALIGN, what, "phys rows must be 16-byte aligned");
    return 0;
}

// a's geometry for n_envs aviaries of D drones, and the launch of pick(EFF) over their CTAs
template <class Args, class Pick>
int dw_launch(const char* what, unsigned effects, int n_envs, int drones_per_env, int substeps, void* stream, Args& a, Pick pick) {
    a.N = (long long)n_envs * drones_per_env;
    a.D = drones_per_env; a.substeps = substeps;
    a.tpb = block_size_for(drones_per_env, kDwTPB);
    const long long per_cta = a.tpb / drones_per_env;
    const unsigned blocks = (unsigned)((n_envs + per_cta - 1) / per_cta);
    return traj_launch<DwTrajEffects>(what, effects, pick, blocks, kDwTPB, 0, (cudaStream_t)stream, a);
}

template <bool VJP>
int launch_dw_traj(const QsParams* p, const QsDynTrajIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                   void* stream, const char* what) {
    if (!p || !io) return fail(QS_ERR_NULL, what, "NULL params / io");
    if (!io->state0 || !io->rpm || !io->states) return fail(QS_ERR_NULL, what, "NULL state0 / rpm / states");
    if (VJP && (!io->g_states || !io->g_rpm || !io->g_state0 || !io->scratch))
        return fail(QS_ERR_NULL, what, "NULL g_states / g_rpm / g_state0 / scratch");
    if (int rc = traj_check_sizes(what, n_envs, drones_per_env, substeps, io->T)) return rc;
    if (int rc = dw_check(what, effects, drones_per_env, io->phys)) return rc;
    DwTrajArgs a;
    memset(&a, 0, sizeof(a));
    a.P = *p; a.io = *io;
    return dw_launch(what, effects, n_envs, drones_per_env, substeps, stream, a, [](auto EFF) {
        return VJP ? dyn_dw_traj_vjp_kernel<decltype(EFF)::value> : dyn_dw_traj_kernel<decltype(EFF)::value>;
    });
}

template <bool VJP>
int launch_dw_ctrl_traj(const QsParams* p, const QsParams* cp, const QsDynCtrlTrajIO* io, int n_envs, int drones_per_env,
                        int substeps, unsigned effects, void* stream, const char* what) {
    if (!p || !cp || !io) return fail(QS_ERR_NULL, what, "NULL params / controller params / io");
    if (!io->state0 || !io->pid0 || !io->target_pos || !io->states || !io->rpm || !io->pid_states)
        return fail(QS_ERR_NULL, what, "NULL state0 / pid0 / target_pos / states / rpm / pid_states");
    if (VJP && (!io->g_states || !io->g_state0 || !io->scratch)) return fail(QS_ERR_NULL, what, "NULL g_states / g_state0 / scratch");
    if (int rc = traj_check_sizes(what, n_envs, drones_per_env, substeps, io->T)) return rc;
    if (!(io->control_timestep > 0.0)) return fail(QS_ERR_SIZE, what, "control_timestep must be > 0");
    if (int rc = dw_check(what, effects, drones_per_env, io->phys)) return rc;
    DwCtrlTrajArgs a;
    memset(&a, 0, sizeof(a));
    a.P = *p; a.CP = *cp; a.io = *io;
    return dw_launch(what, effects, n_envs, drones_per_env, substeps, stream, a, [](auto EFF) {
        return VJP ? dyn_dw_ctrl_traj_vjp_kernel<decltype(EFF)::value> : dyn_dw_ctrl_traj_kernel<decltype(EFF)::value>;
    });
}

}  // namespace
}  // namespace qsi

using namespace qsi;

extern "C" {

int qs_dyn_traj_dw(const QsParams* p, const QsDynTrajIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                   void* stream) {
    return launch_dw_traj<false>(p, io, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_traj_dw");
}

int qs_dyn_traj_dw_vjp(const QsParams* p, const QsDynTrajIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                       void* stream) {
    return launch_dw_traj<true>(p, io, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_traj_dw_vjp");
}

int qs_dyn_ctrl_traj_dw(const QsParams* p, const QsParams* cp, const QsDynCtrlTrajIO* io, int n_envs, int drones_per_env, int substeps,
                        unsigned effects, void* stream) {
    return launch_dw_ctrl_traj<false>(p, cp, io, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_ctrl_traj_dw");
}

int qs_dyn_ctrl_traj_dw_vjp(const QsParams* p, const QsParams* cp, const QsDynCtrlTrajIO* io, int n_envs, int drones_per_env,
                            int substeps, unsigned effects, void* stream) {
    return launch_dw_ctrl_traj<true>(p, cp, io, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_ctrl_traj_dw_vjp");
}

}  // extern "C"
