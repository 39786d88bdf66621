// mppi.cu -- qs_mppi_sample / qs_mppi_update / qs_mppi_commit / qs_mppi_noise: sampling-based trajectory optimisation (MPPI) of
// raw-RPM trajectories for every Physics mode of the DYN family, downwash included (include/quadsim.h, DESIGN.md 4.5.2).
//   mppi_sample_kernel<EFF, BOX>:  J of every sample.  Without downwash one thread per (drone, sample), the samples of a drone
//                                  in neighbouring lanes (as ilqr_line_search_kernel places its step sizes); with downwash whole
//                                  (aviary, sample) groups per 128-thread CTA.
//   mppi_update_kernel<DW, BOX>:   one warp per unit (drone, or aviary with downwash): the weights, then the candidate.
//   mppi_commit_kernel<EFF, BOX>:  rolls out the candidate (per aviary with downwash) and commits it or the best sample.
// Every rollout is mppi_rollout: ilqr_rollout's tick (clip_rpm, dyn_tick_k, round_to_planes) and stage cost, so sample 0's J is
// the nominal's cost bit for bit; with downwash each substep is ctrl_rollout_kernel's (positions through shared memory,
// qs::downwash_fz, one dyn_tick_k substep), so a committed trajectory is CtrlAviary.rollout()'s for the committed rpm.  The
// checks and the launch over PlanEffects are traj_io.cuh's.
#include "qs_common.cuh"
#include "dyn_adjoint.cuh"
#include "lqr_law.cuh"
#include "riccati.cuh"
#include "traj_io.cuh"
#include "mppi.cuh"

namespace qsi {
namespace {

constexpr int kMppiTPB = 128;         // sample and commit CTAs; with downwash whole aviaries of up to 128 drones
constexpr int kUpdWarps = 4;          // units (warps) per update CTA
constexpr int kMaxSamples = 1024;

struct MppiArgs {
    QsParams P;
    QsMppiIO io;
    long long N;
    int D, substeps;
    int tpb;                        // downwash: the threads of a CTA that hold whole groups (D * (128 / D))
};

// The commands of drone i at tick k: of sample s (s >= 0), or the candidate (s < 0) clamped into the box
template <bool BOX>
__device__ __forceinline__ void mppi_tick_command(const MppiArgs& a, double sig, long long i, int k, int s, double v[4]) {
    const QsMppiIO& io = a.io;
    const long long ki = (long long)k * a.N + i;
    double lo[4] = {0, 0, 0, 0}, hi[4] = {0, 0, 0, 0};
    if constexpr (BOX) ld_box(io.rpm_lo, io.rpm_hi, io.per_tick, k, a.N, i, lo, hi);
    if (s < 0) {
        ld4(io.cand, ki, v);
        if constexpr (BOX) {
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] = qs::clampd(v[j], lo[j], hi[j]);
        }
        return;
    }
    ld4(io.rpm, ki, v);
    if (s == 0) return;                                               // eps = 0: the nominal, which lies in the box
    double eps[4];
    qs::mppi_eps(io.seed, k, s, i, io.iteration, eps);
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = qs::mppi_command<BOX>(v[j], sig, eps[j], lo[j], hi[j]);
}

// sig_i = sigma[e] HOVER_RPM of drone i's row
__device__ __forceinline__ double mppi_sig(const MppiArgs& a, const qs::PhysRow& c, long long i) { return a.io.sigma[i / a.D] * c.hover_rpm; }

// The end of tick k of drone i with commands v (after the box) and the clipped uc: the optional stores and the stage cost
__device__ __forceinline__ double mppi_tick_end(const MppiArgs& a, const double* wt, const double Rt[4], const double uref[4], long long i,
                                                int k, const double v[4], qs::Drone& d, bool store) {
    const QsMppiIO& io = a.io;
    const long long N = a.N;
    round_to_planes(d);
    if (store) {
        st_state(io.states + (long long)k * 13 * N, N, i, d);
        double* o = io.rpm + 4 * ((long long)k * N + i);
        o[0] = v[0]; o[1] = v[1]; o[2] = v[2]; o[3] = v[3];
    }
    qs::Drone rd;
    double ref[13], x[13];
    ld_state(io.targets + (long long)k * 13 * N, N, i, rd);
    drone_vec(rd, ref);
    drone_vec(d, x);
    return qs::stage_cost(x, ref, wt + qs::stage_weights(k, io.T), v, uref, Rt);
}

// J of drone i's rollout of sample s (s < 0: the candidate).  With `store` the states and the commands are written, each tick's
// commands over the nominal's after they are read.  With downwash the rollout is one (aviary, sample) group's: thread t holds
// drone i, its group's drones are the threads [b, b + D), every thread of the CTA runs the loop (the barriers) and `live` ones
// compute; each substep is ctrl_rollout_kernel's.  Without downwash every caller is live.
template <int EFF, bool BOX>
__device__ double mppi_rollout(const MppiArgs& a, bool live, long long i, int s, bool store, int t = 0, int b = 0,
                               double* pos_s = nullptr) {
    const QsMppiIO& io = a.io;
    qs::PhysRow c;
    const double* wt = io.weights;
    double Rt[4] = {0, 0, 0, 0}, uref[4] = {0, 0, 0, 0}, sig = 0.0;
    qs::Drone d;
    double up[4] = {0, 0, 0, 0};
    if (live) {
        c = row_of(a, i);
        wt = io.weights + (long long)qs::kWeightsRow * (i / a.D);
        qs::rel_weights(wt, c, Rt);
        ld4(io.rpm_ref, i, uref);
        sig = mppi_sig(a, c, i);
        ld_state(io.state0, a.N, i, d);
        if ((EFF & QS_EFFECT_DRAG) && io.last_rpm) ld4(io.last_rpm, i, up);
    }
    double J = 0.0;
    for (int k = 0; k < io.T; ++k) {
        double v[4], uc[4] = {0, 0, 0, 0}, R_last[9];
        if (live) {
            mppi_tick_command<BOX>(a, sig, i, k, s, v);
            clip_rpm(v, c.max_rpm, uc);
        }
        if constexpr (EFF & QS_EFFECT_DW) {
            for (int ss = 0; ss < a.substeps; ++ss) {
                if (live) { pos_s[3 * t] = d.px; pos_s[3 * t + 1] = d.py; pos_s[3 * t + 2] = d.pz; }
                __syncthreads();
                if (live) {
                    const double fz = qs::downwash_fz(a.P, pos_s, b, a.D, d.px, d.py, d.pz);
                    double rp[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) rp[j] = ss == 0 ? up[j] : uc[j];
                    qs::dyn_tick_k<EFF>(a.P, c, d, uc, rp, fz, 1, R_last);
                }
                __syncthreads();
            }
        } else if (live) {
            qs::dyn_tick_k<EFF>(a.P, c, d, uc, up, 0.0, a.substeps, R_last);
        }
        if (live) {
            J += mppi_tick_end(a, wt, Rt, uref, i, k, v, d, store);
#pragma unroll
            for (int j = 0; j < 4; ++j) up[j] = uc[j];
        }
    }
    return J;
}

template <int EFF, bool BOX>
__global__ void __launch_bounds__(kMppiTPB) mppi_sample_kernel(const __grid_constant__ MppiArgs a) {
    const QsMppiIO& io = a.io;
    const int K = io.K;
    if constexpr (EFF & QS_EFFECT_DW) {
        __shared__ double pos_s[3 * kMppiTPB];
        const DwSlot sl = dw_slot(a, a.N / a.D * K);
        const long long e = sl.G / K;
        const int s = (int)(sl.G - e * K);
        const long long i = e * a.D + sl.q;
        const double J = mppi_rollout<EFF, BOX>(a, sl.live, i, s, false, threadIdx.x, sl.b, pos_s);
        if (sl.live) io.J[(long long)s * a.N + i] = J;
    } else {
        const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
        if (g >= a.N * K) return;
        const long long i = g / K;
        const int s = (int)(g - i * K);
        io.J[(long long)s * a.N + i] = mppi_rollout<EFF, BOX>(a, true, i, s, false);
    }
}

// J of unit u's sample s: the drone's, or with downwash the sum over the aviary's drones in drone order
template <bool DW>
__device__ __forceinline__ double unit_cost(const MppiArgs& a, long long u, int s) {
    const double* Js = a.io.J + (long long)s * a.N;
    if (!DW) return Js[u];
    double j = 0.0;
    for (int q = 0; q < a.D; ++q) j += Js[u * a.D + q];
    return j;
}

template <bool DW, bool BOX>
__global__ void __launch_bounds__(32 * kUpdWarps) mppi_update_kernel(const __grid_constant__ MppiArgs a) {
    extern __shared__ double upd_s[];                                 // per warp: J [K] and w [K] of its unit
    const QsMppiIO& io = a.io;
    const int K = io.K, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long long u = (long long)blockIdx.x * kUpdWarps + wid;
    const long long units = DW ? a.N / a.D : a.N;
    if (u >= units) return;                                           // the whole warp: no CTA-wide barrier below
    double* Ju = upd_s + (size_t)wid * 2 * K;
    double* w = Ju + K;
    for (int s = lane; s < K; s += 32) Ju[s] = unit_cost<DW>(a, u, s);
    __syncwarp();
    // every lane scans the unit's costs in s order (the same bits in every lane)
    const qs::MppiStats st = qs::mppi_stats([&](int s) { return Ju[s]; }, K, io.temperature);
    for (int s = lane; s < K; s += 32) w[s] = qs::mppi_weight(Ju[s], st);
    __syncwarp();
    double wsum = 0.0;
    for (int s = 0; s < K; ++s) wsum += w[s];
    // the entries (tick, drone of the unit): u_c = u + sum_s w_s delta_s / sum_s w_s, delta regenerated from the counter
    const int nd = DW ? a.D : 1;
    const long long i0 = DW ? u * a.D : u;
    for (int idx = lane; idx < io.T * nd; idx += 32) {
        const int k = idx / nd;
        const long long i = i0 + (idx - k * nd);
        const long long ki = (long long)k * a.N + i;
        const qs::PhysRow c = row_of(a, i);
        const double sig = mppi_sig(a, c, i);
        double un[4], lo[4] = {0, 0, 0, 0}, hi[4] = {0, 0, 0, 0};
        ld4(io.rpm, ki, un);
        if constexpr (BOX) ld_box(io.rpm_lo, io.rpm_hi, io.per_tick, k, a.N, i, lo, hi);
        double num[4] = {0, 0, 0, 0};
        for (int s = 1; s < K; ++s) {                                 // delta_0 = 0; a zero weight adds nothing
            const double ws = w[s];
            if (ws == 0.0) continue;
            double eps[4];
            qs::mppi_eps(io.seed, k, s, i, io.iteration, eps);
#pragma unroll
            for (int j = 0; j < 4; ++j) num[j] += ws * qs::mppi_delta<BOX>(un[j], sig, eps[j], lo[j], hi[j]);
        }
        double* o = io.cand + 4 * ki;
#pragma unroll
        for (int j = 0; j < 4; ++j) o[j] = qs::mppi_candidate(un[j], num[j], wsum);
    }
}

// the commit's decision for unit u from the candidate's J: the sample to take, or -1 for the candidate
template <bool DW>
__device__ __forceinline__ int commit_choice(const MppiArgs& a, long long u, double jc) {
    const qs::MppiStats st = qs::mppi_stats([&](int s) { return unit_cost<DW>(a, u, s); }, a.io.K, 1.0);
    return qs::mppi_take_candidate(jc, unit_cost<DW>(a, u, st.best)) ? -1 : st.best;
}
// the candidate clamped into the box as drone i's nominal rpm
template <bool BOX>
__device__ __forceinline__ void store_candidate(const MppiArgs& a, long long i) {
    for (int k = 0; k < a.io.T; ++k) {
        double v[4];
        mppi_tick_command<BOX>(a, 0.0, i, k, -1, v);
        double* o = a.io.rpm + 4 * ((long long)k * a.N + i);
        o[0] = v[0]; o[1] = v[1]; o[2] = v[2]; o[3] = v[3];
    }
}

template <int EFF, bool BOX>
__global__ void __launch_bounds__(kMppiTPB) mppi_commit_kernel(const __grid_constant__ MppiArgs a) {
    const QsMppiIO& io = a.io;
    if constexpr (EFF & QS_EFFECT_DW) {
        __shared__ double pos_s[3 * kMppiTPB];
        __shared__ double jc_s[kMppiTPB];
        const DwSlot sl = dw_slot(a, a.N / a.D);
        const long long e = sl.G, i = e * a.D + sl.q;
        const int t = threadIdx.x;
        if (!io.cand) {                                               // the nominal's own rollout (its rpm stored unchanged)
            const double J = mppi_rollout<EFF, BOX>(a, sl.live, i, 0, true, t, sl.b, pos_s);
            if (sl.live) io.cost_out[i] = J;
            return;
        }
        const double jc = mppi_rollout<EFF, BOX>(a, sl.live, i, -1, false, t, sl.b, pos_s);
        if (sl.live) jc_s[t] = jc;
        __syncthreads();
        int pick = -1;
        if (sl.live) {
            double sum = 0.0;                                         // the aviary's J in drone order
            for (int q = 0; q < a.D; ++q) sum += jc_s[sl.b + q];
            pick = commit_choice<true>(a, e, sum);
            if (io.pick && sl.q == 0) io.pick[e] = pick;
        }
        const double J = mppi_rollout<EFF, BOX>(a, sl.live, i, pick, true, t, sl.b, pos_s);
        if (sl.live) io.cost_out[i] = J;
    } else {
        const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
        if (i >= a.N) return;
        if (!io.cand) {
            io.cost_out[i] = mppi_rollout<EFF, BOX>(a, true, i, 0, true);
            return;
        }
        const double jc = mppi_rollout<EFF, BOX>(a, true, i, -1, false);
        const int pick = commit_choice<false>(a, i, jc);
        io.cost_out[i] = mppi_rollout<EFF, BOX>(a, true, i, pick, true);
        if (io.pick) io.pick[i] = pick;
    }
}

__global__ void mppi_noise_kernel(const QsMppiIO io, long long N) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long TN = (long long)io.T * N;
    if (g >= (long long)io.K * TN) return;
    const int s = (int)(g / TN);
    const long long r = g - s * TN;
    const int k = (int)(r / N);
    qs::mppi_eps(io.seed, k, s, r - k * N, io.iteration, io.noise + 4 * g);
}

enum MppiEntry { kSample, kUpdate, kCommit };

int mppi_check_sizes(const char* what, const QsMppiIO* io, int n_envs, int drones_per_env, int substeps) {
    if (int rc = traj_check_sizes(what, n_envs, drones_per_env, substeps, io->T)) return rc;
    if (io->K < 2 || io->K > kMaxSamples) return fail(QS_ERR_SIZE, what, "K (samples) must be in 2..1024");
    if (io->iteration < 0) return fail(QS_ERR_SIZE, what, "iteration must be >= 0");
    return 0;
}

template <MppiEntry WHICH>
int launch_mppi(const QsParams* p, const QsMppiIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects, void* stream,
                const char* what) {
    if (!p || !io) return fail(QS_ERR_NULL, what, "NULL params / io");
    if (!io->state0 || !io->rpm || !io->targets || !io->weights || !io->rpm_ref || !io->sigma)
        return fail(QS_ERR_NULL, what, "NULL state0 / rpm / targets / weights / rpm_ref / sigma");
    if (WHICH != kCommit && !io->J) return fail(QS_ERR_NULL, what, "NULL J");
    if (WHICH == kUpdate && !io->cand) return fail(QS_ERR_NULL, what, "NULL cand");
    if (WHICH == kCommit && (!io->states || !io->cost_out || (io->cand && !io->J)))
        return fail(QS_ERR_NULL, what, "NULL states / cost_out, or J with cand");
    if (int rc = mppi_check_sizes(what, io, n_envs, drones_per_env, substeps)) return rc;
    if (WHICH == kUpdate && !(isfinite(io->temperature) && io->temperature > 0.0))
        return fail(QS_ERR_SIZE, what, "temperature must be finite and > 0");
    if (io->per_tick != 0 && io->per_tick != 1) return fail(QS_ERR_SIZE, what, "per_tick must be 0 or 1");
    if (!io->rpm_lo != !io->rpm_hi) return fail(QS_ERR_NULL, what, "rpm_lo and rpm_hi are both given or both NULL");
    if (int rc = traj_check_effects(what, effects, io->phys, nullptr, true)) return rc;
    const bool dw = effects & QS_EFFECT_DW;
    if (dw && drones_per_env > kMppiTPB) return fail(QS_ERR_UNSUPPORTED, what, "downwash needs drones_per_env <= 128");
    const long long N = (long long)n_envs * drones_per_env;
    MppiArgs a;
    memset(&a, 0, sizeof(a));
    a.P = *p; a.io = *io;
    a.N = N;
    a.D = drones_per_env; a.substeps = substeps;
    a.tpb = dw ? block_size_for(drones_per_env, kMppiTPB) : kMppiTPB;
    const long long per_cta = dw ? a.tpb / drones_per_env : kMppiTPB;   // groups (downwash) or threads per CTA
    const long long work = WHICH == kUpdate ? 0 : WHICH == kSample ? (dw ? (long long)n_envs * io->K : N * io->K) : (dw ? n_envs : N);
    const long long blocks = WHICH == kUpdate ? ((dw ? n_envs : N) + kUpdWarps - 1) / kUpdWarps : (work + per_cta - 1) / per_cta;
    if (blocks > 0x7fffffffLL) return fail(QS_ERR_SIZE, what, "the grid exceeds 2^31-1 CTAs");
    const size_t smem = WHICH == kUpdate ? (size_t)kUpdWarps * 2 * io->K * sizeof(double) : 0;
    const bool box = io->rpm_lo != nullptr;
    return traj_launch<PlanEffects>(what, effects, [box](auto EFF) {
        return with_bool(box, [](auto BOX) {
            constexpr int E = decltype(EFF)::value;
            constexpr bool B = decltype(BOX)::value;
            return WHICH == kSample ? mppi_sample_kernel<E, B> : WHICH == kUpdate ? mppi_update_kernel<(E & QS_EFFECT_DW) != 0, B> : mppi_commit_kernel<E, B>;
        });
    }, (unsigned)blocks, WHICH == kUpdate ? 32 * kUpdWarps : kMppiTPB, smem, (cudaStream_t)stream, a);
}

}  // namespace
}  // namespace qsi

using namespace qsi;

extern "C" {

int qs_sizeof_mppi_io(void) { return (int)sizeof(QsMppiIO); }

int qs_mppi_sample(const QsParams* p, const QsMppiIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                   void* stream) {
    return launch_mppi<kSample>(p, io, n_envs, drones_per_env, substeps, effects, stream, "qs_mppi_sample");
}

int qs_mppi_update(const QsParams* p, const QsMppiIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                   void* stream) {
    return launch_mppi<kUpdate>(p, io, n_envs, drones_per_env, substeps, effects, stream, "qs_mppi_update");
}

int qs_mppi_commit(const QsParams* p, const QsMppiIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                   void* stream) {
    return launch_mppi<kCommit>(p, io, n_envs, drones_per_env, substeps, effects, stream, "qs_mppi_commit");
}

int qs_mppi_noise(const QsMppiIO* io, int n_envs, int drones_per_env, void* stream) {
    const char* what = "qs_mppi_noise";
    if (!io || !io->noise) return fail(QS_ERR_NULL, what, "NULL io / noise");
    if (int rc = mppi_check_sizes(what, io, n_envs, drones_per_env, 1)) return rc;
    const long long N = (long long)n_envs * drones_per_env, blocks = ((long long)io->K * io->T * N + kMppiTPB - 1) / kMppiTPB;
    if (blocks > 0x7fffffffLL) return fail(QS_ERR_SIZE, what, "the grid exceeds 2^31-1 CTAs");
    mppi_noise_kernel<<<(unsigned)blocks, kMppiTPB, 0, (cudaStream_t)stream>>>(*io, N);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, what);
}

}  // extern "C"
