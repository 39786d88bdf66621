// policy_actor.cuh -- what the policy-trajectory translation units (dyn_policy_traj.cu: the forward and its VJP; dyn_policy_jvp.cu:
// forward mode) share: the CTA's float64 GEMM on the FP64 tensor cores, the actor's forward pass over the CTA's observation rows
// and, on the host, the argument checks and the aviaries per CTA.  A CTA owns M whole aviaries (DESIGN.md 4.5).
#pragma once
#include "qs_common.cuh"
#include "mlp_adjoint.cuh"
#include "traj_io.cuh"

namespace qsi {
namespace {

constexpr int kPolTPB = 256;
constexpr int kPolMG = 8;            // aviaries per CTA come in m-tiles of 8 rows (mma.m8n8k4)
constexpr int kPolMaxM = 16;         // aviaries per CTA at most
constexpr int kPolNT = 4;            // n-tiles a warp carries per pass: one A fragment per m-tile feeds kPolNT products
constexpr size_t kPolSmemMax = 227 * 1024;

// C[r][n] = sum_k X[r][k] Bm(k, n) for the CTA's M rows (X in shared memory, row stride ldx) and n < Nn, with
// Bm(k, n) = W[k * sk + n * sn] read from global memory: (sk, sn) = (Nout, 1) is a layer, (1, Nout) its transpose.  epi(r, n, c)
// receives every element once.  Every thread of the CTA calls it; no barrier inside.
//
// The product runs on the FP64 tensor cores (mma.sync.aligned.m8n8k4.row.col.f64): lane 4 g + t holds A[g][t], B[t][g] and
// C[g][2 t], C[g][2 t + 1].  A warp owns kPolNT n-tiles at a time for all M / 8 m-tiles, so each weight is loaded exactly once
// per CTA and layer (no other warp needs it: staging it through shared memory would add a copy and no reuse) and each A fragment
// feeds kPolNT products.  Built with -DQS_POLICY_GEMM_FMA the same interface runs mlp_adjoint.cuh's plain FMA loop (what the
// host build uses), four rows per thread: the A/B partner of DESIGN.md 4.5's measurement, not a run-time option.
template <class Epi>
__device__ __forceinline__ void cta_gemm(int M, const double* X, int ldx, const double* W, int sk, int sn, int K, int Nn, Epi epi) {
#if defined(QS_POLICY_GEMM_FMA)
    for (int it = threadIdx.x; it < Nn * (M / 4); it += blockDim.x) {
        const int n = it % Nn, g = it / Nn;
        double acc[4] = {0.0, 0.0, 0.0, 0.0};
        for (int k = 0; k < K; ++k) {
            const double w = W[(long long)k * sk + (long long)n * sn];
#pragma unroll
            for (int m = 0; m < 4; ++m) acc[m] = qs::fmad(X[(size_t)(g * 4 + m) * ldx + k], w, acc[m]);
        }
#pragma unroll
        for (int m = 0; m < 4; ++m) epi(g * 4 + m, n, acc[m]);
    }
#else
    const int warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int MT = M / kPolMG;                                   // 1 or 2
    for (int nt0 = warp * kPolNT; nt0 * 8 < Nn; nt0 += nwarps * kPolNT) {
        double c[kPolNT][2][2];
#pragma unroll
        for (int j = 0; j < kPolNT; ++j) c[j][0][0] = c[j][0][1] = c[j][1][0] = c[j][1][1] = 0.0;
        for (int k0 = 0; k0 < K; k0 += 4) {
            const int kk = k0 + t;
            const bool kin = kk < K;
            const double a0 = kin ? X[(size_t)g * ldx + kk] : 0.0;
            const double a1 = (kin && MT > 1) ? X[(size_t)(8 + g) * ldx + kk] : 0.0;
            double bfr[kPolNT];
#pragma unroll
            for (int j = 0; j < kPolNT; ++j) {
                const int n = (nt0 + j) * 8 + g;
                bfr[j] = (kin && n < Nn) ? W[(long long)kk * sk + (long long)n * sn] : 0.0;
            }
#pragma unroll
            for (int j = 0; j < kPolNT; ++j) {
                asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                             : "+d"(c[j][0][0]), "+d"(c[j][0][1]) : "d"(a0), "d"(bfr[j]));
                if (MT > 1)
                    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                                 : "+d"(c[j][1][0]), "+d"(c[j][1][1]) : "d"(a1), "d"(bfr[j]));
            }
        }
#pragma unroll
        for (int j = 0; j < kPolNT; ++j)
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int n = (nt0 + j) * 8 + 2 * t + h;
                    if (mt < MT && n < Nn) epi(mt * 8 + g, n, c[j][mt][h]);
                }
    }
#endif
}

// The actor's hidden layers (and, with `mean`, its output layer) over the CTA's M observation rows (a.io: the actor's layers).  Layer l's activations go
// to act + (keep ? l : l & 1) * M * maxw, row stride maxw.  Every thread of the CTA calls it; it ends on a barrier.
template <class Args>
__device__ void actor_forward(const Args& a, const double* obs, double* act, bool keep, double* mean) {
    const auto& io = a.io;
    const int layers = io.depth + (mean ? 1 : 0);
    const double* x = obs;
    int K = io.in_dim, ldx = io.in_dim;
    for (int l = 0; l < layers; ++l) {
        const bool last = l == io.depth;
        const int Nout = last ? io.out_dim : io.width[l];
        double* dst = last ? mean : act + (size_t)(keep ? l : (l & 1)) * a.M * a.maxw;
        const int ldd = last ? io.out_dim : a.maxw;
        const double* bias = io.b[l];
        const int kind = io.activation;
        cta_gemm(a.M, x, ldx, io.w[l], Nout, 1, K, Nout, [&](int r, int n, double v) {
            v = v + bias[n];
            dst[(size_t)r * ldd + n] = last ? v : qs::mlp_act(kind, v);
        });
        __syncthreads();
        x = dst; K = Nout; ldx = ldd;
    }
}

// the applied RPMs of tick k, from the saved raw action
template <class Args>
__device__ __forceinline__ void applied_rpm(const Args& a, const qs::PhysRow& c, long long i, int k, double raw_a[4], double aa[4],
                                            double raw[4], double u[4]) {
    aa[0] = aa[1] = aa[2] = aa[3] = 0.0;
    for (int j = 0; j < a.A; ++j) {
        raw_a[j] = a.io.actions[((long long)k * a.N + i) * a.A + j];
        aa[j] = qs::clampd(raw_a[j], -1.0, 1.0);
    }
    qs::policy_rpm(a.A, c, aa, raw);
    clip_rpm(raw, c.max_rpm, u);
}

// ---- host: the checks of every policy-trajectory entry point, in this order around its own.  `what` is the entry point's name.
template <class IO>
int policy_check_inputs(const QsParams* p, const IO* io, const char* what) {
    if (!p || !io) return fail(QS_ERR_NULL, what, "NULL params / io");
    if (!io->state0 || !io->action_buffer || !io->log_std || !io->states || !io->actions || !io->obs)
        return fail(QS_ERR_NULL, what, "NULL state0 / action_buffer / log_std / states / actions / obs");
    return 0;
}
// the sizes, the action type, the actor and the effects; maxw: the widest hidden layer.  t_phys: the constants' tangent (forward
// mode) or NULL
template <class IO>
int policy_check_shape(const IO* io, int act_type, int n_envs, int drones_per_env, int substeps, unsigned effects, const double* t_phys,
                       const char* what, int& maxw) {
    if (int rc = traj_check_sizes(what, n_envs, drones_per_env, substeps, io->T)) return rc;
    if (act_type != QS_ACT_RPM && act_type != QS_ACT_ONE_D_RPM)
        return fail(QS_ERR_UNSUPPORTED, what, "only the RPM and ONE_D_RPM actions have an adjoint (PID, VEL and ONE_D_PID run the embedded "
                                              "controller)");
    const int A = act_width(act_type), D = drones_per_env;
    if (io->act_buffer_size <= 0) return fail(QS_ERR_SIZE, what, "act_buffer_size must be > 0");
    if (io->activation != QS_MLP_TANH && io->activation != QS_MLP_RELU) return fail(QS_ERR_ENUM, what, "bad activation");
    if (io->depth < 1 || io->depth > QS_MLP_MAX_HIDDEN) return fail(QS_ERR_SIZE, what, "1 to 4 hidden layers");
    maxw = 0;
    for (int l = 0; l <= io->depth; ++l) {
        if (!io->w[l] || !io->b[l]) return fail(QS_ERR_NULL, what, "NULL weight / bias");
        if (l < io->depth) {
            if (io->width[l] < 1 || io->width[l] > QS_MLP_MAX_WIDTH) return fail(QS_ERR_SIZE, what, "hidden widths must be 1 .. 256");
            maxw = io->width[l] > maxw ? io->width[l] : maxw;
        }
    }
    if (D * A > 32 || D > kPolTPB / kPolMG) return fail(QS_ERR_UNSUPPORTED, what, "up to 32 action outputs (D * A) and 32 drones per aviary");
    if (io->in_dim != D * (12 + io->act_buffer_size * A) || io->out_dim != D * A)
        return fail(QS_ERR_SIZE, what, "in_dim must be D (12 + B A) and out_dim D A");
    return traj_check_effects(what, effects, io->phys, t_phys);
}
// Doubles of shared memory per aviary of the VJP: the observation row, every hidden layer, the mean action's cotangent, two
// cotangent buffers of max(in_dim, maxw) and the history ring.  Every policy-trajectory kernel fits 8 aviaries (or 8 rows of one
// aviary's tangents) where this does, so that no entry point refuses what another accepts.
template <class IO>
size_t policy_vjp_doubles(const IO* io, int D, int A, int maxw) {
    const size_t cw = maxw > io->in_dim ? maxw : io->in_dim;
    return (size_t)io->in_dim + (size_t)io->depth * maxw + io->out_dim + 2 * cw + (size_t)D * io->act_buffer_size * A;
}
// M: aviaries per CTA for `per` doubles of shared memory per aviary, a multiple of kPolMG up to kPolMaxM with M D <= kPolTPB;
// refused where the VJP's 8 aviaries do not fit
template <class IO>
int policy_ctas(const IO* io, int D, int A, int maxw, size_t per, const char* what, int& M) {
    M = (int)(kPolSmemMax / (per * sizeof(double)));
    if (kPolSmemMax / (policy_vjp_doubles(io, D, A, maxw) * sizeof(double)) < (size_t)kPolMG) M = 0;
    M = M < kPolTPB / D ? M : kPolTPB / D;
    M = M < kPolMaxM ? M : kPolMaxM;
    M -= M % kPolMG;
    if (M < kPolMG)
        return fail(QS_ERR_UNSUPPORTED, what, "the observation rows, hidden activations and cotangents of 8 aviaries exceed the 227 KB of "
                                       "shared memory of a CTA (shorten the action buffer with a lower ctrl_freq, or use fewer drones "
                                       "per aviary)");
    return 0;
}

}  // namespace
}  // namespace qsi
