// ilqr_adjoint.cu -- qs_ilqr_adjoint / qs_ilqr_adjoint_rollout: the derivative of a batched iLQR solution (include/quadsim.h,
// DESIGN.md 4.5.1 "Gradients of the solution").  At the returned trajectory the derivative is one more LQR problem with the
// solve's Jacobians and stage Hessians at mu = 0 and the linear terms -g_X (state) and -g_U (command), on the free rotors only.
//   ilqr_adjoint_kernel<EFF, BOX>:         its Riccati pass.  One warp per drone for all T ticks, lane j running column j of
//                                          riccati.cuh's phases on the drone's workspace in shared memory, as
//                                          ilqr_backward_kernel does; no mu ladder (a failed factor sets status).
//   ilqr_adjoint_rollout_kernel<EFF, BOX>: the linear forward pass w_k = k_k + K_k dz_k, dz_{k+1} = F_k [dz_k; w_k] from dz_0 = 0.
//                                          One warp per drone as well: the tick's 13 C-double Jacobian block is one contiguous
//                                          read per warp (thread per drone would read 32 blocks 1.8 to 2.2 KB apart per load),
//                                          and the 17 rows of dz_{k+1} are 17 lanes' dot products.
// BOX = true reads the held rotors from the solve's `active` (nonzero: held, their w is 0); it does not solve a QP.
#include <type_traits>
#include "qs_common.cuh"
#include "dyn_tangent.cuh"
#include "riccati.cuh"
#include "traj_io.cuh"

namespace qsi {
namespace {

constexpr int kAdjWarps = 4;          // drones (warps) per CTA, both kernels

struct IlqrAdjArgs {
    QsParams P;
    QsIlqrAdjointIO io;
    long long N;
    int D;
};

// F = [A | B] of tick k of drone i in the workspace: qs_dyn_tick_jac's block (one coalesced warp read) and with drag the rows
// of the clipped RPMs, as ilqr_backward_kernel builds it
template <int EFF, int NZ>
__device__ __forceinline__ void adj_load_f(const QsIlqrAdjointIO& io, const qs::RicWs<NZ>& w, const qs::PhysRow& c, long long ki,
                                           int lane) {
    constexpr int M = NZ + 4, C = (EFF & QS_EFFECT_DRAG) ? 21 : 17;
    const double* jb = io.jac + ki * 13 * C;
    for (int idx = lane; idx < 13 * C; idx += 32) {
        const int r = idx / C, cc = idx - r * C;
        w.F[r * M + qs::ric_f_col<NZ>(cc)] = jb[idx];
    }
    if (EFF & QS_EFFECT_DRAG) {
        double raw[4], cd[4];
        const double one[4] = {1.0, 1.0, 1.0, 1.0};
        ld4(io.rpm, ki, raw);
        qs::rpm_clip_jvp(raw, c.max_rpm, one, 0.0, cd);
        for (int idx = lane; idx < 4 * M; idx += 32) qs::ric_f_aug(w, idx, cd);
    }
}

// Both kernels keep 3 CTAs (12 warps) per SM, as the backward pass of the solve runs
template <int EFF, bool BOX>
__global__ void __launch_bounds__(32 * kAdjWarps, 3) ilqr_adjoint_kernel(const __grid_constant__ IlqrAdjArgs a) {
    constexpr int NZ = (EFF & QS_EFFECT_DRAG) ? 17 : 13, M = NZ + 4;
    __shared__ double sm[kAdjWarps][qs::RicWs<NZ>::DOUBLES];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long long i = (long long)blockIdx.x * kAdjWarps + wid;
    const long long N = a.N;
    if (i >= N) return;                                               // the whole warp: no CTA-wide barrier below
    const QsIlqrAdjointIO& io = a.io;
    const qs::RicWs<NZ> w = qs::ric_ws<NZ>(sm[wid]);
    const qs::PhysRow c = row_of(a, i);
    const double* wt = io.weights + (long long)qs::kWeightsRow * (i / a.D);
    double Rt[4];
    qs::rel_weights(wt, c, Rt);
    const int T = io.T;
    for (int idx = lane; idx < NZ * NZ; idx += 32) w.V[idx] = 0.0;
    if (lane < NZ) w.vx[lane] = 0.0;
    bool ok = true;
    for (int k = T - 1; k >= 0; --k) {
        const long long ki = (long long)k * N + i;
        __syncwarp();
        if (lane < 13)                                                // phase S: the state after tick k
            qs::ric_stage_adj(w, lane, wt[qs::stage_weights(k, T) + lane], io.g_states[(long long)k * 13 * N + plane_at(N, i, lane)]);
        adj_load_f<EFF, NZ>(io, w, c, ki, lane);
        double gu[4] = {0.0, 0.0, 0.0, 0.0};
        if (io.g_rpm) ld4(io.g_rpm, ki, gu);
        int act[4] = {0, 0, 0, 0};
        if constexpr (BOX) {
#pragma unroll
            for (int j = 0; j < 4; ++j) act[j] = io.active[4 * ki + j] != 0;
        }
        __syncwarp();
        if (lane < M) qs::ric_col_H(w, lane);
        __syncwarp();
        qs::RicBoxGains G;
        if (!qs::ric_gains_adj(w, Rt, gu, act, G)) {                 // the same bits in every lane: a uniform branch
            ok = false;
            break;
        }
        if (lane < NZ) {
            if constexpr (BOX) qs::ric_col_K_box(w, lane, G);
            else qs::ric_col_K(w, lane, G);
        }
        __syncwarp();
        if (lane < NZ) qs::ric_col_V(w, lane, G);
        double* Ko = io.K + ki * 4 * NZ;
        for (int idx = lane; idx < 4 * NZ; idx += 32) Ko[idx] = w.K[idx];
        if (lane < 4) io.k[4 * ki + lane] = G.k[lane];
        __syncwarp();
        if (lane < NZ) qs::ric_col_sym(w, lane);
    }
    if (lane == 0) io.status[i] = ok ? 0 : 1;
}

template <int EFF, bool BOX>
__global__ void __launch_bounds__(32 * kAdjWarps, 3) ilqr_adjoint_rollout_kernel(const __grid_constant__ IlqrAdjArgs a) {
    constexpr int NZ = (EFF & QS_EFFECT_DRAG) ? 17 : 13, M = NZ + 4;
    __shared__ double sm[kAdjWarps][NZ * M + 4 * NZ + M];              // F, K, y = [dz | w]
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long long i = (long long)blockIdx.x * kAdjWarps + wid;
    const long long N = a.N;
    if (i >= N) return;
    const QsIlqrAdjointIO& io = a.io;
    const int T = io.T;
    if (io.status[i] != 0) {                                          // the adjoint had no factor: NaN gradients
        for (int k = 0; k < T; ++k) {
            if (lane < 4) io.w[4 * ((long long)k * N + i) + lane] = NAN;
            if (lane < 13) io.dx[(long long)k * 13 * N + plane_at(N, i, lane)] = NAN;
        }
        return;
    }
    qs::RicWs<NZ> w;
    w.F = sm[wid];
    double* Ks = w.F + NZ * M;
    double* y = Ks + 4 * NZ;
    const qs::PhysRow c = row_of(a, i);
    if (lane < NZ) y[lane] = 0.0;
    for (int k = 0; k < T; ++k) {
        const long long ki = (long long)k * N + i;
        __syncwarp();
        adj_load_f<EFF, NZ>(io, w, c, ki, lane);
        const double* Kg = io.K + ki * 4 * NZ;
        for (int idx = lane; idx < 4 * NZ; idx += 32) Ks[idx] = Kg[idx];
        __syncwarp();
        double v = 0.0;
        if (lane < 4) {
            const bool held = BOX && io.active[4 * ki + lane] != 0;
            v = qs::ric_adj_w<NZ>(Ks + lane * NZ, io.k[4 * ki + lane], y, held);
        }
        __syncwarp();
        if (lane < 4) {
            y[NZ + lane] = v;
            io.w[4 * ki + lane] = v;
        }
        __syncwarp();
        if (lane < NZ) v = qs::ric_adj_next(w, lane, y);
        __syncwarp();
        if (lane < NZ) y[lane] = v;
        if (lane < 13) io.dx[(long long)k * 13 * N + plane_at(N, i, lane)] = v;
    }
}

template <bool ROLLOUT>
int launch_adjoint(const QsParams* p, const QsIlqrAdjointIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                   void* stream, const char* what) {
    if (!p || !io) return fail(QS_ERR_NULL, what, "NULL params / io");
    if (!io->jac || !io->rpm || !io->weights || !io->K || !io->k || !io->status)
        return fail(QS_ERR_NULL, what, "NULL jac / rpm / weights / K / k / status");
    if (!ROLLOUT && !io->g_states) return fail(QS_ERR_NULL, what, "NULL g_states");
    if (ROLLOUT && (!io->w || !io->dx)) return fail(QS_ERR_NULL, what, "NULL w / dx");
    if (int rc = traj_check_sizes(what, n_envs, drones_per_env, substeps, io->T)) return rc;
    if (int rc = traj_check_effects(what, effects, io->phys, nullptr)) return rc;
    const long long N = (long long)n_envs * drones_per_env;
    const long long blocks = (N + kAdjWarps - 1) / kAdjWarps;
    if (blocks > 0x7fffffffLL) return fail(QS_ERR_SIZE, what, "the grid exceeds 2^31-1 CTAs");
    IlqrAdjArgs a;
    memset(&a, 0, sizeof(a));
    a.P = *p; a.io = *io;
    a.N = N;
    a.D = drones_per_env;
    const bool box = io->active != nullptr;
    return traj_launch(what, effects, [box](auto EFF) {
        constexpr int E = decltype(EFF)::value;
        if (ROLLOUT) return box ? ilqr_adjoint_rollout_kernel<E, true> : ilqr_adjoint_rollout_kernel<E, false>;
        return box ? ilqr_adjoint_kernel<E, true> : ilqr_adjoint_kernel<E, false>;
    }, (unsigned)blocks, 32 * kAdjWarps, 0, (cudaStream_t)stream, a);
}

}  // namespace
}  // namespace qsi

using namespace qsi;

extern "C" {

int qs_sizeof_ilqr_adjoint_io(void) { return (int)sizeof(QsIlqrAdjointIO); }

int qs_ilqr_adjoint(const QsParams* p, const QsIlqrAdjointIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                    void* stream) {
    return launch_adjoint<false>(p, io, n_envs, drones_per_env, substeps, effects, stream, "qs_ilqr_adjoint");
}

int qs_ilqr_adjoint_rollout(const QsParams* p, const QsIlqrAdjointIO* io, int n_envs, int drones_per_env, int substeps,
                            unsigned effects, void* stream) {
    return launch_adjoint<true>(p, io, n_envs, drones_per_env, substeps, effects, stream, "qs_ilqr_adjoint_rollout");
}

}  // extern "C"
