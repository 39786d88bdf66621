// ilqr.cu -- qs_ilqr_backward / qs_ilqr_line_search / qs_ilqr_commit: batched iLQR of raw-RPM trajectories of Physics.DYN
// (include/quadsim.h, DESIGN.md 4.5.1), one independent problem per drone, on qs_dyn_tick_jac's per-tick Jacobians.
//   ilqr_backward_kernel<EFF, BOX>:    one warp per drone for all T ticks; lane j runs column j of riccati.cuh's phases on
//                                      the drone's workspace in shared memory.  The tick's Jacobian block is one contiguous
//                                      13 C-double read per warp.
//   ilqr_line_search_kernel<EFF, BOX>: one thread per (drone, step size), the step sizes of a drone in neighbouring lanes so
//                                      that they read its K and k rows together.
//   ilqr_commit_kernel<EFF, BOX>:      one thread per drone.
// The rollouts of the last two are ilqr_rollout, whose tick is dyn_traj_kernel's (clip_rpm, dyn_tick_k, round_to_planes), so a
// committed trajectory is qs_dyn_traj's output for the committed rpm and the commit's J is the line search's J bit for bit.
// BOX = true is the control-limited variant (qs_ilqr_box_*): the backward solves riccati.cuh's box QP per tick and writes the
// held rotors, the rollouts clamp each command to [rpm_lo, rpm_hi] (ld_box's row) before the tick, the stage cost and the
// commit's store.
#include <type_traits>
#include "qs_common.cuh"
#include "dyn_tangent.cuh"
#include "lqr_law.cuh"
#include "riccati.cuh"
#include "traj_io.cuh"

namespace qsi {
namespace {

constexpr int kBwdWarps = 4;          // drones (warps) per backward CTA
constexpr int kIlqrTPB = 128;         // line search and commit
constexpr int kMaxAlpha = 16;
constexpr int kMaxRestarts = 8;

struct IlqrArgs {
    QsParams P;
    QsIlqrIO io;
    long long N;
    int D, substeps;
};
struct IlqrBoxArgs : IlqrArgs {
    const double* lo;               // [N][4], or [T][N][4] with per_tick
    const double* hi;
    signed char* active;            // [T][N][4], nullable
    int per_tick;
};
template <bool BOX>
using IlqrArgsOf = std::conditional_t<BOX, IlqrBoxArgs, IlqrArgs>;

// BOX: at least 3 CTAs (12 warps) per SM, as the unconstrained kernel runs.  Left free, the drag variant takes 196 registers
// and 8 warps per SM, and its backward pass ran 37% longer than with the 24 spilled bytes this bound costs (DESIGN.md 4.5.1).
// 0 leaves the unconstrained kernels as they were.
template <int EFF, bool BOX>
__global__ void __launch_bounds__(32 * kBwdWarps, BOX ? 3 : 0) ilqr_backward_kernel(const __grid_constant__ IlqrArgsOf<BOX> a) {
    constexpr int NZ = (EFF & QS_EFFECT_DRAG) ? 17 : 13, M = NZ + 4, C = (EFF & QS_EFFECT_DRAG) ? 21 : 17;
    __shared__ double sm[kBwdWarps][qs::RicWs<NZ>::DOUBLES];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long long i = (long long)blockIdx.x * kBwdWarps + wid;
    const long long N = a.N;
    if (i >= N) return;                                               // the whole warp: no CTA-wide barrier below
    const QsIlqrIO& io = a.io;
    const qs::RicWs<NZ> w = qs::ric_ws<NZ>(sm[wid]);
    const qs::PhysRow c = row_of(a, i);
    const double* wt = io.weights + (long long)qs::kWeightsRow * (i / a.D);
    double Rt[4], uref[4];
    qs::rel_weights(wt, c, Rt);
    ld4(io.rpm_ref, i, uref);
    const int T = io.T;
    double mu = io.mu[i], dV1 = 0.0, dV2 = 0.0;
    int status = 0;
    for (int restarts = 0;; ++restarts) {
        for (int idx = lane; idx < NZ * NZ; idx += 32) w.V[idx] = 0.0;
        if (lane < NZ) w.vx[lane] = 0.0;
        dV1 = dV2 = 0.0;
        bool ok = true;
        for (int k = T - 1; k >= 0; --k) {
            const long long ki = (long long)k * N + i;
            __syncwarp();
            if (lane < 13) {                                          // phase S: the cost of the state after tick k
                const long long at = (long long)k * 13 * N + plane_at(N, i, lane);
                qs::ric_stage(w, lane, io.states[at] - io.targets[at], wt[qs::stage_weights(k, T) + lane]);
            }
            const double* jb = io.jac + ki * 13 * C;
            for (int idx = lane; idx < 13 * C; idx += 32) {
                const int r = idx / C, cc = idx - r * C;
                w.F[r * M + qs::ric_f_col<NZ>(cc)] = jb[idx];
            }
            double raw[4], du[4];
            ld4(io.rpm, ki, raw);
            if (EFF & QS_EFFECT_DRAG) {
                const double one[4] = {1.0, 1.0, 1.0, 1.0};
                double cd[4];
                qs::rpm_clip_jvp(raw, c.max_rpm, one, 0.0, cd);
                for (int idx = lane; idx < 4 * M; idx += 32) qs::ric_f_aug(w, idx, cd);
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) du[j] = raw[j] - uref[j];
            __syncwarp();
            if (lane < M) qs::ric_col_H(w, lane);
            __syncwarp();
            std::conditional_t<BOX, qs::RicBoxGains, qs::RicGains> G;
            if constexpr (BOX) {
                double lo[4], hi[4];                                  // the box of k: the command's box minus u_nom
                ld_box(a.lo, a.hi, a.per_tick, k, a.N, i, lo, hi);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    lo[j] -= raw[j];
                    hi[j] -= raw[j];
                }
                if (!qs::ric_gains_box(w, Rt, du, lo, hi, mu, G, dV1, dV2)) {   // the same bits in every lane: uniform
                    ok = false;
                    break;
                }
                if (lane < NZ) qs::ric_col_K_box(w, lane, G);
            } else {
                if (!qs::ric_gains(w, Rt, du, mu, G, dV1, dV2)) {      // the same bits in every lane: a uniform branch
                    ok = false;
                    break;
                }
                if (lane < NZ) qs::ric_col_K(w, lane, G);
            }
            __syncwarp();
            if (lane < NZ) qs::ric_col_V(w, lane, G);
            double* Ko = io.K + ki * 4 * NZ;
            for (int idx = lane; idx < 4 * NZ; idx += 32) Ko[idx] = w.K[idx];
            if (lane < 4) io.k[4 * ki + lane] = G.k[lane];
            if constexpr (BOX) {
                if (a.active && lane < 4) a.active[4 * ki + lane] = (signed char)G.act[lane];
            }
            __syncwarp();
            if (lane < NZ) qs::ric_col_sym(w, lane);
        }
        __syncwarp();
        if (ok) break;
        mu = fmax(1e-6, 10.0 * mu);
        if (restarts == kMaxRestarts) {
            status = 1;
            break;
        }
    }
    if (lane == 0) {
        io.mu[i] = mu;
        io.status[i] = status;
        io.dV[2 * i] = dV1;
        io.dV[2 * i + 1] = dV2;
    }
}

// J of the rollout u_k = rpm[k] + alpha k_k + K_k (z_k - z_nom,k) from z_nom,0 (K, k NULL: zero).  With `commit` the rollout
// overwrites tick k's nominal rpm and state after reading them.
template <int EFF, bool BOX>
__device__ __forceinline__ double ilqr_rollout(const IlqrArgsOf<BOX>& a, long long i, double alpha, bool commit) {
    constexpr int NZ = (EFF & QS_EFFECT_DRAG) ? 17 : 13;
    const QsIlqrIO& io = a.io;
    const long long N = a.N;
    const qs::PhysRow c = row_of(a, i);
    const double* wt = io.weights + (long long)qs::kWeightsRow * (i / a.D);
    double Rt[4], uref[4];
    qs::rel_weights(wt, c, Rt);
    ld4(io.rpm_ref, i, uref);
    qs::Drone d, dn;                                                  // the rollout's and the nominal's state before tick k
    ld_state(io.state0, N, i, d);
    dn = d;
    double up[4] = {0, 0, 0, 0}, upn[4] = {0, 0, 0, 0};               // drag: their clipped RPMs of tick k - 1
    if ((EFF & QS_EFFECT_DRAG) && io.last_rpm) {
        ld4(io.last_rpm, i, up);
        ld4(io.last_rpm, i, upn);
    }
    double J = 0.0;
    for (int k = 0; k < io.T; ++k) {
        const long long ki = (long long)k * N + i;
        double raw[4], u[4], uc[4];
        ld4(io.rpm, ki, raw);
        double dz[NZ], x[13], xn[13];
        drone_vec(d, x);
        drone_vec(dn, xn);
#pragma unroll
        for (int r = 0; r < 13; ++r) dz[r] = x[r] - xn[r];
        if constexpr (NZ == 17) {
#pragma unroll
            for (int j = 0; j < 4; ++j) dz[13 + j] = up[j] - upn[j];
        }
        const double* Kk = io.K ? io.K + ki * 4 * NZ : nullptr;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            double v = raw[j];
            if (io.k) v += alpha * io.k[4 * ki + j];
            if (Kk) v += lqr_feedback<NZ>([&](int q) { return Kk[j * NZ + q]; }, dz);
            u[j] = v;
        }
        if constexpr (BOX) {
            double lo[4], hi[4];
            ld_box(a.lo, a.hi, a.per_tick, k, a.N, i, lo, hi);
#pragma unroll
            for (int j = 0; j < 4; ++j) u[j] = qs::clampd(u[j], lo[j], hi[j]);
        }
        if (commit) {
            double* o = io.rpm + 4 * ki;
            o[0] = u[0]; o[1] = u[1]; o[2] = u[2]; o[3] = u[3];
        }
        clip_rpm(u, c.max_rpm, uc);
        double R_last[9];
        qs::dyn_tick_k<EFF>(a.P, c, d, uc, up, 0.0, a.substeps, R_last);
        round_to_planes(d);
        double* sk = io.states + (long long)k * 13 * N;
        ld_state(sk, N, i, dn);                                       // the nominal state after tick k, before a commit's store
        if (commit) st_state(sk, N, i, d);
        qs::Drone rd;
        double ref[13];
        ld_state(io.targets + (long long)k * 13 * N, N, i, rd);
        drone_vec(rd, ref);
        drone_vec(d, x);
        J += qs::stage_cost(x, ref, wt + (k == io.T - 1 ? qs::kWeightsQFinal : qs::kWeightsQ), u, uref, Rt);   // stage_weights
        clip_rpm(raw, c.max_rpm, upn);
#pragma unroll
        for (int j = 0; j < 4; ++j) up[j] = uc[j];
    }
    return J;
}

template <int EFF, bool BOX>
__global__ void __launch_bounds__(kIlqrTPB) ilqr_line_search_kernel(const __grid_constant__ IlqrArgsOf<BOX> a) {
    const QsIlqrIO& io = a.io;
    const int na = io.n_alpha;
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= a.N * na) return;
    const long long i = g / na;
    const int s = (int)(g - i * na);
    double J = INFINITY;
    if (!(io.status && io.status[i]) && !(io.converged && io.converged[i])) J = ilqr_rollout<EFF, BOX>(a, i, io.alpha[s], false);
    io.J[(long long)s * a.N + i] = J;
}

template <int EFF, bool BOX>
__global__ void __launch_bounds__(kIlqrTPB) ilqr_commit_kernel(const __grid_constant__ IlqrArgsOf<BOX> a) {
    const QsIlqrIO& io = a.io;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long N = a.N;
    if (i >= N) return;
    const double Jn = io.cost_in[i];
    if (io.converged[i]) {
        io.cost_out[i] = Jn;
        return;
    }
    const double dV1 = io.dV[2 * i], dV2 = io.dV[2 * i + 1];
    if constexpr (BOX) {
        // k = 0 at every tick (dV2 = 1/2 sum k'Quu k = 0): the nominal is the box QPs' fixed point, typically every rotor held
        // at a bound.  No step can lower J there, so without this the drone would only raise mu until it overflows.
        if (io.status[i] == 0 && dV1 == 0.0 && dV2 == 0.0) {
            io.cost_out[i] = Jn;
            io.converged[i] = 1;
            return;
        }
    }
    int best = -1;
    if (io.status[i] == 0) {
        for (int s = 0; s < io.n_alpha; ++s) {
            const double al = io.alpha[s], Ja = io.J[(long long)s * N + i];
            const double expected = -(al * dV1 + al * al * dV2);
            if (Ja < Jn && Jn - Ja >= 1e-4 * expected && (best < 0 || al > io.alpha[best])) best = s;
        }
    }
    double mu = io.mu[i];
    if (best >= 0) {
        const double Jc = ilqr_rollout<EFF, BOX>(a, i, io.alpha[best], true);
        io.cost_out[i] = Jc;
        mu = mu / 10.0;
        if (mu < 1e-6) mu = 0.0;
        if (Jn - Jc < 1e-9 * Jn) io.converged[i] = 1;
    } else {
        io.cost_out[i] = Jn;
        mu = fmax(1e-6, 10.0 * mu);
    }
    io.mu[i] = mu;
}

enum IlqrEntry { kBackward, kLineSearch, kCommit };

// BOX: io = &box->base (both NULL when box is)
template <IlqrEntry WHICH, bool BOX>
int launch_ilqr(const QsParams* p, const QsIlqrIO* io, const QsIlqrBoxIO* box, int n_envs, int drones_per_env, int substeps,
                unsigned effects, void* stream, const char* what) {
    if (!p || !io) return fail(QS_ERR_NULL, what, "NULL params / io");
    if (BOX && (!box->rpm_lo || !box->rpm_hi)) return fail(QS_ERR_NULL, what, "NULL rpm_lo / rpm_hi");
    if (BOX && box->per_tick != 0 && box->per_tick != 1) return fail(QS_ERR_SIZE, what, "per_tick must be 0 or 1");
    if (!io->state0 || !io->rpm || !io->states || !io->targets || !io->weights || !io->rpm_ref)
        return fail(QS_ERR_NULL, what, "NULL state0 / rpm / states / targets / weights / rpm_ref");
    if (WHICH == kBackward && (!io->jac || !io->mu || !io->K || !io->k || !io->dV || !io->status))
        return fail(QS_ERR_NULL, what, "NULL jac / mu / K / k / dV / status");
    if (WHICH != kBackward && (!io->alpha || !io->J)) return fail(QS_ERR_NULL, what, "NULL alpha / J");
    if (WHICH == kCommit && (!io->mu || !io->dV || !io->status || !io->converged || !io->cost_in || !io->cost_out))
        return fail(QS_ERR_NULL, what, "NULL mu / dV / status / converged / cost_in / cost_out");
    if (int rc = traj_check_sizes(what, n_envs, drones_per_env, substeps, io->T)) return rc;
    if (WHICH != kBackward && (io->n_alpha <= 0 || io->n_alpha > kMaxAlpha))
        return fail(QS_ERR_SIZE, what, "n_alpha must be in 1..16");
    if (int rc = traj_check_effects(what, effects, io->phys, nullptr)) return rc;
    const long long N = (long long)n_envs * drones_per_env;
    const long long blocks = WHICH == kBackward ? (N + kBwdWarps - 1) / kBwdWarps
                             : WHICH == kLineSearch ? (N * io->n_alpha + kIlqrTPB - 1) / kIlqrTPB : (N + kIlqrTPB - 1) / kIlqrTPB;
    if (blocks > 0x7fffffffLL) return fail(QS_ERR_SIZE, what, "the grid exceeds 2^31-1 CTAs");
    IlqrArgsOf<BOX> a;
    memset(&a, 0, sizeof(a));
    a.P = *p; a.io = *io;
    a.N = N;
    a.D = drones_per_env; a.substeps = substeps;
    if constexpr (BOX) {
        a.lo = box->rpm_lo; a.hi = box->rpm_hi;
        a.active = box->active;
        a.per_tick = box->per_tick;
    }
    return traj_launch(what, effects, [](auto EFF) {
        constexpr int E = decltype(EFF)::value;
        return WHICH == kBackward ? ilqr_backward_kernel<E, BOX>
                                  : WHICH == kLineSearch ? ilqr_line_search_kernel<E, BOX> : ilqr_commit_kernel<E, BOX>;
    }, (unsigned)blocks, WHICH == kBackward ? 32 * kBwdWarps : kIlqrTPB, 0, (cudaStream_t)stream, a);
}

}  // namespace
}  // namespace qsi

using namespace qsi;

extern "C" {

int qs_sizeof_ilqr_io(void) { return (int)sizeof(QsIlqrIO); }

int qs_ilqr_backward(const QsParams* p, const QsIlqrIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                     void* stream) {
    return launch_ilqr<kBackward, false>(p, io, nullptr, n_envs, drones_per_env, substeps, effects, stream, "qs_ilqr_backward");
}

int qs_ilqr_line_search(const QsParams* p, const QsIlqrIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                        void* stream) {
    return launch_ilqr<kLineSearch, false>(p, io, nullptr, n_envs, drones_per_env, substeps, effects, stream,
                                           "qs_ilqr_line_search");
}

int qs_ilqr_commit(const QsParams* p, const QsIlqrIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                   void* stream) {
    return launch_ilqr<kCommit, false>(p, io, nullptr, n_envs, drones_per_env, substeps, effects, stream, "qs_ilqr_commit");
}

int qs_sizeof_ilqr_box_io(void) { return (int)sizeof(QsIlqrBoxIO); }

int qs_ilqr_box_backward(const QsParams* p, const QsIlqrBoxIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                         void* stream) {
    return launch_ilqr<kBackward, true>(p, io ? &io->base : nullptr, io, n_envs, drones_per_env, substeps, effects, stream,
                                        "qs_ilqr_box_backward");
}

int qs_ilqr_box_line_search(const QsParams* p, const QsIlqrBoxIO* io, int n_envs, int drones_per_env, int substeps,
                            unsigned effects, void* stream) {
    return launch_ilqr<kLineSearch, true>(p, io ? &io->base : nullptr, io, n_envs, drones_per_env, substeps, effects, stream,
                                          "qs_ilqr_box_line_search");
}

int qs_ilqr_box_commit(const QsParams* p, const QsIlqrBoxIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                       void* stream) {
    return launch_ilqr<kCommit, true>(p, io ? &io->base : nullptr, io, n_envs, drones_per_env, substeps, effects, stream,
                                      "qs_ilqr_box_commit");
}

}  // extern "C"
