// lqr_law.cuh -- the time-varying LQR tracker of an iLQR plan, u_j = u_nom,j + sum_q K_jq (z - z_nom)_q, written once for
// ilqr.cu's feedback rollout, qs_ctrl_rollout_lqr's tracker (rollout_ctrl.cu), the differentiable tracker loop (dyn_lqr_traj.cu)
// and the host harness (tests/host_harness/lqr_traj_host.cpp): the loop state's order, a box's row, the law and its adjoint.
#pragma once
#include "quad_core.cuh"
#if defined(__CUDACC__)
#include "qs_common.cuh"
#endif

namespace qsi {
namespace {

// x = the drone's state in the loop state's order: px py pz qx qy qz qw vx vy vz wx wy wz
QS_HD void drone_vec(const qs::Drone& d, double x[13]) {
    x[0] = d.px; x[1] = d.py; x[2] = d.pz; x[3] = d.qx; x[4] = d.qy; x[5] = d.qz; x[6] = d.qw;
    x[7] = d.vx; x[8] = d.vy; x[9] = d.vz; x[10] = d.wx; x[11] = d.wy; x[12] = d.wz;
}

// the row of drone i's box at plan tick p: [T][N][4] when the box is per tick, else [N][4]
QS_HD long long box_row(int per_tick, long long p, long long N, long long i) { return per_tick ? p * N + i : i; }

// s = sum_{q=0}^{NZ-1} K(q) dz[q], summed in that order from 0.0; K(q) returns K_jq of the caller's row j in its own layout
template <int NZ, class Gain>
QS_HD double lqr_feedback(Gain K, const double* dz) {
    double s = 0.0;
#pragma unroll
    for (int q = 0; q < NZ; ++q) s += K(q) * dz[q];
    return s;
}

// The tracker reads one plan tick of a drone through a view, so that each build keeps its own loads: pl.zn(q) = z_nom_q,
// pl.K(j, q) = K_jq, pl.nom(b): b = rpm_nom, pl.box(lo, hi): false without a box, else its row.
// dz = x in drone_vec's order minus z_nom[0:13], and with NZ = 17 the RPMs applied at the tick before minus z_nom[13:17]
template <int NZ, class Plan>
QS_HD void tracker_dz(const Plan& pl, const qs::Drone& d, const double up[4], double dz[NZ]) {
    double x[13];
    drone_vec(d, x);
#pragma unroll
    for (int q = 0; q < 13; ++q) dz[q] = x[q] - pl.zn(q);
    if constexpr (NZ == 17) {
#pragma unroll
        for (int j = 0; j < 4; ++j) dz[13 + j] = up[j] - pl.zn(13 + j);
    }
}

// The command b = rpm_nom + K dz, clamped to the box when there is one; keep[j]: torch.clamp's gradient passes (lo_j <= b_j <=
// hi_j before the clamp).  The env's clip to [0, MAX_RPM] is the caller's.
template <int NZ, class Plan>
QS_HD void tracker_command(const Plan& pl, const qs::Drone& d, const double up[4], double b[4], bool keep[4]) {
    double dz[NZ];
    tracker_dz<NZ>(pl, d, up, dz);
    pl.nom(b);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        b[j] += lqr_feedback<NZ>([&](int q) { return pl.K(j, q); }, dz);
        keep[j] = true;
    }
    double lo[4], hi[4];
    if (pl.box(lo, hi)) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            keep[j] = !(b[j] < lo[j]) && !(b[j] > hi[j]);
            b[j] = qs::clampd(b[j], lo[j], hi[j]);
        }
    }
}

// The adjoint of u = u_nom + K dz, dz = z - z_nom, for the cotangent lam [4] of u.  The law is linear: the cotangent of u_nom is
// lam itself; gK(j, q, g) receives g = lam_j dz_q, the cotangent of K_jq (K(j, q) returns K_jq); Ktl[q] = sum_j K_jq lam_j,
// summed j = 0..3 from 0.0, is the cotangent of z, and -Ktl that of z_nom.
template <int NZ, class Gain, class GainGrad>
QS_HD void lqr_feedback_vjp(Gain K, const double* dz, const double lam[4], GainGrad gK, double* Ktl) {
#pragma unroll
    for (int q = 0; q < NZ; ++q) Ktl[q] = 0.0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int q = 0; q < NZ; ++q) {
            gK(j, q, lam[j] * dz[q]);
            Ktl[q] += K(j, q) * lam[j];
        }
    }
}

#if defined(__CUDACC__)
// The device view of drone i at plan tick p of a QsDynLqrTrajIO: K and z_nom through the read-only cache, the rest 32-byte loads
template <int NZ, class IO>
struct DevicePlan {
    const IO& io;
    long long N, i, p;
    const double *z, *k;    // z_nom[p][i], K[p][i]
    __device__ __forceinline__ double zn(int q) const { return __ldg(z + q); }
    __device__ __forceinline__ double K(int j, int q) const { return __ldg(k + j * NZ + q); }
    __device__ __forceinline__ void nom(double b[4]) const {
        const D4 un = ld256_nc(io.rpm_nom, p * N + i);
        b[0] = un.x; b[1] = un.y; b[2] = un.z; b[3] = un.w;
    }
    __device__ __forceinline__ bool box(double lo[4], double hi[4]) const {
        if (!io.lo) return false;
        const long long at = box_row(io.per_tick, p, N, i);
        const D4 l4 = ld256_nc(io.lo, at), h4 = ld256_nc(io.hi, at);
        lo[0] = l4.x; lo[1] = l4.y; lo[2] = l4.z; lo[3] = l4.w;
        hi[0] = h4.x; hi[1] = h4.y; hi[2] = h4.z; hi[3] = h4.w;
        return true;
    }
};
template <int NZ, class IO>
__device__ __forceinline__ DevicePlan<NZ, IO> device_plan(const IO& io, long long N, long long i, long long p) {
    return {io, N, i, p, io.z_nom + (p * N + i) * NZ, io.K + (p * N + i) * 4 * NZ};
}
#endif

}  // namespace
}  // namespace qsi
