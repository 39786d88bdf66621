// lqr_law.cuh -- the feedback term of a time-varying LQR tracker, u_j = u_nom,j + sum_q K_jq (z - z_nom)_q: the arithmetic of
// ilqr.cu's feedback rollout (line search, commit) and of qs_ctrl_rollout_lqr's tracker (rollout_ctrl.cu), written once so that
// the tracker flies a plan with the bits the solver committed it with.
#pragma once

namespace qsi {
namespace {

// s = sum_{q=0}^{NZ-1} K(q) dz[q], summed in that order from 0.0; K(q) returns K_jq of the caller's row j in its own layout
template <int NZ, class Gain>
__device__ __forceinline__ double lqr_feedback(Gain K, const double* dz) {
    double s = 0.0;
#pragma unroll
    for (int q = 0; q < NZ; ++q) s += K(q) * dz[q];
    return s;
}

}  // namespace
}  // namespace qsi
