// lqr_law.cuh -- the feedback term of a time-varying LQR tracker, u_j = u_nom,j + sum_q K_jq (z - z_nom)_q: the arithmetic of
// ilqr.cu's feedback rollout (line search, commit), of qs_ctrl_rollout_lqr's tracker (rollout_ctrl.cu) and of the differentiable
// tracker loop (dyn_lqr_traj.cu), written once so that the tracker flies a plan with the bits the solver committed it with; and the
// law's adjoint, which the tracker loop's backward and the host harness (tests/host_harness/lqr_traj_host.cpp) share.
#pragma once
#include "quad_core.cuh"

namespace qsi {
namespace {

// s = sum_{q=0}^{NZ-1} K(q) dz[q], summed in that order from 0.0; K(q) returns K_jq of the caller's row j in its own layout
template <int NZ, class Gain>
QS_HD double lqr_feedback(Gain K, const double* dz) {
    double s = 0.0;
#pragma unroll
    for (int q = 0; q < NZ; ++q) s += K(q) * dz[q];
    return s;
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

}  // namespace
}  // namespace qsi
