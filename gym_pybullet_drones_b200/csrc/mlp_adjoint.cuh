// mlp_adjoint.cuh -- the per-element math of the differentiable policy trajectories (dyn_policy_traj.cu, DESIGN.md 4.5): the
// float64 MLP actor and its transpose, the observation head and its adjoint, the RPM / ONE_D_RPM decode and its adjoint, and the
// tick adjoint that also takes the cotangent of the next observation's ang_v.  Compiled for the sm_90a kernels and for the host
// harness (tests/host_harness/diff_policy_host.cpp); the kernels' GEMMs run on the tensor cores (policy_actor.cuh, cta_gemm), the
// host build and the FMA comparison build use mlp_col / mlp_row_t.
//
// Which derivative (DESIGN.md 4.5):
//   * ReLU: h > 0 passes the gradient (torch.relu); Tanh: 1 - h^2 on the forward's own h;
//   * the action clip follows torch.clamp: the gradient passes for -1 <= raw <= 1 and is zero outside;
//   * rpy = quat_to_euler<false>: each branch of the +-0.99999 gimbal guard is differentiated on the forward's predicate
//     (dyn_adjoint.cuh, quat_to_euler_vjp: the function the controller's adjoint uses);
//   * ang_v = R_last w with R_last = quat_to_matrix_unit (s = 2 (2 - |q|^2)) of the attitude at the start of the tick's last
//     substep: differentiated as written, and its quaternion cotangent enters the tick adjoint at that substep.
#pragma once
#include "dyn_adjoint.cuh"

namespace qs {

// one fused multiply-add on both builds: the dot products of the actor round the same way on the device and on the host
QS_HD double fmad(double a, double b, double c) {
#if defined(__CUDA_ARCH__)
    return __fma_rn(a, b, c);
#else
    return fma(a, b, c);
#endif
}

QS_HD double mlp_act(int kind, double z) { return kind == QS_MLP_RELU ? (z > 0.0 ? z : 0.0) : tanh(z); }
QS_HD double mlp_act_vjp(int kind, double h, double Lh) { return kind == QS_MLP_RELU ? (h > 0.0 ? Lh : 0.0) : (1.0 - h * h) * Lh; }

// acc[m] = b[n] + sum_k x[m][k] W[k][n] for MG rows of x (row stride ldx); W is [K][Nout] row-major
template <int MG>
QS_HD void mlp_col(const double* W, const double* b, int K, int Nout, int n, const double* x, int ldx, double acc[MG]) {
#pragma unroll
    for (int m = 0; m < MG; ++m) acc[m] = b[n];
    for (int k = 0; k < K; ++k) {
        const double w = W[(long long)k * Nout + n];
#pragma unroll
        for (int m = 0; m < MG; ++m) acc[m] = fmad(x[m * ldx + k], w, acc[m]);
    }
}
// acc[m] = sum_n W[k][n] Lz[m][n] for MG rows of Lz (row stride ldz): row k of the transposed layer
template <int MG>
QS_HD void mlp_row_t(const double* W, int Nout, int k, const double* Lz, int ldz, double acc[MG]) {
#pragma unroll
    for (int m = 0; m < MG; ++m) acc[m] = 0.0;
    const double* wr = W + (long long)k * Nout;
    for (int n = 0; n < Nout; ++n) {
        const double w = wr[n];
#pragma unroll
        for (int m = 0; m < MG; ++m) acc[m] = fmad(Lz[m * ldz + n], w, acc[m]);
    }
}

// the 12 kinematic entries of a KIN observation row: pos, rpy, vel, ang_v = R w (BaseRLAviary._computeObs, BaseAviary.py:873)
QS_HD void obs_head(const Drone& d, const double R[9], double o[12]) {
    o[0] = d.px; o[1] = d.py; o[2] = d.pz;
    quat_to_euler<false>(d.qx, d.qy, d.qz, d.qw, o[3], o[4], o[5]);
    o[6] = d.vx; o[7] = d.vy; o[8] = d.vz;
    o[9] = R[0] * d.wx + R[1] * d.wy + R[2] * d.wz;
    o[10] = R[3] * d.wx + R[4] * d.wy + R[5] * d.wz;
    o[11] = R[6] * d.wx + R[7] * d.wy + R[8] * d.wz;
}

// Lq += d R / d q ^T A for R = quat_to_matrix_unit(q) = I + s M(q), s = 2 (2 - |q|^2)
QS_HD void quat_to_matrix_unit_vjp(double qx, double qy, double qz, double qw, const double A[9], double Lq[4]) {
    const double s = 2.0 * (2.0 - (qx * qx + qy * qy + qz * qz + qw * qw));
    const double M[9] = {-(qy * qy + qz * qz), qx * qy - qw * qz, qx * qz + qw * qy,
                         qx * qy + qw * qz, -(qx * qx + qz * qz), qy * qz - qw * qx,
                         qx * qz - qw * qy, qy * qz + qw * qx, -(qx * qx + qy * qy)};
    double Ls = 0.0;
    for (int j = 0; j < 9; ++j) Ls += A[j] * M[j];
    Lq[0] += s * (A[1] * qy + A[2] * qz + A[3] * qy - 2.0 * qx * A[4] - A[5] * qw + A[6] * qz + A[7] * qw - 2.0 * qx * A[8]);
    Lq[1] += s * (-2.0 * qy * A[0] + A[1] * qx + A[2] * qw + A[3] * qx + A[5] * qz - A[6] * qw + A[7] * qz - 2.0 * qy * A[8]);
    Lq[2] += s * (-2.0 * qz * A[0] - A[1] * qw + A[2] * qx + A[3] * qw - 2.0 * qz * A[4] + A[5] * qy + A[6] * qx + A[7] * qy);
    Lq[3] += s * (-A[1] * qz + A[2] * qy + A[3] * qz - A[5] * qx - A[6] * qy + A[7] * qx);
    const double k = -4.0 * Ls;                          // ds/dq = -4 q
    Lq[0] += k * qx; Lq[1] += k * qy; Lq[2] += k * qz; Lq[3] += k * qw;
}

// Adjoint of ang_v = R(q) w for R = quat_to_matrix_unit(q): Lw += R^T Lang, Lq += d(R w)/dq ^T Lang
QS_HD void ang_v_vjp(double qx, double qy, double qz, double qw, const double w[3], const double Lang[3], double Lw[3], double Lq[4]) {
    double R[9], A[9];
    quat_to_matrix_unit(qx, qy, qz, qw, R);
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) { Lw[c] += R[3 * r + c] * Lang[r]; A[3 * r + c] = Lang[r] * w[c]; }
    quat_to_matrix_unit_vjp(qx, qy, qz, qw, A, Lq);
}

// The cotangent of the 12 kinematic entries of an observation row built from the stored state d: pos, vel and (through rpy) the
// quaternion go into L; ang_v's part is returned in Lang, for the adjoint of the tick that produced d (or of the initial state)
QS_HD void obs_head_vjp(const Drone& d, const double Lo[12], Drone& L, double Lang[3]) {
    L.px += Lo[0]; L.py += Lo[1]; L.pz += Lo[2];
    L.vx += Lo[6]; L.vy += Lo[7]; L.vz += Lo[8];
    double Lq[4] = {0.0, 0.0, 0.0, 0.0};
    quat_to_euler_vjp(d.qx, d.qy, d.qz, d.qw, Lo + 3, Lq);
    L.qx += Lq[0]; L.qy += Lq[1]; L.qz += Lq[2]; L.qw += Lq[3];
    Lang[0] = Lo[9]; Lang[1] = Lo[10]; Lang[2] = Lo[11];
}

// The first observation's ang_v = R(q0 / |q0|) w0: its cotangent Lang into L (the cotangent of the initial state d0)
QS_HD void initial_ang_v_vjp(const Drone& d0, const double Lang[3], Drone& L) {
    Drone x0 = d0;
    double inv;
    entry_normalise(x0, inv);
    const double w[3] = {d0.wx, d0.wy, d0.wz};
    double Lw[3] = {0.0, 0.0, 0.0}, Lq[4] = {0.0, 0.0, 0.0, 0.0};
    ang_v_vjp(x0.qx, x0.qy, x0.qz, x0.qw, w, Lang, Lw, Lq);
    L.wx += Lw[0]; L.wy += Lw[1]; L.wz += Lw[2];
    const double dot = x0.qx * Lq[0] + x0.qy * Lq[1] + x0.qz * Lq[2] + x0.qw * Lq[3];
    L.qx += (Lq[0] - x0.qx * dot) * inv; L.qy += (Lq[1] - x0.qy * dot) * inv;
    L.qz += (Lq[2] - x0.qz * dot) * inv; L.qw += (Lq[3] - x0.qw * dot) * inv;
}

// rpm = HOVER_RPM (1 + 0.05 a) in float64 (BaseRLAviary.py:192 / :225): A = 4 one action per motor, A = 1 one for all four
QS_HD void policy_rpm(int A, const PhysRow& c, const double a[4], double rpm[4]) {
#pragma unroll
    for (int j = 0; j < 4; ++j) rpm[j] = c.hover_rpm * (1.0 + 0.05 * a[A == 1 ? 0 : j]);
}
QS_HD void policy_rpm_vjp(int A, const PhysRow& c, const double a[4], const double Lrpm[4], double La[4], double& g_hover) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int s = A == 1 ? 0 : j;
        g_hover += (1.0 + 0.05 * a[s]) * Lrpm[j];
        La[s] += c.hover_rpm * 0.05 * Lrpm[j];
    }
}

// dyn_tick_vjp (dyn_adjoint.cuh) for a tick whose end state also feeds the next observation's ang_v = R_last w_end, R_last the
// attitude at the start of the last substep.  Lang: the cotangent of that ang_v.  Its w part joins L before the tick's adjoint;
// its quaternion part joins L after the last substep's adjoint, where L is the cotangent of that substep's start state.
template <int EFF, class Rec>
QS_HD void dyn_tick_obs_vjp(const QsParams& P, const PhysRow& c, const Drone& d0, const double u[4], const double up[4], int S,
                            Rec& rec, Drone& L, const double Lang[3], double Lu[4], double Lup[4], PhysGrad& G) {
    Drone d = d0;
    {
        double R_last[9];
        dyn_tick_k<EFF>(P, c, d, u, up, 0.0, S, R_last, RecordHook<Rec>{&d, &rec, S - 1});
    }
    Drone x0 = d0;
    double inv;
    entry_normalise(x0, inv);
    Drone xl = x0;
    if (S > 1) rec.load(S - 2, xl);
    const double w_end[3] = {d.wx, d.wy, d.wz};
    double Lw[3] = {0.0, 0.0, 0.0}, Lql[4] = {0.0, 0.0, 0.0, 0.0};
    ang_v_vjp(xl.qx, xl.qy, xl.qz, xl.qw, w_end, Lang, Lw, Lql);
    L.wx += Lw[0]; L.wy += Lw[1]; L.wz += Lw[2];
    const double kk = 2.0 * 3.14159265358979323846;
    const double ds_prev = kk * up[0] / 60.0 + kk * up[1] / 60.0 + kk * up[2] / 60.0 + kk * up[3] / 60.0;
    const double ds_cur = kk * u[0] / 60.0 + kk * u[1] / 60.0 + kk * u[2] / 60.0 + kk * u[3] / 60.0;
    double Lds_prev = 0.0, Lds_cur = 0.0;
    for (int s = S - 1; s >= 0; --s) {
        Drone x;
        if (s == 0) x = x0; else rec.load(s - 1, x);
        substep_vjp<EFF>(P, c, x, u, s == 0 ? ds_prev : ds_cur, L, Lu, s == 0 ? Lds_prev : Lds_cur, G);
        if (s == S - 1) { L.qx += Lql[0]; L.qy += Lql[1]; L.qz += Lql[2]; L.qw += Lql[3]; }
    }
    if (EFF & QS_EFFECT_DRAG) {
#pragma unroll
        for (int i = 0; i < 4; ++i) { Lup[i] += (kk / 60.0) * Lds_prev; Lu[i] += (kk / 60.0) * Lds_cur; }
    }
    const double dot = x0.qx * L.qx + x0.qy * L.qy + x0.qz * L.qz + x0.qw * L.qw;
    L.qx = (L.qx - x0.qx * dot) * inv; L.qy = (L.qy - x0.qy * dot) * inv;
    L.qz = (L.qz - x0.qz * dot) * inv; L.qw = (L.qw - x0.qw * dot) * inv;
}

}  // namespace qs
