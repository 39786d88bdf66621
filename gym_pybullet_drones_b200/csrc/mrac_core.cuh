// mrac_core.cuh -- per-drone math of the MRAC controller (reference: gym_pybullet_drones/control/MRAC.py:109-155), float64,
// compiled into the CUDA kernels (mrac.cu, rollout_ctrl.cu) and, with g++, into the host harness tests/host_harness/mrac_host.cpp.
// The gains are synthesised once per model on the host (control/MRAC.py) and arrive here as QsMracParams.
#pragma once
#include "quad_core.cuh"

namespace qs {

// one controller's adaptive state (include/quadsim.h, QS_MRAC_STATE rows): element q at p[q * stride] -- the [76][N] planes in
// global memory (stride N) or a CTA's [76][tpb] copy in shared memory (stride tpb)
struct MracState {
    double* p;
    long long stride;
    QS_HD double& operator[](int q) const { return p[q * stride]; }
};
constexpr int kMracKr = 48, kMracXm = 64;

// the state vector's ang_v from the float64 planes: getMatrixFromQuaternion(q) w (BaseAviary.py:873 with R_old w = R_new w)
QS_HD void mrac_ang_v(const Drone& d, double a[3]) {
    double R[9];
    quat_to_matrix(d.qx, d.qy, d.qz, d.qw, R);
    a[0] = R[0] * d.wx + R[1] * d.wy + R[2] * d.wz;
    a[1] = R[3] * d.wx + R[4] * d.wy + R[5] * d.wz;
    a[2] = R[6] * d.wx + R[7] * d.wy + R[8] * d.wz;
}

// Rotation.from_euler('XYZ', rpy).inv().apply(v) (MRAC.py:121): R = Rx(roll) Ry(pitch) Rz(yaw) (scipy's intrinsic XYZ applied to
// Bullet's extrinsic angles, a quirk of the reference that is kept), so R^T v = Rz^T Ry^T Rx^T v
QS_HD void mrac_body_rates(double roll, double pitch, double yaw, const double v[3], double w[3]) {
    const double ca = cos(roll), sa = sin(roll), cb = cos(pitch), sb = sin(pitch), cc = cos(yaw), sc = sin(yaw);
    const double x1 = v[0], y1 = ca * v[1] + sa * v[2], z1 = ca * v[2] - sa * v[1];
    const double x2 = cb * x1 - sb * z1, z2 = sb * x1 + cb * z1;
    w[0] = cc * x2 + sc * y1;
    w[1] = cc * y1 - sc * x2;
    w[2] = z2;
}

// MRAC.computeControl for one drone (MRAC.py:109-155).  pos / quat / vel / ang_v: the drone's state as computeControl receives
// it; r = [target_pos, target_rpy, target_vel, target_rpy_rates].  Returns the unclipped rpm[4], pos_e[3], rpy_e[3] and advances
// S (Kx, Kr with the old Kx / Kr in u, then Xm with the old Xm).
QS_HD void mrac_control(const QsMracParams& M, const MracState& S, bool init, double dt, const double pos[3], const double quat[4],
                        const double vel[3], const double ang_v[3], const double r[12], double rpm[4], double pos_e[3],
                        double rpy_e[3]) {
    double roll, pitch, yaw;
    quat_to_euler<false>(quat[0], quat[1], quat[2], quat[3], roll, pitch, yaw);          // :120
    double wb[3];
    mrac_body_rates(roll, pitch, yaw, ang_v, wb);                                          // :121
    const double X[12] = {pos[0], pos[1], pos[2], roll, pitch, yaw, vel[0], vel[1], vel[2], wb[0], wb[1], wb[2]};   // :130
    if (init) {
#pragma unroll
        for (int q = 0; q < 12; ++q) S[kMracXm + q] = X[q];                                // :123-124
    }
    double rt[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {                                                          // :127-128
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < 12; ++k) s += M.Kr_ref[j][k] * r[k];
        rt[j] = -s;
    }
    double u[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {                                                          // :131
        double sx = 0.0, sr = 0.0;
#pragma unroll
        for (int i = 0; i < 12; ++i) sx += S[4 * i + j] * X[i];
#pragma unroll
        for (int i = 0; i < 4; ++i) sr += S[kMracKr + 4 * i + j] * rt[i];
        u[j] = sx + sr;
    }
    double e[12];
#pragma unroll
    for (int q = 0; q < 12; ++q) e[q] = X[q] - S[kMracXm + q];                             // :132
    double ep[4];                                                                          // e^T P Bm
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < 12; ++k) s += e[k] * M.PBm[k][j];
        ep[j] = s;
    }
#pragma unroll
    for (int i = 0; i < 12; ++i) {                                                         // :133, :136
        const double g = -M.gamma_x * X[i];
#pragma unroll
        for (int j = 0; j < 4; ++j) S[4 * i + j] += (g * ep[j]) * dt;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {                                                          // :134, :137
        const double g = -M.gamma_r * rt[i];
#pragma unroll
        for (int j = 0; j < 4; ++j) S[kMracKr + 4 * i + j] += (g * ep[j]) * dt;
    }
    const double thrust = u[0] < 0.0 ? 0.0 : u[0];                                         // :139-140
    const double t0 = clampd(u[1], -3200.0, 3200.0), t1 = clampd(u[2], -3200.0, 3200.0), t2 = clampd(u[3], -3200.0, 3200.0);
    const double tp = (sqrt(thrust / (4.0 * M.kf)) - M.pwm2rpm_const) / M.pwm2rpm_scale;   // :144
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        double pwm = tp + (M.mixer[i][0] * t0 + M.mixer[i][1] * t1 + M.mixer[i][2] * t2);   // :145
        pwm = clampd(pwm, M.min_pwm, M.max_pwm);                                           // :146
        rpm[i] = M.pwm2rpm_scale * pwm + M.pwm2rpm_const;                                  // :147
    }
    pos_e[0] = r[0] - pos[0]; pos_e[1] = r[1] - pos[1]; pos_e[2] = r[2] - pos[2];          // :149
    rpy_e[0] = r[3] - roll; rpy_e[1] = r[4] - pitch; rpy_e[2] = r[5] - yaw;                // :150
    double xd[12];                                                                         // :152-153, with the old Xm
#pragma unroll
    for (int q = 0; q < 12; ++q) {
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < 12; ++k) s += M.Am[q][k] * S[kMracXm + k];
        xd[q] = s;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) xd[8 + j] += M.bm[j] * rt[j];
#pragma unroll
    for (int q = 0; q < 12; ++q) S[kMracXm + q] += xd[q] * dt;
}

}  // namespace qs
