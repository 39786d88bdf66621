// pid_adjoint.cuh -- reverse mode of DSLPIDControl.computeControl (qs::pid_control_k, quad_core.cuh) for the differentiable
// closed-loop trajectories of dyn_ctrl_traj.cu, compiled for the sm_90a kernels and for the host harness
// (tests/host_harness/diff_ctrl_host.cpp).
//
// Which derivative (DESIGN.md 4.5):
//   * every clip follows torch.clamp with constant bounds: the gradient passes for lo <= x <= hi and is zero outside.  That is
//     the integral clips (the nested ipz clip +-2 then +-0.15, irx / iry +-1500 then +-1, irz +-1500), the torque clip +-3200, the
//     PWM clip [MIN_PWM, MAX_PWM] and (in the kernel) the controller's and the env's max_rpm clips (rpm_clip_vjp);
//   * `scalar < 0 ? 0 : scalar` then sqrt: the gradient is zero where scalar <= 0 (at 0 the derivative of sqrt is infinite);
//   * quat_to_euler<false>: each branch of the +-0.99999 gimbal guard is differentiated on the forward's predicate (atan2 / asin,
//     or the 2 atan2 yaw of the guard, whose roll and pitch are constants).  The atan2 of the yaw error only feeds yaw_e, which is
//     not an output of the trajectory, so it has no adjoint;
//   * the rate term (rpy - last_rpy) / dt is differentiated as the forward computes it, with no angle unwrap;
//   * the normalisations of the target thrust direction and of z x x_c are assumed nonzero (the forward is singular there too).
//
// The adjoint recomputes the forward values it needs from the controller's inputs; nothing is stored between the two.
#pragma once
#include "dyn_adjoint.cuh"

#if defined(__CUDACC__)
// out of line on the device: the tick adjoint of dyn_adjoint.cuh already holds most of the register file (DESIGN.md 4.5)
#define QS_HD_NOINLINE inline __host__ __device__ __noinline__
#else
#define QS_HD_NOINLINE inline
#endif

namespace qs {

// One gain set of DSLPIDControl, the 18 columns of QsDynCtrlTrajIO.gains in this order.  The member names are QsParams', so
// pid_control_k reads either.
struct PidGains { double pid_p_for[3], pid_i_for[3], pid_d_for[3], pid_p_tor[3], pid_i_tor[3], pid_d_tor[3]; };

QS_HD PidGains pid_gains_of(const QsParams& P) {
    PidGains g;
    for (int a = 0; a < 3; ++a) {
        g.pid_p_for[a] = P.pid_p_for[a]; g.pid_i_for[a] = P.pid_i_for[a]; g.pid_d_for[a] = P.pid_d_for[a];
        g.pid_p_tor[a] = P.pid_p_tor[a]; g.pid_i_tor[a] = P.pid_i_tor[a]; g.pid_d_tor[a] = P.pid_d_tor[a];
    }
    return g;
}

// the controller's targets of one tick: target_pos, target yaw (target_rpy[2]), target_vel, target_rpy_rates
struct PidTargets { double tp[3], tyaw, tv[3], trr[3]; };

QS_HD bool clamp_passes(double x, double lo, double hi) { return lo <= x && x <= hi; }

// Adjoint of pid_control_k(P, K, st, dt, d.pos, d.quat, d.vel, tg, ...).  Lrpm: the cotangent of the raw RPMs (before any
// max_rpm clip).  Lst: in, the cotangent of the updated controller state; out, of `st` (the state the call started from).  L
// accumulates pos / quat / vel (its rates are not read), Lt the targets (Lt.tyaw the target yaw) and Lg the 18 gains.
QS_HD_NOINLINE void pid_control_vjp(const QsParams& P, const PidGains& K, const PidState& st, double dt, const Drone& d,
                                    const PidTargets& tg, const double Lrpm[4], PidState& Lst, Drone& L, PidTargets& Lt,
                                    double Lg[18]) {
    const double qx = d.qx, qy = d.qy, qz = d.qz, qw = d.qw;
    // ---- forward values, in pid_control_k's order ----
    double R[9];
    quat_to_matrix(qx, qy, qz, qw, R);
    const double e[3] = {tg.tp[0] - d.px, tg.tp[1] - d.py, tg.tp[2] - d.pz};
    const double ev[3] = {tg.tv[0] - d.vx, tg.tv[1] - d.vy, tg.tv[2] - d.vz};
    const double ip0[3] = {st.ipx + e[0] * dt, st.ipy + e[1] * dt, st.ipz + e[2] * dt};
    const double ipz1 = clampd(ip0[2], -2.0, 2.0);
    const double ip[3] = {clampd(ip0[0], -2.0, 2.0), clampd(ip0[1], -2.0, 2.0), clampd(ipz1, -0.15, 0.15)};
    const bool ip_live[3] = {clamp_passes(ip0[0], -2.0, 2.0), clamp_passes(ip0[1], -2.0, 2.0),
                             clamp_passes(ip0[2], -2.0, 2.0) && clamp_passes(ipz1, -0.15, 0.15)};
    const double tt[3] = {K.pid_p_for[0] * e[0] + K.pid_i_for[0] * ip[0] + K.pid_d_for[0] * ev[0],
                          K.pid_p_for[1] * e[1] + K.pid_i_for[1] * ip[1] + K.pid_d_for[1] * ev[1],
                          K.pid_p_for[2] * e[2] + K.pid_i_for[2] * ip[2] + K.pid_d_for[2] * ev[2] + P.pid_gravity};
    const double scalar = tt[0] * R[2] + tt[1] * R[5] + tt[2] * R[8];
    const double sc = scalar < 0.0 ? 0.0 : scalar;
    const double root = sqrt(sc / (4.0 * P.pid_kf));
    const double thrust = (root - P.pid_pwm2rpm_const) / P.pid_pwm2rpm_scale;
    const double tn = sqrt(tt[0] * tt[0] + tt[1] * tt[1] + tt[2] * tt[2]);
    const double z[3] = {tt[0] / tn, tt[1] / tn, tt[2] / tn};
    const double cx = cos(tg.tyaw), cy = sin(tg.tyaw);
    const double y0[3] = {z[1] * 0.0 - z[2] * cy, z[2] * cx - z[0] * 0.0, z[0] * cy - z[1] * cx};
    const double yn = sqrt(y0[0] * y0[0] + y0[1] * y0[1] + y0[2] * y0[2]);
    const double y[3] = {y0[0] / yn, y0[1] / yn, y0[2] / yn};
    const double x[3] = {y[1] * z[2] - y[2] * z[1], y[2] * z[0] - y[0] * z[2], y[0] * z[1] - y[1] * z[0]};
    // T = Rd, columns x, y, z: T[j][c]
    const double T[9] = {x[0], y[0], z[0], x[1], y[1], z[1], x[2], y[2], z[2]};
    double rpy[3];
    quat_to_euler<false>(qx, qy, qz, qw, rpy[0], rpy[1], rpy[2]);
    double re[3];
    {
        #define QS_TtR(i, k) (T[0 + i] * R[0 + k] + T[3 + i] * R[3 + k] + T[6 + i] * R[6 + k])
        #define QS_RtT(i, k) (R[0 + i] * T[0 + k] + R[3 + i] * T[3 + k] + R[6 + i] * T[6 + k])
        re[0] = QS_TtR(2, 1) - QS_RtT(2, 1);
        re[1] = QS_TtR(0, 2) - QS_RtT(0, 2);
        re[2] = QS_TtR(1, 0) - QS_RtT(1, 0);
        #undef QS_TtR
        #undef QS_RtT
    }
    const double last[3] = {st.lr, st.lp, st.ly};
    const double ir_in[3] = {st.irx, st.iry, st.irz};
    double rr[3], ir[3], qt[3];
    bool ir_live[3], q_live[3];
    for (int a = 0; a < 3; ++a) {
        rr[a] = tg.trr[a] - (rpy[a] - last[a]) / dt;
        const double ir0 = ir_in[a] - re[a] * dt;
        const double ir1 = clampd(ir0, -1500.0, 1500.0);
        ir[a] = a < 2 ? clampd(ir1, -1.0, 1.0) : ir1;
        ir_live[a] = clamp_passes(ir0, -1500.0, 1500.0) && (a == 2 || clamp_passes(ir1, -1.0, 1.0));
        qt[a] = -K.pid_p_tor[a] * re[a] + K.pid_d_tor[a] * rr[a] + K.pid_i_tor[a] * ir[a];
        q_live[a] = clamp_passes(qt[a], -3200.0, 3200.0);
    }
    const double qc[3] = {clampd(qt[0], -3200.0, 3200.0), clampd(qt[1], -3200.0, 3200.0), clampd(qt[2], -3200.0, 3200.0)};

    // ---- reverse ----
    // rpm = scale pwm + const, pwm = clip(thrust + mixer qc)
    double Lthrust = 0.0, Lqc[3] = {0.0, 0.0, 0.0};
    for (int j = 0; j < 4; ++j) {
        const double pwm = thrust + (P.pid_mixer[j][0] * qc[0] + P.pid_mixer[j][1] * qc[1] + P.pid_mixer[j][2] * qc[2]);
        const double Lpwm = clamp_passes(pwm, P.pid_min_pwm, P.pid_max_pwm) ? P.pid_pwm2rpm_scale * Lrpm[j] : 0.0;
        Lthrust += Lpwm;
        for (int a = 0; a < 3; ++a) Lqc[a] += P.pid_mixer[j][a] * Lpwm;
    }
    // torques, rate and integral terms
    double Lre[3], Lrpy[3] = {Lst.lr, Lst.lp, Lst.ly};
    double Lir_old[3];
    for (int a = 0; a < 3; ++a) {
        const double Lq = q_live[a] ? Lqc[a] : 0.0;
        Lg[9 + a] += -re[a] * Lq;
        Lg[12 + a] += ir[a] * Lq;
        Lg[15 + a] += rr[a] * Lq;
        Lre[a] = -K.pid_p_tor[a] * Lq;
        const double Lrr = K.pid_d_tor[a] * Lq;
        const double Lir = K.pid_i_tor[a] * Lq + (a == 0 ? Lst.irx : a == 1 ? Lst.iry : Lst.irz);
        const double Lir0 = ir_live[a] ? Lir : 0.0;
        Lir_old[a] = Lir0;
        Lre[a] -= dt * Lir0;
        Lt.trr[a] += Lrr;
        Lrpy[a] -= Lrr / dt;
        Lst.lr = a == 0 ? Lrr / dt : Lst.lr;
        Lst.lp = a == 1 ? Lrr / dt : Lst.lp;
        Lst.ly = a == 2 ? Lrr / dt : Lst.ly;
    }
    Lst.irx = Lir_old[0]; Lst.iry = Lir_old[1]; Lst.irz = Lir_old[2];
    // rot_e = (E[2][1], E[0][2], E[1][0]) of E = T^T R - R^T T
    double LT[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, LR[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int j = 0; j < 3; ++j) {
        // rex = sum_j T[j][2] R[j][1] - R[j][2] T[j][1]
        LT[3 * j + 2] += Lre[0] * R[3 * j + 1]; LR[3 * j + 1] += Lre[0] * T[3 * j + 2];
        LR[3 * j + 2] -= Lre[0] * T[3 * j + 1]; LT[3 * j + 1] -= Lre[0] * R[3 * j + 2];
        // rey = sum_j T[j][0] R[j][2] - R[j][0] T[j][2]
        LT[3 * j + 0] += Lre[1] * R[3 * j + 2]; LR[3 * j + 2] += Lre[1] * T[3 * j + 0];
        LR[3 * j + 0] -= Lre[1] * T[3 * j + 2]; LT[3 * j + 2] -= Lre[1] * R[3 * j + 0];
        // rez = sum_j T[j][1] R[j][0] - R[j][1] T[j][0]
        LT[3 * j + 1] += Lre[2] * R[3 * j + 0]; LR[3 * j + 0] += Lre[2] * T[3 * j + 1];
        LR[3 * j + 1] -= Lre[2] * T[3 * j + 0]; LT[3 * j + 0] -= Lre[2] * R[3 * j + 1];
    }
    double Lx[3] = {LT[0], LT[3], LT[6]}, Ly[3] = {LT[1], LT[4], LT[7]}, Lz[3] = {LT[2], LT[5], LT[8]};
    // x = y x z: Ly += z x Lx, Lz += Lx x y
    Ly[0] += z[1] * Lx[2] - z[2] * Lx[1]; Ly[1] += z[2] * Lx[0] - z[0] * Lx[2]; Ly[2] += z[0] * Lx[1] - z[1] * Lx[0];
    Lz[0] += Lx[1] * y[2] - Lx[2] * y[1]; Lz[1] += Lx[2] * y[0] - Lx[0] * y[2]; Lz[2] += Lx[0] * y[1] - Lx[1] * y[0];
    // y = y0 / |y0|
    const double yd = y[0] * Ly[0] + y[1] * Ly[1] + y[2] * Ly[2];
    const double Ly0[3] = {(Ly[0] - y[0] * yd) / yn, (Ly[1] - y[1] * yd) / yn, (Ly[2] - y[2] * yd) / yn};
    // y0 = z x c, c = (cos tyaw, sin tyaw, 0): Lz += c x Ly0, Lc = Ly0 x z
    Lz[0] += cy * Ly0[2]; Lz[1] += -cx * Ly0[2]; Lz[2] += cx * Ly0[1] - cy * Ly0[0];
    const double Lcx = Ly0[1] * z[2] - Ly0[2] * z[1], Lcy = Ly0[2] * z[0] - Ly0[0] * z[2];
    Lt.tyaw += -cy * Lcx + cx * Lcy;
    // z = tt / |tt|
    const double zd = z[0] * Lz[0] + z[1] * Lz[1] + z[2] * Lz[2];
    double Ltt[3] = {(Lz[0] - z[0] * zd) / tn, (Lz[1] - z[1] * zd) / tn, (Lz[2] - z[2] * zd) / tn};
    // thrust = (sqrt(max(scalar, 0) / (4 kf)) - const) / scale; zero gradient where scalar <= 0
    const double Lscalar = scalar > 0.0 ? Lthrust / P.pid_pwm2rpm_scale * (0.5 / root) / (4.0 * P.pid_kf) : 0.0;
    Ltt[0] += Lscalar * R[2]; Ltt[1] += Lscalar * R[5]; Ltt[2] += Lscalar * R[8];
    LR[2] += Lscalar * tt[0]; LR[5] += Lscalar * tt[1]; LR[8] += Lscalar * tt[2];
    // tt = P_FOR e + I_FOR ip + D_FOR ev (+ gravity), ip = clip(st.ip + e dt)
    const double Lip_new[3] = {Lst.ipx, Lst.ipy, Lst.ipz};
    double Lip_old[3];
    for (int a = 0; a < 3; ++a) {
        Lg[a] += e[a] * Ltt[a];
        Lg[3 + a] += ip[a] * Ltt[a];
        Lg[6 + a] += ev[a] * Ltt[a];
        const double Lip0 = ip_live[a] ? K.pid_i_for[a] * Ltt[a] + Lip_new[a] : 0.0;
        Lip_old[a] = Lip0;
        const double Le = K.pid_p_for[a] * Ltt[a] + dt * Lip0;
        const double Lev = K.pid_d_for[a] * Ltt[a];
        Lt.tp[a] += Le;
        Lt.tv[a] += Lev;
        if (a == 0) { L.px -= Le; L.vx -= Lev; } else if (a == 1) { L.py -= Le; L.vy -= Lev; } else { L.pz -= Le; L.vz -= Lev; }
    }
    Lst.ipx = Lip_old[0]; Lst.ipy = Lip_old[1]; Lst.ipz = Lip_old[2];
    // rpy = quat_to_euler<false>(q), on the forward's branch
    double Lqe[4] = {0.0, 0.0, 0.0, 0.0};
    quat_to_euler_vjp(qx, qy, qz, qw, Lrpy, Lqe);
    double LX = Lqe[0], LY = Lqe[1], LZ = Lqe[2], LW = Lqe[3];
    // R = I + s M(q), s = 2 / |q|^2 (quat_to_matrix)
    {
        const double dq = qx * qx + qy * qy + qz * qz + qw * qw;
        const double s = 2.0 / dq;
        const double M[9] = {-(qy * qy + qz * qz), qx * qy - qw * qz, qx * qz + qw * qy,
                             qx * qy + qw * qz, -(qx * qx + qz * qz), qy * qz - qw * qx,
                             qx * qz - qw * qy, qy * qz + qw * qx, -(qx * qx + qy * qy)};
        double Ls = 0.0;
        for (int j = 0; j < 9; ++j) Ls += LR[j] * M[j];
        const double* A = LR;
        LX += s * (A[1] * qy + A[2] * qz + A[3] * qy - 2.0 * qx * A[4] - A[5] * qw + A[6] * qz + A[7] * qw - 2.0 * qx * A[8]);
        LY += s * (-2.0 * qy * A[0] + A[1] * qx + A[2] * qw + A[3] * qx + A[5] * qz - A[6] * qw + A[7] * qz - 2.0 * qy * A[8]);
        LZ += s * (-2.0 * qz * A[0] - A[1] * qw + A[2] * qx + A[3] * qw - 2.0 * qz * A[4] + A[5] * qy + A[6] * qx + A[7] * qy);
        LW += s * (-A[1] * qz + A[2] * qy + A[3] * qz - A[5] * qx - A[6] * qy + A[7] * qx);
        const double k = -4.0 * Ls / (dq * dq);          // ds/dq = -4 q / |q|^4
        LX += k * qx; LY += k * qy; LZ += k * qz; LW += k * qw;
    }
    L.qx += LX; L.qy += LY; L.qz += LZ; L.qw += LW;
}

}  // namespace qs
