// pid_tangent.cuh -- forward mode (the tangent) of DSLPIDControl.computeControl (qs::pid_control_k, quad_core.cuh) for the
// closed-loop JVP and Jacobian kernels of dyn_ctrl_jvp.cu, compiled for the sm_90a kernels and for the host harness
// (tests/host_harness/ctrl_jvp_host.cpp).
//
// Every derivative decision is the transpose of pid_adjoint.cuh's (DESIGN.md 4.5), so that <J v, w> = <v, J^T w> holds per drone:
//   * every clip follows torch.clamp with constant bounds: the tangent passes for lo <= x <= hi and is zero outside (the nested
//     integral clips, the torque clip +-3200, the PWM clip);
//   * the tangent of `scalar < 0 ? 0 : scalar` then sqrt is zero where scalar <= 0;
//   * quat_to_euler<false> is differentiated on the forward's branch of the +-0.99999 gimbal guard (quat_to_euler_jvp);
//   * the rate term (rpy - last_rpy) / dt has no angle unwrap;
//   * the quaternion is read as stored, unnormalised: R = I + (2 / |q|^2) M(q) carries the tangent of |q|, and the Euler angles
//     are those of the unnormalised quaternion;
//   * the atan2 of the yaw error only feeds yaw_e, which is not an output of the trajectory: it carries no tangent.
#pragma once
#include "dyn_tangent.cuh"
#include "pid_adjoint.cuh"

namespace qs {

// Tangent of pid_control_k(P, K, st, dt, d.pos, d.quat, d.vel, tg, ...).  tK / t_st / t_d / t_tg: the tangents of the gains, of
// the controller state the call starts from, of the drone (pos, quat, vel are read) and of the targets.  Out: t_rpm, the tangent
// of the raw RPMs (before any max_rpm clip), and t_out, of the updated controller state.
QS_HD_NOINLINE void pid_control_jvp(const QsParams& P, const PidGains& K, const PidState& st, double dt, const Drone& d,
                                    const PidTargets& tg, const PidGains& tK, const PidState& t_st, const Drone& t_d,
                                    const PidTargets& t_tg, double t_rpm[4], PidState& t_out) {
    const double qx = d.qx, qy = d.qy, qz = d.qz, qw = d.qw;
    const double dqx = t_d.qx, dqy = t_d.qy, dqz = t_d.qz, dqw = t_d.qw;
    // R = I + s M(q), s = 2 / |q|^2 (quat_to_matrix), and its tangent
    double R[9], dR[9];
    quat_to_matrix(qx, qy, qz, qw, R);
    {
        const double dq = qx * qx + qy * qy + qz * qz + qw * qw;
        const double s = 2.0 / dq;
        const double ds = -4.0 * (qx * dqx + qy * dqy + qz * dqz + qw * dqw) / (dq * dq);
        const double M[9] = {-(qy * qy + qz * qz), qx * qy - qw * qz, qx * qz + qw * qy,
                             qx * qy + qw * qz, -(qx * qx + qz * qz), qy * qz - qw * qx,
                             qx * qz - qw * qy, qy * qz + qw * qx, -(qx * qx + qy * qy)};
        const double dM[9] = {-2.0 * (qy * dqy + qz * dqz), dqx * qy + qx * dqy - dqw * qz - qw * dqz,
                              dqx * qz + qx * dqz + dqw * qy + qw * dqy,
                              dqx * qy + qx * dqy + dqw * qz + qw * dqz, -2.0 * (qx * dqx + qz * dqz),
                              dqy * qz + qy * dqz - dqw * qx - qw * dqx,
                              dqx * qz + qx * dqz - dqw * qy - qw * dqy, dqy * qz + qy * dqz + dqw * qx + qw * dqx,
                              -2.0 * (qx * dqx + qy * dqy)};
        for (int j = 0; j < 9; ++j) dR[j] = ds * M[j] + s * dM[j];
    }
    // position loop
    const double e[3] = {tg.tp[0] - d.px, tg.tp[1] - d.py, tg.tp[2] - d.pz};
    const double ev[3] = {tg.tv[0] - d.vx, tg.tv[1] - d.vy, tg.tv[2] - d.vz};
    const double de[3] = {t_tg.tp[0] - t_d.px, t_tg.tp[1] - t_d.py, t_tg.tp[2] - t_d.pz};
    const double dev[3] = {t_tg.tv[0] - t_d.vx, t_tg.tv[1] - t_d.vy, t_tg.tv[2] - t_d.vz};
    const double ip0[3] = {st.ipx + e[0] * dt, st.ipy + e[1] * dt, st.ipz + e[2] * dt};
    const double ipz1 = clampd(ip0[2], -2.0, 2.0);
    const double ip[3] = {clampd(ip0[0], -2.0, 2.0), clampd(ip0[1], -2.0, 2.0), clampd(ipz1, -0.15, 0.15)};
    const bool ip_live[3] = {clamp_passes(ip0[0], -2.0, 2.0), clamp_passes(ip0[1], -2.0, 2.0),
                             clamp_passes(ip0[2], -2.0, 2.0) && clamp_passes(ipz1, -0.15, 0.15)};
    const double t_ip_in[3] = {t_st.ipx, t_st.ipy, t_st.ipz};
    // the forward values in pid_control_k's operation order, so that every decision is taken on the same bits
    const double tt[3] = {K.pid_p_for[0] * e[0] + K.pid_i_for[0] * ip[0] + K.pid_d_for[0] * ev[0],
                          K.pid_p_for[1] * e[1] + K.pid_i_for[1] * ip[1] + K.pid_d_for[1] * ev[1],
                          K.pid_p_for[2] * e[2] + K.pid_i_for[2] * ip[2] + K.pid_d_for[2] * ev[2] + P.pid_gravity};
    double dtt[3], dip[3];
    for (int a = 0; a < 3; ++a) {
        dip[a] = ip_live[a] ? t_ip_in[a] + de[a] * dt : 0.0;
        dtt[a] =tK.pid_p_for[a] * e[a] + K.pid_p_for[a] * de[a] + tK.pid_i_for[a] * ip[a] + K.pid_i_for[a] * dip[a] +
                 tK.pid_d_for[a] * ev[a] + K.pid_d_for[a] * dev[a];
    }
    const double scalar = tt[0] * R[2] + tt[1] * R[5] + tt[2] * R[8];
    const double sc = scalar < 0.0 ? 0.0 : scalar;
    const double root = sqrt(sc / (4.0 * P.pid_kf));
    const double thrust = (root - P.pid_pwm2rpm_const) / P.pid_pwm2rpm_scale;
    const double dscalar = dtt[0] * R[2] + dtt[1] * R[5] + dtt[2] * R[8] + tt[0] * dR[2] + tt[1] * dR[5] + tt[2] * dR[8];
    const double dthrust = scalar > 0.0 ? dscalar / P.pid_pwm2rpm_scale * (0.5 / root) / (4.0 * P.pid_kf) : 0.0;
    // target attitude: z = tt / |tt|, y = z x c / |z x c|, x = y x z, c = (cos tyaw, sin tyaw, 0)
    const double tn = sqrt(tt[0] * tt[0] + tt[1] * tt[1] + tt[2] * tt[2]);
    const double z[3] = {tt[0] / tn, tt[1] / tn, tt[2] / tn};
    const double zd = z[0] * dtt[0] + z[1] * dtt[1] + z[2] * dtt[2];
    const double dz[3] = {(dtt[0] - z[0] * zd) / tn, (dtt[1] - z[1] * zd) / tn, (dtt[2] - z[2] * zd) / tn};
    const double cx = cos(tg.tyaw), cy = sin(tg.tyaw);
    const double dcx = -cy * t_tg.tyaw, dcy = cx * t_tg.tyaw;
    const double y0[3] = {z[1] * 0.0 - z[2] * cy, z[2] * cx - z[0] * 0.0, z[0] * cy - z[1] * cx};
    const double dy0[3] = {-dz[2] * cy - z[2] * dcy, dz[2] * cx + z[2] * dcx, dz[0] * cy + z[0] * dcy - dz[1] * cx - z[1] * dcx};
    const double yn = sqrt(y0[0] * y0[0] + y0[1] * y0[1] + y0[2] * y0[2]);
    const double y[3] = {y0[0] / yn, y0[1] / yn, y0[2] / yn};
    const double yd = y[0] * dy0[0] + y[1] * dy0[1] + y[2] * dy0[2];
    const double dy[3] = {(dy0[0] - y[0] * yd) / yn, (dy0[1] - y[1] * yd) / yn, (dy0[2] - y[2] * yd) / yn};
    const double x[3] = {y[1] * z[2] - y[2] * z[1], y[2] * z[0] - y[0] * z[2], y[0] * z[1] - y[1] * z[0]};
    const double dx[3] = {dy[1] * z[2] + y[1] * dz[2] - dy[2] * z[1] - y[2] * dz[1],
                          dy[2] * z[0] + y[2] * dz[0] - dy[0] * z[2] - y[0] * dz[2],
                          dy[0] * z[1] + y[0] * dz[1] - dy[1] * z[0] - y[1] * dz[0]};
    // T = Rd, columns x, y, z: T[3 j + c]
    const double T[9] = {x[0], y[0], z[0], x[1], y[1], z[1], x[2], y[2], z[2]};
    const double dT[9] = {dx[0], dy[0], dz[0], dx[1], dy[1], dz[1], dx[2], dy[2], dz[2]};
    // rot_e = (E[2][1], E[0][2], E[1][0]) of E = T^T R - R^T T: re[a] = sum_j T[j][i] R[j][k] - R[j][i] T[j][k]
    double re[3], dre[3];
    {
        #define QS_TtR(i, k) (T[0 + i] * R[0 + k] + T[3 + i] * R[3 + k] + T[6 + i] * R[6 + k])
        #define QS_RtT(i, k) (R[0 + i] * T[0 + k] + R[3 + i] * T[3 + k] + R[6 + i] * T[6 + k])
        re[0] = QS_TtR(2, 1) - QS_RtT(2, 1);
        re[1] = QS_TtR(0, 2) - QS_RtT(0, 2);
        re[2] = QS_TtR(1, 0) - QS_RtT(1, 0);
        #undef QS_TtR
        #undef QS_RtT
        const int I[3] = {2, 0, 1}, Kc[3] = {1, 2, 0};
        for (int a = 0; a < 3; ++a) {
            const int i = I[a], k = Kc[a];
            double dv = 0.0;
            for (int j = 0; j < 3; ++j)
                dv += dT[3 * j + i] * R[3 * j + k] + T[3 * j + i] * dR[3 * j + k] - dR[3 * j + i] * T[3 * j + k] - R[3 * j + i] * dT[3 * j + k];
            dre[a] = dv;
        }
    }
    // attitude loop
    double rpy[3], drpy[3] = {0.0, 0.0, 0.0};
    quat_to_euler<false>(qx, qy, qz, qw, rpy[0], rpy[1], rpy[2]);
    const double tq[4] = {dqx, dqy, dqz, dqw};
    quat_to_euler_jvp(qx, qy, qz, qw, tq, drpy);
    const double last[3] = {st.lr, st.lp, st.ly}, t_last[3] = {t_st.lr, t_st.lp, t_st.ly};
    const double ir_in[3] = {st.irx, st.iry, st.irz}, t_ir_in[3] = {t_st.irx, t_st.iry, t_st.irz};
    double dqc[3], qc[3], dir[3];
    for (int a = 0; a < 3; ++a) {
        const double rr = tg.trr[a] - (rpy[a] - last[a]) / dt;
        const double drr = t_tg.trr[a] - (drpy[a] - t_last[a]) / dt;
        const double ir0 = ir_in[a] - re[a] * dt;
        const double ir1 = clampd(ir0, -1500.0, 1500.0);
        const double ir = a < 2 ? clampd(ir1, -1.0, 1.0) : ir1;
        const bool ir_live = clamp_passes(ir0, -1500.0, 1500.0) && (a == 2 || clamp_passes(ir1, -1.0, 1.0));
        dir[a] = ir_live ? t_ir_in[a] - dre[a] * dt : 0.0;
        const double qt = -K.pid_p_tor[a] * re[a] + K.pid_d_tor[a] * rr + K.pid_i_tor[a] * ir;
        const double dqt = -tK.pid_p_tor[a] * re[a] - K.pid_p_tor[a] * dre[a] + tK.pid_d_tor[a] * rr + K.pid_d_tor[a] * drr +
                           tK.pid_i_tor[a] * ir + K.pid_i_tor[a] * dir[a];
        qc[a] = clampd(qt, -3200.0, 3200.0);
        dqc[a] = clamp_passes(qt, -3200.0, 3200.0) ? dqt : 0.0;
    }
    // rpm = scale pwm + const, pwm = clip(thrust + mixer qc)
    for (int j = 0; j < 4; ++j) {
        const double pwm = thrust + (P.pid_mixer[j][0] * qc[0] + P.pid_mixer[j][1] * qc[1] + P.pid_mixer[j][2] * qc[2]);
        const double dpwm = dthrust + (P.pid_mixer[j][0] * dqc[0] + P.pid_mixer[j][1] * dqc[1] + P.pid_mixer[j][2] * dqc[2]);
        t_rpm[j] = clamp_passes(pwm, P.pid_min_pwm, P.pid_max_pwm) ? P.pid_pwm2rpm_scale * dpwm : 0.0;
    }
    t_out.ipx = dip[0]; t_out.ipy = dip[1]; t_out.ipz = dip[2];
    t_out.lr = drpy[0]; t_out.lp = drpy[1]; t_out.ly = drpy[2];
    t_out.irx = dir[0]; t_out.iry = dir[1]; t_out.irz = dir[2];
}

}  // namespace qs
