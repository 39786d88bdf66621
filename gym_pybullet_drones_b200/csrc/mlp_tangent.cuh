// mlp_tangent.cuh -- forward mode (the tangent) of one tick of the policy loop (dyn_policy_jvp.cu, DESIGN.md 4.5): the actor's
// activation derivative, the observation head, the action clip and the RPM / ONE_D_RPM decode, and the physics tick that also
// gives the tangent of the next observation's ang_v.  Compiled for the sm_90a kernels and for the host harness
// (tests/host_harness/policy_jvp_host.cpp).
//
// Every derivative decision is the transpose of mlp_adjoint.cuh's, so that <J v, w> = <v, J^T w> holds per aviary:
//   * ReLU passes the tangent where h > 0; Tanh multiplies it by 1 - h^2 on the forward's own h;
//   * the action clip follows torch.clamp: the tangent passes for -1 <= raw <= 1;
//   * rpy is differentiated on the forward's branch of the gimbal guard (dyn_tangent.cuh, quat_to_euler_jvp);
//   * ang_v = R_last w: its tangent goes through the attitude at the start of the tick's last substep, for the first
//     observation through the normalised initial attitude;
//   * HOVER_RPM (phys column 12) enters through the decode, MAX_RPM (column 13) through the env's clip.
#pragma once
#include "dyn_tangent.cuh"
#include "mlp_adjoint.cuh"

namespace qs {

QS_HD double mlp_act_jvp(int kind, double h, double t) { return kind == QS_MLP_RELU ? (h > 0.0 ? t : 0.0) : (1.0 - h * h) * t; }

// the tangent of clip(raw, -1, 1), the transpose of the VJP's mask
QS_HD double action_clip_jvp(double raw, double t) { return (raw < -1.0 || raw > 1.0) ? 0.0 : t; }

// t_ang = d(R(q) w) = R(q) t_w + (dR/dq t_q) w for R = quat_to_matrix_unit(q) = I + s M(q), s = 2 (2 - |q|^2): the transpose of
// ang_v_vjp
QS_HD void ang_v_jvp(double x, double y, double z, double w, const double v[3], const double t_q[4], const double t_v[3], double t_ang[3]) {
    double R[9];
    quat_to_matrix_unit(x, y, z, w, R);
    const double dx = t_q[0], dy = t_q[1], dz = t_q[2], dw = t_q[3];
    const double s = 2.0 * (2.0 - (x * x + y * y + z * z + w * w)), ds = -4.0 * (x * dx + y * dy + z * dz + w * dw);
    const double M[9] = {-(y * y + z * z), x * y - w * z, x * z + w * y,
                         x * y + w * z, -(x * x + z * z), y * z - w * x,
                         x * z - w * y, y * z + w * x, -(x * x + y * y)};
    const double dM[9] = {-2.0 * (y * dy + z * dz), dx * y + x * dy - dw * z - w * dz, dx * z + x * dz + dw * y + w * dy,
                          dx * y + x * dy + dw * z + w * dz, -2.0 * (x * dx + z * dz), dy * z + y * dz - dw * x - w * dx,
                          dx * z + x * dz - dw * y - w * dy, dy * z + y * dz + dw * x + w * dx, -2.0 * (x * dx + y * dy)};
    for (int r = 0; r < 3; ++r) {
        double acc = 0.0;
        for (int c = 0; c < 3; ++c) acc += R[3 * r + c] * t_v[c] + (s * dM[3 * r + c] + ds * M[3 * r + c]) * v[c];
        t_ang[r] = acc;
    }
}

// The tangent of the 12 kinematic entries of an observation row built from the stored state d (obs_head): pos, rpy (from the
// quaternion's tangent), vel, and ang_v's tangent t_ang, which the loop carries (the transpose of obs_head_vjp)
QS_HD void obs_head_jvp(const Drone& d, const Drone& t, const double t_ang[3], double t_o[12]) {
    t_o[0] = t.px; t_o[1] = t.py; t_o[2] = t.pz;
    const double t_q[4] = {t.qx, t.qy, t.qz, t.qw};
    double t_rpy[3] = {0.0, 0.0, 0.0};
    quat_to_euler_jvp(d.qx, d.qy, d.qz, d.qw, t_q, t_rpy);
    t_o[3] = t_rpy[0]; t_o[4] = t_rpy[1]; t_o[5] = t_rpy[2];
    t_o[6] = t.vx; t_o[7] = t.vy; t_o[8] = t.vz;
    t_o[9] = t_ang[0]; t_o[10] = t_ang[1]; t_o[11] = t_ang[2];
}

// The tangent of the first observation's ang_v = R(q0 / |q0|) w0 along the tangent t of the stored initial state d0 (the
// transpose of initial_ang_v_vjp)
QS_HD void initial_ang_v_jvp(const Drone& d0, const Drone& t, double t_ang[3]) {
    Drone x0 = d0;
    double inv;
    entry_normalise(x0, inv);
    const double dot = x0.qx * t.qx + x0.qy * t.qy + x0.qz * t.qz + x0.qw * t.qw;
    const double t_q[4] = {(t.qx - x0.qx * dot) * inv, (t.qy - x0.qy * dot) * inv, (t.qz - x0.qz * dot) * inv, (t.qw - x0.qw * dot) * inv};
    const double w[3] = {d0.wx, d0.wy, d0.wz}, t_w[3] = {t.wx, t.wy, t.wz};
    ang_v_jvp(x0.qx, x0.qy, x0.qz, x0.qw, w, t_q, t_w, t_ang);
}

// the tangent of rpm = HOVER_RPM (1 + 0.05 a) along the clipped action's tangent t_a and HOVER_RPM's t_hover (the transpose of
// policy_rpm_vjp)
QS_HD void policy_rpm_jvp(int A, const PhysRow& c, const double a[4], const double t_a[4], double t_hover, double t_rpm[4]) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int s = A == 1 ? 0 : j;
        t_rpm[j] = (1.0 + 0.05 * a[s]) * t_hover + c.hover_rpm * 0.05 * t_a[s];
    }
}

// dyn_tick_k's `between` hook of dyn_tick_obs_jvp: TangentHook, and before the last substep's tangent step the start state of
// that substep and its tangent
template <int EFF>
struct LastStartHook {
    TangentHook<EFF> step;
    int last;
    Drone* xl;
    Drone* tl;
    QS_HD void operator()(int s) const {
        if (s == last) { *xl = *step.x; *tl = *step.t; }
        step(s);
    }
};

// dyn_tick_jvp (dyn_tangent.cuh) for a tick whose end state also feeds the next observation's ang_v = R_last w_end, R_last the
// attitude at the start of the last substep: the transpose of dyn_tick_obs_vjp.  d / t / tc / tu / tup as dyn_tick_jvp (the
// primal is dyn_tick_k's bits); t_ang: out, the tangent of that ang_v.
template <int EFF>
QS_HD void dyn_tick_obs_jvp(const QsParams& P, const PhysRow& c, const PhysRow& tc, Drone& d, const double u[4], const double up[4],
                            int S, Drone& t, const double tu[4], const double tup[4], double t_ang[3]) {
    Drone x = d;
    double inv;
    entry_normalise(x, inv);
    const double dot = x.qx * t.qx + x.qy * t.qy + x.qz * t.qz + x.qw * t.qw;
    t.qx = (t.qx - x.qx * dot) * inv; t.qy = (t.qy - x.qy * dot) * inv;
    t.qz = (t.qz - x.qz * dot) * inv; t.qw = (t.qw - x.qw * dot) * inv;
    const double kk = 2.0 * 3.14159265358979323846;
    double tds_prev = 0.0, tds_cur = 0.0;
    if (EFF & QS_EFFECT_DRAG) {
#pragma unroll
        for (int i = 0; i < 4; ++i) { tds_prev += (kk / 60.0) * tup[i]; tds_cur += (kk / 60.0) * tu[i]; }
    }
    Drone xl = x, tl = t;
    double R_last[9];
    dyn_tick_k<EFF>(P, c, d, u, up, 0.0, S, R_last,
                    LastStartHook<EFF>{TangentHook<EFF>{&P, &c, &tc, &d, &x, &t, u, tu, drag_sum(up), drag_sum(u), tds_prev, tds_cur},
                                       S - 1, &xl, &tl});
    const double w_end[3] = {d.wx, d.wy, d.wz}, t_w[3] = {t.wx, t.wy, t.wz};
    const double t_ql[4] = {tl.qx, tl.qy, tl.qz, tl.qw};
    ang_v_jvp(xl.qx, xl.qy, xl.qz, xl.qw, w_end, t_ql, t_w, t_ang);
}

// The tangent of one drone's part of a policy tick after the actor: the action clip, the decode, the env's clip and the physics.
// raw / t_raw: the raw action and its tangent (A entries); d: in, the stored start state, out, the end state; t: its tangent in and
// out; up / t_up: drag's previous applied RPMs and their tangent; tc: the constants' tangent.  Out: t_a, the clipped action's
// tangent (what enters the history), t_u, the applied RPMs' tangent, t_ang, the next observation's ang_v tangent.
template <int EFF>
QS_HD void policy_tick_jvp(const QsParams& P, const PhysRow& c, const PhysRow& tc, int A, int S, const double raw[4], const double t_raw[4],
                           Drone& d, Drone& t, const double up[4], const double t_up[4], double t_a[4], double t_u[4], double t_ang[3]) {
    double aa[4] = {0.0, 0.0, 0.0, 0.0}, rpm[4], u[4], t_rpm[4];
    t_a[0] = t_a[1] = t_a[2] = t_a[3] = 0.0;
    for (int j = 0; j < A; ++j) {
        aa[j] = clampd(raw[j], -1.0, 1.0);
        t_a[j] = action_clip_jvp(raw[j], t_raw[j]);
    }
    policy_rpm(A, c, aa, rpm);
#pragma unroll
    for (int j = 0; j < 4; ++j) u[j] = clampd(rpm[j], 0.0, c.max_rpm);
    policy_rpm_jvp(A, c, aa, t_a, tc.hover_rpm, t_rpm);
    rpm_clip_jvp(rpm, c.max_rpm, t_rpm, tc.max_rpm, t_u);
    dyn_tick_obs_jvp<EFF>(P, c, tc, d, u, up, S, t, t_u, t_up, t_ang);
}

}  // namespace qs
