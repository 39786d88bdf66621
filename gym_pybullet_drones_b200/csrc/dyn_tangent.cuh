// dyn_tangent.cuh -- forward mode (the tangent) of one control tick of Physics.DYN (qs::dyn_tick_k, quad_core.cuh) for the JVP
// and Jacobian kernels of dyn_jvp.cu, compiled for the sm_90a kernels and for the host harness (tests/host_harness/jvp_host.cpp).
//
// Every derivative decision is the transpose of dyn_adjoint.cuh's (DESIGN.md 4.5), so that <J v, w> = <v, J^T w> holds per drone:
//   * _integrateQ's exponential map is differentiated everywhere (half_angle_grad), also where the forward takes np.isclose's
//     identity;
//   * the quaternion renormalisation on tick entry is part of the function; the rounding on exit (round_to_planes) is the identity;
//   * the RPM clip follows torch.clamp (rpm_clip_jvp): raw's tangent passes for 0 <= raw <= MAX_RPM, MAX_RPM's is taken above it;
//   * the ground-effect height clip uses the forward's `hz < clip` predicate; the upright switch is held constant;
//   * drag's first substep reads the previous tick's clipped RPMs `up`, later substeps the current ones.
//
// The tick's tangent runs dyn_tick_k itself with a `between` hook (TangentHook) that keeps the previous substep's end state in
// registers and advances the tangent over each substep as it completes: the primal is dyn_tick_k's bits and nothing is recorded.
// The tangent of the constants is a PhysRow of tangents (QsState.phys column order; hover_rpm's does not enter a tick).
#pragma once
#include "dyn_adjoint.cuh"

namespace qs {

// The tangent of clip(raw, 0, max_rpm) (CtrlAviary.py:140), the transpose of rpm_clip_vjp: t_raw passes for 0 <= raw <= max,
// t_max is taken for raw > max, nothing below 0
QS_HD void rpm_clip_jvp(const double raw[4], double max_rpm, const double t_raw[4], double t_max, double t_u[4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) t_u[i] = raw[i] > max_rpm ? t_max : (raw[i] < 0.0 ? 0.0 : t_raw[i]);
}

// t_rpy += d rpy / d q  t_q for rpy = quat_to_euler<false>(q), on the forward's branch of the +-0.99999 gimbal guard: the
// transpose of quat_to_euler_vjp (in the guard roll and pitch are constants and yaw = 2 atan2(x, -y) or 2 atan2(-x, y))
QS_HD void quat_to_euler_jvp(double qx, double qy, double qz, double qw, const double t_q[4], double t_rpy[3]) {
    const double sarg = -2.0 * (qx * qz - qw * qy);
    const double dx = t_q[0], dy = t_q[1], dz = t_q[2], dw = t_q[3];
    if (sarg <= -0.99999 || sarg >= 0.99999) {
        const double r2 = qx * qx + qy * qy;
        t_rpy[2] += (-2.0 * qy / r2) * dx + (2.0 * qx / r2) * dy;
    } else {
        const double ra = 2.0 * (qy * qz + qw * qx), rb = qw * qw - qx * qx - qy * qy + qz * qz;
        const double ya = 2.0 * (qx * qy + qw * qz), yb = qw * qw + qx * qx - qy * qy - qz * qz;
        const double n_r = ra * ra + rb * rb, n_y = ya * ya + yb * yb;
        const double dra = 2.0 * (qw * dx + qz * dy + qy * dz + qx * dw), drb = 2.0 * (-qx * dx - qy * dy + qz * dz + qw * dw);
        const double dsarg = 2.0 * (-qz * dx + qw * dy - qx * dz + qy * dw);
        const double dya = 2.0 * (qy * dx + qx * dy + qw * dz + qz * dw), dyb = 2.0 * (qx * dx - qy * dy - qz * dz + qw * dw);
        t_rpy[0] += (rb * dra - ra * drb) / n_r;
        t_rpy[1] += dsarg / sqrt(1.0 - sarg * sarg);
        t_rpy[2] += (yb * dya - ya * dyb) / n_y;
    }
}

// Tangent of one substep of dyn_tick_k<EFF> from its start state x with (clipped) rpm u and drag sum ds.  t: in, the tangent of
// x; out, of the substep's end state.  tc / tu / tds: the tangents of the constants, of u and of ds.
template <int EFF>
QS_HD void substep_jvp(const QsParams& P, const PhysRow& c, const PhysRow& tc, const Drone& x, const double u[4], double ds,
                       Drone& t, const double tu[4], double tds) {
    const double dt = P.dt, dt_m = dt * c.inv_m;
    const double X = x.qx, Y = x.qy, Z = x.qz, W = x.qw;
    const double dX = t.qx, dY = t.qy, dZ = t.qz, dW = t.qw;
    // the rotation entries (unit quaternion: Bullet's s = 2) and their tangents
    const double r02 = 2.0 * (X * Z + W * Y), r12 = 2.0 * (Y * Z - W * X), r22 = 1.0 - 2.0 * (X * X + Y * Y);
    const double r20 = 2.0 * (X * Z - W * Y), r21 = 2.0 * (Y * Z + W * X);
    const double d02 = 2.0 * (dX * Z + X * dZ + dW * Y + W * dY), d12 = 2.0 * (dY * Z + Y * dZ - dW * X - W * dX);
    const double d22 = -4.0 * (X * dX + Y * dY);
    const double d20 = 2.0 * (dX * Z + X * dZ - dW * Y - W * dY), d21 = 2.0 * (dY * Z + Y * dZ + dW * X + W * dX);
    bool up = false;
    if (EFF & QS_EFFECT_GND) up = upright(-2.0 * (X * Z - W * Y), 2.0 * (Y * Z + W * X), W * W - X * X - Y * Y + Z * Z);
    const double gcoef = P.gnd_eff_coeff;
    // forces and torques
    double thrust = 0.0, sxf = 0.0, syf = 0.0, tz = 0.0, d_thrust = 0.0, d_sxf = 0.0, d_syf = 0.0, d_tz = 0.0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const double u2 = u[i] * u[i], d_u2 = 2.0 * u[i] * tu[i];
        const double f0 = u2 * c.kf, d_f0 = d_u2 * c.kf + u2 * tc.kf;
        double fg = f0, d_fg = d_f0;
        if ((EFF & QS_EFFECT_GND) && up) {
            const double hz = x.pz + r20 * P.prop_xyz[i][0] + r21 * P.prop_xyz[i][1] + r22 * P.prop_xyz[i][2];
            const bool live = !(hz < P.gnd_eff_h_clip);
            const double hh = live ? hz : P.gnd_eff_h_clip;
            const double rr = P.prop_radius / (4.0 * hh);
            const double e = gcoef * (rr * rr);
            fg += f0 * e;
            d_fg += d_f0 * e;
            if (live) {
                const double d_hz = t.pz + d20 * P.prop_xyz[i][0] + d21 * P.prop_xyz[i][1] + d22 * P.prop_xyz[i][2];
                d_fg += -(rr / hh) * (2.0 * f0 * gcoef * rr) * d_hz;
            }
        }
        thrust += fg; sxf += P.sx[i] * fg; syf += P.sy[i] * fg;
        d_thrust += d_fg; d_sxf += P.sx[i] * d_fg; d_syf += P.sy[i] * d_fg;
        tz += P.sz[i] * (u2 * c.km);
        d_tz += P.sz[i] * (d_u2 * c.km + u2 * tc.km);
    }
    const double tx = sxf * c.kx, ty = syf * c.ky;
    const double d_tx = d_sxf * c.kx + sxf * tc.kx, d_ty = d_syf * c.ky + syf * tc.ky;
    double F[3] = {r02 * thrust, r12 * thrust, r22 * thrust - c.gravity};
    double dF[3] = {d02 * thrust + r02 * d_thrust, d12 * thrust + r12 * d_thrust, d22 * thrust + r22 * d_thrust - tc.gravity};
    const double v[3] = {x.vx, x.vy, x.vz}, dv[3] = {t.vx, t.vy, t.vz};
    if (EFF & QS_EFFECT_DRAG) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            F[a] += -P.drag_coeff[a] * ds * v[a];
            dF[a] -= P.drag_coeff[a] * (tds * v[a] + ds * dv[a]);
        }
    }
    // w' = w + dt J^-1 (torques - w x Jw)
    const double g21 = c.j[2] - c.j[1], g02 = c.j[0] - c.j[2], g10 = c.j[1] - c.j[0];
    const double d_g21 = tc.j[2] - tc.j[1], d_g02 = tc.j[0] - tc.j[2], d_g10 = tc.j[1] - tc.j[0];
    const double tt[3] = {tx - g21 * (x.wy * x.wz), ty - g02 * (x.wz * x.wx), tz - g10 * (x.wx * x.wy)};
    const double d_tt[3] = {d_tx - d_g21 * (x.wy * x.wz) - g21 * (t.wy * x.wz + x.wy * t.wz),
                            d_ty - d_g02 * (x.wz * x.wx) - g02 * (t.wz * x.wx + x.wz * t.wx),
                            d_tz - d_g10 * (x.wx * x.wy) - g10 * (t.wx * x.wy + x.wx * t.wy)};
    const double w[3] = {x.wx, x.wy, x.wz}, dw[3] = {t.wx, t.wy, t.wz};
    double wn[3], d_wn[3], d_vn[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        wn[a] = w[a] + dt * c.j_inv[a] * tt[a];
        d_wn[a] = dw[a] + dt * (tc.j_inv[a] * tt[a] + c.j_inv[a] * d_tt[a]);
        d_vn[a] = dv[a] + dt_m * dF[a] + dt * tc.inv_m * F[a];        // v' = v + dt/M F
    }
    // p' = p + dt v'
    t.px += dt * d_vn[0]; t.py += dt * d_vn[1]; t.pz += dt * d_vn[2];
    t.vx = d_vn[0]; t.vy = d_vn[1]; t.vz = d_vn[2];
    t.wx = d_wn[0]; t.wy = d_wn[1]; t.wz = d_wn[2];
    // q' = C q + S Omega(w') q
    const double p = wn[0], q = wn[1], r = wn[2], dp = d_wn[0], dq = d_wn[1], dr = d_wn[2];
    double C, S, dC, dS;
    half_angle_grad(p * p + q * q + r * r, dt, C, S, dC, dS);
    const double d_n2 = 2.0 * (p * dp + q * dq + r * dr);
    const double tC = dC * d_n2, tS = dS * d_n2;
    const double m0 = r * Y - q * Z + p * W, m1 = -r * X + p * Z + q * W, m2 = q * X - p * Y + r * W, m3 = -p * X - q * Y - r * Z;
    const double dm0 = dr * Y + r * dY - dq * Z - q * dZ + dp * W + p * dW;
    const double dm1 = -dr * X - r * dX + dp * Z + p * dZ + dq * W + q * dW;
    const double dm2 = dq * X + q * dX - dp * Y - p * dY + dr * W + r * dW;
    const double dm3 = -dp * X - p * dX - dq * Y - q * dY - dr * Z - r * dZ;
    t.qx = tC * X + C * dX + tS * m0 + S * dm0;
    t.qy = tC * Y + C * dY + tS * m1 + S * dm1;
    t.qz = tC * Z + C * dZ + tS * m2 + S * dm2;
    t.qw = tC * W + C * dW + tS * m3 + S * dm3;
}

// dyn_tick_k's `between` hook of the tick tangent: after substep s, advance the tangent over it from the substep's start state
// (held in *x) and keep the end state (*d) as the next substep's start
template <int EFF>
struct TangentHook {
    const QsParams* P;
    const PhysRow* c;
    const PhysRow* tc;
    const Drone* d;
    Drone* x;
    Drone* t;
    const double* u;
    const double* tu;
    double ds_prev, ds_cur, tds_prev, tds_cur;
    QS_HD void operator()(int s) const {
        substep_jvp<EFF>(*P, *c, *tc, *x, u, s == 0 ? ds_prev : ds_cur, *t, tu, s == 0 ? tds_prev : tds_cur);
        *x = *d;
    }
};

// Tangent of dyn_tick_k<EFF>(P, c, d, u, up, 0, S, .).  d: in, the tick-start state as stored (before the entry renormalisation);
// out, dyn_tick_k's end state (its bits).  t: in, the tangent of the stored start state; out, of the end state (the exit rounding
// round_to_planes passes it unchanged).  tc / tu / tup: the tangents of the constants, of the clipped RPMs u and of drag's
// previous clipped RPMs up.
template <int EFF>
QS_HD void dyn_tick_jvp(const QsParams& P, const PhysRow& c, const PhysRow& tc, Drone& d, const double u[4], const double up[4],
                        int S, Drone& t, const double tu[4], const double tup[4]) {
    Drone x = d;
    double inv;
    entry_normalise(x, inv);
    // q_hat = q / |q|: t_hat = (t - q_hat (q_hat . t)) / |q|
    const double dot = x.qx * t.qx + x.qy * t.qy + x.qz * t.qz + x.qw * t.qw;
    t.qx = (t.qx - x.qx * dot) * inv; t.qy = (t.qy - x.qy * dot) * inv;
    t.qz = (t.qz - x.qz * dot) * inv; t.qw = (t.qw - x.qw * dot) * inv;
    const double kk = 2.0 * 3.14159265358979323846;
    double tds_prev = 0.0, tds_cur = 0.0;
    if (EFF & QS_EFFECT_DRAG) {
#pragma unroll
        for (int i = 0; i < 4; ++i) { tds_prev += (kk / 60.0) * tup[i]; tds_cur += (kk / 60.0) * tu[i]; }
    }
    double R_last[9];
    dyn_tick_k<EFF>(P, c, d, u, up, 0.0, S, R_last,
                    TangentHook<EFF>{&P, &c, &tc, &d, &x, &t, u, tu, drag_sum(up), drag_sum(u), tds_prev, tds_cur});
}

}  // namespace qs
