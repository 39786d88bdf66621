// dyn_adjoint.cuh -- reverse mode of one control tick of Physics.DYN (qs::dyn_tick_k, quad_core.cuh) for the differentiable
// trajectories of dyn_traj.cu, compiled for the sm_90a kernels and for the host harness (tests/host_harness/diff_host.cpp).
//
// Which derivative (DESIGN.md 4.5):
//   * _integrateQ: the exponential map q' = (cos th I + sin(th)/|w| Omega(w)) q is differentiated everywhere, also where the forward
//     takes np.isclose(|w|, 0)'s identity (there the two differ by at most |w| dt / 2 in value, and the identity's zero derivative
//     would leave a hovering drone's attitude blind to differential RPM).
//   * the quaternion renormalisation on tick entry is part of the function (so the state's quaternion cotangent has no radial part);
//     the one on tick exit (store_drone) acts on a unit quaternion whose derivative is tangent, so its VJP is the identity there.
//   * the ground-effect height clip and the upright switch use the forward's predicates; the switch has no derivative.
//   * the RPM clip (rpm_clip_vjp) follows torch.clamp: the gradient passes for 0 <= rpm <= MAX_RPM and goes to MAX_RPM above it.
//
// The tick's adjoint recomputes the substeps with dyn_tick_k itself, recording each substep's end state through its `between` hook
// into a caller-provided record (global scratch in the kernel, a host array in the harness), then runs the substep adjoints in
// reverse.  Gradients with respect to the constants are accumulated into the 16 columns of a QsState.phys row (PhysGrad).
#pragma once
#include "quad_core.cuh"

namespace qs {

// d/d(constants of the row) in QsState.phys column order: inv_m, gravity, kf, km, kx, ky, j[3], j_inv[3], hover_rpm, max_rpm, pad[2]
struct PhysGrad { double g[16]; };

QS_HD PhysRow phys_row_of(const QsParams& P) {
    PhysRow c;
    c.inv_m = P.inv_m; c.gravity = P.gravity; c.kf = P.kf; c.km = P.km; c.kx = P.kx; c.ky = P.ky;
    for (int k = 0; k < 3; ++k) { c.j[k] = P.j[k]; c.j_inv[k] = P.j_inv[k]; }
    c.hover_rpm = P.hover_rpm; c.max_rpm = P.max_rpm;
    return c;
}

// cos(theta), sin(theta)/|w| (half_angle_terms) and their derivatives with respect to n2 = |w|^2.  With t = theta^2 = n2 h^2:
// dC/dn2 = h^2 dC/dt, dS/dn2 = h^3 dsinc/dt; below t = 1/4 both are 8-term series in t (next terms < 1e-19), no sqrt at w = 0.
QS_HD void half_angle_grad(double n2, double dt, double& c, double& s, double& dc, double& ds) {
    half_angle_terms(n2, dt, c, s);
    const double h = 0.5 * dt;
    const double t = n2 * h * h;
    if (t < 0.25) {
        // dC/dt = sum_{k=1..8} (-1)^k k t^(k-1) / (2k)!
        double pc = 8.0 / 20922789888000.0;                  // k=8  +8/16!
        pc = pc * t - 7.0 / 87178291200.0;                   // k=7  -7/14!
        pc = pc * t + 6.0 / 479001600.0;                     // k=6  +6/12!
        pc = pc * t - 5.0 / 3628800.0;                       // k=5  -5/10!
        pc = pc * t + 4.0 / 40320.0;                         // k=4  +4/8!
        pc = pc * t - 3.0 / 720.0;                           // k=3  -3/6!
        pc = pc * t + 2.0 / 24.0;                            // k=2  +2/4!
        pc = pc * t - 0.5;                                   // k=1  -1/2!
        // dsinc/dt = sum_{k=1..8} (-1)^k k t^(k-1) / (2k+1)!
        double ps = 8.0 / 355687428096000.0;                 // k=8  +8/17!
        ps = ps * t - 7.0 / 1307674368000.0;                 // k=7  -7/15!
        ps = ps * t + 6.0 / 6227020800.0;                    // k=6  +6/13!
        ps = ps * t - 5.0 / 39916800.0;                      // k=5  -5/11!
        ps = ps * t + 4.0 / 362880.0;                        // k=4  +4/9!
        ps = ps * t - 3.0 / 5040.0;                          // k=3  -3/7!
        ps = ps * t + 2.0 / 120.0;                           // k=2  +2/5!
        ps = ps * t - 1.0 / 6.0;                             // k=1  -1/3!
        dc = pc * (h * h);
        ds = ps * (h * h * h);
    } else {
        const double n = sqrt(n2);
        const double th = n * h;
        dc = -sin(th) * h / (2.0 * n);
        ds = (h * cos(th) - s) / (2.0 * n2);
    }
}

// clip(raw, 0, max_rpm) (CtrlAviary.py:140) with torch.clamp's gradient: g_raw = L for 0 <= raw <= max, g_max += L for raw > max
QS_HD void rpm_clip_vjp(const double raw[4], double max_rpm, const double L[4], double g_raw[4], double& g_max) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const bool above = raw[i] > max_rpm, below = raw[i] < 0.0;
        g_raw[i] = (above || below) ? 0.0 : L[i];
        if (above) g_max += L[i];
    }
}

// Adjoint of one substep of dyn_tick_k<EFF> from its start state x with (clipped) rpm u and drag sum ds.  L: in, the cotangent of
// the substep's end state; out, of x.  Lu / Lds / G accumulate.  With QS_EFFECT_DW, fz is the substep's downwash force along body
// z (held constant here) and *Lfz receives its cotangent, the cotangent of the thrust scalar.
template <int EFF>
QS_HD void substep_vjp(const QsParams& P, const PhysRow& c, const Drone& x, const double u[4], double ds, Drone& L, double Lu[4],
                       double& Lds, PhysGrad& G, double fz = 0.0, double* Lfz = nullptr) {
    const double dt = P.dt, dt_m = dt * c.inv_m;
    const double X = x.qx, Y = x.qy, Z = x.qz, W = x.qw;
    // ---- forward values of the substep (unit quaternion: Bullet's s = 2) ----
    const double r02 = 2.0 * (X * Z + W * Y), r12 = 2.0 * (Y * Z - W * X), r22 = 1.0 - 2.0 * (X * X + Y * Y);
    const double r20 = 2.0 * (X * Z - W * Y), r21 = 2.0 * (Y * Z + W * X);
    double fg[4], rr[4], hh[4];
    bool hz_live[4] = {false, false, false, false};
    bool up = false;
    const double gcoef = P.gnd_eff_coeff;
#pragma unroll
    for (int i = 0; i < 4; ++i) { fg[i] = u[i] * u[i] * c.kf; rr[i] = 0.0; hh[i] = 1.0; }
    if (EFF & QS_EFFECT_GND) {
        up = upright(-2.0 * (X * Z - W * Y), 2.0 * (Y * Z + W * X), W * W - X * X - Y * Y + Z * Z);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const double hz = x.pz + r20 * P.prop_xyz[i][0] + r21 * P.prop_xyz[i][1] + r22 * P.prop_xyz[i][2];
            hz_live[i] = !(hz < P.gnd_eff_h_clip);
            hh[i] = hz_live[i] ? hz : P.gnd_eff_h_clip;
            rr[i] = P.prop_radius / (4.0 * hh[i]);
            if (up) fg[i] += u[i] * u[i] * c.kf * gcoef * (rr[i] * rr[i]);
        }
    }
    double thrust = 0.0, sxf = 0.0, syf = 0.0, tz = 0.0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        thrust += fg[i]; sxf += P.sx[i] * fg[i]; syf += P.sy[i] * fg[i]; tz += P.sz[i] * (u[i] * u[i] * c.km);
    }
    const double tx = sxf * c.kx, ty = syf * c.ky;
    double F[3] = {r02 * thrust, r12 * thrust, r22 * thrust - c.gravity};
    if (EFF & QS_EFFECT_DRAG) {
        F[0] += -P.drag_coeff[0] * ds * x.vx; F[1] += -P.drag_coeff[1] * ds * x.vy; F[2] += -P.drag_coeff[2] * ds * x.vz;
    }
    if (EFF & QS_EFFECT_DW) { F[0] += r02 * fz; F[1] += r12 * fz; F[2] += r22 * fz; }
    const double g21 = c.j[2] - c.j[1], g02 = c.j[0] - c.j[2], g10 = c.j[1] - c.j[0];
    const double tt[3] = {tx - g21 * (x.wy * x.wz), ty - g02 * (x.wz * x.wx), tz - g10 * (x.wx * x.wy)};
    const double wn[3] = {x.wx + dt * c.j_inv[0] * tt[0], x.wy + dt * c.j_inv[1] * tt[1], x.wz + dt * c.j_inv[2] * tt[2]};
    const double p = wn[0], q = wn[1], r = wn[2];
    double C, S, dC, dS;
    half_angle_grad(p * p + q * q + r * r, dt, C, S, dC, dS);
    // Omega(w) q of _integrateQ
    const double m0 = r * Y - q * Z + p * W, m1 = -r * X + p * Z + q * W, m2 = q * X - p * Y + r * W, m3 = -p * X - q * Y - r * Z;

    // ---- reverse ----
    const double Lq0 = L.qx, Lq1 = L.qy, Lq2 = L.qz, Lq3 = L.qw;
    // q' = C q + S Omega(w') q
    const double LC = Lq0 * X + Lq1 * Y + Lq2 * Z + Lq3 * W, LS = Lq0 * m0 + Lq1 * m1 + Lq2 * m2 + Lq3 * m3;
    const double k2 = 2.0 * (LC * dC + LS * dS);
    double Lw[3];
    Lw[0] = L.wx + k2 * p + S * (Lq0 * W + Lq1 * Z - Lq2 * Y - Lq3 * X);
    Lw[1] = L.wy + k2 * q + S * (-Lq0 * Z + Lq1 * W + Lq2 * X - Lq3 * Y);
    Lw[2] = L.wz + k2 * r + S * (Lq0 * Y - Lq1 * X + Lq2 * W - Lq3 * Z);
    double LX = C * Lq0 + S * (-r * Lq1 + q * Lq2 - p * Lq3);
    double LY = C * Lq1 + S * (r * Lq0 - p * Lq2 - q * Lq3);
    double LZ = C * Lq2 + S * (-q * Lq0 + p * Lq1 - r * Lq3);
    double LW = C * Lq3 + S * (p * Lq0 + q * Lq1 + r * Lq2);
    // p' = p + dt v'
    double Lv[3] = {L.vx + dt * L.px, L.vy + dt * L.py, L.vz + dt * L.pz};
    double Lpz = L.pz;
    // w' = w + dt J^-1 tt
    double Ltt[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) { Ltt[a] = dt * c.j_inv[a] * Lw[a]; G.g[9 + a] += dt * Lw[a] * tt[a]; }
    double Lwx = Lw[0] - g02 * x.wz * Ltt[1] - g10 * x.wy * Ltt[2];
    double Lwy = Lw[1] - g21 * x.wz * Ltt[0] - g10 * x.wx * Ltt[2];
    double Lwz = Lw[2] - g21 * x.wy * Ltt[0] - g02 * x.wx * Ltt[1];
    const double Lg21 = -(x.wy * x.wz) * Ltt[0], Lg02 = -(x.wz * x.wx) * Ltt[1], Lg10 = -(x.wx * x.wy) * Ltt[2];
    G.g[6] += Lg02 - Lg10; G.g[7] += Lg10 - Lg21; G.g[8] += Lg21 - Lg02;
    // v' = v + dt/M F
    const double LF[3] = {dt_m * Lv[0], dt_m * Lv[1], dt_m * Lv[2]};
    G.g[0] += dt * (Lv[0] * F[0] + Lv[1] * F[1] + Lv[2] * F[2]);
    G.g[1] -= LF[2];
    if (EFF & QS_EFFECT_DRAG) {
        Lds -= P.drag_coeff[0] * x.vx * LF[0] + P.drag_coeff[1] * x.vy * LF[1] + P.drag_coeff[2] * x.vz * LF[2];
        Lv[0] -= P.drag_coeff[0] * ds * LF[0]; Lv[1] -= P.drag_coeff[1] * ds * LF[1]; Lv[2] -= P.drag_coeff[2] * ds * LF[2];
    }
    const double LT = r02 * LF[0] + r12 * LF[1] + r22 * LF[2];
    if (EFF & QS_EFFECT_DW) *Lfz = LT;                    // F = R[:,2] (T + fz) - g e_z: fz's cotangent is the thrust's
    const double tf = (EFF & QS_EFFECT_DW) ? thrust + fz : thrust;
    double Lr02 = tf * LF[0], Lr12 = tf * LF[1], Lr22 = tf * LF[2], Lr20 = 0.0, Lr21 = 0.0;
    // forces and torques
    G.g[4] += Ltt[0] * sxf; G.g[5] += Ltt[1] * syf;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const double u2 = u[i] * u[i];
        const double Lfg = LT + c.kx * P.sx[i] * Ltt[0] + c.ky * P.sy[i] * Ltt[1];
        Lu[i] += 2.0 * u[i] * (c.kf * Lfg + c.km * P.sz[i] * Ltt[2]);
        G.g[2] += u2 * Lfg;
        G.g[3] += P.sz[i] * u2 * Ltt[2];
        if ((EFF & QS_EFFECT_GND) && up) {
            const double e = gcoef * (rr[i] * rr[i]);
            Lu[i] += 2.0 * u[i] * c.kf * e * Lfg;
            G.g[2] += u2 * e * Lfg;
            if (hz_live[i]) {
                const double Lhz = -(rr[i] / hh[i]) * (2.0 * u2 * c.kf * gcoef * rr[i] * Lfg);
                Lpz += Lhz;
                Lr20 += P.prop_xyz[i][0] * Lhz; Lr21 += P.prop_xyz[i][1] * Lhz; Lr22 += P.prop_xyz[i][2] * Lhz;
            }
        }
    }
    // the rotation entries as functions of the quaternion
    LX += 2.0 * (Z * Lr02 - W * Lr12 - 2.0 * X * Lr22 + Z * Lr20 + W * Lr21);
    LY += 2.0 * (W * Lr02 + Z * Lr12 - 2.0 * Y * Lr22 - W * Lr20 + Z * Lr21);
    LZ += 2.0 * (X * Lr02 + Y * Lr12 + X * Lr20 + Y * Lr21);
    LW += 2.0 * (Y * Lr02 - X * Lr12 - Y * Lr20 + X * Lr21);
    L.pz = Lpz;                                          // L.px, L.py pass through
    L.qx = LX; L.qy = LY; L.qz = LZ; L.qw = LW;
    L.vx = Lv[0]; L.vy = Lv[1]; L.vz = Lv[2];
    L.wx = Lwx; L.wy = Lwy; L.wz = Lwz;
}

// Records the end state of substeps 0 .. S-2 (the start states of substeps 1 .. S-1) during the recomputation.
template <class Rec>
struct RecordHook {
    Drone* d;
    Rec* rec;
    int last;
    QS_HD void operator()(int s) const { if (s < last) rec->store(s, *d); }
};

// The tick's entry renormalisation, as dyn_tick_k evaluates it
QS_HD void entry_normalise(Drone& d, double& inv) {
    const double n2 = quat_norm2(d.qx, d.qy, d.qz, d.qw);
#if defined(__CUDA_ARCH__)
    inv = rsqrt(n2);
#else
    inv = 1.0 / sqrt(n2);
#endif
    d.qx *= inv; d.qy *= inv; d.qz *= inv; d.qw *= inv;
}

// The VJP of entry_normalise at its output xn (inv = 1 / |q|): q_hat = q / |q| gives L_q = (L_hat - q_hat (q_hat . L_hat)) / |q|
QS_HD void entry_normalise_vjp(const Drone& xn, double inv, Drone& L) {
    const double dot = xn.qx * L.qx + xn.qy * L.qy + xn.qz * L.qz + xn.qw * L.qw;
    L.qx = (L.qx - xn.qx * dot) * inv; L.qy = (L.qy - xn.qy * dot) * inv;
    L.qz = (L.qz - xn.qz * dot) * inv; L.qw = (L.qw - xn.qw * dot) * inv;
}

// drag's sum of the rotor speeds over four clipped RPMs (rad/s), as dyn_tick_k evaluates it
QS_HD double drag_sum(const double r[4]) {
    const double kk = 2.0 * 3.14159265358979323846;
    return kk * r[0] / 60.0 + kk * r[1] / 60.0 + kk * r[2] / 60.0 + kk * r[3] / 60.0;
}

// Adjoint of dyn_tick_k<EFF>(P, c, d, u, up, 0, S, .) from the tick-start state d0 (as stored: before the entry renormalisation).
// L: in, the cotangent of the tick's end state; out, of d0.  Lu / Lup (drag's previous RPMs) / G accumulate.  `rec` holds S - 1
// drones: rec.store(s, d) / rec.load(s, d).
template <int EFF, class Rec>
QS_HD void dyn_tick_vjp(const QsParams& P, const PhysRow& c, const Drone& d0, const double u[4], const double up[4], int S, Rec& rec,
                        Drone& L, double Lu[4], double Lup[4], PhysGrad& G) {
    {
        Drone d = d0;
        double R_last[9];
        dyn_tick_k<EFF>(P, c, d, u, up, 0.0, S, R_last, RecordHook<Rec>{&d, &rec, S - 1});
    }
    Drone x0 = d0;
    double inv;
    entry_normalise(x0, inv);
    const double kk = 2.0 * 3.14159265358979323846;
    const double ds_prev = drag_sum(up), ds_cur = drag_sum(u);
    double Lds_prev = 0.0, Lds_cur = 0.0;
    for (int s = S - 1; s >= 0; --s) {
        Drone x;
        if (s == 0) x = x0; else rec.load(s - 1, x);
        substep_vjp<EFF>(P, c, x, u, s == 0 ? ds_prev : ds_cur, L, Lu, s == 0 ? Lds_prev : Lds_cur, G);
    }
    if (EFF & QS_EFFECT_DRAG) {
#pragma unroll
        for (int i = 0; i < 4; ++i) { Lup[i] += (kk / 60.0) * Lds_prev; Lu[i] += (kk / 60.0) * Lds_cur; }
    }
    entry_normalise_vjp(x0, inv, L);
}

// ---- downwash (DESIGN.md 4.5, downwash adjoint) -------------------------------------------------------------------------------
// An aviary tick with downwash runs its S substeps one dyn_tick_k<EFF>(., fz, 1, .) call at a time, fz = downwash_fz of the
// substep's start positions, so each substep renormalises the quaternion on entry and every drone's substep depends on the
// positions of its aviary.  The adjoint of substep s is two phases around a barrier: dw_substep_vjp (drone-local, fz held
// constant) gives lambda, the cotangent of the drone's fz; downwash_pos_vjp then adds the pair terms to the positions' cotangents
// from the lambdas of the whole aviary.

// Adjoint of one downwash substep from x as recorded (before its entry renormalisation), with clipped rpm u, drag sum ds and
// the pair force fz.  L: in, the cotangent of the end state; out, of x without the pair terms.  Lu / Lds / G accumulate.
// Returns lambda.
template <int EFF>
QS_HD double dw_substep_vjp(const QsParams& P, const PhysRow& c, const Drone& x, const double u[4], double ds, double fz, Drone& L,
                            double Lu[4], double& Lds, PhysGrad& G) {
    Drone xn = x;
    double inv, lam = 0.0;
    entry_normalise(xn, inv);
    substep_vjp<EFF>(P, c, xn, u, ds, L, Lu, Lds, G, fz, &lam);
    entry_normalise_vjp(xn, inv, L);                     // touches the quaternion only: the pair terms below touch positions only
    return lam;
}

// The pair terms of drone q's position cotangent: pos[3 (b + k) + c] are the positions of the aviary's D drones at the substep's
// start and lam[b + k] the cotangents of their fz.  For a receiver i and a source k, fz_i += p(z_k - z_i, (x_k - x_i)^2 +
// (y_k - y_i)^2) wherever downwash_acts holds (the forward's predicate and operands), so drone q gets -lam_q dp for the sources
// over it (its receiver terms, summed in drone order) and then +lam_i dp for the receivers under it (its source terms, in drone
// order).  No atomics: each drone sums its own terms.
QS_HD void downwash_pos_vjp(const QsParams& P, const double* pos, const double* lam, int b, int D, int q, Drone& L) {
    const double* pq = pos + 3 * (b + q);
    const double lq = lam[b + q];
    double gx = 0.0, gy = 0.0, gz = 0.0;
    for (int k = 0; k < D; ++k) {                        // q the receiver, k the source
        const double* pk = pos + 3 * (b + k);
        const double dz = pk[2] - pq[2];
        const double dx = pk[0] - pq[0], dy = pk[1] - pq[1];
        const double dxy2 = dx * dx + dy * dy;
        if (downwash_acts(dz, dxy2)) {
            double g_dz, g_dxy2;
            downwash_pair_grad(P, dz, dxy2, g_dz, g_dxy2);
            gx -= lq * (2.0 * dx * g_dxy2); gy -= lq * (2.0 * dy * g_dxy2); gz -= lq * g_dz;
        }
    }
    for (int k = 0; k < D; ++k) {                        // k the receiver, q the source
        const double* pk = pos + 3 * (b + k);
        const double dz = pq[2] - pk[2];
        const double dx = pq[0] - pk[0], dy = pq[1] - pk[1];
        const double dxy2 = dx * dx + dy * dy;
        if (downwash_acts(dz, dxy2)) {
            double g_dz, g_dxy2;
            downwash_pair_grad(P, dz, dxy2, g_dz, g_dxy2);
            const double lk = lam[b + k];
            gx += lk * (2.0 * dx * g_dxy2); gy += lk * (2.0 * dy * g_dxy2); gz += lk * g_dz;
        }
    }
    L.px += gx; L.py += gy; L.pz += gz;
}

// Lq += d rpy / d q ^T Lrpy for rpy = quat_to_euler<false>(q), on the forward's branch of the +-0.99999 gimbal guard
// (the controller's adjoint, pid_adjoint.cuh, and the policy loop's observation head, mlp_adjoint.cuh)
QS_HD void quat_to_euler_vjp(double qx, double qy, double qz, double qw, const double Lrpy[3], double Lq[4]) {
    const double sarg = -2.0 * (qx * qz - qw * qy);
    if (sarg <= -0.99999 || sarg >= 0.99999) {
        // roll and pitch are constants; yaw = 2 atan2(x, -y) or 2 atan2(-x, y): the same derivative
        const double r2 = qx * qx + qy * qy;
        Lq[0] += Lrpy[2] * (-2.0 * qy / r2);
        Lq[1] += Lrpy[2] * (2.0 * qx / r2);
    } else {
        const double ra = 2.0 * (qy * qz + qw * qx), rb = qw * qw - qx * qx - qy * qy + qz * qz;
        const double ya = 2.0 * (qx * qy + qw * qz), yb = qw * qw + qx * qx - qy * qy - qz * qz;
        const double n_r = ra * ra + rb * rb, n_y = ya * ya + yb * yb;
        const double Lra = Lrpy[0] * rb / n_r, Lrb = -Lrpy[0] * ra / n_r;
        const double Ls = Lrpy[1] / sqrt(1.0 - sarg * sarg);
        const double Lya = Lrpy[2] * yb / n_y, Lyb = -Lrpy[2] * ya / n_y;
        Lq[0] += 2.0 * (qw * Lra - qx * Lrb - qz * Ls + qy * Lya + qx * Lyb);
        Lq[1] += 2.0 * (qz * Lra - qy * Lrb + qw * Ls + qx * Lya - qy * Lyb);
        Lq[2] += 2.0 * (qy * Lra + qz * Lrb - qx * Ls + qw * Lya - qz * Lyb);
        Lq[3] += 2.0 * (qx * Lra + qw * Lrb + qy * Ls + qz * Lya + qw * Lyb);
    }
}

}  // namespace qs
