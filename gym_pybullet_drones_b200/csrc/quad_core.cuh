// quad_core.cuh -- per-drone math of the Physics.DYN hot path, written once and compiled both for the
// sm_90a kernels (quadsim.cu) and for the host-side unit harness (tests/host_harness).
//
// New implementation of the behaviour of (paths relative to gym_pybullet_drones/ in the reference):
//   envs/BaseAviary.py:815-892   _dynamics + _integrateQ
//   envs/BaseAviary.py:715-811   _groundEffect / _drag / _downwash force models (as explicit DYN+ terms)
//   envs/BaseRLAviary.py:160-239 action decoding
//   control/DSLPIDControl.py:82-259 cascaded PID
//   pybullet helpers getMatrixFromQuaternion / getEulerFromQuaternion (Bullet's published algorithm)
//
// Numerics: the reference is float64 end to end.  Here the state lives in HBM as float32 planes and is
// advanced in float64 registers; see DESIGN.md ("precision") for the measurements behind that choice.
#pragma once
#include <math.h>
#include "../../include/quadsim.h"

#if defined(__CUDACC__)
#define QS_HD __host__ __device__ __forceinline__
#else
#define QS_HD inline
#endif

namespace qs {

struct Drone {          // one drone's kinematic state in registers
    double px, py, pz;
    double qx, qy, qz, qw;   // Bullet order x,y,z,w
    double vx, vy, vz;
    double wx, wy, wz;       // body rates (`rpy_rates`)
};

struct Derived {        // outputs that are recomputed every tick, never fed back
    double roll, pitch, yaw;
    double ax, ay, az;       // ang_v = R_old * w_new  (BaseAviary.py:873)
};

// ---- float32 <-> float64 helpers -------------------------------------------------------------
// float32 product/sum with one rounding each and no FMA contraction: NumPy evaluates
// `1 + 0.05*action` on float32 actions in float32 (NEP 50 weak scalars; reference pins numpy ^2.2).
QS_HD float f32_mul(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    volatile float r = a * b; return r;
#endif
}
QS_HD float f32_add(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    volatile float r = a + b; return r;
#endif
}
QS_HD float f32_div(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fdiv_rn(a, b);
#else
    volatile float r = a / b; return r;
#endif
}
QS_HD float f32_sqrt(float a) {
#if defined(__CUDA_ARCH__)
    return __fsqrt_rn(a);
#else
    volatile float r = sqrtf(a); return r;
#endif
}

QS_HD double clampd(double v, double lo, double hi) { return v < lo ? lo : (v > hi ? hi : v); }

// |q|^2 with a fixed operation order and explicit fused multiply-adds (the library is built with -fmad=false, so nothing
// else is fused): the renormalised quaternion must be the same bits in every kernel that advances the state
QS_HD double quat_norm2(double x, double y, double z, double w) {
#if defined(__CUDA_ARCH__)
    return __fma_rn(w, w, __fma_rn(z, z, __fma_rn(y, y, __dmul_rn(x, x))));
#else
    return fma(w, w, fma(z, z, fma(y, y, x * x)));
#endif
}

// ---- Bullet quaternion helpers ---------------------------------------------------------------
// getMatrixFromQuaternion (btMatrix3x3::setRotation): row-major R, implicit normalisation by s = 2/|q|^2.
QS_HD void quat_to_matrix(double x, double y, double z, double w, double R[9]) {
    const double d = x * x + y * y + z * z + w * w;
    const double s = 2.0 / d;
    const double xs = x * s, ys = y * s, zs = z * s;
    const double wx = w * xs, wy = w * ys, wz = w * zs;
    const double xx = x * xs, xy = x * ys, xz = x * zs;
    const double yy = y * ys, yz = y * zs, zz = z * zs;
    R[0] = 1.0 - (yy + zz); R[1] = xy - wz;         R[2] = xz + wy;
    R[3] = xy + wz;         R[4] = 1.0 - (xx + zz); R[5] = yz - wx;
    R[6] = xz - wy;         R[7] = yz + wx;         R[8] = 1.0 - (xx + yy);
}

// the same for a quaternion that is unit to rounding (|q|^2 = 1 + e, |e| ~ 1e-15): s = 2/|q|^2 = 2(2 - |q|^2) + O(e^2), no division
QS_HD void quat_to_matrix_unit(double x, double y, double z, double w, double R[9]) {
    const double d = x * x + y * y + z * z + w * w;
    const double s = 2.0 * (2.0 - d);
    const double xs = x * s, ys = y * s, zs = z * s;
    const double wx = w * xs, wy = w * ys, wz = w * zs;
    const double xx = x * xs, xy = x * ys, xz = x * zs;
    const double yy = y * ys, yz = y * zs, zz = z * zs;
    R[0] = 1.0 - (yy + zz); R[1] = xy - wz;         R[2] = xz + wy;
    R[3] = xy + wz;         R[4] = 1.0 - (xx + zz); R[5] = yz - wx;
    R[6] = xz - wy;         R[7] = yz + wx;         R[8] = 1.0 - (xx + yy);
}

// getEulerFromQuaternion: ZYX roll/pitch/yaw with the +-0.99999 gimbal guard, no normalisation.
template <bool F32>
QS_HD void quat_to_euler(double x, double y, double z, double w, double& roll, double& pitch, double& yaw) {
    const double sqx = x * x, sqy = y * y, sqz = z * z, squ = w * w;
    const double sarg = -2.0 * (x * z - w * y);
    const double HALF_PI = 1.57079632679489661923;
    if (sarg <= -0.99999) {
        roll = 0.0; pitch = -HALF_PI;
        yaw = F32 ? 2.0 * (double)atan2f((float)x, (float)-y) : 2.0 * atan2(x, -y);
    } else if (sarg >= 0.99999) {
        roll = 0.0; pitch = HALF_PI;
        yaw = F32 ? 2.0 * (double)atan2f((float)-x, (float)y) : 2.0 * atan2(-x, y);
    } else if (F32) {
        roll = (double)atan2f((float)(2.0 * (y * z + w * x)), (float)(squ - sqx - sqy + sqz));
        pitch = (double)asinf((float)sarg);
        yaw = (double)atan2f((float)(2.0 * (x * y + w * z)), (float)(squ + sqx - sqy - sqz));
    } else {
        roll = atan2(2.0 * (y * z + w * x), squ - sqx - sqy + sqz);
        pitch = asin(sarg);
        yaw = atan2(2.0 * (x * y + w * z), squ + sqx - sqy - sqz);
    }
}

// cos(theta) and sin(theta)/|w| for theta = |w| dt/2, from n2 = |w|^2 -- both are even in theta, so for the
// small angles of a 240 Hz substep they are 5- or 8-term series in theta^2 (truncation < 2^-53 in both ranges):
// no sqrt, no division, no range reduction.  Large rates fall back to sqrt/sincos.
QS_HD void half_angle_terms(double n2, double dt, double& c, double& s_over_n) {
    const double h = 0.5 * dt;
    const double t = n2 * h * h;                 // theta^2
    if (t < 0.0078125) {
        // theta^2 < 1/128 (|w| < 42 rad/s at 240 Hz): 5 terms are exact to double rounding (next terms t^5/10! < 8e-18)
        double pc = 1.0 / 40320.0;                           // k=4  +1/8!
        pc = pc * t - 1.0 / 720.0;                           // k=3  -1/6!
        pc = pc * t + 1.0 / 24.0;                            // k=2  +1/4!
        pc = pc * t - 0.5;                                   // k=1  -1/2!
        c = pc * t + 1.0;                                    // k=0
        double ps = 1.0 / 362880.0;                          // k=4  +1/9!
        ps = ps * t - 1.0 / 5040.0;                          // k=3  -1/7!
        ps = ps * t + 1.0 / 120.0;                           // k=2  +1/5!
        ps = ps * t - 1.0 / 6.0;                             // k=1  -1/3!
        ps = ps * t + 1.0;                                   // k=0
        s_over_n = ps * h;
    } else if (t < 0.25) {
        // cos(theta) = sum_{k=0..7} (-1)^k t^k/(2k)!
        double pc = -1.0 / 87178291200.0;                    // k=7  -1/14!
        pc = pc * t + 1.0 / 479001600.0;                     // k=6  +1/12!
        pc = pc * t - 1.0 / 3628800.0;                       // k=5  -1/10!
        pc = pc * t + 1.0 / 40320.0;                         // k=4  +1/8!
        pc = pc * t - 1.0 / 720.0;                           // k=3  -1/6!
        pc = pc * t + 1.0 / 24.0;                            // k=2  +1/4!
        pc = pc * t - 0.5;                                   // k=1  -1/2!
        c = pc * t + 1.0;                                    // k=0
        // sinc(theta) = sum_{k=0..7} (-1)^k t^k/(2k+1)!
        double ps = -1.0 / 1307674368000.0;                  // k=7  -1/15!
        ps = ps * t + 1.0 / 6227020800.0;                    // k=6  +1/13!
        ps = ps * t - 1.0 / 39916800.0;                      // k=5  -1/11!
        ps = ps * t + 1.0 / 362880.0;                        // k=4  +1/9!
        ps = ps * t - 1.0 / 5040.0;                          // k=3  -1/7!
        ps = ps * t + 1.0 / 120.0;                           // k=2  +1/5!
        ps = ps * t - 1.0 / 6.0;                             // k=1  -1/3!
        ps = ps * t + 1.0;                                   // k=0
        s_over_n = ps * h;                                   // sin(theta)/|w| = (dt/2) sinc(theta)
    } else {
        const double n = sqrt(n2);
        const double th = n * h;
        c = cos(th);
        s_over_n = sin(th) / n;
    }
}

// _integrateQ (BaseAviary.py:879-892): q' = (cos(th) I + (sin(th)/|w|) Omega(w)) q, identity if np.isclose(|w|,0).
QS_HD void integrate_q(Drone& d, double dt) {
    const double p = d.wx, q = d.wy, r = d.wz;
    const double n2 = p * p + q * q + r * r;
    if (n2 <= 1e-16) return;                     // |w| <= 1e-8  == np.isclose(|w|, 0) (atol 1e-8)
    double c, s;
    half_angle_terms(n2, dt, c, s);
    const double x = d.qx, y = d.qy, z = d.qz, w = d.qw;
    d.qx = c * x + s * (r * y - q * z + p * w);
    d.qy = c * y + s * (-r * x + p * z + q * w);
    d.qz = c * z + s * (q * x - p * y + r * w);
    d.qw = c * w + s * (-p * x - q * y - r * z);
}

// ---- one control tick of Physics.DYN ----------------------------------------------------------
// `substeps` x _dynamics with constant rpm.  EFF = compile-time set of DYN+ terms.
// rpm_prev = last_clipped_action: drag uses the previous tick's rpm in substep 0 and the current rpm
// afterwards, because the reference refreshes last_clipped_action inside the substep loop (BaseAviary.py:372).
// dw_fz = downwash force along body z for this substep (host launches one substep per call when DW is on).
// `between` is called after every substep with its index (the fused kernels poll an asynchronous copy there).
struct NoHook { QS_HD void operator()(int) const {} };

// The drone's physical constants -- M (as 1/M), GRAVITY, KF, KM, the arm inside kx/ky, J, J^-1, HOVER_RPM, MAX_RPM -- come
// from `c`: the QsParams themselves (one drone for the whole batch), or the aviary's PhysRow when QsState.phys is set.
// Everything else (time step, mixing signs, DYN+ coefficients, task, embedded controller) always comes from P.
struct PhysRow { double inv_m, gravity, kf, km, kx, ky, j[3], j_inv[3], hover_rpm, max_rpm; };

template <int EFF, class K, class Hook = NoHook>
QS_HD void dyn_tick_k(const QsParams& P, const K& c, Drone& d, const double rpm[4], const double rpm_prev[4], double dw_fz,
                      int substeps, double R_last[9], Hook between = Hook()) {
    const double dt = P.dt;
    const double dt_m = dt * c.inv_m;                                                // v += dt * (F / M)  (:858,:860)
    double f[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) f[i] = rpm[i] * rpm[i] * c.kf;                       // :838
    // z torque (:842-845); sz carries the -1,+1,-1,+1 pattern (negated for RACE)
    const double zt0 = rpm[0] * rpm[0] * c.km, zt1 = rpm[1] * rpm[1] * c.km,
                 zt2 = rpm[2] * rpm[2] * c.km, zt3 = rpm[3] * rpm[3] * c.km;
    const double tz = P.sz[0] * zt0 + P.sz[1] * zt1 + P.sz[2] * zt2 + P.sz[3] * zt3;
    double thrust = f[0] + f[1] + f[2] + f[3];                                       // :839
    double tx = (P.sx[0] * f[0] + P.sx[1] * f[1] + P.sx[2] * f[2] + P.sx[3] * f[3]) * c.kx;   // :846-854
    double ty = (P.sy[0] * f[0] + P.sy[1] * f[1] + P.sy[2] * f[2] + P.sy[3] * f[3]) * c.ky;
    double drag_sum = 0.0;
    if (EFF & QS_EFFECT_DRAG) {                                                      // :773
        const double k = 2.0 * 3.14159265358979323846;
        drag_sum = k * rpm_prev[0] / 60.0 + k * rpm_prev[1] / 60.0 + k * rpm_prev[2] / 60.0 + k * rpm_prev[3] / 60.0;
    }
    // Unit quaternion on entry: the planes hold a float32-rounded unit quaternion (|q|^2 = 1 +- 1e-7); after this
    // |q|^2 - 1 ~ 1e-16 for the whole tick (_integrateQ is norm preserving), so Bullet's s = 2/|q|^2 is evaluated as
    // 2(2 - |q|^2), exact to (|q|^2-1)^2 -- one DFMA instead of a double-precision division per substep.
    {
        const double n2 = quat_norm2(d.qx, d.qy, d.qz, d.qw);
#if defined(__CUDA_ARCH__)
        const double inv = rsqrt(n2);
#else
        const double inv = 1.0 / sqrt(n2);
#endif
        d.qx *= inv; d.qy *= inv; d.qz *= inv; d.qw *= inv;
    }
    double q0x = d.qx, q0y = d.qy, q0z = d.qz, q0w = d.qw;                           // attitude at the start of the last substep
    // per-tick constants of the Euler step: dt*J^-1, the gyroscopic differences (w x Jw for a diagonal J), dt/M*gravity
    const double dj0 = dt * c.j_inv[0], dj1 = dt * c.j_inv[1], dj2 = dt * c.j_inv[2];
    const double g21 = c.j[2] - c.j[1], g02 = c.j[0] - c.j[2], g10 = c.j[1] - c.j[0];
    const double gm = dt_m * c.gravity;
    const double tm2 = 2.0 * (dt_m * thrust), tmg = dt_m * thrust - gm;             // EFF == 0: thrust is constant over the tick
    for (int s = 0; s < substeps; ++s) {
        q0x = d.qx; q0y = d.qy; q0z = d.qz; q0w = d.qw;
        const double x = d.qx, y = d.qy, z = d.qz, w = d.qw;
        // Bullet's s = 2/|q|^2 (:836): |q|^2 = 1 to 1e-16 for the whole tick (unit on entry, _integrateQ is norm preserving)
        double r02 = 0.0, r12 = 0.0, r22 = 0.0, xs = 0.0, ys = 0.0, zs = 0.0;
        if (EFF != 0) {
            xs = x + x; ys = y + y; zs = z + z;
            // third column and third row of R
            r02 = x * zs + w * ys; r12 = y * zs - w * xs; r22 = 1.0 - (x * xs + y * ys);
        }
        if (EFF & QS_EFFECT_GND) {                                                   // :715-750 on the substep-start state
            const double r20 = x * zs - w * ys, r21 = y * zs + w * xs;
            const double sarg = -2.0 * (x * z - w * y);
            const double ra = 2.0 * (y * z + w * x);
            const double rb = w * w - x * x - y * y + z * z;
            // |roll| < pi/2 and |pitch| < pi/2 (:742) without trig: roll = atan2(ra, rb), pitch = asin(sarg) w/ guard
            const bool upright = (sarg > -0.99999) && (sarg < 0.99999) && (rb > 0.0 || (rb == 0.0 && ra == 0.0));
            double g[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const double hz = d.pz + r20 * P.prop_xyz[i][0] + r21 * P.prop_xyz[i][1] + r22 * P.prop_xyz[i][2];
                const double h = hz < P.gnd_eff_h_clip ? P.gnd_eff_h_clip : hz;       // :739-740
                const double rr = P.prop_radius / (4.0 * h);
                g[i] = upright ? rpm[i] * rpm[i] * c.kf * P.gnd_eff_coeff * (rr * rr) : 0.0;   // :741
            }
            const double f0 = f[0] + g[0], f1 = f[1] + g[1], f2 = f[2] + g[2], f3 = f[3] + g[3];
            thrust = f0 + f1 + f2 + f3;
            tx = (P.sx[0] * f0 + P.sx[1] * f1 + P.sx[2] * f2 + P.sx[3] * f3) * c.kx;
            ty = (P.sy[0] * f0 + P.sy[1] * f1 + P.sy[2] * f2 + P.sy[3] * f3) * c.ky;
        }
        if (EFF == 0) {
            // v += dt (R[:,2] thrust - [0,0,GRAVITY]) / M   (:840-841,:858,:860) with R[:,2] = (2(xz+wy), 2(yz-wx), 1-2(xx+yy)):
            // the factor 2 rides on the per-tick constant, the column itself is never formed (10 instead of 14 operations)
            d.vx = d.vx + (x * z + w * y) * tm2;
            d.vy = d.vy + (y * z - w * x) * tm2;
            d.vz = (d.vz + tmg) - (x * x + y * y) * tm2;
        } else {
            double fx = r02 * thrust, fy = r12 * thrust, fz = r22 * thrust - c.gravity;  // :840-841
            if (EFF & QS_EFFECT_DRAG) {                                                  // world force = -DRAG_COEFF*sum (.) vel
                fx += (-1.0 * P.drag_coeff[0] * drag_sum) * d.vx;
                fy += (-1.0 * P.drag_coeff[1] * drag_sum) * d.vy;
                fz += (-1.0 * P.drag_coeff[2] * drag_sum) * d.vz;
                if (s == 0) {
                    const double k = 2.0 * 3.14159265358979323846;
                    drag_sum = k * rpm[0] / 60.0 + k * rpm[1] / 60.0 + k * rpm[2] / 60.0 + k * rpm[3] / 60.0;
                }
            }
            if (EFF & QS_EFFECT_DW) { fx += r02 * dw_fz; fy += r12 * dw_fz; fz += r22 * dw_fz; }
            d.vx = d.vx + dt_m * fx;                                                     // :858,:860
            d.vy = d.vy + dt_m * fy;
            d.vz = d.vz + dt_m * fz;
        }
        // w' = J^-1 (torques - w x (J w))  (:856-857); for the diagonal J: (w x Jw)_x = (Jz - Jy) wy wz, cyclic
        const double ttx = tx - g21 * (d.wy * d.wz);
        const double tty = ty - g02 * (d.wz * d.wx);
        const double ttz = tz - g10 * (d.wx * d.wy);
        d.wx = d.wx + dj0 * ttx;                                                     // :861
        d.wy = d.wy + dj1 * tty;
        d.wz = d.wz + dj2 * ttz;
        d.px = d.px + dt * d.vx;                                                     // :862
        d.py = d.py + dt * d.vy;
        d.pz = d.pz + dt * d.vz;
        integrate_q(d, dt);                                                          // :863
        between(s);
    }
    quat_to_matrix_unit(q0x, q0y, q0z, q0w, R_last);                                 // R used by :873 (ang_v = R_old w_new)
}

template <int EFF, class Hook = NoHook>
QS_HD void dyn_tick(const QsParams& P, Drone& d, const double rpm[4], const double rpm_prev[4], double dw_fz,
                    int substeps, double R_last[9], Hook between = Hook()) {
    dyn_tick_k<EFF>(P, P, d, rpm, rpm_prev, dw_fz, substeps, R_last, between);
}

template <bool RPY_F32>
QS_HD void derive(const Drone& d, const double R_last[9], Derived& o) {
    quat_to_euler<RPY_F32>(d.qx, d.qy, d.qz, d.qw, o.roll, o.pitch, o.yaw);          // :518
    o.ax = R_last[0] * d.wx + R_last[1] * d.wy + R_last[2] * d.wz;                   // :873
    o.ay = R_last[3] * d.wx + R_last[4] * d.wy + R_last[5] * d.wz;
    o.az = R_last[6] * d.wx + R_last[7] * d.wy + R_last[8] * d.wz;
}

// ---- DSLPIDControl -----------------------------------------------------------------------------
struct PidState { double ipx, ipy, ipz, lr, lp, ly, irx, iry, irz; };   // integral_pos_e, last_rpy, integral_rpy_e

// computeControl (control/DSLPIDControl.py:82-145).  Returns rpm[4], pos_e[3], yaw_e; updates st.
QS_HD void pid_control(const QsParams& P, PidState& st, double dt,
                       double px, double py, double pz, double qx, double qy, double qz, double qw,
                       double vx, double vy, double vz,
                       double tpx, double tpy, double tpz, double tyaw,
                       double tvx, double tvy, double tvz, double trr0, double trr1, double trr2,
                       double rpm[4], double pos_e[3], double& yaw_e) {
    double R[9];
    quat_to_matrix(qx, qy, qz, qw, R);                                               // :187
    const double ex = tpx - px, ey = tpy - py, ez = tpz - pz;                        // :188
    const double evx = tvx - vx, evy = tvy - vy, evz = tvz - vz;                     // :189
    st.ipx = clampd(st.ipx + ex * dt, -2.0, 2.0);                                    // :190-191
    st.ipy = clampd(st.ipy + ey * dt, -2.0, 2.0);
    st.ipz = clampd(clampd(st.ipz + ez * dt, -2.0, 2.0), -0.15, 0.15);               // :192
    double ttx = P.pid_p_for[0] * ex + P.pid_i_for[0] * st.ipx + P.pid_d_for[0] * evx;          // :194-196
    double tty = P.pid_p_for[1] * ey + P.pid_i_for[1] * st.ipy + P.pid_d_for[1] * evy;
    double ttz = P.pid_p_for[2] * ez + P.pid_i_for[2] * st.ipz + P.pid_d_for[2] * evz + P.pid_gravity;
    double scalar = ttx * R[2] + tty * R[5] + ttz * R[8];                            // :197
    if (scalar < 0.0) scalar = 0.0;
    const double thrust = (sqrt(scalar / (4.0 * P.pid_kf)) - P.pid_pwm2rpm_const) / P.pid_pwm2rpm_scale;   // :198
    const double tn = sqrt(ttx * ttx + tty * tty + ttz * ttz);
    const double zx = ttx / tn, zy = tty / tn, zz = ttz / tn;                        // :199
    const double cx = cos(tyaw), cy = sin(tyaw);                                     // :200 (x_c = [cos, sin, 0])
    double yx = zy * 0.0 - zz * cy, yy = zz * cx - zx * 0.0, yz = zx * cy - zy * cx; // z_ax x x_c
    const double yn = sqrt(yx * yx + yy * yy + yz * yz);
    yx /= yn; yy /= yn; yz /= yn;                                                    // :201
    const double xx = yy * zz - yz * zy, xy = yz * zx - yx * zz, xz = yx * zy - yy * zx;   // y x z (:202)
    // target_rotation columns = [x_ax y_ax z_ax] (:203): Rd[r][c]
    const double Rd[9] = {xx, yx, zx, xy, yy, zy, xz, yz, zz};
    // The reference converts Rd to intrinsic-XYZ Euler angles (scipy as_euler('XYZ'), :205) and, in the attitude loop,
    // straight back to a matrix (from_euler('XYZ').as_quat() -> from_quat().as_matrix(), :242-244).  That round trip is
    // the identity on rotation matrices (also in gimbal lock, where only the angle split is ambiguous), so the target
    // rotation used below IS Rd; of the three angles only c = atan2(-Rd[0][1], Rd[0][0]) is ever consumed (yaw error, :145).
    const double ec = atan2(-Rd[1], Rd[0]);
    pos_e[0] = ex; pos_e[1] = ey; pos_e[2] = ez;
    const double* T = Rd;
    double roll, pitch, yaw;
    quat_to_euler<false>(qx, qy, qz, qw, roll, pitch, yaw);                          // :241
    // E = T^T R - R^T T ; rot_e = (E[2][1], E[0][2], E[1][0])  (:245-246)
    #define QS_TtR(i, k) (T[0 + i] * R[0 + k] + T[3 + i] * R[3 + k] + T[6 + i] * R[6 + k])
    #define QS_RtT(i, k) (R[0 + i] * T[0 + k] + R[3 + i] * T[3 + k] + R[6 + i] * T[6 + k])
    const double rex = QS_TtR(2, 1) - QS_RtT(2, 1);
    const double rey = QS_TtR(0, 2) - QS_RtT(0, 2);
    const double rez = QS_TtR(1, 0) - QS_RtT(1, 0);
    #undef QS_TtR
    #undef QS_RtT
    const double rrx = trr0 - (roll - st.lr) / dt;                                   // :247 (no angle unwrap)
    const double rry = trr1 - (pitch - st.lp) / dt;
    const double rrz = trr2 - (yaw - st.ly) / dt;
    st.lr = roll; st.lp = pitch; st.ly = yaw;                                        // :248
    st.irx = clampd(clampd(st.irx - rex * dt, -1500.0, 1500.0), -1.0, 1.0);          // :249-251
    st.iry = clampd(clampd(st.iry - rey * dt, -1500.0, 1500.0), -1.0, 1.0);
    st.irz = clampd(st.irz - rez * dt, -1500.0, 1500.0);
    double q0 = -P.pid_p_tor[0] * rex + P.pid_d_tor[0] * rrx + P.pid_i_tor[0] * st.irx;      // :253-255
    double q1 = -P.pid_p_tor[1] * rey + P.pid_d_tor[1] * rry + P.pid_i_tor[1] * st.iry;
    double q2 = -P.pid_p_tor[2] * rez + P.pid_d_tor[2] * rrz + P.pid_i_tor[2] * st.irz;
    q0 = clampd(q0, -3200.0, 3200.0); q1 = clampd(q1, -3200.0, 3200.0); q2 = clampd(q2, -3200.0, 3200.0);   // :256
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        double pwm = thrust + (P.pid_mixer[i][0] * q0 + P.pid_mixer[i][1] * q1 + P.pid_mixer[i][2] * q2);   // :257
        pwm = clampd(pwm, P.pid_min_pwm, P.pid_max_pwm);                             // :258
        rpm[i] = P.pid_pwm2rpm_scale * pwm + P.pid_pwm2rpm_const;                    // :259
    }
    yaw_e = ec - yaw;                                                                // :145
}

// ---- action decoding (BaseRLAviary._preprocessAction, envs/BaseRLAviary.py:160-239) -----------------
// `a` = this drone's float32 action; `der` = the cached kinematics the reference reads through
// _getDroneStateVector (rpy from the end of the previous tick).  PID variants update `pst`.
// HOVER_RPM and MAX_RPM come from `c` (see dyn_tick_k); the embedded controller keeps P's constants (BaseRLAviary.py:76).
template <bool PIDACT, class K>
QS_HD void decode_action_k(const QsParams& P, const K& c, int act_type, const float a[4], const Drone& d, double cur_yaw,
                           PidState& pst, double rpm[4]) {
    if (act_type == QS_ACT_RPM) {                                                    // :192
#pragma unroll
        for (int i = 0; i < 4; ++i) rpm[i] = c.hover_rpm * (double)f32_add(1.0f, f32_mul(0.05f, a[i]));
    } else if (act_type == QS_ACT_ONE_D_RPM) {                                       // :225
        const double v = c.hover_rpm * (double)f32_add(1.0f, f32_mul(0.05f, a[0]));
        rpm[0] = rpm[1] = rpm[2] = rpm[3] = v;
    } else if (act_type == QS_ACT_RAW_RPM) {                                         // CtrlAviary.py:140
#pragma unroll
        for (int i = 0; i < 4; ++i) rpm[i] = clampd((double)a[i], 0.0, c.max_rpm);
    } else if (PIDACT) {
        double tpx, tpy, tpz, tyaw = 0.0, tvx = 0.0, tvy = 0.0, tvz = 0.0;
        if (act_type == QS_ACT_PID) {                                                // :194-207, _calculateNextStep :1108-1150
            const double dx = (double)a[0] - d.px, dy = (double)a[1] - d.py, dz = (double)a[2] - d.pz;
            const double dist = sqrt(dx * dx + dy * dy + dz * dz);
            if (dist <= 1.0) { tpx = (double)a[0]; tpy = (double)a[1]; tpz = (double)a[2]; }
            else { tpx = d.px + dx / dist * 1.0; tpy = d.py + dy / dist * 1.0; tpz = d.pz + dz / dist * 1.0; }
        } else if (act_type == QS_ACT_VEL) {                                         // :209-223 (float32 arithmetic on the action)
            tpx = d.px; tpy = d.py; tpz = d.pz; tyaw = cur_yaw;
            const float n = f32_sqrt(f32_add(f32_add(f32_mul(a[0], a[0]), f32_mul(a[1], a[1])), f32_mul(a[2], a[2])));
            float ux = 0.f, uy = 0.f, uz = 0.f;
            if (n != 0.f) { ux = f32_div(a[0], n); uy = f32_div(a[1], n); uz = f32_div(a[2], n); }
            const float sp = f32_mul((float)P.speed_limit, fabsf(a[3]));
            tvx = (double)f32_mul(sp, ux); tvy = (double)f32_mul(sp, uy); tvz = (double)f32_mul(sp, uz);
        } else {                                                                     // ONE_D_PID :227-235
            tpx = d.px + 0.1 * 0.0; tpy = d.py + 0.1 * 0.0; tpz = d.pz + 0.1 * (double)a[0];
        }
        double pe[3], ye;
        pid_control(P, pst, P.ctrl_dt, d.px, d.py, d.pz, d.qx, d.qy, d.qz, d.qw, d.vx, d.vy, d.vz,
                    tpx, tpy, tpz, tyaw, tvx, tvy, tvz, 0.0, 0.0, 0.0, rpm, pe, ye);
    }
}

template <bool PIDACT>
QS_HD void decode_action(const QsParams& P, int act_type, const float a[4], const Drone& d, double cur_yaw,
                         PidState& pst, double rpm[4]) {
    decode_action_k<PIDACT>(P, P, act_type, a, d, cur_yaw, pst, rpm);
}

// ---- task: Hover / MultiHover per-drone terms ----------------------------------------------------
struct TaskTerms { double reward, dist; bool out_of_bounds; };

QS_HD TaskTerms hover_terms(const QsParams& P, const Drone& d, const Derived& o, double tx, double ty, double tz) {
    const double ex = tx - d.px, ey = ty - d.py, ez = tz - d.pz;
    const double n = sqrt(ex * ex + ey * ey + ez * ez);                              // HoverAviary.py:77
    const double n2 = n * n;
    TaskTerms t;
    const double r = 2.0 - n2 * n2;
    t.reward = r > 0.0 ? r : 0.0;                                                    // max(0, 2 - |e|^4)
    t.dist = n;
    t.out_of_bounds = fabs(d.px) > P.xy_bound || fabs(d.py) > P.xy_bound || d.pz > P.z_bound ||
                      fabs(o.roll) > P.tilt_bound || fabs(o.pitch) > P.tilt_bound;   // HoverAviary.py:109-111
    return t;
}

// ---- downwash pair term (BaseAviary.py:798-803) ----------------------------------------------------
QS_HD double downwash_pair(const QsParams& P, double dz, double dxy2) {
    // caller guarantees dz > 0 and dxy2 < 100
    const double rr = P.prop_radius / (4.0 * dz);
    const double alpha = P.dw_coeff[0] * (rr * rr);
    const double beta = P.dw_coeff[1] * dz + P.dw_coeff[2];
    const double u = sqrt(dxy2) / beta;
    return -alpha * exp(-0.5 * (u * u));
}

}  // namespace qs
