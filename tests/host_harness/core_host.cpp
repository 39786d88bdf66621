// TEST INFRASTRUCTURE: compiles gym_pybullet_drones_b200/csrc/quad_core.cuh (the per-drone math of the CUDA
// kernels) as plain host C++ so the `-m "not gpu"` suite can check the same source against the oracle before
// any GPU time is spent.  It keeps the kernel's state layout: float64 planes ([pos|w.x] [quat] [vel|w.y] of [n][4], then
// w.z [n]) loaded into registers, one control tick, quaternion renormalised, stored back.
// Never linked into or imported by the product package.
#include <cmath>
#include <cstring>
#include "../../gym_pybullet_drones_b200/csrc/quad_core.cuh"

namespace {
void load(const double* planes, long long N, long long i, qs::Drone& d) {
    const double* p0 = planes + 4 * i; const double* p1 = planes + 4 * (N + i); const double* p2 = planes + 4 * (2 * N + i);
    d.px = p0[0]; d.py = p0[1]; d.pz = p0[2];
    d.qx = p1[0]; d.qy = p1[1]; d.qz = p1[2]; d.qw = p1[3];
    d.vx = p2[0]; d.vy = p2[1]; d.vz = p2[2];
    d.wx = p0[3]; d.wy = p2[3]; d.wz = planes[12 * N + i];
}
void store(double* planes, long long N, long long i, qs::Drone& d) {
    const double inv = 1.0 / std::sqrt(qs::quat_norm2(d.qx, d.qy, d.qz, d.qw));
    d.qx *= inv; d.qy *= inv; d.qz *= inv; d.qw *= inv;
    double* p0 = planes + 4 * i; double* p1 = planes + 4 * (N + i); double* p2 = planes + 4 * (2 * N + i);
    p0[0] = d.px; p0[1] = d.py; p0[2] = d.pz; p0[3] = d.wx;
    p1[0] = d.qx; p1[1] = d.qy; p1[2] = d.qz; p1[3] = d.qw;
    p2[0] = d.vx; p2[1] = d.vy; p2[2] = d.vz; p2[3] = d.wy;
    planes[12 * N + i] = d.wz;
}
template <int EFF>
void tick_all(const QsParams& P, double* planes, int n, const float* act, int A, int act_type, int substeps,
              double* last_rpm, double* pid, double* rec) {
    for (long long i = 0; i < n; ++i) {
        qs::Drone d; load(planes, n, i, d);
        float a[4] = {0, 0, 0, 0};
        for (int k = 0; k < A; ++k) a[k] = act[i * A + k];
        qs::PidState ps = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        if (pid) { ps.ipx = pid[i]; ps.ipy = pid[n + i]; ps.ipz = pid[2 * n + i]; ps.lr = pid[3 * n + i]; ps.lp = pid[4 * n + i];
                   ps.ly = pid[5 * n + i]; ps.irx = pid[6 * n + i]; ps.iry = pid[7 * n + i]; ps.irz = pid[8 * n + i]; }
        double rpm[4], rpm_prev[4] = {last_rpm[4 * i], last_rpm[4 * i + 1], last_rpm[4 * i + 2], last_rpm[4 * i + 3]};
        double yaw = 0, r_, p_;
        if (act_type == QS_ACT_VEL) qs::quat_to_euler<false>(d.qx, d.qy, d.qz, d.qw, r_, p_, yaw);
        qs::decode_action<true>(P, act_type, a, d, yaw, ps, rpm);
        double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
        qs::dyn_tick<EFF>(P, d, rpm, rpm_prev, 0.0, substeps, R);
        qs::Derived o; qs::derive<false>(d, R, o);
        store(planes, n, i, d);
        for (int k = 0; k < 4; ++k) last_rpm[4 * i + k] = rpm[k];
        if (pid) { pid[i] = ps.ipx; pid[n + i] = ps.ipy; pid[2 * n + i] = ps.ipz; pid[3 * n + i] = ps.lr;
                   pid[4 * n + i] = ps.lp; pid[5 * n + i] = ps.ly; pid[6 * n + i] = ps.irx; pid[7 * n + i] = ps.iry; pid[8 * n + i] = ps.irz; }
        if (rec) {
            double* r = rec + i * 23;
            r[0] = d.px; r[1] = d.py; r[2] = d.pz; r[3] = d.qx; r[4] = d.qy; r[5] = d.qz; r[6] = d.qw;
            r[7] = o.roll; r[8] = o.pitch; r[9] = o.yaw; r[10] = d.vx; r[11] = d.vy; r[12] = d.vz;
            r[13] = o.ax; r[14] = o.ay; r[15] = o.az; r[16] = d.wx; r[17] = d.wy; r[18] = d.wz;
            r[19] = rpm[0]; r[20] = rpm[1]; r[21] = rpm[2]; r[22] = rpm[3];
        }
    }
}
}  // namespace

extern "C" {
// one control tick for n independent drones; rec = [n][23] float64 (pos3 quat4 rpy3 vel3 ang_v3 w3 rpm4) or NULL
void hh_tick(const QsParams* P, double* planes, int n, const float* act, int A, int act_type, int substeps, unsigned effects,
             double* last_rpm, double* pid, double* rec) {
    switch (effects & 3u) {
        case 0: tick_all<0>(*P, planes, n, act, A, act_type, substeps, last_rpm, pid, rec); break;
        case 1: tick_all<1>(*P, planes, n, act, A, act_type, substeps, last_rpm, pid, rec); break;
        case 2: tick_all<2>(*P, planes, n, act, A, act_type, substeps, last_rpm, pid, rec); break;
        case 3: tick_all<3>(*P, planes, n, act, A, act_type, substeps, last_rpm, pid, rec); break;
    }
}
// DSLPIDControl.computeControl on float64 inputs; st = [9] float64 state in/out
void hh_pid(const QsParams* P, double* st, double dt, const double* pos, const double* quat, const double* vel,
            const double* tpos, double tyaw, const double* tvel, const double* trr, double* rpm, double* pos_e, double* yaw_e) {
    qs::PidState s = {st[0], st[1], st[2], st[3], st[4], st[5], st[6], st[7], st[8]};
    qs::pid_control(*P, s, dt, pos[0], pos[1], pos[2], quat[0], quat[1], quat[2], quat[3], vel[0], vel[1], vel[2],
                    tpos[0], tpos[1], tpos[2], tyaw, tvel[0], tvel[1], tvel[2], trr[0], trr[1], trr[2], rpm, pos_e, *yaw_e);
    st[0] = s.ipx; st[1] = s.ipy; st[2] = s.ipz; st[3] = s.lr; st[4] = s.lp; st[5] = s.ly; st[6] = s.irx; st[7] = s.iry; st[8] = s.irz;
}
// getEulerFromQuaternion of the kernels for n quaternions [n][4] (x,y,z,w) -> rpy [n][3]; f32 = the RPY_F32 variant
void hh_quat_to_euler(const double* q, int n, int f32, double* rpy) {
    for (int i = 0; i < n; ++i) {
        const double* v = q + 4 * i; double* r = rpy + 3 * i;
        if (f32) qs::quat_to_euler<true>(v[0], v[1], v[2], v[3], r[0], r[1], r[2]);
        else qs::quat_to_euler<false>(v[0], v[1], v[2], v[3], r[0], r[1], r[2]);
    }
}
// the ground-effect switch of dyn_tick_k on n quaternions -> out[n] (0/1)
void hh_upright(const double* q, int n, unsigned char* out) {
    for (int i = 0; i < n; ++i) {
        const double x = q[4 * i], y = q[4 * i + 1], z = q[4 * i + 2], w = q[4 * i + 3];
        out[i] = qs::upright(-2.0 * (x * z - w * y), 2.0 * (y * z + w * x), w * w - x * x - y * y + z * z) ? 1 : 0;
    }
}
// hover_terms on n drones: pos [n][3], quat [n][4], target [n][3]; the task's angles come from derive<f32> as in the kernels.
// out [n][5]: reward, dist, out_of_bounds, roll, pitch (the angles the kernel reports)
void hh_hover_terms(const QsParams* P, const double* pos, const double* quat, const double* tgt, int n, int f32, double* out) {
    const double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    for (int i = 0; i < n; ++i) {
        qs::Drone d = {pos[3 * i], pos[3 * i + 1], pos[3 * i + 2], quat[4 * i], quat[4 * i + 1], quat[4 * i + 2], quat[4 * i + 3],
                       0, 0, 0, 0, 0, 0};
        qs::Derived o;
        if (f32) qs::derive<true>(d, R, o); else qs::derive<false>(d, R, o);
        const qs::TaskTerms t = qs::hover_terms(*P, d, o, tgt[3 * i], tgt[3 * i + 1], tgt[3 * i + 2]);
        double* r = out + 5 * i;
        r[0] = t.reward; r[1] = t.dist; r[2] = t.out_of_bounds ? 1.0 : 0.0; r[3] = o.roll; r[4] = o.pitch;
    }
}
double hh_downwash_pair(const QsParams* P, double dz, double dxy2) { return qs::downwash_pair(*P, dz, dxy2); }
int hh_downwash_acts(double dz, double dxy2) { return qs::downwash_acts(dz, dxy2); }
double hh_downwash_fz(const QsParams* P, const double* pos, int b, int D, double px, double py, double pz) {
    return qs::downwash_fz(*P, pos, b, D, px, py, pz);
}
void hh_half_angle(double n2, double dt, double* c, double* s) { qs::half_angle_terms(n2, dt, *c, *s); }
}
