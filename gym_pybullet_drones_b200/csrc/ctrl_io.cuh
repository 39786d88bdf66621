// ctrl_io.cuh -- what the closed-loop translation units (dyn_ctrl_traj.cu, dyn_ctrl_jvp.cu) share on top of traj_io.cuh: the
// aviary's gain set, the tick's targets and the controller call with the two max_rpm clips of the QS_CTRL_TRACK tick.  `Args`
// holds the controller's QsParams CP, the drones per aviary D and an io with gains, control_timestep and the target pointers.
#pragma once
#include "pid_adjoint.cuh"
#include "traj_io.cuh"

namespace qsi {
namespace {

// the 18 gains of one row of QsDynCtrlTrajIO.gains' layout
__device__ __forceinline__ qs::PidGains gains_row(const double* g) {
    qs::PidGains k;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        k.pid_p_for[c] = g[c]; k.pid_i_for[c] = g[3 + c]; k.pid_d_for[c] = g[6 + c];
        k.pid_p_tor[c] = g[9 + c]; k.pid_i_tor[c] = g[12 + c]; k.pid_d_tor[c] = g[15 + c];
    }
    return k;
}
// the gain set of drone i: its aviary's row of io.gains, or the controller's own
template <class Args>
__device__ __forceinline__ qs::PidGains gains_of(const Args& a, long long i) {
    if (!a.io.gains) return qs::pid_gains_of(a.CP);
    return gains_row(a.io.gains + 18 * (i / a.D));
}
__device__ __forceinline__ void ld3(const double* p, long long i, double v[3]) {
    if (p) { v[0] = p[3 * i]; v[1] = p[3 * i + 1]; v[2] = p[3 * i + 2]; } else { v[0] = v[1] = v[2] = 0.0; }
}
// the tick's targets of drone i from target_pos [T][N][3] and the constant target_vel / target_rpy (its yaw) / target_rpy_rates
// [N][3], each nullable = zeros
__device__ __forceinline__ qs::PidTargets targets_from(const double* tp, const double* tv, const double* trpy, const double* trr,
                                                       long long N, long long i, int k) {
    qs::PidTargets t;
    ld3(tp, (long long)k * N + i, t.tp);
    ld3(tv, i, t.tv);
    double r[3];
    ld3(trpy, i, r);
    t.tyaw = r[2];
    ld3(trr, i, t.trr);
    return t;
}
template <class IO>
__device__ __forceinline__ qs::PidTargets targets_of(const IO& io, long long N, long long i, int k) {
    return targets_from(io.target_pos, io.target_vel, io.target_rpy, io.target_rpy_rates, N, i, k);
}

// computeControlFromEnv + the two clips of the TRACK tick: the raw controller RPMs, the controller's clip u1, the applied u
template <class Args>
__device__ __forceinline__ void control(const Args& a, const qs::PidGains& K, qs::PidState& st, const qs::Drone& d,
                                        const qs::PidTargets& t, double mr, double raw[4], double u1[4], double u[4]) {
    double pe[3], ye;
    qs::pid_control_k(a.CP, K, st, a.io.control_timestep, d.px, d.py, d.pz, d.qx, d.qy, d.qz, d.qw, d.vx, d.vy, d.vz,
                      t.tp[0], t.tp[1], t.tp[2], t.tyaw, t.tv[0], t.tv[1], t.tv[2], t.trr[0], t.trr[1], t.trr[2], raw, pe, ye);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        u1[j] = qs::clampd(raw[j], 0.0, a.CP.max_rpm);
        u[j] = qs::clampd(u1[j], 0.0, mr);
    }
}

}  // namespace
}  // namespace qsi
