// TEST INFRASTRUCTURE: compiles gym_pybullet_drones_b200/csrc/pid_adjoint.cuh with quad_core.cuh's pid_control_k and
// dyn_adjoint.cuh (the code of the closed-loop differentiable-trajectory kernels, dyn_ctrl_traj.cu) as plain host C++, so the
// `-m "not gpu"` suite can hold one closed-loop tick's VJP to the torch reference (tests/diff_pid_ref.py).  One tick is the
// kernel's: pid_control_k, the controller's max_rpm clip, the env's clip, dyn_tick_k; its VJP is the kernel's backward step.
// Never linked into or imported by the product package.
#include <cmath>
#include "../../gym_pybullet_drones_b200/csrc/pid_adjoint.cuh"
#include "harness.h"

namespace {
qs::PidGains gains_from(const double* g) {
    qs::PidGains k;
    for (int a = 0; a < 3; ++a) {
        k.pid_p_for[a] = g[a]; k.pid_i_for[a] = g[3 + a]; k.pid_d_for[a] = g[6 + a];
        k.pid_p_tor[a] = g[9 + a]; k.pid_i_tor[a] = g[12 + a]; k.pid_d_tor[a] = g[15 + a];
    }
    return k;
}
qs::PidState pid_from(const double* s) { return qs::PidState{s[0], s[1], s[2], s[3], s[4], s[5], s[6], s[7], s[8]}; }
void pid_to(const qs::PidState& p, double* s) {
    const double v[9] = {p.ipx, p.ipy, p.ipz, p.lr, p.lp, p.ly, p.irx, p.iry, p.irz};
    for (int k = 0; k < 9; ++k) s[k] = v[k];
}

template <int EFF>
void ctrl_tick_vjp(const QsParams& P, const QsParams& CP, const double* row, const double* gains, int S, double dt,
                   const double* state, const double* pid, const double* tg, const double* up, const double* g_out,
                   const double* g_rpm, const double* g_pid, double* out, double* u_out, double* pid_out, double* g_state,
                   double* g_pid0, double* g_tg, double* g_up, double* g_row, double* g_gains) {
    const qs::PhysRow c = row_from(P, row);
    const qs::PidGains K = gains_from(gains);
    const qs::Drone d0 = drone_from(state);
    const qs::PidState st0 = pid_from(pid);
    const qs::PidTargets t = {{tg[0], tg[1], tg[2]}, tg[3], {tg[4], tg[5], tg[6]}, {tg[7], tg[8], tg[9]}};
    // forward, as dyn_ctrl_traj_kernel
    qs::PidState st = st0;
    double raw[4], u1[4], u[4], pe[3], ye;
    qs::pid_control_k(CP, K, st, dt, d0.px, d0.py, d0.pz, d0.qx, d0.qy, d0.qz, d0.qw, d0.vx, d0.vy, d0.vz,
                      t.tp[0], t.tp[1], t.tp[2], t.tyaw, t.tv[0], t.tv[1], t.tv[2], t.trr[0], t.trr[1], t.trr[2], raw, pe, ye);
    for (int j = 0; j < 4; ++j) { u1[j] = qs::clampd(raw[j], 0.0, CP.max_rpm); u[j] = qs::clampd(u1[j], 0.0, c.max_rpm); }
    qs::Drone d = d0;
    double R_last[9];
    qs::dyn_tick_k<EFF>(P, c, d, u, up, 0.0, S, R_last);
    drone_to(d, out);
    for (int j = 0; j < 4; ++j) u_out[j] = u[j];
    pid_to(st, pid_out);
    // backward, as one step of dyn_ctrl_traj_vjp_kernel
    HostRec rec;
    rec.v.resize(S > 1 ? S - 1 : 1);
    qs::Drone L = drone_from(g_out);
    double Lu[4] = {g_rpm[0], g_rpm[1], g_rpm[2], g_rpm[3]}, Lup[4] = {0, 0, 0, 0};
    qs::PhysGrad G;
    for (int j = 0; j < 16; ++j) G.g[j] = 0.0;
    qs::dyn_tick_vjp<EFF>(P, c, d0, u, up, S, rec, L, Lu, Lup, G);
    double Lu1[4], Lraw[4], g_cmax = 0.0;
    qs::rpm_clip_vjp(u1, c.max_rpm, Lu, Lu1, G.g[13]);
    qs::rpm_clip_vjp(raw, CP.max_rpm, Lu1, Lraw, g_cmax);
    qs::PidState Ls = pid_from(g_pid);
    qs::PidTargets Lt = {{0, 0, 0}, 0, {0, 0, 0}, {0, 0, 0}};
    for (int j = 0; j < 18; ++j) g_gains[j] = 0.0;
    qs::pid_control_vjp(CP, K, st0, dt, d0, t, Lraw, Ls, L, Lt, g_gains);
    drone_to(L, g_state);
    pid_to(Ls, g_pid0);
    const double lt[10] = {Lt.tp[0], Lt.tp[1], Lt.tp[2], Lt.tyaw, Lt.tv[0], Lt.tv[1], Lt.tv[2], Lt.trr[0], Lt.trr[1], Lt.trr[2]};
    for (int j = 0; j < 10; ++j) g_tg[j] = lt[j];
    for (int j = 0; j < 4; ++j) g_up[j] = Lup[j];
    for (int j = 0; j < 16; ++j) g_row[j] = G.g[j];
}
}  // namespace

extern "C" {
// One closed-loop tick and its VJP for n drones.  Per drone: row [16], gains [18], state [13], pid [9], targets [10] (target_pos,
// target yaw, target_vel, target_rpy_rates), up = drag's previous applied rpm [4]; cotangents g_out [13] (end state), g_rpm [4]
// (applied rpm), g_pid [9] (updated controller state).  Out: the end state [13] (before store_drone's rounding), the applied rpm
// [4], the updated controller state [9], and the gradients of state [13], pid [9], targets [10], up [4], row [16], gains [18].
void dh_ctrl_tick_vjp(const QsParams* P, const QsParams* CP, unsigned effects, int S, double dt, int n, const double* rows,
                      const double* gains, const double* state, const double* pid, const double* tg, const double* up,
                      const double* g_out, const double* g_rpm, const double* g_pid, double* out, double* u_out, double* pid_out,
                      double* g_state, double* g_pid0, double* g_tg, double* g_up, double* g_row, double* g_gains) {
    with_effects(effects, [&](auto EFF) {
        for (int i = 0; i < n; ++i)
            ctrl_tick_vjp<decltype(EFF)::value>(*P, *CP, rows + 16 * i, gains + 18 * i, S, dt, state + 13 * i, pid + 9 * i, tg + 10 * i,
                                                up + 4 * i, g_out + 13 * i, g_rpm + 4 * i, g_pid + 9 * i, out + 13 * i, u_out + 4 * i,
                                                pid_out + 9 * i, g_state + 13 * i, g_pid0 + 9 * i, g_tg + 10 * i, g_up + 4 * i,
                                                g_row + 16 * i, g_gains + 18 * i);
    });
}
}
