// TEST INFRASTRUCTURE: compiles gym_pybullet_drones_b200/csrc/pid_tangent.cuh with dyn_tangent.cuh (the closed-loop tick tangent
// of the JVP and Jacobian kernels, dyn_ctrl_jvp.cu) as plain host C++, so the `-m "not gpu"` suite can hold one closed-loop
// tick's tangent to the torch reference (tests/diff_pid_ref.py + tests/diff_ref.py under torch.func.jacfwd) and to the transpose
// of the host-built closed-loop adjoint (diff_ctrl_host.cpp).  One tick is the kernel's: pid_control_k, the controller's max_rpm
// clip, the env's clip, dyn_tick_k.  Never linked into or imported by the product package.
#include "../../gym_pybullet_drones_b200/csrc/pid_tangent.cuh"
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
qs::PidTargets targets_from(const double* tg) {
    return qs::PidTargets{{tg[0], tg[1], tg[2]}, tg[3], {tg[4], tg[5], tg[6]}, {tg[7], tg[8], tg[9]}};
}

template <int EFF>
void ctrl_tick_jvp(const QsParams& P, const QsParams& CP, const double* row, const double* gains, int S, double dt, const double* state,
                   const double* pid, const double* tg, const double* up, const double* t_row, const double* t_gains,
                   const double* t_state, const double* t_pid, const double* t_tg, const double* t_up, double* out, double* u_out,
                   double* pid_out, double* t_out, double* t_u_out, double* t_pid_out) {
    const qs::PhysRow c = row_from(P, row), tc = row_from(P, t_row);
    const qs::PidGains K = gains_from(gains), tK = gains_from(t_gains);
    qs::Drone d = drone_from(state), td = drone_from(t_state);
    const qs::PidState st0 = pid_from(pid);
    const qs::PidTargets t = targets_from(tg), t_t = targets_from(t_tg);
    // forward, as dyn_ctrl_traj_kernel
    qs::PidState st = st0;
    double raw[4], u1[4], u[4], pe[3], ye;
    qs::pid_control_k(CP, K, st, dt, d.px, d.py, d.pz, d.qx, d.qy, d.qz, d.qw, d.vx, d.vy, d.vz,
                      t.tp[0], t.tp[1], t.tp[2], t.tyaw, t.tv[0], t.tv[1], t.tv[2], t.trr[0], t.trr[1], t.trr[2], raw, pe, ye);
    for (int j = 0; j < 4; ++j) { u1[j] = qs::clampd(raw[j], 0.0, CP.max_rpm); u[j] = qs::clampd(u1[j], 0.0, c.max_rpm); }
    pid_to(st, pid_out);
    // tangent, as dyn_ctrl_jvp.cu's ctrl_tick_jvp
    double t_raw[4], t_u1[4], t_u[4];
    qs::PidState t_st;
    qs::pid_control_jvp(CP, K, st0, dt, d, t, tK, pid_from(t_pid), td, t_t, t_raw, t_st);
    qs::rpm_clip_jvp(raw, CP.max_rpm, t_raw, 0.0, t_u1);
    qs::rpm_clip_jvp(u1, c.max_rpm, t_u1, tc.max_rpm, t_u);
    qs::dyn_tick_jvp<EFF>(P, c, tc, d, u, up, S, td, t_u, t_up);
    drone_to(d, out);
    drone_to(td, t_out);
    pid_to(t_st, t_pid_out);
    for (int j = 0; j < 4; ++j) { u_out[j] = u[j]; t_u_out[j] = t_u[j]; }
}
}  // namespace

extern "C" {
// One closed-loop tick and its tangent for n drones.  Per drone: row [16], gains [18], state [13], pid [9], targets [10]
// (target_pos, target yaw, target_vel, target_rpy_rates), up = drag's previous applied rpm [4], and a tangent of each in the
// same layout.  Out: the end state [13] (before store_drone's rounding), the applied rpm [4], the updated controller state [9]
// and their tangents.
void cj_ctrl_tick_jvp(const QsParams* P, const QsParams* CP, unsigned effects, int S, double dt, int n, const double* rows,
                      const double* gains, const double* state, const double* pid, const double* tg, const double* up,
                      const double* t_rows, const double* t_gains, const double* t_state, const double* t_pid, const double* t_tg,
                      const double* t_up, double* out, double* u_out, double* pid_out, double* t_out, double* t_u, double* t_pid_out) {
    with_effects(effects, [&](auto EFF) {
        for (int i = 0; i < n; ++i)
            ctrl_tick_jvp<decltype(EFF)::value>(*P, *CP, rows + 16 * i, gains + 18 * i, S, dt, state + 13 * i, pid + 9 * i, tg + 10 * i,
                                                up + 4 * i, t_rows + 16 * i, t_gains + 18 * i, t_state + 13 * i, t_pid + 9 * i,
                                                t_tg + 10 * i, t_up + 4 * i, out + 13 * i, u_out + 4 * i, pid_out + 9 * i,
                                                t_out + 13 * i, t_u + 4 * i, t_pid_out + 9 * i);
    });
}
}
