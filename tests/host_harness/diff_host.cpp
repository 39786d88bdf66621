// TEST INFRASTRUCTURE: compiles gym_pybullet_drones_b200/csrc/dyn_adjoint.cuh and quad_core.cuh's dyn_tick_k (the code of the
// differentiable-trajectory kernels, dyn_traj.cu) as plain host C++, so the `-m "not gpu"` suite can hold one tick's VJP to the
// torch reference (tests/diff_ref.py).  A drone is 13 doubles: pos, quat (x, y, z, w), vel, rpy_rates.  Never linked into or
// imported by the product package.
#include <cmath>
#include "../../gym_pybullet_drones_b200/csrc/dyn_adjoint.cuh"
#include "harness.h"

namespace {
template <int EFF>
void tick_vjp(const QsParams& P, const qs::PhysRow& c, int S, const double* state, const double* raw, const double* up,
              const double* g_out, double* out, double* g_state, double* g_raw, double* g_up, double* g_row) {
    double u[4];
    for (int j = 0; j < 4; ++j) u[j] = qs::clampd(raw[j], 0.0, c.max_rpm);
    const qs::Drone d0 = drone_from(state);
    qs::Drone d = d0;
    double R_last[9];
    qs::dyn_tick_k<EFF>(P, c, d, u, up, 0.0, S, R_last);
    drone_to(d, out);
    HostRec rec;
    rec.v.resize(S > 1 ? S - 1 : 1);
    qs::Drone L = drone_from(g_out);
    double Lu[4] = {0, 0, 0, 0}, Lup[4] = {0, 0, 0, 0};
    qs::PhysGrad G;
    for (int j = 0; j < 16; ++j) G.g[j] = 0.0;
    qs::dyn_tick_vjp<EFF>(P, c, d0, u, up, S, rec, L, Lu, Lup, G);
    qs::rpm_clip_vjp(raw, c.max_rpm, Lu, g_raw, G.g[13]);
    drone_to(L, g_state);
    for (int j = 0; j < 4; ++j) g_up[j] = Lup[j];
    for (int j = 0; j < 16; ++j) g_row[j] = G.g[j];
}
}  // namespace

extern "C" {
// One control tick and its VJP for n drones: state [n][13], raw rpm (unclipped) [n][4], up = drag's previous clipped rpm [n][4],
// rows [n][16] (nullable = QsParams' constants), g_out [n][13] -> out [n][13] (the end state, before store_drone's rounding),
// g_state [n][13], g_raw [n][4], g_up [n][4], g_row [n][16].  effects: 0, GND, DRAG or GND|DRAG.
void dh_tick_vjp(const QsParams* P, const double* rows, unsigned effects, int S, int n, const double* state, const double* raw,
                 const double* up, const double* g_out, double* out, double* g_state, double* g_raw, double* g_up, double* g_row) {
    with_effects(effects, [&](auto EFF) {
        for (int i = 0; i < n; ++i)
            tick_vjp<decltype(EFF)::value>(*P, row_from(*P, rows ? rows + 16 * i : nullptr), S, state + 13 * i, raw + 4 * i, up + 4 * i,
                                           g_out + 13 * i, out + 13 * i, g_state + 13 * i, g_raw + 4 * i, g_up + 4 * i, g_row + 16 * i);
    });
}
// half_angle_grad: c, s, dc/dn2, ds/dn2 for n values of n2
void dh_half_angle_grad(const double* n2, int n, double dt, double* out) {
    for (int i = 0; i < n; ++i) qs::half_angle_grad(n2[i], dt, out[4 * i], out[4 * i + 1], out[4 * i + 2], out[4 * i + 3]);
}
}
