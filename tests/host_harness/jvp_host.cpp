// TEST INFRASTRUCTURE: compiles gym_pybullet_drones_b200/csrc/dyn_tangent.cuh (the tick tangent of the JVP and Jacobian kernels,
// dyn_jvp.cu) as plain host C++, so the `-m "not gpu"` suite can hold one tick's tangent to the torch reference (tests/diff_ref.py
// under torch.func.jacfwd) and to the transpose of the host-built adjoint (diff_host.cpp).  A drone is 13 doubles: pos, quat
// (x, y, z, w), vel, rpy_rates.  Never linked into or imported by the product package.
#include "../../gym_pybullet_drones_b200/csrc/dyn_tangent.cuh"
#include "harness.h"

namespace {
template <int EFF>
void tick_jvp(const QsParams& P, const qs::PhysRow& c, const qs::PhysRow& tc, int S, const double* state, const double* raw,
              const double* up, const double* t_state, const double* t_raw, const double* t_up, double* out, double* t_out) {
    double u[4], tu[4];
    for (int j = 0; j < 4; ++j) u[j] = qs::clampd(raw[j], 0.0, c.max_rpm);
    qs::rpm_clip_jvp(raw, c.max_rpm, t_raw, tc.max_rpm, tu);
    qs::Drone d = drone_from(state), t = drone_from(t_state);
    qs::dyn_tick_jvp<EFF>(P, c, tc, d, u, up, S, t, tu, t_up);
    drone_to(d, out);
    drone_to(t, t_out);
}
}  // namespace

extern "C" {
// One control tick and its tangent for n drones: state [n][13], raw rpm (unclipped) [n][4], up = drag's previous clipped rpm
// [n][4], rows [n][16] (nullable = QsParams' constants) and the tangents t_state [n][13], t_raw [n][4], t_up [n][4], t_rows
// [n][16] -> out [n][13] (the end state, before store_drone's rounding), t_out [n][13].  effects: 0, GND, DRAG or GND|DRAG.
void jh_tick_jvp(const QsParams* P, const double* rows, unsigned effects, int S, int n, const double* state, const double* raw,
                 const double* up, const double* t_state, const double* t_raw, const double* t_up, const double* t_rows, double* out,
                 double* t_out) {
    with_effects(effects, [&](auto EFF) {
        for (int i = 0; i < n; ++i)
            tick_jvp<decltype(EFF)::value>(*P, row_from(*P, rows ? rows + 16 * i : nullptr), row_from(*P, t_rows + 16 * i), S, state + 13 * i,
                                           raw + 4 * i, up + 4 * i, t_state + 13 * i, t_raw + 4 * i, t_up + 4 * i, out + 13 * i, t_out + 13 * i);
    });
}
}
