// TEST INFRASTRUCTURE: compiles gym_pybullet_drones_b200/csrc/dyn_tangent.cuh (the tick tangent of the JVP and Jacobian kernels,
// dyn_jvp.cu) as plain host C++, so the `-m "not gpu"` suite can hold one tick's tangent to the torch reference (tests/diff_ref.py
// under torch.func.jacfwd) and to the transpose of the host-built adjoint (diff_host.cpp).  A drone is 13 doubles: pos, quat
// (x, y, z, w), vel, rpy_rates.  Never linked into or imported by the product package.
#include "../../gym_pybullet_drones_b200/csrc/dyn_tangent.cuh"

namespace {
qs::PhysRow row_from(const QsParams& P, const double* r) {
    if (!r) return qs::phys_row_of(P);
    qs::PhysRow c;
    c.inv_m = r[0]; c.gravity = r[1]; c.kf = r[2]; c.km = r[3]; c.kx = r[4]; c.ky = r[5];
    for (int k = 0; k < 3; ++k) { c.j[k] = r[6 + k]; c.j_inv[k] = r[9 + k]; }
    c.hover_rpm = r[12]; c.max_rpm = r[13];
    return c;
}

qs::Drone drone_from(const double* s) {
    return qs::Drone{s[0], s[1], s[2], s[3], s[4], s[5], s[6], s[7], s[8], s[9], s[10], s[11], s[12]};
}
void drone_to(const qs::Drone& d, double* s) {
    const double v[13] = {d.px, d.py, d.pz, d.qx, d.qy, d.qz, d.qw, d.vx, d.vy, d.vz, d.wx, d.wy, d.wz};
    for (int k = 0; k < 13; ++k) s[k] = v[k];
}

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
    for (int i = 0; i < n; ++i) {
        const qs::PhysRow c = row_from(*P, rows ? rows + 16 * i : nullptr);
        qs::PhysRow tc = row_from(*P, t_rows + 16 * i);
        auto f = effects == 0 ? tick_jvp<0> : effects == QS_EFFECT_GND ? tick_jvp<QS_EFFECT_GND>
               : effects == QS_EFFECT_DRAG ? tick_jvp<QS_EFFECT_DRAG> : tick_jvp<3>;
        f(*P, c, tc, S, state + 13 * i, raw + 4 * i, up + 4 * i, t_state + 13 * i, t_raw + 4 * i, t_up + 4 * i, out + 13 * i,
          t_out + 13 * i);
    }
}
}
