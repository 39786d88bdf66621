// TEST INFRASTRUCTURE: what the host harnesses of the differentiable trajectories (diff_host.cpp, diff_ctrl_host.cpp,
// diff_policy_host.cpp, jvp_host.cpp) share.  A drone is 13 doubles: pos, quat (x, y, z, w), vel, rpy_rates; a row is the 16
// doubles of QsState.phys.  Never linked into or imported by the product package.
#pragma once
#include <type_traits>
#include <vector>
#include "../../gym_pybullet_drones_b200/csrc/dyn_adjoint.cuh"

namespace {
// the substep record of the tick adjoint, in host memory
struct HostRec {
    std::vector<qs::Drone> v;
    void store(int s, const qs::Drone& d) { v[s] = d; }
    void load(int s, qs::Drone& d) const { d = v[s]; }
};

// the constants of a row, or where r is NULL the constants of P
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

// f(std::integral_constant<int, EFF>{}) for the effect set `effects`: 0, GND, DRAG or GND|DRAG
template <class F>
void with_effects(unsigned effects, F&& f) {
    if (effects == 0) f(std::integral_constant<int, 0>{});
    else if (effects == QS_EFFECT_GND) f(std::integral_constant<int, QS_EFFECT_GND>{});
    else if (effects == QS_EFFECT_DRAG) f(std::integral_constant<int, QS_EFFECT_DRAG>{});
    else f(std::integral_constant<int, QS_EFFECT_GND | QS_EFFECT_DRAG>{});
}
}  // namespace
