// TEST INFRASTRUCTURE: compiles gym_pybullet_drones_b200/csrc/lqr_law.cuh (the tracker's law and its adjoint) with dyn_adjoint.cuh
// (the tick, its adjoint and the RPM clip's) as plain host C++, so the `-m "not gpu"` suite can hold one tracker tick's VJP to the
// torch reference (tests/ilqr_tracker_ref.py + tests/diff_ref.py).  One tick is dyn_lqr_traj.cu's: dz, the law, the optional box,
// the env's clip, dyn_tick_k; its VJP is the kernel's backward step.  Never linked into or imported by the product package.
#include <cmath>
#include "../../gym_pybullet_drones_b200/csrc/lqr_law.cuh"
#include "harness.h"

namespace {
// one drone's plan tick in host arrays, as lqr_law.cuh's tracker reads it
template <int NZ>
struct HostPlan {
    const double *z_nom, *k, *rpm_nom, *lo, *hi;
    double zn(int q) const { return z_nom[q]; }
    double K(int j, int q) const { return k[j * NZ + q]; }
    void nom(double b[4]) const {
        for (int j = 0; j < 4; ++j) b[j] = rpm_nom[j];
    }
    bool box(double l[4], double h[4]) const {
        if (!lo) return false;
        for (int j = 0; j < 4; ++j) { l[j] = lo[j]; h[j] = hi[j]; }
        return true;
    }
};

template <int EFF, int NZ>
void lqr_tick_vjp(const QsParams& P, const double* row, int S, const double* state, const double* up, const double* rpm_nom,
                  const double* K, const double* z_nom, const double* lo, const double* hi, const double* g_out, const double* g_rpm,
                  double* out, double* u_out, double* g_state, double* g_up, double* g_row, double* g_rpm_nom, double* g_K,
                  double* g_z_nom) {
    const qs::PhysRow c = row_from(P, row);
    const qs::Drone d0 = drone_from(state);
    // forward, as one tick of dyn_lqr_traj_kernel: the shared tracker_command, then the env's clip
    const HostPlan<NZ> pl = {z_nom, K, rpm_nom, lo, hi};
    double b[4], u[4];
    bool keep[4];
    qsi::tracker_command<NZ>(pl, d0, up, b, keep);
    for (int j = 0; j < 4; ++j) u[j] = qs::clampd(b[j], 0.0, c.max_rpm);
    qs::Drone d = d0;
    double R_last[9];
    qs::dyn_tick_k<EFF>(P, c, d, u, up, 0.0, S, R_last);
    drone_to(d, out);
    for (int j = 0; j < 4; ++j) u_out[j] = u[j];
    // backward, as one step of dyn_lqr_traj_vjp_kernel
    HostRec rec;
    rec.v.resize(S > 1 ? S - 1 : 1);
    qs::Drone L = drone_from(g_out);
    double Lu[4] = {g_rpm[0], g_rpm[1], g_rpm[2], g_rpm[3]}, Lup[4] = {0, 0, 0, 0};
    qs::PhysGrad G;
    for (int j = 0; j < 16; ++j) G.g[j] = 0.0;
    qs::dyn_tick_vjp<EFF>(P, c, d0, u, up, S, rec, L, Lu, Lup, G);
    double lam[4], dz[NZ], Ktl[NZ];
    qsi::tracker_dz<NZ>(pl, d0, up, dz);
    qs::rpm_clip_vjp(b, c.max_rpm, Lu, lam, G.g[13]);
    for (int j = 0; j < 4; ++j) lam[j] = keep[j] ? lam[j] : 0.0;
    qsi::lqr_feedback_vjp<NZ>([&](int j, int q) { return pl.K(j, q); }, dz, lam, [&](int j, int q, double g) { g_K[j * NZ + q] = g; },
                              Ktl);
    double gs[13];
    drone_to(L, gs);
    for (int q = 0; q < 13; ++q) g_state[q] = gs[q] + Ktl[q];
    for (int j = 0; j < 4; ++j) g_up[j] = Lup[j];
    if constexpr (NZ == 17) {
        for (int j = 0; j < 4; ++j) g_up[j] += Ktl[13 + j];
    }
    for (int q = 0; q < NZ; ++q) g_z_nom[q] = -Ktl[q];
    for (int j = 0; j < 4; ++j) g_rpm_nom[j] = lam[j];
    for (int j = 0; j < 16; ++j) g_row[j] = G.g[j];
}
}  // namespace

extern "C" {
// One tracker tick and its VJP for n drones.  Per drone: row [16], state [13], up = the RPMs applied at the tick before [4] (drag's
// and dz's), rpm_nom [4], K [4][nz], z_nom [nz], lo / hi [4] (both NULL: no box); cotangents g_out [13] (end state) and g_rpm [4]
// (applied RPMs).  Out: the end state [13] (before the quaternion rounding of the store), the applied RPMs [4], and the gradients
// of state [13], up [4], row [16], rpm_nom [4], K [4][nz], z_nom [nz].
void lh_tick_vjp(const QsParams* P, unsigned effects, int S, int nz, int n, const double* rows, const double* state, const double* up,
                 const double* rpm_nom, const double* K, const double* z_nom, const double* lo, const double* hi, const double* g_out,
                 const double* g_rpm, double* out, double* u_out, double* g_state, double* g_up, double* g_row, double* g_rpm_nom,
                 double* g_K, double* g_z_nom) {
    with_effects(effects, [&](auto EFF) {
        for (int i = 0; i < n; ++i) {
            auto one = [&](auto NZ) {
                constexpr int Z = decltype(NZ)::value;
                lqr_tick_vjp<decltype(EFF)::value, Z>(*P, rows + 16 * i, S, state + 13 * i, up + 4 * i, rpm_nom + 4 * i, K + 4 * Z * i,
                                                      z_nom + Z * i, lo ? lo + 4 * i : nullptr, hi ? hi + 4 * i : nullptr, g_out + 13 * i,
                                                      g_rpm + 4 * i, out + 13 * i, u_out + 4 * i, g_state + 13 * i, g_up + 4 * i,
                                                      g_row + 16 * i, g_rpm_nom + 4 * i, g_K + 4 * Z * i, g_z_nom + Z * i);
            };
            if (nz == 17) one(std::integral_constant<int, 17>{});
            else one(std::integral_constant<int, 13>{});
        }
    });
}
}
