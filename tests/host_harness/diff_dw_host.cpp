// TEST INFRASTRUCTURE: compiles the downwash adjoint of dyn_adjoint.cuh (dw_substep_vjp, downwash_pos_vjp, quad_core.cuh's
// downwash_pair_grad) and the substeps of dyn_dw_traj.cu as plain host C++, phase by phase, where the kernels place a barrier
// between two phases and the harness finishes a phase for every drone of the aviary before the next one.  The `-m "not gpu"`
// suite holds one aviary tick's VJP to the torch reference (tests/diff_dw_ref.py).  A drone is 13 doubles: pos, quat (x, y, z,
// w), vel, rpy_rates.  Never linked into or imported by the product package.
#include <cmath>
#include <vector>
#include "harness.h"

namespace {
template <int EFF>
void aviary_tick_vjp(const QsParams& P, const std::vector<qs::PhysRow>& c, int S, int D, const double* state, const double* raw,
                     const double* up, const double* g_out, double* out, double* g_state, double* g_raw, double* g_up, double* g_row) {
    std::vector<double> u(4 * D), pos(3 * D), lam(D);
    for (int q = 0; q < D; ++q)
        for (int j = 0; j < 4; ++j) u[4 * q + j] = qs::clampd(raw[4 * q + j], 0.0, c[q].max_rpm);
    std::vector<qs::Drone> d0(D), d(D);
    std::vector<HostRec> rec(D);
    for (int q = 0; q < D; ++q) {
        d0[q] = d[q] = drone_from(state + 13 * q);
        rec[q].v.resize(S > 1 ? S - 1 : 1);
    }
    // the forward: dyn_dw_traj.cu's dw_tick, recording each substep's end state (the VJP's recomputation)
    for (int s = 0; s < S; ++s) {
        for (int q = 0; q < D; ++q) { pos[3 * q] = d[q].px; pos[3 * q + 1] = d[q].py; pos[3 * q + 2] = d[q].pz; }
        for (int q = 0; q < D; ++q) {
            const double fz = qs::downwash_fz(P, pos.data(), 0, D, d[q].px, d[q].py, d[q].pz);
            double rp[4], R_last[9];
            for (int j = 0; j < 4; ++j) rp[j] = s == 0 ? up[4 * q + j] : u[4 * q + j];
            qs::dyn_tick_k<EFF>(P, c[q], d[q], &u[4 * q], rp, fz, 1, R_last);
            if (s < S - 1) rec[q].store(s, d[q]);
        }
    }
    // the reverse: dw_tick_vjp
    std::vector<qs::Drone> L(D);
    std::vector<qs::PhysGrad> G(D);
    std::vector<double> Lu(4 * D, 0.0), Lup(4 * D, 0.0), Lds_prev(D, 0.0), Lds_cur(D, 0.0);
    for (int q = 0; q < D; ++q) {
        drone_to(d[q], out + 13 * q);
        L[q] = drone_from(g_out + 13 * q);
        for (int j = 0; j < 16; ++j) G[q].g[j] = 0.0;
    }
    for (int s = S - 1; s >= 0; --s) {
        std::vector<qs::Drone> x(D);
        for (int q = 0; q < D; ++q) {
            x[q] = d0[q];
            if (s > 0) rec[q].load(s - 1, x[q]);
            pos[3 * q] = x[q].px; pos[3 * q + 1] = x[q].py; pos[3 * q + 2] = x[q].pz;
        }
        for (int q = 0; q < D; ++q) {
            const double fz = qs::downwash_fz(P, pos.data(), 0, D, x[q].px, x[q].py, x[q].pz);
            const double ds = qs::drag_sum(s == 0 ? up + 4 * q : &u[4 * q]);
            lam[q] = qs::dw_substep_vjp<EFF>(P, c[q], x[q], &u[4 * q], ds, fz, L[q], &Lu[4 * q], s == 0 ? Lds_prev[q] : Lds_cur[q], G[q]);
        }
        for (int q = 0; q < D; ++q) qs::downwash_pos_vjp(P, pos.data(), lam.data(), 0, D, q, L[q]);
    }
    const double kk = 2.0 * 3.14159265358979323846;
    for (int q = 0; q < D; ++q) {
        if (EFF & QS_EFFECT_DRAG)
            for (int j = 0; j < 4; ++j) { Lup[4 * q + j] += (kk / 60.0) * Lds_prev[q]; Lu[4 * q + j] += (kk / 60.0) * Lds_cur[q]; }
        qs::rpm_clip_vjp(raw + 4 * q, c[q].max_rpm, &Lu[4 * q], g_raw + 4 * q, G[q].g[13]);
        drone_to(L[q], g_state + 13 * q);
        for (int j = 0; j < 4; ++j) g_up[4 * q + j] = Lup[4 * q + j];
        for (int j = 0; j < 16; ++j) g_row[16 * q + j] = G[q].g[j];
    }
}
}  // namespace

extern "C" {
// One aviary tick of D drones with downwash and its VJP, per drone: state [D][13], raw rpm (unclipped) [D][4], up = drag's
// previous clipped rpm [D][4], rows [D][16] (nullable = QsParams' constants), g_out [D][13] -> out [D][13] (the end state, before
// round_to_planes), g_state [D][13], g_raw [D][4], g_up [D][4], g_row [D][16].  effects: DW or GND|DRAG|DW.
void ddh_tick_vjp(const QsParams* P, const double* rows, unsigned effects, int S, int D, const double* state, const double* raw,
                  const double* up, const double* g_out, double* out, double* g_state, double* g_raw, double* g_up, double* g_row) {
    std::vector<qs::PhysRow> c(D);
    for (int q = 0; q < D; ++q) c[q] = row_from(*P, rows ? rows + 16 * q : nullptr);
    if (effects == QS_EFFECT_DW)
        aviary_tick_vjp<QS_EFFECT_DW>(*P, c, S, D, state, raw, up, g_out, out, g_state, g_raw, g_up, g_row);
    else
        aviary_tick_vjp<QS_EFFECT_GND | QS_EFFECT_DRAG | QS_EFFECT_DW>(*P, c, S, D, state, raw, up, g_out, out, g_state, g_raw, g_up,
                                                                        g_row);
}
// downwash_pair_grad for n pairs (dz, dxy2) that act: out [n][2] = (dp/d(dz), dp/d(dxy2))
void ddh_pair_grad(const QsParams* P, const double* dz, const double* dxy2, int n, double* out) {
    for (int i = 0; i < n; ++i) qs::downwash_pair_grad(*P, dz[i], dxy2[i], out[2 * i], out[2 * i + 1]);
}
}
