// TEST INFRASTRUCTURE: compiles the control-limited backward tick of gym_pybullet_drones_b200/csrc/riccati.cuh (the phases of
// qs_ilqr_box_backward, ilqr.cu) as plain host C++, so the `-m "not gpu"` suite can hold the box QP to float64 references
// (tests/ilqr_box_ref.py) and the device to the host bit for bit.  The phases run column by column in the order of the kernel's
// lanes.  Never linked into or imported by the product package.
#include <vector>
#include "../../gym_pybullet_drones_b200/csrc/riccati.cuh"

namespace {
template <int NZ>
int pass(int T, const double* F, const double* dx, const double* W, const double* Rt, const double* du, const double* lo,
         const double* hi, double mu, double* V, double* vx, double* K, double* k, double* dV, int* act) {
    constexpr int M = NZ + 4;
    std::vector<double> buf(qs::RicWs<NZ>::DOUBLES, 0.0);
    const qs::RicWs<NZ> w = qs::ric_ws<NZ>(buf.data());
    for (int j = 0; j < NZ * NZ; ++j) w.V[j] = V[j];
    for (int j = 0; j < NZ; ++j) w.vx[j] = vx[j];
    double d1 = 0.0, d2 = 0.0;
    for (int t = T - 1; t >= 0; --t) {
        for (int j = 0; j < 13; ++j) qs::ric_stage(w, j, dx[13 * t + j], W[13 * t + j]);
        for (int j = 0; j < NZ * M; ++j) w.F[j] = F[(long long)NZ * M * t + j];
        for (int j = 0; j < M; ++j) qs::ric_col_H(w, j);
        qs::RicBoxGains G;
        if (!qs::ric_gains_box(w, Rt, du + 4 * t, lo + 4 * t, hi + 4 * t, mu, G, d1, d2)) return t + 1;
        for (int j = 0; j < NZ; ++j) qs::ric_col_K_box(w, j, G);
        for (int j = 0; j < NZ; ++j) qs::ric_col_V(w, j, G);
        for (int j = 0; j < 4 * NZ; ++j) K[4 * NZ * t + j] = w.K[j];
        for (int j = 0; j < 4; ++j) {
            k[4 * t + j] = G.k[j];
            act[4 * t + j] = G.act[j];
        }
        for (int j = 0; j < NZ; ++j) qs::ric_col_sym(w, j);
    }
    for (int j = 0; j < NZ * NZ; ++j) V[j] = w.V[j];
    for (int j = 0; j < NZ; ++j) vx[j] = w.vx[j];
    dV[0] = d1;
    dV[1] = d2;
    return 0;
}
}  // namespace

extern "C" {
// The k of one tick as ric_gains_box takes it from a = Quu_mu [4][4] and g = Qu [4] on the box lo <= x <= hi: chol4 of a, the
// unconstrained x when it lies in the box, otherwise box_qp.  Out: x [4], Lf [16], act [4].  Returns 0 on the fast path, 1 + the
// box QP's iterations, -1 when the free block has no factor, -2 when a has none.
int ih_box_solve(const double* a, const double* g, const double* lo, const double* hi, double* x, double* Lf, int* act) {
    double L[16];
    if (!qs::chol4(a, L)) return -2;
    qs::chol4_neg_solve(L, g, x);
    if (qs::box_inside(x, lo, hi)) {
        for (int q = 0; q < 16; ++q) Lf[q] = L[q];
        for (int j = 0; j < 4; ++j) act[j] = 0;
        return 0;
    }
    const int it = qs::box_qp(a, g, lo, hi, x, Lf, act);
    return it < 0 ? -1 : 1 + it;
}
// box_qp alone (no fast path): its iterations, or -1
int ih_box_qp(const double* a, const double* g, const double* lo, const double* hi, double* x, double* Lf, int* act) {
    return qs::box_qp(a, g, lo, hi, x, Lf, act);
}
// x = -a^-1 g by chol4 and chol4_neg_solve (ric_gains' k); 0, or -1 when a has no factor
int ih_chol_solve(const double* a, const double* g, double* x) {
    double L[16];
    if (!qs::chol4(a, L)) return -1;
    qs::chol4_neg_solve(L, g, x);
    return 0;
}
// ih_backward_pass of ilqr_host.cpp with the box phases: lo, hi [T][4] the box of k at each tick (the command's box minus u_nom).
// Out as there, and act [T][4].
int ih_box_backward_pass(int nz, int T, const double* F, const double* dx, const double* W, const double* Rt, const double* du,
                         const double* lo, const double* hi, double mu, double* V, double* vx, double* K, double* k, double* dV,
                         int* act) {
    return nz == 13 ? pass<13>(T, F, dx, W, Rt, du, lo, hi, mu, V, vx, K, k, dV, act)
                    : pass<17>(T, F, dx, W, Rt, du, lo, hi, mu, V, vx, K, k, dV, act);
}
}
