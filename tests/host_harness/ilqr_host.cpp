// TEST INFRASTRUCTURE: compiles gym_pybullet_drones_b200/csrc/riccati.cuh (the backward tick of qs_ilqr_backward, ilqr.cu) as
// plain host C++, so the `-m "not gpu"` suite can hold the Riccati recursion to a float64 restatement (tests/ilqr_ref.py) and to
// the discrete algebraic Riccati equation.  The phases run column by column in the order of the kernel's lanes.  Never linked
// into or imported by the product package.
#include <vector>
#include "../../gym_pybullet_drones_b200/csrc/riccati.cuh"

namespace {
template <int NZ>
int pass(int T, const double* F, const double* dx, const double* W, const double* Rt, const double* du, double mu, double* V,
         double* vx, double* K, double* k, double* dV) {
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
        qs::RicGains G;
        if (!qs::ric_gains(w, Rt, du + 4 * t, mu, G, d1, d2)) return t + 1;
        for (int j = 0; j < NZ; ++j) qs::ric_col_K(w, j, G);
        for (int j = 0; j < NZ; ++j) qs::ric_col_V(w, j, G);
        for (int j = 0; j < 4 * NZ; ++j) K[4 * NZ * t + j] = w.K[j];
        for (int j = 0; j < 4; ++j) k[4 * t + j] = G.k[j];
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
// T ticks of the backward pass, t = T-1 .. 0, for one drone: F [T][nz][nz + 4] = [A | B] of each tick, the stage cost's
// dx = x - r [T][13] and weights W [T][13] of the state after tick t, Rt [4], du = u - u_ref [T][4], mu.  V [nz][nz] and vx [nz]:
// in, the value at the state after the last tick; out, at the state before tick 0.  Out: K [T][4][nz], k [T][4], dV [2].
// Returns 0, or 1 + the tick whose regularised Quu has no Cholesky factor.
int ih_backward_pass(int nz, int T, const double* F, const double* dx, const double* W, const double* Rt, const double* du, double mu,
                     double* V, double* vx, double* K, double* k, double* dV) {
    return nz == 13 ? pass<13>(T, F, dx, W, Rt, du, mu, V, vx, K, k, dV) : pass<17>(T, F, dx, W, Rt, du, mu, V, vx, K, k, dV);
}
// J of one tick, qs::stage_cost
double ih_stage_cost(const double* x, const double* ref, const double* W, const double* u, const double* uref, const double* Rt) {
    return qs::stage_cost(x, ref, W, u, uref, Rt);
}
}
