// TEST INFRASTRUCTURE: compiles the adjoint LQR of the solution's derivative (the phases of qs_ilqr_adjoint and
// qs_ilqr_adjoint_rollout, ilqr_adjoint.cu, from gym_pybullet_drones_b200/csrc/riccati.cuh) as plain host C++, so the
// `-m "not gpu"` suite can hold it to a dense float64 solve (tests/ilqr_grad_ref.py) and the device to the host bit for bit.
// The phases run column by column in the order of the kernels' lanes.  Never linked into or imported by the product package.
#include <vector>
#include "../../gym_pybullet_drones_b200/csrc/riccati.cuh"

namespace {
template <int NZ>
int pass(int T, const double* F, const double* W, const double* Rt, const double* gx, const double* gu, const int* act,
         double* K, double* k) {
    constexpr int M = NZ + 4;
    std::vector<double> buf(qs::RicWs<NZ>::DOUBLES, 0.0);
    const qs::RicWs<NZ> w = qs::ric_ws<NZ>(buf.data());
    for (int t = T - 1; t >= 0; --t) {
        for (int j = 0; j < 13; ++j) qs::ric_stage_adj(w, j, W[13 * t + j], gx[13 * t + j]);
        for (int j = 0; j < NZ * M; ++j) w.F[j] = F[(long long)NZ * M * t + j];
        for (int j = 0; j < M; ++j) qs::ric_col_H(w, j);
        const int none[4] = {0, 0, 0, 0};
        qs::RicBoxGains G;
        if (!qs::ric_gains_adj(w, Rt, gu + 4 * t, act ? act + 4 * t : none, G)) return t + 1;
        for (int j = 0; j < NZ; ++j) {
            if (act) qs::ric_col_K_box(w, j, G);
            else qs::ric_col_K(w, j, G);
        }
        for (int j = 0; j < NZ; ++j) qs::ric_col_V(w, j, G);
        for (int j = 0; j < 4 * NZ; ++j) K[4 * NZ * t + j] = w.K[j];
        for (int j = 0; j < 4; ++j) k[4 * t + j] = G.k[j];
        for (int j = 0; j < NZ; ++j) qs::ric_col_sym(w, j);
    }
    return 0;
}

template <int NZ>
void rollout(int T, const double* F, const double* K, const double* k, const int* act, double* wo, double* dz) {
    constexpr int M = NZ + 4;
    std::vector<double> buf(NZ * M);
    qs::RicWs<NZ> w;
    w.F = buf.data();
    double y[M] = {}, nxt[NZ];
    for (int t = 0; t < T; ++t) {
        for (int j = 0; j < NZ * M; ++j) w.F[j] = F[(long long)NZ * M * t + j];
        double v[4];
        for (int j = 0; j < 4; ++j) v[j] = qs::ric_adj_w<NZ>(K + 4 * NZ * t + NZ * j, k[4 * t + j], y, act && act[4 * t + j] != 0);
        for (int j = 0; j < 4; ++j) {
            y[NZ + j] = v[j];
            wo[4 * t + j] = v[j];
        }
        for (int r = 0; r < NZ; ++r) nxt[r] = qs::ric_adj_next(w, r, y);
        for (int r = 0; r < NZ; ++r) {
            y[r] = nxt[r];
            dz[NZ * t + r] = nxt[r];
        }
    }
}
}  // namespace

extern "C" {
// The adjoint's Riccati pass over T ticks of one drone: F [T][nz][nz + 4] = [A | B], W [T][13] the stage weights of the state
// after tick t, Rt [4], gx [T][13] and gu [T][4] the cotangents, act [T][4] the held rotors (nonzero) or NULL (none, and the
// unconstrained phase K).  Out: K [T][4][nz], k [T][4].  Returns 0, or 1 + the tick whose free block has no factor.
int ih_adjoint_pass(int nz, int T, const double* F, const double* W, const double* Rt, const double* gx, const double* gu,
                    const int* act, double* K, double* k) {
    return nz == 13 ? pass<13>(T, F, W, Rt, gx, gu, act, K, k) : pass<17>(T, F, W, Rt, gx, gu, act, K, k);
}
// The adjoint's linear rollout from dz_0 = 0: out w [T][4] and dz [T][nz] (dz_{t+1}: row t)
void ih_adjoint_rollout(int nz, int T, const double* F, const double* K, const double* k, const int* act, double* w, double* dz) {
    if (nz == 13) rollout<13>(T, F, K, k, act, w, dz);
    else rollout<17>(T, F, K, k, act, w, dz);
}
}
