// TEST INFRASTRUCTURE: compiles gym_pybullet_drones_b200/csrc/mlp_tangent.cuh (the policy loop's tick tangent of the JVP and
// Jacobian kernels, dyn_policy_jvp.cu) as plain host C++, so the `-m "not gpu"` suite can hold one aviary tick's tangent to the
// torch reference (tests/diff_policy_ref.py under torch.func.jacfwd) and to the transpose of the host-built adjoint
// (diff_policy_host.cpp).  The tick takes the observation's ang_v as part of the loop state, as the Jacobian kernel's z_k does;
// the actor and its tangent run the plain FMA loop.  Never linked into or imported by the product package.
#include <cmath>
#include <vector>
#include "../../gym_pybullet_drones_b200/csrc/mlp_tangent.cuh"
#include "harness.h"

namespace {
template <int EFF>
void tick_jvp(const QsParams& P, int S, int D, int A, int B, int act, int depth, const int* width, const double* const* W,
              const double* const* bias, const double* log_std, const double* noise, const double* row, const double* state,
              const double* ang, const double* hist, const double* up, const double* t_row, const double* t_state, const double* t_ang,
              const double* t_hist, const double* t_up, const double* t_raw_in, double* out_state, double* out_ang, double* out_hist,
              double* out_u, double* out_raw, double* t_out_state, double* t_out_ang, double* t_out_hist, double* t_out_u,
              double* t_out_raw) {
    const qs::PhysRow c = row_from(P, row), tc = row_from(P, t_row);
    const int od = 12 + B * A, in = D * od, out = D * A;
    const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    std::vector<double> obs(in), t_obs(in);
    for (int d = 0; d < D; ++d) {
        const qs::Drone x = drone_from(state + 13 * d), tx = drone_from(t_state + 13 * d);
        qs::obs_head(x, I, &obs[d * od]);
        for (int j = 0; j < 3; ++j) obs[d * od + 9 + j] = ang[3 * d + j];
        qs::obs_head_jvp(x, tx, t_ang + 3 * d, &t_obs[d * od]);
        for (int j = 0; j < B * A; ++j) { obs[d * od + 12 + j] = hist[d * B * A + j]; t_obs[d * od + 12 + j] = t_hist[d * B * A + j]; }
    }
    // the actor and its tangent, layer by layer
    std::vector<double> x = obs, tx = t_obs;
    int K = in;
    for (int l = 0; l <= depth; ++l) {
        const bool last = l == depth;
        const int Nout = last ? out : width[l];
        std::vector<double> y(Nout), ty(Nout), zero(Nout, 0.0);
        for (int n = 0; n < Nout; ++n) {
            double acc[1], tacc[1];
            qs::mlp_col<1>(W[l], bias[l], K, Nout, n, x.data(), K, acc);
            qs::mlp_col<1>(W[l], zero.data(), K, Nout, n, tx.data(), K, tacc);
            y[n] = last ? acc[0] : qs::mlp_act(act, acc[0]);
            ty[n] = last ? tacc[0] : qs::mlp_act_jvp(act, y[n], tacc[0]);
        }
        x = y; tx = ty; K = Nout;
    }
    for (int n = 0; n < out; ++n) {
        out_raw[n] = noise ? x[n] + exp(log_std[n]) * noise[n] : x[n];
        t_out_raw[n] = tx[n] + t_raw_in[n];
    }
    for (int d = 0; d < D; ++d) {
        double raw[4] = {0, 0, 0, 0}, t_raw[4] = {0, 0, 0, 0}, t_a[4], t_u[4], aa[4] = {0, 0, 0, 0}, rpm[4];
        for (int j = 0; j < A; ++j) { raw[j] = out_raw[d * A + j]; t_raw[j] = t_out_raw[d * A + j]; aa[j] = qs::clampd(raw[j], -1.0, 1.0); }
        qs::policy_rpm(A, c, aa, rpm);
        for (int j = 0; j < 4; ++j) out_u[4 * d + j] = qs::clampd(rpm[j], 0.0, c.max_rpm);
        qs::Drone dd = drone_from(state + 13 * d), td = drone_from(t_state + 13 * d);
        {
            qs::Drone e = dd;
            double R_last[9];
            qs::dyn_tick_k<EFF>(P, c, e, out_u + 4 * d, up + 4 * d, 0.0, S, R_last);
            for (int r = 0; r < 3; ++r) out_ang[3 * d + r] = R_last[3 * r] * e.wx + R_last[3 * r + 1] * e.wy + R_last[3 * r + 2] * e.wz;
        }
        qs::policy_tick_jvp<EFF>(P, c, tc, A, S, raw, t_raw, dd, td, up + 4 * d, t_up + 4 * d, t_a, t_u, t_out_ang + 3 * d);
        drone_to(dd, out_state + 13 * d);
        drone_to(td, t_out_state + 13 * d);
        for (int j = 0; j < 4; ++j) t_out_u[4 * d + j] = t_u[j];
        for (int j = 0; j < (B - 1) * A; ++j) {
            out_hist[d * B * A + j] = hist[d * B * A + j + A];
            t_out_hist[d * B * A + j] = t_hist[d * B * A + j + A];
        }
        for (int j = 0; j < A; ++j) { out_hist[d * B * A + (B - 1) * A + j] = aa[j]; t_out_hist[d * B * A + (B - 1) * A + j] = t_a[j]; }
    }
}
}  // namespace

extern "C" {
// One aviary tick of the policy loop and its tangent for D drones, the loop state per drone being the stored state [13], the
// observation's ang_v [3], the history [B][A] and drag's previous applied rpm up [4].  row [16] the aviary's constants, noise [D A]
// or NULL; a tangent of each (t_row of the constants, t_raw_in [D A] added to the raw action).  Out: the end state (before
// store_drone's rounding), the next observation's ang_v, the next history, the applied rpm, the raw action, and their tangents.
void pj_tick_jvp(const QsParams* P, unsigned effects, int S, int D, int A, int B, int act, int depth, const int* width,
                 const double* const* W, const double* const* bias, const double* log_std, const double* noise, const double* row,
                 const double* state, const double* ang, const double* hist, const double* up, const double* t_row, const double* t_state,
                 const double* t_ang, const double* t_hist, const double* t_up, const double* t_raw_in, double* out_state, double* out_ang,
                 double* out_hist, double* out_u, double* out_raw, double* t_out_state, double* t_out_ang, double* t_out_hist,
                 double* t_out_u, double* t_out_raw) {
    with_effects(effects, [&](auto EFF) {
        tick_jvp<decltype(EFF)::value>(*P, S, D, A, B, act, depth, width, W, bias, log_std, noise, row, state, ang, hist, up, t_row,
                                       t_state, t_ang, t_hist, t_up, t_raw_in, out_state, out_ang, out_hist, out_u, out_raw, t_out_state,
                                       t_out_ang, t_out_hist, t_out_u, t_out_raw);
    });
}
}
