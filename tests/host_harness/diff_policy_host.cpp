// TEST INFRASTRUCTURE: compiles gym_pybullet_drones_b200/csrc/mlp_adjoint.cuh (with dyn_adjoint.cuh and quad_core.cuh: the math
// of the differentiable policy trajectories, dyn_policy_traj.cu) as plain host C++, so the `-m "not gpu"` suite can hold one
// aviary tick of the policy loop and its VJP to the torch reference (tests/diff_policy_ref.py).  The tick is the kernel's:
// observation rows, the actor (plain FMA loop), sample / clip / history shift / decode, the env's clip, dyn_tick_k; its VJP is one
// step of dyn_policy_traj_vjp_kernel, with the next tick's demands (ang_v and history cotangents) as inputs.  Never linked into
// or imported by the product package.
#include <cmath>
#include <vector>
#include "../../gym_pybullet_drones_b200/csrc/mlp_adjoint.cuh"
#include "harness.h"

namespace {
template <int EFF>
void tick_vjp(const QsParams& P, int S, int D, int A, int B, int act, int depth, const int* width, const double* const* W,
              const double* const* bias, const double* log_std, const double* noise, const double* row, const double* state,
              const double* Rq, const double* hist, const double* up, const double* g_end, const double* g_raw_out,
              const double* Lang_next, const double* g_hist_next, double* out_state, double* out_raw, double* out_hist,
              double* out_qlast, double* g_state, double* g_Rq, double* g_hist, double* g_up, double* g_row, double* g_raw) {
    const qs::PhysRow c = row_from(P, row);
    const int od = 12 + B * A, in = D * od, out = D * A;
    // ---- forward ----
    std::vector<double> obs(in);
    for (int d = 0; d < D; ++d) {
        double R[9];
        const double* q = Rq + 4 * d;
        qs::quat_to_matrix_unit(q[0], q[1], q[2], q[3], R);
        qs::obs_head(drone_from(state + 13 * d), R, &obs[d * od]);
        for (int j = 0; j < B * A; ++j) obs[d * od + 12 + j] = hist[d * B * A + j];
    }
    std::vector<std::vector<double>> h(depth);
    const double* x = obs.data();
    int K = in;
    for (int l = 0; l < depth; ++l) {
        h[l].resize(width[l]);
        for (int n = 0; n < width[l]; ++n) {
            double acc[1];
            qs::mlp_col<1>(W[l], bias[l], K, width[l], n, x, K, acc);
            h[l][n] = qs::mlp_act(act, acc[0]);
        }
        x = h[l].data(); K = width[l];
    }
    std::vector<double> raw(out), a(out);
    for (int n = 0; n < out; ++n) {
        double acc[1];
        qs::mlp_col<1>(W[depth], bias[depth], K, out, n, x, K, acc);
        raw[n] = noise ? acc[0] + exp(log_std[n]) * noise[n] : acc[0];
        a[n] = qs::clampd(raw[n], -1.0, 1.0);
        out_raw[n] = raw[n];
    }
    std::vector<double> gz(out), g_rowacc(16, 0.0);
    std::vector<qs::Drone> Ls(D);
    for (int d = 0; d < D; ++d) {
        for (int j = 0; j < (B - 1) * A; ++j) out_hist[d * B * A + j] = hist[d * B * A + j + A];
        double aa[4] = {0, 0, 0, 0}, rpm[4], u[4];
        for (int j = 0; j < A; ++j) { aa[j] = a[d * A + j]; out_hist[d * B * A + (B - 1) * A + j] = aa[j]; }
        qs::policy_rpm(A, c, aa, rpm);
        for (int j = 0; j < 4; ++j) u[j] = qs::clampd(rpm[j], 0.0, c.max_rpm);
        const qs::Drone d0 = drone_from(state + 13 * d);
        HostRec rec;
        rec.v.resize(S > 1 ? S - 1 : 1);
        {
            qs::Drone dd = d0;
            double R_last[9];
            qs::dyn_tick_k<EFF>(P, c, dd, u, up + 4 * d, 0.0, S, R_last, qs::RecordHook<HostRec>{&dd, &rec, S - 1});
            drone_to(dd, out_state + 13 * d);
            qs::Drone xl = d0;
            double inv;
            qs::entry_normalise(xl, inv);
            if (S > 1) rec.load(S - 2, xl);
            out_qlast[4 * d] = xl.qx; out_qlast[4 * d + 1] = xl.qy; out_qlast[4 * d + 2] = xl.qz; out_qlast[4 * d + 3] = xl.qw;
        }
        // ---- backward, as one step of dyn_policy_traj_vjp_kernel ----
        qs::Drone L = drone_from(g_end + 13 * d);
        double Lu[4] = {0, 0, 0, 0}, Lup[4] = {0, 0, 0, 0};
        qs::PhysGrad G;
        for (int j = 0; j < 16; ++j) G.g[j] = 0.0;
        qs::dyn_tick_obs_vjp<EFF>(P, c, d0, u, up + 4 * d, S, rec, L, Lang_next + 3 * d, Lu, Lup, G);
        double Lrpm[4], La[4] = {0, 0, 0, 0};
        qs::rpm_clip_vjp(rpm, c.max_rpm, Lu, Lrpm, G.g[13]);
        qs::policy_rpm_vjp(A, c, aa, Lrpm, La, G.g[12]);
        for (int j = 0; j < A; ++j) {
            const double la = La[j] + g_hist_next[d * B * A + (B - 1) * A + j];
            const double r = raw[d * A + j];
            gz[d * A + j] = ((r < -1.0 || r > 1.0) ? 0.0 : la) + g_raw_out[d * A + j];
            g_raw[d * A + j] = gz[d * A + j];
        }
        Ls[d] = L;
        for (int j = 0; j < 4; ++j) g_up[4 * d + j] = Lup[j];
        for (int j = 0; j < 16; ++j) g_rowacc[j] += G.g[j];
    }
    std::vector<double> src = gz;
    int Nout = out;
    for (int l = depth; l >= 0; --l) {
        const int Kl = l == 0 ? in : width[l - 1];
        std::vector<double> dst(Kl);
        for (int k = 0; k < Kl; ++k) {
            double acc[1];
            qs::mlp_row_t<1>(W[l], Nout, k, src.data(), Nout, acc);
            dst[k] = l == 0 ? acc[0] : qs::mlp_act_vjp(act, h[l - 1][k], acc[0]);
        }
        src = dst; Nout = Kl;
    }
    for (int d = 0; d < D; ++d) {
        const qs::Drone d0 = drone_from(state + 13 * d);
        const double* Lo = &src[d * od];
        double Lang[3];
        qs::obs_head_vjp(d0, Lo, Ls[d], Lang);
        const double w[3] = {d0.wx, d0.wy, d0.wz};
        double Lw[3] = {0, 0, 0}, Lq[4] = {0, 0, 0, 0};
        const double* q = Rq + 4 * d;
        qs::ang_v_vjp(q[0], q[1], q[2], q[3], w, Lang, Lw, Lq);
        Ls[d].wx += Lw[0]; Ls[d].wy += Lw[1]; Ls[d].wz += Lw[2];
        drone_to(Ls[d], g_state + 13 * d);
        for (int j = 0; j < 4; ++j) g_Rq[4 * d + j] = Lq[j];
        for (int j = 0; j < B * A; ++j) g_hist[d * B * A + j] = Lo[12 + j] + (j >= A ? g_hist_next[d * B * A + j - A] : 0.0);
    }
    for (int j = 0; j < 16; ++j) g_row[j] = g_rowacc[j];
}
}  // namespace

extern "C" {
// One aviary tick of the policy loop and its VJP for D drones.  state [D][13], Rq [D][4] (the attitude R_last is taken of), hist
// [D][B][A], up [D][4], noise [D A] or NULL; cotangents g_end [D][13] (end state), g_raw_out [D A] (the returned raw action),
// Lang_next [D][3] (the next observation's ang_v = R(q_last) w_end) and g_hist_next [D][B][A] (the next history).  Out: the end
// state (before store_drone's rounding), raw, the next history, q_last [D][4]; gradients of state, Rq, hist, up, row [16] and
// g_raw [D A], the whole cotangent of the raw action (the actor's parameter gradients follow from it).
void dph_tick_vjp(const QsParams* P, unsigned effects, int S, int D, int A, int B, int act, int depth, const int* width,
                  const double* const* W, const double* const* bias, const double* log_std, const double* noise, const double* row,
                  const double* state, const double* Rq, const double* hist, const double* up, const double* g_end,
                  const double* g_raw_out, const double* Lang_next, const double* g_hist_next, double* out_state, double* out_raw,
                  double* out_hist, double* out_qlast, double* g_state, double* g_Rq, double* g_hist, double* g_up, double* g_row,
                  double* g_raw) {
    with_effects(effects, [&](auto EFF) {
        tick_vjp<decltype(EFF)::value>(*P, S, D, A, B, act, depth, width, W, bias, log_std, noise, row, state, Rq, hist, up, g_end,
                                       g_raw_out, Lang_next, g_hist_next, out_state, out_raw, out_hist, out_qlast, g_state, g_Rq, g_hist,
                                       g_up, g_row, g_raw);
    });
}
}
