// riccati.cuh -- one tick of the iLQR backward pass (qs_ilqr_backward, ilqr.cu; DESIGN.md 4.5.1), the 4x4 Cholesky solve it
// factors Quu with and the quadratic stage cost, compiled for the sm_90a kernels and for the host harness
// (tests/host_harness/ilqr_host.cpp).
//
// The tick works on a per-drone workspace (RicWs) and is split into column phases: phase(ws, j) touches column j of its
// outputs only and reads what earlier phases wrote.  On the device lane j of the drone's warp runs column j with a __syncwarp
// between phases; on the host a loop over j runs each phase.  Both take the same operations in the same order, so they give
// the same bits.  Matrices are row-major.  z = the loop state (n_z = NZ entries: x, and with drag the clipped previous RPMs),
// M = NZ + 4 columns [z | u].
#pragma once
#include "quad_core.cuh"

namespace qs {

// One aviary's row of QsIlqrIO.weights: [Q 13 | Q_final 13 | R 4]
constexpr int kWeightsQ = 0, kWeightsQFinal = 13, kWeightsR = 26, kWeightsRow = 30;
// the offset in the row of the state weights of the state after tick k of T: Q, or Q_final after the last tick
QS_HD int stage_weights(int k, int T) { return k == T - 1 ? kWeightsQFinal : kWeightsQ; }
// Rt = R / HOVER_RPM^2 of the drone's row
QS_HD void rel_weights(const double* wt, const PhysRow& c, double Rt[4]) {
    const double h2 = c.hover_rpm * c.hover_rpm;
#pragma unroll
    for (int j = 0; j < 4; ++j) Rt[j] = wt[kWeightsR + j] / h2;
}

template <int NZ>
struct RicWs {
    static constexpr int M = NZ + 4;
    static constexpr int DOUBLES = NZ * M + M * M + NZ * NZ + NZ + M + 4 * NZ;
    double* F;      // [NZ][M] d z_{k+1} / d (z_k, u_k): [A | B]
    double* H;      // [M][M] F' V_xx F (phase H); rows < NZ of columns < NZ then hold the unsymmetrised new V_xx (phase V)
    double* V;      // [NZ][NZ] V_xx of z_{k+1}, then of z_k
    double* vx;     // [NZ] V_x of z_{k+1}, then of z_k
    double* g;      // [M] F' V_x: Qx, then B'V_x
    double* K;      // [4][NZ] this tick's feedback gain
};
// the workspace carved from DOUBLES doubles at p
template <int NZ>
QS_HD RicWs<NZ> ric_ws(double* p) {
    constexpr int M = NZ + 4;
    RicWs<NZ> w;
    w.F = p; w.H = w.F + NZ * M; w.V = w.H + M * M; w.vx = w.V + NZ * NZ; w.g = w.vx + NZ; w.K = w.g + M;
    return w;
}

// Column c of F for column c of qs_dyn_tick_jac's tick block (C = 17, or 21 with drag): the state columns stay, the raw RPMs
// become the u columns NZ..NZ+3 and drag's previous clipped RPMs (jac columns 17..20) the z columns 13..16
template <int NZ>
QS_HD int ric_f_col(int c) { return NZ == 13 ? c : (c < 13 ? c : (c < 17 ? c + 4 : c - 4)); }

// Rows 13..NZ-1 of F (drag): z_{k+1}'s previous RPMs are this tick's clipped u_k, d/du = the clip's derivative cd
template <int NZ>
QS_HD void ric_f_aug(const RicWs<NZ>& w, int idx, const double cd[4]) {
    constexpr int M = NZ + 4;
    const int r = idx / M, c = idx - r * M;
    w.F[(13 + r) * M + c] = c == NZ + r ? cd[r] : 0.0;
}

// Phase S (j < 13): the stage cost 1/2 wj (x_j - r_j)^2 of z_{k+1}'s state component j
template <int NZ>
QS_HD void ric_stage(const RicWs<NZ>& w, int j, double dx, double wj) {
    w.V[j * NZ + j] += wj;
    w.vx[j] += wj * dx;
}

// Phase H (j < M): column j of H = F' V_xx F and g_j = (F' V_x)_j
template <int NZ>
QS_HD void ric_col_H(const RicWs<NZ>& w, int j) {
    constexpr int M = NZ + 4;
    double f[NZ], p[NZ];
    double gj = 0.0;
#pragma unroll
    for (int s = 0; s < NZ; ++s) {
        f[s] = w.F[s * M + j];
        gj += f[s] * w.vx[s];
    }
    w.g[j] = gj;
#pragma unroll
    for (int r = 0; r < NZ; ++r) {
        double acc = 0.0;
#pragma unroll
        for (int s = 0; s < NZ; ++s) acc += w.V[r * NZ + s] * f[s];
        p[r] = acc;
    }
#pragma unroll 1
    for (int i = 0; i < M; ++i) {
        double acc = 0.0;
#pragma unroll
        for (int r = 0; r < NZ; ++r) acc += w.F[r * M + i] * p[r];
        w.H[i * M + j] = acc;
    }
}

// Lower Cholesky factor L (row-major, upper part unused) of the 4x4 a; false when a pivot is not > 0 (or not finite)
QS_HD bool chol4(const double a[16], double L[16]) {
    bool ok = true;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int j = 0; j <= i; ++j) {
            double s = a[i * 4 + j];
#pragma unroll
            for (int q = 0; q < j; ++q) s -= L[i * 4 + q] * L[j * 4 + q];
            if (i == j) {
                ok = ok && s > 0.0 && s < INFINITY;
                L[i * 4 + i] = sqrt(s);
            } else {
                L[i * 4 + j] = s / L[j * 4 + j];
            }
        }
    }
    return ok;
}
// x = -(L L')^-1 b
QS_HD void chol4_neg_solve(const double L[16], const double b[4], double x[4]) {
    double y[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        double s = b[i];
#pragma unroll
        for (int q = 0; q < i; ++q) s -= L[i * 4 + q] * y[q];
        y[i] = s / L[i * 4 + i];
    }
#pragma unroll
    for (int i = 3; i >= 0; --i) {
        double s = y[i];
#pragma unroll
        for (int q = i + 1; q < 4; ++q) s -= L[q * 4 + i] * x[q];
        x[i] = s / L[i * 4 + i];
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) x[i] = -x[i];
}

// What every column needs after phase H: Quu (unregularised, symmetrised), its regularised factor, Qu and k
struct RicGains {
    double Quu[16], L[16], Qu[4], k[4];
};

// Phase G (every lane, the same bits): Quu = Rt + B'V_xx B, Qu = Rt du + B'V_x, Quu_mu = Quu + mu diag(Quu) = L L',
// k = -Quu_mu^-1 Qu; dV1 += k'Qu, dV2 += 1/2 k'Quu k.  false when Quu_mu is not positive definite.
template <int NZ>
QS_HD bool ric_gains(const RicWs<NZ>& w, const double Rt[4], const double du[4], double mu, RicGains& G, double& dV1, double& dV2) {
    constexpr int M = NZ + 4;
    double a[16];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            double q = 0.5 * (w.H[(NZ + i) * M + NZ + j] + w.H[(NZ + j) * M + NZ + i]);
            if (i == j) q += Rt[i];
            G.Quu[i * 4 + j] = q;
            a[i * 4 + j] = i == j ? q + mu * q : q;
        }
        G.Qu[i] = Rt[i] * du[i] + w.g[NZ + i];
    }
    if (!chol4(a, G.L)) return false;
    chol4_neg_solve(G.L, G.Qu, G.k);
    double d1 = 0.0, d2 = 0.0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        double qk = 0.0;
#pragma unroll
        for (int j = 0; j < 4; ++j) qk += G.Quu[i * 4 + j] * G.k[j];
        d1 += G.k[i] * G.Qu[i];
        d2 += G.k[i] * qk;
    }
    dV1 += d1;
    dV2 += 0.5 * d2;
    return true;
}

// Phase K (j < NZ): column j of K = -Quu_mu^-1 Qux and V_x,j = Qx_j + K_j'Quu k + K_j'Qu + Qux_j'k (Tassa's form, Quu
// unregularised)
template <int NZ>
QS_HD void ric_col_K(const RicWs<NZ>& w, int j, const RicGains& G) {
    constexpr int M = NZ + 4;
    double qux[4], kj[4];
#pragma unroll
    for (int a = 0; a < 4; ++a) qux[a] = w.H[(NZ + a) * M + j];
    chol4_neg_solve(G.L, qux, kj);
    double v = w.g[j];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        double qk = 0.0;
#pragma unroll
        for (int b = 0; b < 4; ++b) qk += G.Quu[a * 4 + b] * G.k[b];
        v += kj[a] * qk + kj[a] * G.Qu[a] + qux[a] * G.k[a];
        w.K[a * NZ + j] = kj[a];
    }
    w.vx[j] = v;
}

// Phase V (j < NZ, after every column of K): column j of Qxx + K'Quu K + K'Qux + Qux'K into H's column j
template <int NZ>
QS_HD void ric_col_V(const RicWs<NZ>& w, int j, const RicGains& G) {
    constexpr int M = NZ + 4;
    double t[4], kj[4];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        kj[a] = w.K[a * NZ + j];
        double qk = 0.0;
#pragma unroll
        for (int b = 0; b < 4; ++b) qk += G.Quu[a * 4 + b] * w.K[b * NZ + j];
        t[a] = qk + w.H[(NZ + a) * M + j];
    }
#pragma unroll 1
    for (int i = 0; i < NZ; ++i) {
        double v = w.H[i * M + j];
#pragma unroll
        for (int a = 0; a < 4; ++a) v += w.K[a * NZ + i] * t[a] + w.H[(NZ + a) * M + i] * kj[a];
        w.H[i * M + j] = v;
    }
}

// Phase Y (j < NZ, after every column of phase V): column j of V_xx = (H + H') / 2
template <int NZ>
QS_HD void ric_col_sym(const RicWs<NZ>& w, int j) {
    constexpr int M = NZ + 4;
#pragma unroll 1
    for (int i = 0; i < NZ; ++i) w.V[i * NZ + j] = 0.5 * (w.H[i * M + j] + w.H[j * M + i]);
}

// ---- Control limits (qs_ilqr_box_backward): the tick's k solves min 1/2 k'Quu_mu k + Qu'k subject to lo <= k <= hi, where
// lo, hi = the box of the raw command minus u_nom.  The unconstrained k of ric_gains is kept when it lies in the box (with
// today's K: a problem whose bounds never bind gives ric_gains' bits); otherwise a projected-Newton box QP (Tassa, Mansard &
// Todorov, ICRA 2014) runs from clamp(0).  Its constants:
constexpr int kBoxMaxIter = 100;        // projected-Newton iterations
constexpr double kBoxArmijo = 0.1;      // a step is accepted when (f(x_new) - f(x)) / (step s'grad) >= kBoxArmijo
constexpr double kBoxStepDec = 0.6;     // the line search's step factor
constexpr double kBoxMinStep = 1e-22;   // the line search gives up below this step
constexpr double kBoxGradTol = 1e-12;   // converged when every free |grad_j| <= kBoxGradTol (|g_j| + sum_q |a_jq x_q|)

// true when lo <= x <= hi (false for a NaN entry)
QS_HD bool box_inside(const double x[4], const double lo[4], const double hi[4]) {
    bool in = true;
#pragma unroll
    for (int j = 0; j < 4; ++j) in = in && lo[j] <= x[j] && x[j] <= hi[j];
    return in;
}

// 1/2 x'a x + g'x
QS_HD double box_value(const double a[16], const double g[4], const double x[4]) {
    double f = 0.0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        double ax = 0.0;
#pragma unroll
        for (int j = 0; j < 4; ++j) ax += a[i * 4 + j] * x[j];
        f += x[i] * (g[i] + 0.5 * ax);
    }
    return f;
}

// The projected-Newton box QP: x = argmin 1/2 x'a x + g'x subject to lo <= x <= hi, a symmetric positive definite, lo <= hi.
// act[j] = -1 / +1 where x_j is held at lo_j / hi_j (x at the bound with the gradient pointing out of the box), 0 free.  Lf =
// the Cholesky factor of a's free block embedded in a 4x4 with identity rows and columns on the held dimensions, so that
// chol4_neg_solve with a right-hand side that is 0 on them solves the free block alone.  Returns the iterations taken, or -1
// when the free block has no factor.
QS_HD int box_qp(const double a[16], const double g[4], const double lo[4], const double hi[4], double x[4], double Lf[16],
                 int act[4]) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        x[j] = clampd(0.0, lo[j], hi[j]);
        act[j] = 0;
    }
    double f = box_value(a, g, x);
    bool factored = false;
    int it = 0;
    for (; it < kBoxMaxIter; ++it) {
        double gr[4];
        bool changed = !factored, held = true, small = true;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            double s = g[i], sc = fabs(g[i]);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                s += a[i * 4 + j] * x[j];
                sc += fabs(a[i * 4 + j] * x[j]);
            }
            gr[i] = s;
            const int na = (x[i] == lo[i] && s > 0.0) ? -1 : ((x[i] == hi[i] && s < 0.0) ? 1 : 0);
            changed = changed || na != act[i];
            act[i] = na;
            held = held && na != 0;
            small = small && (na != 0 || fabs(s) <= kBoxGradTol * sc);
        }
        if (held) {
#pragma unroll
            for (int q = 0; q < 16; ++q) Lf[q] = (q % 5 == 0) ? 1.0 : 0.0;
            return it;
        }
        if (changed) {
            double e[16];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
#pragma unroll
                for (int j = 0; j < 4; ++j) e[i * 4 + j] = (act[i] == 0 && act[j] == 0) ? a[i * 4 + j] : (i == j ? 1.0 : 0.0);
            }
            if (!chol4(e, Lf)) return -1;
            factored = true;
        }
        if (small) return it;
        // the Newton step of the free block with the held entries fixed: x_f + s_f = -a_ff^-1 (g_f + a_fh x_h)
        double r[4], s[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            double v = g[i];
#pragma unroll
            for (int j = 0; j < 4; ++j) v += act[j] != 0 ? a[i * 4 + j] * x[j] : 0.0;
            r[i] = act[i] != 0 ? 0.0 : v;
        }
        chol4_neg_solve(Lf, r, s);
        double sg = 0.0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            s[j] = act[j] != 0 ? 0.0 : s[j] - x[j];
            sg += s[j] * gr[j];
        }
        if (!(sg < 0.0)) return it;                                   // no descent left: rounding
        double step = 1.0, xc[4], fc;
        for (;;) {                                                    // Armijo backtracking along the projected arc
#pragma unroll
            for (int j = 0; j < 4; ++j) xc[j] = clampd(x[j] + step * s[j], lo[j], hi[j]);
            fc = box_value(a, g, xc);
            if ((fc - f) / (step * sg) >= kBoxArmijo) break;
            step *= kBoxStepDec;
            if (step < kBoxMinStep) return it;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) x[j] = xc[j];
        f = fc;
    }
    return it;
}

// What every column needs after phase G of the box backward: RicGains with k the box QP's, the factor Lf that K is solved
// with (L on the fast path) and the held rotors
struct RicBoxGains : RicGains {
    double Lf[16];
    int act[4];
};

// Phase G of the box backward (every lane, the same bits): ric_gains, then k as above for the box [lo, hi] of k, and dV1 +=
// k'Qu, dV2 += 1/2 k'Quu k with that k.  false when Quu_mu or its free block is not positive definite.
template <int NZ>
QS_HD bool ric_gains_box(const RicWs<NZ>& w, const double Rt[4], const double du[4], const double lo[4], const double hi[4],
                         double mu, RicBoxGains& G, double& dV1, double& dV2) {
    double d1 = 0.0, d2 = 0.0;
    if (!ric_gains(w, Rt, du, mu, G, d1, d2)) return false;
    if (box_inside(G.k, lo, hi)) {                                    // the fast path: ric_gains' k, K from its factor
#pragma unroll
        for (int q = 0; q < 16; ++q) G.Lf[q] = G.L[q];
#pragma unroll
        for (int j = 0; j < 4; ++j) G.act[j] = 0;
        dV1 += d1;
        dV2 += d2;
        return true;
    }
    double a[16];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int j = 0; j < 4; ++j) a[i * 4 + j] = i == j ? G.Quu[i * 4 + j] + mu * G.Quu[i * 4 + j] : G.Quu[i * 4 + j];
    }
    if (box_qp(a, G.Qu, lo, hi, G.k, G.Lf, G.act) < 0) return false;
    d1 = d2 = 0.0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        double qk = 0.0;
#pragma unroll
        for (int j = 0; j < 4; ++j) qk += G.Quu[i * 4 + j] * G.k[j];
        d1 += G.k[i] * G.Qu[i];
        d2 += G.k[i] * qk;
    }
    dV1 += d1;
    dV2 += 0.5 * d2;
    return true;
}

// Phase K of the box backward (j < NZ): ric_col_K with K's free rows -(Quu_mu,ff)^-1 Qux,f from Lf and its held rows 0
template <int NZ>
QS_HD void ric_col_K_box(const RicWs<NZ>& w, int j, const RicBoxGains& G) {
    constexpr int M = NZ + 4;
    double qux[4], rhs[4], kj[4];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        qux[a] = w.H[(NZ + a) * M + j];
        rhs[a] = G.act[a] != 0 ? 0.0 : qux[a];
    }
    chol4_neg_solve(G.Lf, rhs, kj);
    double v = w.g[j];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        if (G.act[a] != 0) kj[a] = 0.0;
        double qk = 0.0;
#pragma unroll
        for (int b = 0; b < 4; ++b) qk += G.Quu[a * 4 + b] * G.k[b];
        v += kj[a] * qk + kj[a] * G.Qu[a] + qux[a] * G.k[a];
        w.K[a * NZ + j] = kj[a];
    }
    w.vx[j] = v;
}

// ---- The adjoint LQR of the solution's derivative (qs_ilqr_adjoint, ilqr_adjoint.cu; DESIGN.md 4.5.1): the solve's stage
// Hessians at mu = 0 with the linear terms -g_X (state) and -g_U (command), on the free rotors only.  Its phases S and G are
// below; phases H, K, V and Y are the solve's (ric_col_H, ric_col_K / ric_col_K_box, ric_col_V, ric_col_sym).

// Phase S of the adjoint (j < 13): the stage 1/2 wj dx_j^2 - gx dx_j of z_{k+1}'s state component j
template <int NZ>
QS_HD void ric_stage_adj(const RicWs<NZ>& w, int j, double wj, double gx) {
    w.V[j * NZ + j] += wj;
    w.vx[j] -= gx;
}

// Phase G of the adjoint (every lane, the same bits): Quu = Rt + B'V_xx B as ric_gains takes it, Qu = -gu + B'V_x, and the
// factor of Quu's free block embedded in a 4x4 with identity rows and columns on the held rotors (act[j] != 0; all free: Quu's
// own factor, bit for bit ric_gains' at mu = 0); k = -Quu_ff^-1 Qu_f, 0 on held rotors.  G.L = G.Lf.  false when the free
// block is not positive definite.
template <int NZ>
QS_HD bool ric_gains_adj(const RicWs<NZ>& w, const double Rt[4], const double gu[4], const int act[4], RicBoxGains& G) {
    constexpr int M = NZ + 4;
    double e[16], rhs[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            double q = 0.5 * (w.H[(NZ + i) * M + NZ + j] + w.H[(NZ + j) * M + NZ + i]);
            if (i == j) q += Rt[i];
            G.Quu[i * 4 + j] = q;
            e[i * 4 + j] = (act[i] == 0 && act[j] == 0) ? q : (i == j ? 1.0 : 0.0);
        }
        G.Qu[i] = w.g[NZ + i] - gu[i];
        G.act[i] = act[i];
        rhs[i] = act[i] != 0 ? 0.0 : G.Qu[i];
    }
    if (!chol4(e, G.Lf)) return false;
    chol4_neg_solve(G.Lf, rhs, G.k);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if (act[i] != 0) G.k[i] = 0.0;
    }
#pragma unroll
    for (int q = 0; q < 16; ++q) G.L[q] = G.Lf[q];
    return true;
}

// The adjoint's linear rollout, one tick: w_j = k_j + K_j dz (0 on held rotors), K_j dz summed in q order from 0.0
template <int NZ>
QS_HD double ric_adj_w(const double* Kj, double kj, const double* dz, bool held) {
    double s = 0.0;
#pragma unroll
    for (int q = 0; q < NZ; ++q) s += Kj[q] * dz[q];
    return held ? 0.0 : kj + s;
}
// Row r (< NZ) of dz_{k+1} = F [dz; w]: y = [dz | w] (M entries), summed in column order from 0.0
template <int NZ>
QS_HD double ric_adj_next(const RicWs<NZ>& w, int r, const double* y) {
    constexpr int M = NZ + 4;
    double s = 0.0;
#pragma unroll
    for (int c = 0; c < M; ++c) s += w.F[r * M + c] * y[c];
    return s;
}

// 1/2 (sum_r W_r (x_r - ref_r)^2 + sum_j Rt_j (u_j - uref_j)^2): the cost of one tick, x and ref in the order pos, quat, vel,
// rpy_rates
QS_HD double stage_cost(const double x[13], const double ref[13], const double W[13], const double u[4], const double uref[4],
                        const double Rt[4]) {
    double s = 0.0;
#pragma unroll
    for (int r = 0; r < 13; ++r) {
        const double e = x[r] - ref[r];
        s += W[r] * (e * e);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const double e = u[j] - uref[j];
        s += Rt[j] * (e * e);
    }
    return 0.5 * s;
}

}  // namespace qs
