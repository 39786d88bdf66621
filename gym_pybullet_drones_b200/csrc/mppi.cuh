// mppi.cuh -- the rules of one MPPI iteration (qs_mppi_*, mppi.cu; DESIGN.md 4.5.2) that do not touch the dynamics: the noise
// of a (tick, sample, drone, iteration), a sample's command, the importance weights, the candidate and the commit's choice.
// Compiled for the sm_90a kernels and for the host harness (tests/host_harness/mppi_host.cpp), so the host tests check the
// code the kernels run.
#pragma once
#include "philox.cuh"

namespace qs {

// eps[4]: the standard normals of drone `id` at tick k of sample s in iteration `it`; Philox4x32-10 with key (seed low, seed
// high) and counter (k, s, id, 2 it + h) gives rotors 2h and 2h + 1, the last word in unsigned arithmetic (every it in
// [0, 2^31) has its own counter).  Sample 0 is the nominal: eps = 0.
QS_HD void mppi_eps(unsigned long long seed, int k, int s, long long id, int it, double eps[4]) {
    if (s == 0) {
        eps[0] = eps[1] = eps[2] = eps[3] = 0.0;
        return;
    }
    const uint32_t key[2] = {(uint32_t)(seed & 0xffffffffull), (uint32_t)(seed >> 32)};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const uint32_t ctr[4] = {(uint32_t)k, (uint32_t)s, (uint32_t)id, 2u * (uint32_t)it + (uint32_t)h};   // no int overflow
        uint32_t w[4];
        philox4x32_10(ctr, key, w);
        box_muller(w, eps[2 * h], eps[2 * h + 1]);
    }
}

// the sample's raw command from the nominal u and the scaled noise sig * eps: u + sig eps, with the box clamped into [lo, hi]
template <bool BOX>
QS_HD double mppi_command(double u, double sig, double eps, double lo, double hi) {
    const double v = u + sig * eps;
    return BOX ? clampd(v, lo, hi) : v;
}
// the perturbation the update averages: the clamped command minus the nominal where the box binds, sig eps elsewhere (so a box
// that never binds gives the unboxed bits)
template <bool BOX>
QS_HD double mppi_delta(double u, double sig, double eps, double lo, double hi) {
    const double d = sig * eps;
    if (!BOX) return d;
    const double v = u + d, c = clampd(v, lo, hi);
    return c == v ? d : c - u;
}

// A unit's sample costs J_0 .. J_{K-1}, scanned in s order: J_min and the mean over the finite ones, the lowest s with J_min
// (0 when none is finite) and lambda = temperature (mean - J_min).
struct MppiStats {
    double jmin, lambda;
    int best, finite;
};
template <class Cost>
QS_HD MppiStats mppi_stats(Cost J, int K, double temperature) {
    MppiStats st = {INFINITY, 0.0, 0, 0};
    double sum = 0.0;
    for (int s = 0; s < K; ++s) {
        const double j = J(s);
        if (!isfinite(j)) continue;
        if (j < st.jmin) {
            st.jmin = j;
            st.best = s;
        }
        sum += j;
        ++st.finite;
    }
    if (st.finite > 0) st.lambda = temperature * (sum / st.finite - st.jmin);
    return st;
}
// w_s = exp(-(J_s - J_min) / lambda); 1 for every finite J_s when lambda = 0; 0 for a non-finite J_s
QS_HD double mppi_weight(double j, const MppiStats& st) {
    if (!isfinite(j)) return 0.0;
    if (st.lambda == 0.0) return 1.0;
    return exp(-(j - st.jmin) / st.lambda);
}
// u_c = u + sum_s w_s delta_s / sum_s w_s (num = the weighted sum); the nominal when no weight is positive
QS_HD double mppi_candidate(double u, double num, double wsum) { return wsum > 0.0 ? u + num / wsum : u; }
// the commit keeps the candidate when its cost is no worse than the best sample's (false for a NaN on either side)
QS_HD bool mppi_take_candidate(double jc, double jbest) { return jc <= jbest; }

}  // namespace qs
