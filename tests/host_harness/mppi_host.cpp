// TEST INFRASTRUCTURE: compiles the rules of one MPPI iteration (gym_pybullet_drones_b200/csrc/philox.cuh and mppi.cuh: the
// noise, the weights, the candidate and the commit's choice of qs_mppi_update / qs_mppi_commit, mppi.cu) as plain host C++, so
// the `-m "not gpu"` suite can hold them to the float64 restatement tests/mppi_ref.py.  Never linked into or imported by the
// product package.
#include <vector>
#include "../../gym_pybullet_drones_b200/csrc/mppi.cuh"

extern "C" {

void mppi_philox(const uint32_t* ctr, const uint32_t* key, uint32_t* out) { qs::philox4x32_10(ctr, key, out); }

void mppi_box_muller(const uint32_t* w, double* z) { qs::box_muller(w, z[0], z[1]); }

void mppi_eps_host(unsigned long long seed, int k, int s, long long id, int it, double* eps) { qs::mppi_eps(seed, k, s, id, it, eps); }

// qs_mppi_update for one unit with the perturbations given: J [K], delta [K][n] (delta_0 = 0, as the kernel assumes), u [n] ->
// w [K], cand [n]; returns the best sample of the scan
int mppi_update_host(const double* J, int K, double temperature, const double* delta, const double* u, int n, double* w, double* cand) {
    const qs::MppiStats st = qs::mppi_stats([&](int s) { return J[s]; }, K, temperature);
    for (int s = 0; s < K; ++s) w[s] = qs::mppi_weight(J[s], st);
    double wsum = 0.0;
    for (int s = 0; s < K; ++s) wsum += w[s];
    for (int e = 0; e < n; ++e) {
        double num = 0.0;
        for (int s = 1; s < K; ++s) {
            if (w[s] == 0.0) continue;
            num += w[s] * delta[(long long)s * n + e];
        }
        cand[e] = qs::mppi_candidate(u[e], num, wsum);
    }
    return st.best;
}

// qs_mppi_commit's choice for a unit: -1 keeps the candidate of cost jc, else the sample taken
int mppi_commit_host(double jc, const double* J, int K) {
    const qs::MppiStats st = qs::mppi_stats([&](int s) { return J[s]; }, K, 1.0);
    return qs::mppi_take_candidate(jc, J[st.best]) ? -1 : st.best;
}

// mppi_delta / mppi_command of one entry
double mppi_delta_host(double u, double sig, double eps, double lo, double hi, int box) {
    return box ? qs::mppi_delta<true>(u, sig, eps, lo, hi) : qs::mppi_delta<false>(u, sig, eps, lo, hi);
}

}  // extern "C"
