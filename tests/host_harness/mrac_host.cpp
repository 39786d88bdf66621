// TEST INFRASTRUCTURE: compiles gym_pybullet_drones_b200/csrc/mrac_core.cuh (the MRAC math of the CUDA kernels) as plain host
// C++ so the `-m "not gpu"` suite can check it against the reference's fixtures and the NumPy oracle.  The adaptive state keeps
// the kernels' layout: [76][n] float64 planes.  Never linked into or imported by the product package.
#include <cmath>
#include "../../gym_pybullet_drones_b200/csrc/mrac_core.cuh"

extern "C" {
// MRAC.computeControl for n drones (qs_mrac_control on the host): pos / vel / ang_v [n][3], quat [n][4], r [n][12] targets;
// rpm [n][4], pos_e / rpy_e [n][3] float64 out; state [76][n] in/out
void hh_mrac(const QsMracParams* M, double* state, int n, int init, double dt, const double* pos, const double* quat,
             const double* vel, const double* angv, const double* r, double* rpm, double* pos_e, double* rpy_e) {
    for (long long i = 0; i < n; ++i) {
        const qs::MracState S = {state + i, n};
        qs::mrac_control(*M, S, init != 0, dt, pos + 3 * i, quat + 4 * i, vel + 3 * i, angv + 3 * i, r + 12 * i, rpm + 4 * i,
                         pos_e + 3 * i, rpy_e + 3 * i);
    }
}
// the state vector's ang_v as the kernels rebuild it from the planes: quat [n][4], w [n][3] -> ang_v [n][3]
void hh_mrac_ang_v(const double* quat, const double* w, int n, double* out) {
    for (int i = 0; i < n; ++i) {
        qs::Drone d = {0, 0, 0, quat[4 * i], quat[4 * i + 1], quat[4 * i + 2], quat[4 * i + 3], 0, 0, 0, w[3 * i], w[3 * i + 1], w[3 * i + 2]};
        qs::mrac_ang_v(d, out + 3 * i);
    }
}
int hh_sizeof_mrac_params(void) { return (int)sizeof(QsMracParams); }
}
