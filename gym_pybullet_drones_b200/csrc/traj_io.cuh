// traj_io.cuh -- device-side loads and stores of the differentiable-trajectory kernels (dyn_traj.cu, dyn_ctrl_traj.cu): states
// in the planes layout and the substep record of the tick adjoint.
#pragma once
#include "qs_common.cuh"

namespace qsi {
namespace {

// A state of 13 N doubles in the planes layout.  Plain 8-byte accesses: entry k of a trajectory starts at 13 k N doubles, which
// is not 16-byte aligned for odd N.
__device__ __forceinline__ void ld_state(const double* s, long long N, long long i, qs::Drone& d) {
    d.px = s[4 * i]; d.py = s[4 * i + 1]; d.pz = s[4 * i + 2]; d.wx = s[4 * i + 3];
    d.qx = s[4 * (N + i)]; d.qy = s[4 * (N + i) + 1]; d.qz = s[4 * (N + i) + 2]; d.qw = s[4 * (N + i) + 3];
    d.vx = s[4 * (2 * N + i)]; d.vy = s[4 * (2 * N + i) + 1]; d.vz = s[4 * (2 * N + i) + 2]; d.wy = s[4 * (2 * N + i) + 3];
    d.wz = s[12 * N + i];
}
__device__ __forceinline__ void st_state(double* s, long long N, long long i, const qs::Drone& d) {
    s[4 * i] = d.px; s[4 * i + 1] = d.py; s[4 * i + 2] = d.pz; s[4 * i + 3] = d.wx;
    s[4 * (N + i)] = d.qx; s[4 * (N + i) + 1] = d.qy; s[4 * (N + i) + 2] = d.qz; s[4 * (N + i) + 3] = d.qw;
    s[4 * (2 * N + i)] = d.vx; s[4 * (2 * N + i) + 1] = d.vy; s[4 * (2 * N + i) + 2] = d.vz; s[4 * (2 * N + i) + 3] = d.wy;
    s[12 * N + i] = d.wz;
}
__device__ __forceinline__ void ld4(const double* p, long long i, double v[4]) {
    v[0] = p[4 * i]; v[1] = p[4 * i + 1]; v[2] = p[4 * i + 2]; v[3] = p[4 * i + 3];
}

// the substep states of one tick in the caller's [S][13][N] scratch
struct ScratchRec {
    double* base;
    long long N, i;
    __device__ void store(int s, const qs::Drone& d) const {
        double* p = base + (long long)s * 13 * N + i;
        p[0] = d.px; p[N] = d.py; p[2 * N] = d.pz; p[3 * N] = d.qx; p[4 * N] = d.qy; p[5 * N] = d.qz; p[6 * N] = d.qw;
        p[7 * N] = d.vx; p[8 * N] = d.vy; p[9 * N] = d.vz; p[10 * N] = d.wx; p[11 * N] = d.wy; p[12 * N] = d.wz;
    }
    __device__ void load(int s, qs::Drone& d) const {
        const double* p = base + (long long)s * 13 * N + i;
        d.px = p[0]; d.py = p[N]; d.pz = p[2 * N]; d.qx = p[3 * N]; d.qy = p[4 * N]; d.qz = p[5 * N]; d.qw = p[6 * N];
        d.vx = p[7 * N]; d.vy = p[8 * N]; d.vz = p[9 * N]; d.wx = p[10 * N]; d.wy = p[11 * N]; d.wz = p[12 * N];
    }
};

}  // namespace
}  // namespace qsi
