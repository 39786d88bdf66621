// dyn_traj.cu -- qs_dyn_traj / qs_dyn_traj_vjp: differentiable raw-RPM trajectories of Physics.DYN (include/quadsim.h,
// DESIGN.md 4.5).  One thread per drone for all T ticks.  The forward is qs_dyn_substeps(QS_FLAG_ACTION_F64)'s arithmetic
// (dyn_tick_k, then the quaternion rounding of store_drone) tick after tick; the backward walks the ticks in reverse, reloading
// each tick's start state from the forward's output and running dyn_adjoint.cuh's tick adjoint.
#include "qs_common.cuh"
#include "dyn_adjoint.cuh"

namespace qsi {
namespace {

constexpr int kTrajTPB = 128;

struct TrajArgs {
    QsParams P;
    QsDynTrajIO io;
    long long N;
    int D, substeps;
};

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

__device__ __forceinline__ qs::PhysRow row_of(const TrajArgs& a, long long i) {
    return a.io.phys ? load_phys(a.io.phys, i / a.D) : qs::phys_row_of(a.P);
}

__device__ __forceinline__ void clip_rpm(const double raw[4], double max_rpm, double u[4]) {
#pragma unroll
    for (int j = 0; j < 4; ++j) u[j] = qs::clampd(raw[j], 0.0, max_rpm);            // CtrlAviary.py:140
}

template <int EFF>
__global__ void __launch_bounds__(kTrajTPB) dyn_traj_kernel(const __grid_constant__ TrajArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long N = a.N;
    if (i >= N) return;
    const QsDynTrajIO& io = a.io;
    const qs::PhysRow c = row_of(a, i);
    qs::Drone d;
    ld_state(io.state0, N, i, d);
    double up[4] = {0, 0, 0, 0}, u[4], raw[4];
    if ((EFF & QS_EFFECT_DRAG) && io.last_rpm) ld4(io.last_rpm, i, up);
    for (int k = 0; k < io.T; ++k) {
        ld4(io.rpm, (long long)k * N + i, raw);
        clip_rpm(raw, c.max_rpm, u);
        double R_last[9];
        qs::dyn_tick_k<EFF>(a.P, c, d, u, up, 0.0, a.substeps, R_last);
        round_to_planes(d);
        st_state(io.states + (long long)k * 13 * N, N, i, d);
#pragma unroll
        for (int j = 0; j < 4; ++j) up[j] = u[j];
    }
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

template <int EFF>
__global__ void __launch_bounds__(kTrajTPB) dyn_traj_vjp_kernel(const __grid_constant__ TrajArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long N = a.N;
    if (i >= N) return;
    const QsDynTrajIO& io = a.io;
    const qs::PhysRow c = row_of(a, i);
    ScratchRec rec = {io.scratch, N, i};
    qs::PhysGrad G;
#pragma unroll
    for (int j = 0; j < 16; ++j) G.g[j] = 0.0;
    qs::Drone L = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    double Lup_next[4] = {0, 0, 0, 0};          // drag: the cotangent of this tick's clipped RPMs from tick k + 1's first substep
    for (int k = io.T - 1; k >= 0; --k) {
        qs::Drone g;
        ld_state(io.g_states + (long long)k * 13 * N, N, i, g);
        L.px += g.px; L.py += g.py; L.pz += g.pz; L.qx += g.qx; L.qy += g.qy; L.qz += g.qz; L.qw += g.qw;
        L.vx += g.vx; L.vy += g.vy; L.vz += g.vz; L.wx += g.wx; L.wy += g.wy; L.wz += g.wz;
        qs::Drone d0;
        ld_state(k == 0 ? io.state0 : io.states + (long long)(k - 1) * 13 * N, N, i, d0);
        double raw[4], u[4], up[4] = {0, 0, 0, 0};
        ld4(io.rpm, (long long)k * N + i, raw);
        clip_rpm(raw, c.max_rpm, u);
        if (EFF & QS_EFFECT_DRAG) {
            if (k > 0) {
                double rp[4];
                ld4(io.rpm, (long long)(k - 1) * N + i, rp);
                clip_rpm(rp, c.max_rpm, up);
            } else if (io.last_rpm) {
                ld4(io.last_rpm, i, up);
            }
        }
        double Lu[4] = {Lup_next[0], Lup_next[1], Lup_next[2], Lup_next[3]}, Lup[4] = {0, 0, 0, 0};
        qs::dyn_tick_vjp<EFF>(a.P, c, d0, u, up, a.substeps, rec, L, Lu, Lup, G);
        double gr[4];
        qs::rpm_clip_vjp(raw, c.max_rpm, Lu, gr, G.g[13]);
        double* o = io.g_rpm + 4 * ((long long)k * N + i);
        o[0] = gr[0]; o[1] = gr[1]; o[2] = gr[2]; o[3] = gr[3];
#pragma unroll
        for (int j = 0; j < 4; ++j) Lup_next[j] = Lup[j];
    }
    st_state(io.g_state0, N, i, L);
    if (io.g_last_rpm) {
        double* o = io.g_last_rpm + 4 * i;
        o[0] = Lup_next[0]; o[1] = Lup_next[1]; o[2] = Lup_next[2]; o[3] = Lup_next[3];
    }
    if (io.g_phys) {
        double* o = io.g_phys + 16 * i;
#pragma unroll
        for (int j = 0; j < 16; ++j) o[j] = G.g[j];
    }
}

template <bool VJP>
int launch_traj(const QsParams* p, const QsDynTrajIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                void* stream, const char* what) {
    if (!p || !io) return fail(QS_ERR_NULL, VJP ? "qs_dyn_traj_vjp: NULL params / io" : "qs_dyn_traj: NULL params / io");
    if (!io->state0 || !io->rpm || !io->states) return fail(QS_ERR_NULL, "qs_dyn_traj: NULL state0 / rpm / states");
    if (VJP && (!io->g_states || !io->g_rpm || !io->g_state0 || !io->scratch))
        return fail(QS_ERR_NULL, "qs_dyn_traj_vjp: NULL g_states / g_rpm / g_state0 / scratch");
    if (n_envs <= 0 || drones_per_env <= 0 || substeps <= 0 || io->T <= 0)
        return fail(QS_ERR_SIZE, "qs_dyn_traj: n_envs, drones_per_env, substeps and T must be > 0");
    if ((long long)n_envs * drones_per_env > 0x7fffffffLL) return fail(QS_ERR_SIZE, "qs_dyn_traj: n_envs * drones_per_env exceeds 2^31-1");
    if (effects & ~7u) return fail(QS_ERR_ENUM, "qs_dyn_traj: bad effects");
    if (effects & QS_EFFECT_DW) return fail(QS_ERR_UNSUPPORTED, "qs_dyn_traj: downwash couples the drones pairwise and has no adjoint here");
    if (io->phys && !aligned16(io->phys)) return fail(QS_ERR_ALIGN, "qs_dyn_traj: phys rows must be 16-byte aligned");
    TrajArgs a;
    memset(&a, 0, sizeof(a));
    a.P = *p; a.io = *io;
    a.N = (long long)n_envs * drones_per_env;
    a.D = drones_per_env; a.substeps = substeps;
    const unsigned blocks = (unsigned)((a.N + kTrajTPB - 1) / kTrajTPB);
    cudaStream_t s = (cudaStream_t)stream;
    // the checks above leave TrajEffects only (no bit above 7, no DW)
    with_int(TrajEffects{}, (int)effects, [&](auto EFF) {
        auto* k = VJP ? dyn_traj_vjp_kernel<decltype(EFF)::value> : dyn_traj_kernel<decltype(EFF)::value>;
        k<<<blocks, kTrajTPB, 0, s>>>(a);
    });
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, what);
}

}  // namespace
}  // namespace qsi

using namespace qsi;

extern "C" {

int qs_sizeof_dyn_traj_io(void) { return (int)sizeof(QsDynTrajIO); }

int qs_dyn_traj(const QsParams* p, const QsDynTrajIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects, void* stream) {
    return launch_traj<false>(p, io, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_traj launch");
}

int qs_dyn_traj_vjp(const QsParams* p, const QsDynTrajIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                    void* stream) {
    return launch_traj<true>(p, io, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_traj_vjp launch");
}

}  // extern "C"
