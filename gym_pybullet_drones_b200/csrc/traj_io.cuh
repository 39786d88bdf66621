// traj_io.cuh -- what the differentiable-trajectory translation units (dyn_traj.cu, dyn_ctrl_traj.cu, dyn_policy_traj.cu,
// dyn_jvp.cu, dyn_ctrl_jvp.cu, dyn_dw_traj.cu) and the planners (ilqr.cu, mppi.cu) share: device-side loads and stores of states
// in the planes layout, a box's row, the substep record of the tick adjoint, the per-drone inputs and outputs of a tick, the
// downwash CTA's groups, and on the host the argument checks and the launch over an effect list.
#pragma once
#include "qs_common.cuh"
#include "lqr_law.cuh"

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
// the index of state component j (drone_vec's order: pos, quat x y z w, vel, rpy_rates) of drone i in a state of 13 N doubles
__device__ __forceinline__ long long plane_at(long long N, long long i, int j) {
    if (j < 3) return 4 * i + j;
    if (j < 7) return 4 * (N + i) + (j - 3);
    if (j < 10) return 4 * (2 * N + i) + (j - 7);
    if (j == 10) return 4 * i + 3;
    if (j == 11) return 4 * (2 * N + i) + 3;
    return 12 * N + i;
}
// L += entry i of a stored [13 N] cotangent
__device__ __forceinline__ void add_state(const double* s, long long N, long long i, qs::Drone& L) {
    qs::Drone g;
    ld_state(s, N, i, g);
    L.px += g.px; L.py += g.py; L.pz += g.pz; L.qx += g.qx; L.qy += g.qy; L.qz += g.qz; L.qw += g.qw;
    L.vx += g.vx; L.vy += g.vy; L.vz += g.vz; L.wx += g.wx; L.wy += g.wy; L.wz += g.wz;
}
__device__ __forceinline__ void ld4(const double* p, long long i, double v[4]) {
    v[0] = p[4 * i]; v[1] = p[4 * i + 1]; v[2] = p[4 * i + 2]; v[3] = p[4 * i + 3];
}
// the box [lo, hi] of the raw command of drone i at tick k: row box_row(per_tick, k, N, i) of rpm_lo and rpm_hi
__device__ __forceinline__ void ld_box(const double* rpm_lo, const double* rpm_hi, int per_tick, int k, long long N, long long i,
                                       double lo[4], double hi[4]) {
    const long long at = box_row(per_tick, k, N, i);
    ld4(rpm_lo, at, lo);
    ld4(rpm_hi, at, hi);
}

// The constants of drone i (a.D drones per aviary): its aviary's row of `phys`, or where `phys` is NULL what `fallback()` returns
template <class Args, class Fallback>
__device__ __forceinline__ qs::PhysRow aviary_row(const Args& a, const double* phys, long long i, Fallback fallback) {
    if (phys) return load_phys(phys, i / a.D);
    return fallback();
}
// the row of a.io.phys, or the constants of a.P
template <class Args>
__device__ __forceinline__ qs::PhysRow row_of(const Args& a, long long i) {
    return aviary_row(a, a.io.phys, i, [&] { return qs::phys_row_of(a.P); });
}
// the tangent of the constants (forward mode): the row of a.io.t_phys, or zero
template <class Args>
__device__ __forceinline__ qs::PhysRow t_row_of(const Args& a, long long i) {
    return aviary_row(a, a.io.t_phys, i, [] {
        qs::PhysRow z;
        z.inv_m = z.gravity = z.kf = z.km = z.kx = z.ky = z.hover_rpm = z.max_rpm = 0.0;
        for (int k = 0; k < 3; ++k) z.j[k] = z.j_inv[k] = 0.0;
        return z;
    });
}

__device__ __forceinline__ void clip_rpm(const double raw[4], double max_rpm, double u[4]) {
#pragma unroll
    for (int j = 0; j < 4; ++j) u[j] = qs::clampd(raw[j], 0.0, max_rpm);            // CtrlAviary.py:140
}

__device__ __forceinline__ qs::PhysGrad zero_phys_grad() {
    qs::PhysGrad G;
#pragma unroll
    for (int j = 0; j < 16; ++j) G.g[j] = 0.0;
    return G;
}

// The primal inputs of tick k of drone i of a raw-RPM trajectory (a.io a QsDynTrajIO or QsDynTrajJvpIO): the stored start state,
// the raw and clipped RPMs and drag's previous clipped RPMs
template <int EFF, class Args>
__device__ __forceinline__ void tick_inputs(const Args& a, double max_rpm, long long i, int k, qs::Drone& d, double raw[4], double u[4],
                                            double up[4]) {
    const auto& io = a.io;
    const long long N = a.N;
    ld_state(k == 0 ? io.state0 : io.states + (long long)(k - 1) * 13 * N, N, i, d);
    ld4(io.rpm, (long long)k * N + i, raw);
    clip_rpm(raw, max_rpm, u);
    up[0] = up[1] = up[2] = up[3] = 0.0;
    if (EFF & QS_EFFECT_DRAG) {
        if (k > 0) {
            double rp[4];
            ld4(io.rpm, (long long)(k - 1) * N + i, rp);
            clip_rpm(rp, max_rpm, up);
        } else if (io.last_rpm) {
            ld4(io.last_rpm, i, up);
        }
    }
}

// The end of a VJP kernel after its g_state0: the cotangents of drag's RPMs before tick 0 (g_last_rpm) and of the drone's
// constants (g_phys), each where the caller asked for it
template <class IO>
__device__ __forceinline__ void store_start_grads(const IO& io, long long i, const double Lup[4], const qs::PhysGrad& G) {
    if (io.g_last_rpm) {
        double* o = io.g_last_rpm + 4 * i;
        o[0] = Lup[0]; o[1] = Lup[1]; o[2] = Lup[2]; o[3] = Lup[3];
    }
    if (io.g_phys) {
        double* o = io.g_phys + 16 * i;
#pragma unroll
        for (int j = 0; j < 16; ++j) o[j] = G.g[j];
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

// The downwash CTA (whole groups of a.D drones in its first a.tpb threads) and thread t's group in it: the unit index G (aviary,
// or aviary * K + sample for mppi's sample kernel), the first thread b of the group, the drone q of the group, and whether t holds
// a drone of a live group
struct DwSlot {
    long long G;
    int b, q;
    bool live;
};
template <class Args>
__device__ __forceinline__ DwSlot dw_slot(const Args& a, long long groups) {
    const int t = threadIdx.x, g = t / a.D;
    DwSlot sl;
    sl.G = (long long)blockIdx.x * (a.tpb / a.D) + g;
    sl.b = g * a.D;
    sl.q = t - sl.b;
    sl.live = t < a.tpb && sl.G < groups;
    return sl;
}

// ---- host: the checks every entry point makes, in this order around its own, and the launch.  `what` is the entry point's name.
inline int traj_check_sizes(const char* what, int n_envs, int drones_per_env, int substeps, int T) {
    if (n_envs <= 0 || drones_per_env <= 0 || substeps <= 0 || T <= 0)
        return fail(QS_ERR_SIZE, what, "n_envs, drones_per_env, substeps and T must be > 0");
    if ((long long)n_envs * drones_per_env > 0x7fffffffLL) return fail(QS_ERR_SIZE, what, "n_envs * drones_per_env exceeds 2^31-1");
    return 0;
}
// leaves TrajEffects only, or with `dw` PlanEffects: no bit above 7, downwash only where allowed and then only alone or with both
inline int traj_check_effects(const char* what, unsigned effects, const double* phys, const double* t_phys, bool dw = false) {
    if (effects & ~7u) return fail(QS_ERR_ENUM, what, "bad effects");
    if (!dw && (effects & QS_EFFECT_DW))
        return fail(QS_ERR_UNSUPPORTED, what, "downwash couples the drones pairwise and has no derivative here");
    if (dw && !with_int(PlanEffects{}, (int)effects, [](auto) {}))
        return fail(QS_ERR_UNSUPPORTED, what, "supports no DYN+ effect, GND, DRAG, GND|DRAG, DW or all three");
    if (phys && !aligned16(phys)) return fail(QS_ERR_ALIGN, what, "phys rows must be 16-byte aligned");
    if (t_phys && !aligned16(t_phys)) return fail(QS_ERR_ALIGN, what, "t_phys rows must be 16-byte aligned");
    return 0;
}
// pick(EFF)<<<blocks, threads, smem, s>>>(a) for the checked effect set of the list Effects; above 48 KB of shared memory the
// kernel's limit is raised first
template <class Effects = TrajEffects, class Pick, class Args>
int traj_launch(const char* what, unsigned effects, Pick pick, unsigned blocks, int threads, size_t smem, cudaStream_t s, const Args& a) {
    cudaError_t e = cudaSuccess;
    with_int(Effects{}, (int)effects, [&](auto EFF) {
        auto* k = pick(EFF);
        if (smem > 48 * 1024) e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess) k<<<blocks, threads, smem, s>>>(a);
    });
    if (e == cudaSuccess) e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, what);
}

}  // namespace
}  // namespace qsi
