// dyn_lqr_traj.cu -- qs_dyn_lqr_traj / qs_dyn_lqr_traj_vjp: differentiable trajectories of an iLQR plan's time-varying LQR tracker
// around Physics.DYN (include/quadsim.h, DESIGN.md 4.5).  One thread per drone for all T ticks.  The forward is the QS_CTRL_LQR tick
// of ctrl_rollout_kernel (lqr_law.cuh's tracker_command, the env's clip, dyn_tick_k, round_to_planes) in the same order;
// the backward walks the ticks in reverse, reloading each tick's start state and the applied RPMs of the tick before from the
// forward's outputs, and runs dyn_adjoint.cuh's tick adjoint, the two clip adjoints and the law's adjoint.  n_z is a template
// parameter, so dz, the K rows and K^T lambda are registers, never runtime-indexed local arrays.
#include "qs_common.cuh"
#include "dyn_adjoint.cuh"
#include "lqr_law.cuh"
#include "traj_io.cuh"

namespace qsi {
namespace {

constexpr int kLqrTrajTPB = 128;

struct LqrTrajArgs {
    QsParams P;
    QsDynLqrTrajIO io;
    long long N;
    int D, substeps;
};

// lqr_law.cuh's tracker_dz and tracker_command, written out for dyn_lqr_traj_vjp_kernel: through the plan view that kernel, at
// the register cap, took other registers.  The forward kernel calls tracker_command.
template <int NZ>
__device__ __forceinline__ void vjp_dz(const QsDynLqrTrajIO& io, long long N, long long i, long long p, const qs::Drone& d,
                                        const double up[4], double dz[NZ]) {
    const double* zn = io.z_nom + (p * N + i) * NZ;
    const double x[13] = {d.px, d.py, d.pz, d.qx, d.qy, d.qz, d.qw, d.vx, d.vy, d.vz, d.wx, d.wy, d.wz};
#pragma unroll
    for (int q = 0; q < 13; ++q) dz[q] = x[q] - __ldg(zn + q);
    if constexpr (NZ == 17) {
#pragma unroll
        for (int j = 0; j < 4; ++j) dz[13 + j] = up[j] - __ldg(zn + 13 + j);
    }
}

template <int NZ>
__device__ __forceinline__ void vjp_command(const QsDynLqrTrajIO& io, long long N, long long i, long long p, const qs::Drone& d,
                                                const double up[4], double max_rpm, double b[4], bool keep[4], double u[4]) {
    double dz[NZ];
    vjp_dz<NZ>(io, N, i, p, d, up, dz);
    const D4 un = ld256_nc(io.rpm_nom, p * N + i);
    b[0] = un.x; b[1] = un.y; b[2] = un.z; b[3] = un.w;
    const double* Kp = io.K + (p * N + i) * 4 * NZ;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const double* Kj = Kp + j * NZ;
        b[j] += lqr_feedback<NZ>([&](int q) { return __ldg(Kj + q); }, dz);
        keep[j] = true;
    }
    if (io.lo) {
        const long long at = io.per_tick ? p * N + i : i;
        const D4 l4 = ld256_nc(io.lo, at), h4 = ld256_nc(io.hi, at);
        const double lo[4] = {l4.x, l4.y, l4.z, l4.w}, hi[4] = {h4.x, h4.y, h4.z, h4.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            keep[j] = !(b[j] < lo[j]) && !(b[j] > hi[j]);
            b[j] = qs::clampd(b[j], lo[j], hi[j]);
        }
    }
    clip_rpm(b, max_rpm, u);                                                          // CtrlAviary.py:140
}

template <int EFF, int NZ>
__global__ void __launch_bounds__(kLqrTrajTPB) dyn_lqr_traj_kernel(const __grid_constant__ LqrTrajArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long N = a.N;
    if (i >= N) return;
    const QsDynLqrTrajIO& io = a.io;
    const qs::PhysRow c = row_of(a, i);
    qs::Drone d;
    ld_state(io.state0, N, i, d);
    double up[4] = {0, 0, 0, 0}, b[4], u[4];
    bool keep[4];
    if (((EFF & QS_EFFECT_DRAG) || NZ == 17) && io.last_rpm) ld4(io.last_rpm, i, up);
    for (int k = 0; k < io.T; ++k) {
        tracker_command<NZ>(device_plan<NZ>(io, N, i, (long long)io.tick0 + k), d, up, b, keep);
        clip_rpm(b, c.max_rpm, u);                                                    // CtrlAviary.py:140
        double R_last[9];
        qs::dyn_tick_k<EFF>(a.P, c, d, u, up, 0.0, a.substeps, R_last);
        round_to_planes(d);
        st_state(io.states + (long long)k * 13 * N, N, i, d);
        double* o = io.rpm + 4 * ((long long)k * N + i);
#pragma unroll
        for (int j = 0; j < 4; ++j) { o[j] = u[j]; up[j] = u[j]; }
    }
}

template <int EFF, int NZ>
__global__ void __launch_bounds__(kLqrTrajTPB) dyn_lqr_traj_vjp_kernel(const __grid_constant__ LqrTrajArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long N = a.N;
    if (i >= N) return;
    const QsDynLqrTrajIO& io = a.io;
    const qs::PhysRow c = row_of(a, i);
    ScratchRec rec = {io.scratch, N, i};
    qs::PhysGrad G = zero_phys_grad();
    qs::Drone L = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    double Lup_next[4] = {0, 0, 0, 0};     // the cotangent of this tick's applied RPMs from tick k + 1 (drag, and dz with NZ = 17)
    for (int k = io.T - 1; k >= 0; --k) {
        add_state(io.g_states + (long long)k * 13 * N, N, i, L);
        qs::Drone d0;
        ld_state(k == 0 ? io.state0 : io.states + (long long)(k - 1) * 13 * N, N, i, d0);
        double up[4] = {0, 0, 0, 0};
        if ((EFF & QS_EFFECT_DRAG) || NZ == 17) {
            if (k > 0) ld4(io.rpm, (long long)(k - 1) * N + i, up);
            else if (io.last_rpm) ld4(io.last_rpm, i, up);
        }
        const long long p = (long long)io.tick0 + k;
        double b[4], u[4];
        bool keep[4];
        vjp_command<NZ>(io, N, i, p, d0, up, c.max_rpm, b, keep, u);
        double Lu[4] = {Lup_next[0], Lup_next[1], Lup_next[2], Lup_next[3]}, Lup[4] = {0, 0, 0, 0};
        if (io.g_rpm) {
            double gr[4];
            ld4(io.g_rpm, (long long)k * N + i, gr);
#pragma unroll
            for (int j = 0; j < 4; ++j) Lu[j] += gr[j];
        }
        qs::dyn_tick_vjp<EFF>(a.P, c, d0, u, up, a.substeps, rec, L, Lu, Lup, G);
        // the env's clip (gradient to the row's MAX_RPM), then the box as torch.clamp (its bounds are constants)
        double lam[4];
        qs::rpm_clip_vjp(b, c.max_rpm, Lu, lam, G.g[13]);
#pragma unroll
        for (int j = 0; j < 4; ++j) lam[j] = keep[j] ? lam[j] : 0.0;
        // the law's adjoint at plan tick p: dz recomputed here rather than held across the tick's adjoint
        double dz[NZ], Ktl[NZ];
        vjp_dz<NZ>(io, N, i, p, d0, up, dz);
        const long long pi = p * N + i;
        const double* Kp = io.K + pi * 4 * NZ;
        double* gK = io.g_K ? io.g_K + pi * 4 * NZ : nullptr;
        lqr_feedback_vjp<NZ>([&](int j, int q) { return __ldg(Kp + j * NZ + q); }, dz, lam,
                             [&](int j, int q, double g) { if (gK) gK[j * NZ + q] = g; }, Ktl);
        if (io.g_rpm_nom) {
            double* o = io.g_rpm_nom + 4 * pi;
            o[0] = lam[0]; o[1] = lam[1]; o[2] = lam[2]; o[3] = lam[3];
        }
        if (io.g_z_nom) {
            double* o = io.g_z_nom + pi * NZ;
#pragma unroll
            for (int q = 0; q < NZ; ++q) o[q] = -Ktl[q];
        }
        L.px += Ktl[0]; L.py += Ktl[1]; L.pz += Ktl[2]; L.qx += Ktl[3]; L.qy += Ktl[4]; L.qz += Ktl[5]; L.qw += Ktl[6];
        L.vx += Ktl[7]; L.vy += Ktl[8]; L.vz += Ktl[9]; L.wx += Ktl[10]; L.wy += Ktl[11]; L.wz += Ktl[12];
        if constexpr (NZ == 17) {
#pragma unroll
            for (int j = 0; j < 4; ++j) Lup[j] += Ktl[13 + j];
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) Lup_next[j] = Lup[j];
    }
    st_state(io.g_state0, N, i, L);
    store_start_grads(io, i, Lup_next, G);
}

template <bool VJP>
int launch_lqr_traj(const QsParams* p, const QsDynLqrTrajIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                    void* stream, const char* what) {
    if (!p || !io) return fail(QS_ERR_NULL, what, "NULL params / io");
    if (!io->state0 || !io->K || !io->z_nom || !io->rpm_nom || !io->states || !io->rpm)
        return fail(QS_ERR_NULL, what, "NULL state0 / K / z_nom / rpm_nom / states / rpm");
    if (VJP && (!io->g_states || !io->g_state0 || !io->scratch)) return fail(QS_ERR_NULL, what, "NULL g_states / g_state0 / scratch");
    if (int rc = traj_check_sizes(what, n_envs, drones_per_env, substeps, io->T)) return rc;
    if (int rc = traj_check_effects(what, effects, io->phys, nullptr)) return rc;
    if (io->n_z != 13 && io->n_z != 17) return fail(QS_ERR_SIZE, what, "n_z must be 13 or 17");
    if (io->tick0 < 0 || (long long)io->tick0 + io->T > io->T_plan)
        return fail(QS_ERR_SIZE, what, "the ticks [tick0, tick0 + T) must lie in the plan [0, T_plan)");
    if (!io->lo != !io->hi) return fail(QS_ERR_NULL, what, "lo and hi are both given or both NULL");
    if (io->per_tick != 0 && io->per_tick != 1) return fail(QS_ERR_SIZE, what, "per_tick must be 0 or 1");
    if (!aligned32(io->rpm_nom) || (io->lo && (!aligned32(io->lo) || !aligned32(io->hi))))
        return fail(QS_ERR_ALIGN, what, "rpm_nom, lo and hi must be 32-byte aligned");
    LqrTrajArgs a;
    memset(&a, 0, sizeof(a));
    a.P = *p; a.io = *io;
    a.N = (long long)n_envs * drones_per_env;
    a.D = drones_per_env; a.substeps = substeps;
    const unsigned blocks = (unsigned)((a.N + kLqrTrajTPB - 1) / kLqrTrajTPB);
    const bool nz17 = io->n_z == 17;
    return traj_launch(what, effects, [nz17](auto EFF) {
        constexpr int E = decltype(EFF)::value;
        if (VJP) return nz17 ? dyn_lqr_traj_vjp_kernel<E, 17> : dyn_lqr_traj_vjp_kernel<E, 13>;
        return nz17 ? dyn_lqr_traj_kernel<E, 17> : dyn_lqr_traj_kernel<E, 13>;
    }, blocks, kLqrTrajTPB, 0, (cudaStream_t)stream, a);
}

}  // namespace
}  // namespace qsi

using namespace qsi;

extern "C" {

int qs_sizeof_dyn_lqr_traj_io(void) { return (int)sizeof(QsDynLqrTrajIO); }

int qs_dyn_lqr_traj(const QsParams* p, const QsDynLqrTrajIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                    void* stream) {
    return launch_lqr_traj<false>(p, io, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_lqr_traj");
}

int qs_dyn_lqr_traj_vjp(const QsParams* p, const QsDynLqrTrajIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                        void* stream) {
    return launch_lqr_traj<true>(p, io, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_lqr_traj_vjp");
}

}  // extern "C"
