// dyn_traj.cu -- qs_dyn_traj / qs_dyn_traj_vjp: differentiable raw-RPM trajectories of Physics.DYN (include/quadsim.h,
// DESIGN.md 4.5).  One thread per drone for all T ticks.  The forward is qs_dyn_substeps(QS_FLAG_ACTION_F64)'s arithmetic
// (dyn_tick_k, then the quaternion rounding of store_drone) tick after tick; the backward walks the ticks in reverse, reloading
// each tick's start state from the forward's output and running dyn_adjoint.cuh's tick adjoint.
#include "qs_common.cuh"
#include "dyn_adjoint.cuh"
#include "traj_io.cuh"

namespace qsi {
namespace {

constexpr int kTrajTPB = 128;

struct TrajArgs {
    QsParams P;
    QsDynTrajIO io;
    long long N;
    int D, substeps;
};

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

template <int EFF>
__global__ void __launch_bounds__(kTrajTPB) dyn_traj_vjp_kernel(const __grid_constant__ TrajArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long N = a.N;
    if (i >= N) return;
    const QsDynTrajIO& io = a.io;
    const qs::PhysRow c = row_of(a, i);
    ScratchRec rec = {io.scratch, N, i};
    qs::PhysGrad G = zero_phys_grad();
    qs::Drone L = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    double Lup_next[4] = {0, 0, 0, 0};          // drag: the cotangent of this tick's clipped RPMs from tick k + 1's first substep
    for (int k = io.T - 1; k >= 0; --k) {
        // add_state and tick_inputs written out: through the helpers ptxas allocates this kernel's registers differently
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
    store_start_grads(io, i, Lup_next, G);
}

template <bool VJP>
int launch_traj(const QsParams* p, const QsDynTrajIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                void* stream, const char* what) {
    if (!p || !io) return fail(QS_ERR_NULL, what, "NULL params / io");
    if (!io->state0 || !io->rpm || !io->states) return fail(QS_ERR_NULL, what, "NULL state0 / rpm / states");
    if (VJP && (!io->g_states || !io->g_rpm || !io->g_state0 || !io->scratch))
        return fail(QS_ERR_NULL, what, "NULL g_states / g_rpm / g_state0 / scratch");
    if (int rc = traj_check_sizes(what, n_envs, drones_per_env, substeps, io->T)) return rc;
    if (int rc = traj_check_effects(what, effects, io->phys, nullptr)) return rc;
    TrajArgs a;
    memset(&a, 0, sizeof(a));
    a.P = *p; a.io = *io;
    a.N = (long long)n_envs * drones_per_env;
    a.D = drones_per_env; a.substeps = substeps;
    const unsigned blocks = (unsigned)((a.N + kTrajTPB - 1) / kTrajTPB);
    return traj_launch(what, effects, [](auto EFF) {
        return VJP ? dyn_traj_vjp_kernel<decltype(EFF)::value> : dyn_traj_kernel<decltype(EFF)::value>;
    }, blocks, kTrajTPB, 0, (cudaStream_t)stream, a);
}

}  // namespace
}  // namespace qsi

using namespace qsi;

extern "C" {

int qs_sizeof_dyn_traj_io(void) { return (int)sizeof(QsDynTrajIO); }

int qs_dyn_traj(const QsParams* p, const QsDynTrajIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects, void* stream) {
    return launch_traj<false>(p, io, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_traj");
}

int qs_dyn_traj_vjp(const QsParams* p, const QsDynTrajIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                    void* stream) {
    return launch_traj<true>(p, io, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_traj_vjp");
}

}  // extern "C"
