// dyn_jvp.cu -- qs_dyn_traj_jvp / qs_dyn_tick_jac: forward mode of the raw-RPM trajectories of qs_dyn_traj (include/quadsim.h,
// DESIGN.md 4.5) on dyn_tangent.cuh's tick tangent.  Tick k restarts its primal from the forward's stored state k-1, as
// qs_dyn_traj_vjp does, so the trajectory is linearised at the forward's bits and no substep record is needed.
//   dyn_traj_jvp_kernel<EFF>: one thread per drone for all T ticks, the tangent carried in registers.
//   dyn_tick_jac_kernel<EFF>: one thread per (tick, drone, column), the tick's tangent along one unit input.
#include "qs_common.cuh"
#include "dyn_tangent.cuh"
#include "traj_io.cuh"

namespace qsi {
namespace {

constexpr int kJvpTPB = 128;

struct JvpArgs {
    QsParams P;
    QsDynTrajJvpIO io;
    long long N;
    int D, substeps;
};

template <int EFF>
__global__ void __launch_bounds__(kJvpTPB) dyn_traj_jvp_kernel(const __grid_constant__ JvpArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long N = a.N;
    if (i >= N) return;
    const QsDynTrajJvpIO& io = a.io;
    const qs::PhysRow c = row_of(a, i), tc = t_row_of(a, i);
    qs::Drone t = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (io.t_state0) ld_state(io.t_state0, N, i, t);
    double tup[4] = {0, 0, 0, 0};          // drag: the tangent of the previous tick's clipped RPMs
    if ((EFF & QS_EFFECT_DRAG) && io.t_last_rpm) ld4(io.t_last_rpm, i, tup);
    for (int k = 0; k < io.T; ++k) {
        qs::Drone d;
        double raw[4], u[4], up[4], t_raw[4] = {0, 0, 0, 0}, tu[4];
        tick_inputs<EFF>(a, c.max_rpm, i, k, d, raw, u, up);
        if (io.t_rpm) ld4(io.t_rpm, (long long)k * N + i, t_raw);
        qs::rpm_clip_jvp(raw, c.max_rpm, t_raw, tc.max_rpm, tu);
        qs::dyn_tick_jvp<EFF>(a.P, c, tc, d, u, up, a.substeps, t, tu, tup);
        st_state(io.t_states + (long long)k * 13 * N, N, i, t);
#pragma unroll
        for (int j = 0; j < 4; ++j) tup[j] = tu[j];
    }
}

// columns of one tick's Jacobian: the 13 state components, the 4 raw RPMs and, with drag, the 4 previous clipped RPMs
constexpr int jac_cols(unsigned effects) { return (effects & QS_EFFECT_DRAG) ? 21 : 17; }

template <int EFF>
__global__ void __launch_bounds__(kJvpTPB) dyn_tick_jac_kernel(const __grid_constant__ JvpArgs a) {
    constexpr int C = (EFF & QS_EFFECT_DRAG) ? 21 : 17;
    const long long N = a.N;
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;      // = ((k N + i) C + col): the output's own order
    if (g >= (long long)a.io.T * N * C) return;
    const long long ki = g / C;
    const int col = (int)(g - ki * C);
    const int k = (int)(ki / N);
    const long long i = ki - (long long)k * N;
    const qs::PhysRow c = row_of(a, i), tc = t_row_of(a, i);       // t_phys is NULL: the constants carry no tangent here
    qs::Drone d;
    double raw[4], u[4], up[4];
    tick_inputs<EFF>(a, c.max_rpm, i, k, d, raw, u, up);
    // the unit tangent of column col
    qs::Drone t = {col == 0 ? 1.0 : 0.0, col == 1 ? 1.0 : 0.0, col == 2 ? 1.0 : 0.0, col == 3 ? 1.0 : 0.0, col == 4 ? 1.0 : 0.0,
                   col == 5 ? 1.0 : 0.0, col == 6 ? 1.0 : 0.0, col == 7 ? 1.0 : 0.0, col == 8 ? 1.0 : 0.0, col == 9 ? 1.0 : 0.0,
                   col == 10 ? 1.0 : 0.0, col == 11 ? 1.0 : 0.0, col == 12 ? 1.0 : 0.0};
    double t_raw[4], tup[4], tu[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) { t_raw[j] = col == 13 + j ? 1.0 : 0.0; tup[j] = col == 17 + j ? 1.0 : 0.0; }
    qs::rpm_clip_jvp(raw, c.max_rpm, t_raw, 0.0, tu);
    qs::dyn_tick_jvp<EFF>(a.P, c, tc, d, u, up, a.substeps, t, tu, tup);
    double* o = a.io.jac + g + 12LL * C * ki;                      // ((k N + i) 13 + r) C + col at r = 0
    o[0] = t.px; o[C] = t.py; o[2 * C] = t.pz; o[3 * C] = t.qx; o[4 * C] = t.qy; o[5 * C] = t.qz; o[6 * C] = t.qw;
    o[7 * C] = t.vx; o[8 * C] = t.vy; o[9 * C] = t.vz; o[10 * C] = t.wx; o[11 * C] = t.wy; o[12 * C] = t.wz;
}

template <bool JAC>
int launch_jvp(const QsParams* p, const QsDynTrajJvpIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
               void* stream, const char* what) {
    if (!p || !io) return fail(QS_ERR_NULL, what, "NULL params / io");
    if (!io->state0 || !io->rpm || !io->states) return fail(QS_ERR_NULL, what, "NULL state0 / rpm / states");
    if (JAC ? !io->jac : !io->t_states) return fail(QS_ERR_NULL, what, JAC ? "NULL jac" : "NULL t_states");
    if (int rc = traj_check_sizes(what, n_envs, drones_per_env, substeps, io->T)) return rc;
    if (int rc = traj_check_effects(what, effects, io->phys, io->t_phys)) return rc;
    const long long N = (long long)n_envs * drones_per_env;
    const long long threads = JAC ? (long long)io->T * N * jac_cols(effects) : N;
    const long long blocks = (threads + kJvpTPB - 1) / kJvpTPB;
    if (blocks > 0x7fffffffLL) return fail(QS_ERR_SIZE, what, "T * N * columns exceeds 2^31-1 CTAs of 128 threads");
    JvpArgs a;
    memset(&a, 0, sizeof(a));
    a.P = *p; a.io = *io;
    if (JAC) a.io.t_phys = nullptr;                                  // the Jacobian's columns are the state and RPM inputs only
    a.N = N;
    a.D = drones_per_env; a.substeps = substeps;
    return traj_launch(what, effects, [](auto EFF) {
        return JAC ? dyn_tick_jac_kernel<decltype(EFF)::value> : dyn_traj_jvp_kernel<decltype(EFF)::value>;
    }, (unsigned)blocks, kJvpTPB, 0, (cudaStream_t)stream, a);
}

}  // namespace
}  // namespace qsi

using namespace qsi;

extern "C" {

int qs_sizeof_dyn_traj_jvp_io(void) { return (int)sizeof(QsDynTrajJvpIO); }

int qs_dyn_traj_jvp(const QsParams* p, const QsDynTrajJvpIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                    void* stream) {
    return launch_jvp<false>(p, io, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_traj_jvp");
}

int qs_dyn_tick_jac(const QsParams* p, const QsDynTrajJvpIO* io, int n_envs, int drones_per_env, int substeps, unsigned effects,
                    void* stream) {
    return launch_jvp<true>(p, io, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_tick_jac");
}

}  // extern "C"
