// dyn_ctrl_jvp.cu -- qs_dyn_ctrl_traj_jvp / qs_dyn_ctrl_tick_jac: forward mode of the closed-loop trajectories of qs_dyn_ctrl_traj
// (include/quadsim.h, DESIGN.md 4.5) on pid_tangent.cuh's controller tangent and dyn_tangent.cuh's tick tangent.  Tick k restarts
// its primal from the forward's stored state k-1 and controller state pid_states[k], as qs_dyn_ctrl_traj_vjp does, so the loop is
// linearised at the forward's bits and nothing is recorded.
//   dyn_ctrl_traj_jvp_kernel<EFF>: one thread per drone for all T ticks, the tangent carried in registers.
//   dyn_ctrl_tick_jac_kernel<EFF>: one thread per (tick, drone, column), the tick's tangent along one unit input.
#include "qs_common.cuh"
#include "pid_tangent.cuh"
#include "ctrl_io.cuh"

namespace qsi {
namespace {

constexpr int kCtrlJvpTPB = 128;

struct CtrlJvpArgs {
    QsParams P;          // the env: physics, MAX_RPM clip
    QsParams CP;         // the DSLPIDControl's own constants
    QsDynCtrlTrajJvpIO io;
    long long N;
    int D, substeps;
};

// the tangent of drone i's gain set: its aviary's row of io.t_gains, or zero
__device__ __forceinline__ qs::PidGains t_gains_of(const CtrlJvpArgs& a, long long i) {
    if (a.io.t_gains) return gains_row(a.io.t_gains + 18 * (i / a.D));
    qs::PidGains z;
#pragma unroll
    for (int c = 0; c < 3; ++c) z.pid_p_for[c] = z.pid_i_for[c] = z.pid_d_for[c] = z.pid_p_tor[c] = z.pid_i_tor[c] = z.pid_d_tor[c] = 0.0;
    return z;
}

// The primal inputs of tick k of drone i: the stored start state d, the controller state st the tick starts from, the targets,
// the raw / controller-clipped / applied RPMs and drag's previous applied RPMs up
template <int EFF>
__device__ __forceinline__ void ctrl_tick_inputs(const CtrlJvpArgs& a, const qs::PidGains& K, const qs::PhysRow& c, long long i, int k,
                                                 qs::Drone& d, qs::PidState& st, qs::PidTargets& t, double raw[4], double u1[4],
                                                 double u[4], double up[4]) {
    const QsDynCtrlTrajJvpIO& io = a.io;
    const long long N = a.N;
    ld_state(k == 0 ? io.state0 : io.states + (long long)(k - 1) * 13 * N, N, i, d);
    load_pid(io.pid_states + (long long)k * 9 * N, N, i, st);
    t = targets_of(io, N, i, k);
    {
        qs::PidState s = st;
        control(a, K, s, d, t, c.max_rpm, raw, u1, u);
    }
    up[0] = up[1] = up[2] = up[3] = 0.0;
    if (EFF & QS_EFFECT_DRAG) {
        if (k > 0) ld4(io.rpm, (long long)(k - 1) * N + i, up);
        else if (io.last_rpm) ld4(io.last_rpm, i, up);
    }
}

// The tangent of one closed-loop tick: the controller, its max_rpm clip (a constant of the controller), the env's clip (the row's
// MAX_RPM, tangent tc.max_rpm) and the physics.  In: t (the stored start state), t_st (the controller state), t_up (drag's
// previous applied RPMs).  Out: t (the end state), t_st (the updated controller state), t_u (the applied RPMs).
template <int EFF>
__device__ __forceinline__ void ctrl_tick_jvp(const CtrlJvpArgs& a, const qs::PidGains& K, const qs::PhysRow& c, const qs::PhysRow& tc,
                                              qs::Drone& d, const qs::PidState& st, const qs::PidTargets& t, const double raw[4],
                                              const double u1[4], const double u[4], const double up[4], const qs::PidGains& tK,
                                              const qs::PidTargets& t_t, qs::Drone& td, qs::PidState& t_st, const double t_up[4],
                                              double t_u[4]) {
    double t_raw[4], t_u1[4];
    qs::PidState t_new;
    qs::pid_control_jvp(a.CP, K, st, a.io.control_timestep, d, t, tK, t_st, td, t_t, t_raw, t_new);
    t_st = t_new;
    qs::rpm_clip_jvp(raw, a.CP.max_rpm, t_raw, 0.0, t_u1);
    qs::rpm_clip_jvp(u1, c.max_rpm, t_u1, tc.max_rpm, t_u);
    qs::dyn_tick_jvp<EFF>(a.P, c, tc, d, u, up, a.substeps, td, t_u, t_up);
}

template <int EFF>
__global__ void __launch_bounds__(kCtrlJvpTPB) dyn_ctrl_traj_jvp_kernel(const __grid_constant__ CtrlJvpArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long N = a.N;
    if (i >= N) return;
    const QsDynCtrlTrajJvpIO& io = a.io;
    const qs::PhysRow c = row_of(a, i), tc = t_row_of(a, i);
    const qs::PidGains K = gains_of(a, i);
    const qs::PidGains tK = t_gains_of(a, i);
    qs::Drone td = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (io.t_state0) ld_state(io.t_state0, N, i, td);
    qs::PidState t_st = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (io.t_pid0) load_pid(io.t_pid0, N, i, t_st);
    double t_up[4] = {0, 0, 0, 0};          // drag: the tangent of the previous tick's applied RPMs
    if ((EFF & QS_EFFECT_DRAG) && io.t_last_rpm) ld4(io.t_last_rpm, i, t_up);
    for (int k = 0; k < io.T; ++k) {
        qs::Drone d;
        qs::PidState st;
        qs::PidTargets t;
        double raw[4], u1[4], u[4], up[4], t_u[4];
        ctrl_tick_inputs<EFF>(a, K, c, i, k, d, st, t, raw, u1, u, up);
        const qs::PidTargets t_t = targets_from(io.t_target_pos, io.t_target_vel, io.t_target_rpy, io.t_target_rpy_rates, N, i, k);
        ctrl_tick_jvp<EFF>(a, K, c, tc, d, st, t, raw, u1, u, up, tK, t_t, td, t_st, t_up, t_u);
        st_state(io.t_states + (long long)k * 13 * N, N, i, td);
        double* o = io.t_rpm + 4 * ((long long)k * N + i);
#pragma unroll
        for (int j = 0; j < 4; ++j) { o[j] = t_u[j]; t_up[j] = t_u[j]; }
    }
}

// columns of one tick's Jacobian: x_k (13), s_k (9), with drag u_{k-1} (4), target_pos[k] (3); rows x_{k+1} (13), s_{k+1} (9), u_k (4)
constexpr int ctrl_jac_cols(unsigned effects) { return (effects & QS_EFFECT_DRAG) ? 29 : 25; }
constexpr int kCtrlJacRows = 26;

template <int EFF>
__global__ void __launch_bounds__(kCtrlJvpTPB) dyn_ctrl_tick_jac_kernel(const __grid_constant__ CtrlJvpArgs a) {
    constexpr int C = (EFF & QS_EFFECT_DRAG) ? 29 : 25;
    constexpr int TP = C - 3;                                        // the first target_pos column
    const long long N = a.N;
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;      // = ((k N + i) C + col): the output's own order
    if (g >= (long long)a.io.T * N * C) return;
    const long long ki = g / C;
    const int col = (int)(g - ki * C);
    const int k = (int)(ki / N);
    const long long i = ki - (long long)k * N;
    const qs::PhysRow c = row_of(a, i), tc = t_row_of(a, i);       // t_phys is NULL: the constants carry no tangent here
    const qs::PidGains K = gains_of(a, i);
    const qs::PidGains tK = t_gains_of(a, i);          // t_gains is NULL here too
    qs::Drone d;
    qs::PidState st;
    qs::PidTargets t;
    double raw[4], u1[4], u[4], up[4], t_u[4];
    ctrl_tick_inputs<EFF>(a, K, c, i, k, d, st, t, raw, u1, u, up);
    // the unit tangent of column col
    auto e = [col](int j) { return col == j ? 1.0 : 0.0; };
    qs::Drone td = {e(0), e(1), e(2), e(3), e(4), e(5), e(6), e(7), e(8), e(9), e(10), e(11), e(12)};
    qs::PidState t_st = {e(13), e(14), e(15), e(16), e(17), e(18), e(19), e(20), e(21)};
    double t_up[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) t_up[j] = (EFF & QS_EFFECT_DRAG) ? e(22 + j) : 0.0;
    const qs::PidTargets t_t = {{e(TP), e(TP + 1), e(TP + 2)}, 0.0, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}};
    ctrl_tick_jvp<EFF>(a, K, c, tc, d, st, t, raw, u1, u, up, tK, t_t, td, t_st, t_up, t_u);
    double* o = a.io.jac + g + (long long)(kCtrlJacRows - 1) * C * ki;  // ((k N + i) 26 + r) C + col at r = 0
    o[0] = td.px; o[C] = td.py; o[2 * C] = td.pz; o[3 * C] = td.qx; o[4 * C] = td.qy; o[5 * C] = td.qz; o[6 * C] = td.qw;
    o[7 * C] = td.vx; o[8 * C] = td.vy; o[9 * C] = td.vz; o[10 * C] = td.wx; o[11 * C] = td.wy; o[12 * C] = td.wz;
    o[13 * C] = t_st.ipx; o[14 * C] = t_st.ipy; o[15 * C] = t_st.ipz; o[16 * C] = t_st.lr; o[17 * C] = t_st.lp;
    o[18 * C] = t_st.ly; o[19 * C] = t_st.irx; o[20 * C] = t_st.iry; o[21 * C] = t_st.irz;
    o[22 * C] = t_u[0]; o[23 * C] = t_u[1]; o[24 * C] = t_u[2]; o[25 * C] = t_u[3];
}

template <bool JAC>
int launch_ctrl_jvp(const QsParams* p, const QsParams* cp, const QsDynCtrlTrajJvpIO* io, int n_envs, int drones_per_env,
                    int substeps, unsigned effects, void* stream, const char* what) {
    if (!p || !cp || !io) return fail(QS_ERR_NULL, what, "NULL params / controller params / io");
    if (!io->state0 || !io->pid0 || !io->target_pos || !io->states || !io->rpm || !io->pid_states)
        return fail(QS_ERR_NULL, what, "NULL state0 / pid0 / target_pos / states / rpm / pid_states");
    if (JAC ? !io->jac : (!io->t_states || !io->t_rpm)) return fail(QS_ERR_NULL, what, JAC ? "NULL jac" : "NULL t_states / t_rpm");
    if (int rc = traj_check_sizes(what, n_envs, drones_per_env, substeps, io->T)) return rc;
    if (!(io->control_timestep > 0.0)) return fail(QS_ERR_SIZE, what, "control_timestep must be > 0");
    if (int rc = traj_check_effects(what, effects, io->phys, io->t_phys)) return rc;
    const long long N = (long long)n_envs * drones_per_env;
    const long long threads = JAC ? (long long)io->T * N * ctrl_jac_cols(effects) : N;
    const long long blocks = (threads + kCtrlJvpTPB - 1) / kCtrlJvpTPB;
    if (blocks > 0x7fffffffLL) return fail(QS_ERR_SIZE, what, "T * N * columns exceeds 2^31-1 CTAs of 128 threads");
    CtrlJvpArgs a;
    memset(&a, 0, sizeof(a));
    a.P = *p; a.CP = *cp; a.io = *io;
    if (JAC) a.io.t_phys = a.io.t_gains = nullptr;                  // the Jacobian's columns are z_k and target_pos[k] only
    a.N = N;
    a.D = drones_per_env; a.substeps = substeps;
    return traj_launch(what, effects, [](auto EFF) {
        return JAC ? dyn_ctrl_tick_jac_kernel<decltype(EFF)::value> : dyn_ctrl_traj_jvp_kernel<decltype(EFF)::value>;
    }, (unsigned)blocks, kCtrlJvpTPB, 0, (cudaStream_t)stream, a);
}

}  // namespace
}  // namespace qsi

using namespace qsi;

extern "C" {

int qs_sizeof_dyn_ctrl_traj_jvp_io(void) { return (int)sizeof(QsDynCtrlTrajJvpIO); }

int qs_dyn_ctrl_traj_jvp(const QsParams* p, const QsParams* cp, const QsDynCtrlTrajJvpIO* io, int n_envs, int drones_per_env,
                         int substeps, unsigned effects, void* stream) {
    return launch_ctrl_jvp<false>(p, cp, io, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_ctrl_traj_jvp");
}

int qs_dyn_ctrl_tick_jac(const QsParams* p, const QsParams* cp, const QsDynCtrlTrajJvpIO* io, int n_envs, int drones_per_env,
                         int substeps, unsigned effects, void* stream) {
    return launch_ctrl_jvp<true>(p, cp, io, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_ctrl_tick_jac");
}

}  // extern "C"
