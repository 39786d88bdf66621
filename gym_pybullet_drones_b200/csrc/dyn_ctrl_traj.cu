// dyn_ctrl_traj.cu -- qs_dyn_ctrl_traj / qs_dyn_ctrl_traj_vjp: differentiable closed-loop trajectories of a DSLPIDControl around
// Physics.DYN (include/quadsim.h, DESIGN.md 4.5).  One thread per drone for all T ticks.  The forward is the QS_CTRL_TRACK tick of
// ctrl_rollout_kernel (pid_control, the controller's max_rpm clip, the env's clip, dyn_tick_k, round_to_planes) in the same order;
// the backward walks the ticks in reverse, reloading each tick's start state and controller state from the forward's outputs and
// running dyn_adjoint.cuh's tick adjoint, the two clip adjoints and pid_adjoint.cuh's controller adjoint.
#include "qs_common.cuh"
#include "ctrl_io.cuh"

namespace qsi {
namespace {

constexpr int kCtrlTrajTPB = 128;

struct CtrlTrajArgs {
    QsParams P;          // the env: physics, MAX_RPM clip
    QsParams CP;         // the DSLPIDControl's own constants (gains unless io.gains, model, g, max_rpm)
    QsDynCtrlTrajIO io;
    long long N;
    int D, substeps;
};

template <int EFF>
__global__ void __launch_bounds__(kCtrlTrajTPB) dyn_ctrl_traj_kernel(const __grid_constant__ CtrlTrajArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long N = a.N;
    if (i >= N) return;
    const QsDynCtrlTrajIO& io = a.io;
    const qs::PhysRow c = row_of(a, i);
    const qs::PidGains K = gains_of(a, i);
    qs::Drone d;
    ld_state(io.state0, N, i, d);
    qs::PidState st;
    load_pid(io.pid0, N, i, st);
    double up[4] = {0, 0, 0, 0}, raw[4], u1[4], u[4];
    if ((EFF & QS_EFFECT_DRAG) && io.last_rpm) ld4(io.last_rpm, i, up);
    for (int k = 0; k < io.T; ++k) {
        store_pid(io.pid_states + (long long)k * 9 * N, N, i, st);
        control(a, K, st, d, targets_of(io, N, i, k), c.max_rpm, raw, u1, u);
        double R_last[9];
        qs::dyn_tick_k<EFF>(a.P, c, d, u, up, 0.0, a.substeps, R_last);
        round_to_planes(d);
        st_state(io.states + (long long)k * 13 * N, N, i, d);
        double* o = io.rpm + 4 * ((long long)k * N + i);
#pragma unroll
        for (int j = 0; j < 4; ++j) { o[j] = u[j]; up[j] = u[j]; }
    }
}

template <int EFF>
__global__ void __launch_bounds__(kCtrlTrajTPB) dyn_ctrl_traj_vjp_kernel(const __grid_constant__ CtrlTrajArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long N = a.N;
    if (i >= N) return;
    const QsDynCtrlTrajIO& io = a.io;
    const qs::PhysRow c = row_of(a, i);
    const qs::PidGains K = gains_of(a, i);
    ScratchRec rec = {io.scratch, N, i};
    qs::PhysGrad G = zero_phys_grad();
    double Lg[18];
#pragma unroll
    for (int j = 0; j < 18; ++j) Lg[j] = 0.0;
    qs::PidTargets Lt = {{0, 0, 0}, 0, {0, 0, 0}, {0, 0, 0}};
    qs::Drone L = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    qs::PidState Ls = {0, 0, 0, 0, 0, 0, 0, 0, 0};      // the cotangent of the controller state after tick k
    double Lup_next[4] = {0, 0, 0, 0};                 // drag: the cotangent of this tick's applied RPMs from tick k + 1
    for (int k = io.T - 1; k >= 0; --k) {
        add_state(io.g_states + (long long)k * 13 * N, N, i, L);
        qs::Drone d0;
        ld_state(k == 0 ? io.state0 : io.states + (long long)(k - 1) * 13 * N, N, i, d0);
        qs::PidState st0;
        load_pid(io.pid_states + (long long)k * 9 * N, N, i, st0);
        const qs::PidTargets t = targets_of(io, N, i, k);
        double raw[4], u1[4], u[4], up[4] = {0, 0, 0, 0};
        {
            qs::PidState st = st0;
            control(a, K, st, d0, t, c.max_rpm, raw, u1, u);
        }
        if (EFF & QS_EFFECT_DRAG) {
            if (k > 0) ld4(io.rpm, (long long)(k - 1) * N + i, up);
            else if (io.last_rpm) ld4(io.last_rpm, i, up);
        }
        double Lu[4] = {Lup_next[0], Lup_next[1], Lup_next[2], Lup_next[3]}, Lup[4] = {0, 0, 0, 0};
        if (io.g_rpm_out) {
            double gr[4];
            ld4(io.g_rpm_out, (long long)k * N + i, gr);
#pragma unroll
            for (int j = 0; j < 4; ++j) Lu[j] += gr[j];
        }
        qs::dyn_tick_vjp<EFF>(a.P, c, d0, u, up, a.substeps, rec, L, Lu, Lup, G);
        // the env's clip (gradient to the row's MAX_RPM), then the controller's (its max_rpm is a constant of the controller)
        double Lu1[4], Lraw[4], g_cmax = 0.0;
        qs::rpm_clip_vjp(u1, c.max_rpm, Lu, Lu1, G.g[13]);
        qs::rpm_clip_vjp(raw, a.CP.max_rpm, Lu1, Lraw, g_cmax);
        Lt.tp[0] = Lt.tp[1] = Lt.tp[2] = 0.0;             // target_pos is per tick: its cotangent is written, not carried
        qs::pid_control_vjp(a.CP, K, st0, io.control_timestep, d0, t, Lraw, Ls, L, Lt, Lg);
        if (io.g_target_pos) {
            double* o = io.g_target_pos + 3 * ((long long)k * N + i);
            o[0] = Lt.tp[0]; o[1] = Lt.tp[1]; o[2] = Lt.tp[2];
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) Lup_next[j] = Lup[j];
    }
    st_state(io.g_state0, N, i, L);
    if (io.g_pid0) store_pid(io.g_pid0, N, i, Ls);
    auto st3 = [&](double* p, const double v[3]) { if (p) { p[3 * i] = v[0]; p[3 * i + 1] = v[1]; p[3 * i + 2] = v[2]; } };
    st3(io.g_target_vel, Lt.tv);
    st3(io.g_target_rpy_rates, Lt.trr);
    const double ly[3] = {0.0, 0.0, Lt.tyaw};
    st3(io.g_target_rpy, ly);
    store_start_grads(io, i, Lup_next, G);
    if (io.g_gains) {
        double* o = io.g_gains + 18 * i;
#pragma unroll
        for (int j = 0; j < 18; ++j) o[j] = Lg[j];
    }
}

template <bool VJP>
int launch_ctrl_traj(const QsParams* p, const QsParams* cp, const QsDynCtrlTrajIO* io, int n_envs, int drones_per_env,
                     int substeps, unsigned effects, void* stream, const char* what) {
    if (!p || !cp || !io) return fail(QS_ERR_NULL, what, "NULL params / controller params / io");
    if (!io->state0 || !io->pid0 || !io->target_pos || !io->states || !io->rpm || !io->pid_states)
        return fail(QS_ERR_NULL, what, "NULL state0 / pid0 / target_pos / states / rpm / pid_states");
    if (VJP && (!io->g_states || !io->g_state0 || !io->scratch)) return fail(QS_ERR_NULL, what, "NULL g_states / g_state0 / scratch");
    if (int rc = traj_check_sizes(what, n_envs, drones_per_env, substeps, io->T)) return rc;
    if (!(io->control_timestep > 0.0)) return fail(QS_ERR_SIZE, what, "control_timestep must be > 0");
    if (int rc = traj_check_effects(what, effects, io->phys, nullptr)) return rc;
    CtrlTrajArgs a;
    memset(&a, 0, sizeof(a));
    a.P = *p; a.CP = *cp; a.io = *io;
    a.N = (long long)n_envs * drones_per_env;
    a.D = drones_per_env; a.substeps = substeps;
    const unsigned blocks = (unsigned)((a.N + kCtrlTrajTPB - 1) / kCtrlTrajTPB);
    return traj_launch(what, effects, [](auto EFF) {
        return VJP ? dyn_ctrl_traj_vjp_kernel<decltype(EFF)::value> : dyn_ctrl_traj_kernel<decltype(EFF)::value>;
    }, blocks, kCtrlTrajTPB, 0, (cudaStream_t)stream, a);
}

}  // namespace
}  // namespace qsi

using namespace qsi;

extern "C" {

int qs_sizeof_dyn_ctrl_traj_io(void) { return (int)sizeof(QsDynCtrlTrajIO); }

int qs_dyn_ctrl_traj(const QsParams* p, const QsParams* cp, const QsDynCtrlTrajIO* io, int n_envs, int drones_per_env, int substeps,
                     unsigned effects, void* stream) {
    return launch_ctrl_traj<false>(p, cp, io, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_ctrl_traj");
}

int qs_dyn_ctrl_traj_vjp(const QsParams* p, const QsParams* cp, const QsDynCtrlTrajIO* io, int n_envs, int drones_per_env,
                         int substeps, unsigned effects, void* stream) {
    return launch_ctrl_traj<true>(p, cp, io, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_ctrl_traj_vjp");
}

}  // extern "C"
