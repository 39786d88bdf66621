// dyn_policy_traj.cu -- qs_dyn_policy_traj / qs_dyn_policy_traj_vjp: differentiable trajectories of an MLP actor driving
// Physics.DYN through the RPM / ONE_D_RPM decode (include/quadsim.h, DESIGN.md 4.5).  A CTA owns M whole aviaries for all T ticks:
// their observation rows live in shared memory (the action history is shifted in place), the actor runs as a float64 GEMM chain
// over the M rows on the FP64 tensor cores (cta_gemm, policy_actor.cuh), and one thread per drone runs the decode and the physics.  The backward walks the ticks in reverse: it reloads the tick's
// observation and start state from the forward's outputs, recomputes the hidden activations with the forward's own
// actor_forward, runs mlp_adjoint.cuh's tick adjoint, collects the action's cotangent (physics + the returned action + what later
// observations sent back through the history, a ring of B cotangents per drone in shared memory), and pushes it through the
// transposed actor to the observation's cotangent.
#include "policy_actor.cuh"

namespace qsi {
namespace {

struct PolArgs {
    QsParams P;
    QsDynPolicyTrajIO io;
    long long N;
    int E, D, A, substeps;
    int M;                          // aviaries per CTA, a multiple of kPolMG with M * D <= kPolTPB
    int maxw, cw;                   // widest hidden layer; max(maxw, in_dim): the row stride of the cotangent buffers
};

// The transposed actor: gz [M][out_dim] (the cotangent of the mean action) down to the observation's cotangent, which it
// returns: [M] rows of stride cw in one of the two buffers.  `act` holds every hidden layer (actor_forward, keep).  Ends on a barrier.
__device__ const double* actor_transpose(const PolArgs& a, const double* act, const double* gz, double* c0, double* c1) {
    const QsDynPolicyTrajIO& io = a.io;
    const double* src = gz;
    int Nout = io.out_dim, lds = io.out_dim;
    for (int l = io.depth; l >= 0; --l) {
        const int K = l == 0 ? io.in_dim : io.width[l - 1];
        double* dst = (l & 1) ? c1 : c0;
        const double* h = l == 0 ? nullptr : act + (size_t)(l - 1) * a.M * a.maxw;
        const int kind = io.activation, cw = a.cw, maxw = a.maxw;
        cta_gemm(a.M, src, lds, io.w[l], 1, Nout, Nout, K, [&](int r, int k, double v) {
            dst[(size_t)r * cw + k] = h ? qs::mlp_act_vjp(kind, h[(size_t)r * maxw + k], v) : v;
        });
        __syncthreads();
        src = dst; Nout = K; lds = cw;
    }
    return src;
}

template <int EFF>
__global__ void __launch_bounds__(kPolTPB) dyn_policy_traj_kernel(const __grid_constant__ PolArgs a) {
    extern __shared__ double pol_sm[];
    const QsDynPolicyTrajIO& io = a.io;
    const int M = a.M, D = a.D, A = a.A, B = io.act_buffer_size, in = io.in_dim, out = io.out_dim, od = 12 + B * A;
    double* obs = pol_sm;
    double* act = obs + (size_t)M * in;
    double* mean = act + (size_t)2 * M * a.maxw;
    const int e0 = blockIdx.x * M, Mv = min(M, a.E - e0), tid = threadIdx.x;
    const bool live = tid < Mv * D;
    const long long N = a.N, i = (long long)e0 * D + tid;
    const int m = tid / D, dd = tid % D;
    for (int j = tid; j < M * in; j += blockDim.x) obs[j] = 0.0;        // the rows of a partial CTA's missing aviaries stay zero
    __syncthreads();
    qs::PhysRow c = qs::phys_row_of(a.P);
    qs::Drone d = {0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0};
    double up[4] = {0, 0, 0, 0}, R[9];
    double* row = obs + (size_t)tid * od;                                 // aviary m's row is D drone rows: m * in + dd * od
    if (live) {
        c = row_of(a, i);
        ld_state(io.state0, N, i, d);
        if ((EFF & QS_EFFECT_DRAG) && io.last_rpm) ld4(io.last_rpm, i, up);
        qs::Drone x0 = d;
        double inv;
        qs::entry_normalise(x0, inv);
        qs::quat_to_matrix_unit(x0.qx, x0.qy, x0.qz, x0.qw, R);
        for (int j = 0; j < B * A; ++j) row[12 + j] = io.action_buffer[i * B * A + j];
    }
    for (int k = 0; k < io.T; ++k) {
        if (live) qs::obs_head(d, R, row);
        __syncthreads();
        double* og = io.obs + ((long long)k * a.E + e0) * in;
        for (int j = tid; j < Mv * in; j += blockDim.x) og[j] = obs[j];
        actor_forward(a, obs, act, false, mean);
        if (live) {
            double aa[4] = {0, 0, 0, 0}, raw[4], u[4];
            for (int j = 0; j < A; ++j) {
                const int col = dd * A + j;
                double r = mean[m * out + col];
                if (io.noise) r = r + exp(io.log_std[col]) * io.noise[((long long)k * a.E + e0 + m) * out + col];
                io.actions[((long long)k * N + i) * A + j] = r;
                aa[j] = qs::clampd(r, -1.0, 1.0);
            }
            for (int j = 0; j < (B - 1) * A; ++j) row[12 + j] = row[12 + j + A];
            for (int j = 0; j < A; ++j) row[12 + (B - 1) * A + j] = aa[j];
            qs::policy_rpm(A, c, aa, raw);
            clip_rpm(raw, c.max_rpm, u);
            qs::dyn_tick_k<EFF>(a.P, c, d, u, up, 0.0, a.substeps, R);
            round_to_planes(d);
            st_state(io.states + (long long)k * 13 * N, N, i, d);
#pragma unroll
            for (int j = 0; j < 4; ++j) up[j] = u[j];
        }
    }
}

template <int EFF>
__global__ void __launch_bounds__(kPolTPB) dyn_policy_traj_vjp_kernel(const __grid_constant__ PolArgs a) {
    extern __shared__ double pol_sm[];
    const QsDynPolicyTrajIO& io = a.io;
    const int M = a.M, D = a.D, A = a.A, B = io.act_buffer_size, in = io.in_dim, out = io.out_dim, od = 12 + B * A;
    double* obs = pol_sm;
    double* act = obs + (size_t)M * in;
    double* gz = act + (size_t)io.depth * M * a.maxw;
    double* c0 = gz + (size_t)M * out;
    double* c1 = c0 + (size_t)M * a.cw;
    double* ring = c1 + (size_t)M * a.cw;                              // [M * D][B][A]: slot j mod B holds action j's cotangent
    const int e0 = blockIdx.x * M, Mv = min(M, a.E - e0), tid = threadIdx.x;
    const bool live = tid < Mv * D;
    const long long N = a.N, i = (long long)e0 * D + tid;
    const int m = tid / D, dd = tid % D;
    for (int j = tid; j < M * in; j += blockDim.x) obs[j] = 0.0;
    for (int j = tid; j < M * out; j += blockDim.x) gz[j] = 0.0;
    for (int j = tid; j < M * D * B * A; j += blockDim.x) ring[j] = 0.0;
    __syncthreads();
    const qs::PhysRow c = live ? row_of(a, i) : qs::phys_row_of(a.P);
    ScratchRec rec = {io.scratch, N, i};
    qs::PhysGrad G = zero_phys_grad();
    qs::Drone L = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    double Lup_next[4] = {0, 0, 0, 0};          // drag: the cotangent of this tick's clipped RPMs from tick k + 1's first substep
    double Lang[3] = {0, 0, 0};                 // the cotangent of ang_v in observation k + 1
    double* hist = ring + (size_t)tid * B * A;
    for (int k = io.T - 1; k >= 0; --k) {
        const double* og = io.obs + ((long long)k * a.E + e0) * in;
        for (int j = tid; j < Mv * in; j += blockDim.x) obs[j] = og[j];
        __syncthreads();
        actor_forward(a, obs, act, true, nullptr);
        qs::Drone d0 = {0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0};
        if (live) {
            add_state(io.g_states + (long long)k * 13 * N, N, i, L);
            ld_state(k == 0 ? io.state0 : io.states + (long long)(k - 1) * 13 * N, N, i, d0);
            double ra[4], aa[4], raw[4], u[4], up[4] = {0, 0, 0, 0};
            applied_rpm(a, c, i, k, ra, aa, raw, u);
            if (EFF & QS_EFFECT_DRAG) {
                if (k > 0) {
                    double ra1[4], aa1[4], raw1[4];
                    applied_rpm(a, c, i, k - 1, ra1, aa1, raw1, up);
                } else if (io.last_rpm) {
                    ld4(io.last_rpm, i, up);
                }
            }
            double Lu[4] = {Lup_next[0], Lup_next[1], Lup_next[2], Lup_next[3]}, Lup[4] = {0, 0, 0, 0};
            qs::dyn_tick_obs_vjp<EFF>(a.P, c, d0, u, up, a.substeps, rec, L, Lang, Lu, Lup, G);
            double Lraw[4], La[4] = {0, 0, 0, 0};
            qs::rpm_clip_vjp(raw, c.max_rpm, Lu, Lraw, G.g[13]);
            qs::policy_rpm_vjp(A, c, aa, Lraw, La, G.g[12]);
            for (int j = 0; j < A; ++j) {
                double& slot = hist[(k % B) * A + j];
                const double la = La[j] + slot;
                slot = 0.0;
                double gr = (ra[j] < -1.0 || ra[j] > 1.0) ? 0.0 : la;
                const long long o = ((long long)k * N + i) * A + j;
                if (io.g_actions) gr += io.g_actions[o];
                io.g_raw[o] = gr;
                gz[m * out + dd * A + j] = gr;
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) Lup_next[j] = Lup[j];
        }
        __syncthreads();
        const double* Lobs = actor_transpose(a, act, gz, c0, c1);
        if (live) {
            const double* Lo = Lobs + (size_t)m * a.cw + dd * od;
            qs::obs_head_vjp(d0, Lo, L, Lang);
            for (int b = 0; b < B; ++b) {
                const int s = ((k - B + b) % B + B) % B;
                for (int j = 0; j < A; ++j) hist[s * A + j] += Lo[12 + b * A + j];
            }
        }
        __syncthreads();
    }
    if (!live) return;
    {
        qs::Drone d0;
        ld_state(io.state0, N, i, d0);
        qs::initial_ang_v_vjp(d0, Lang, L);
    }
    st_state(io.g_state0, N, i, L);
    store_start_grads(io, i, Lup_next, G);
    if (io.g_action_buffer)
        for (int j = 0; j < B * A; ++j) io.g_action_buffer[i * B * A + j] = hist[j];
}

template <bool VJP>
int launch_policy_traj(const QsParams* p, const QsDynPolicyTrajIO* io, int act_type, int n_envs, int drones_per_env, int substeps,
                       unsigned effects, void* stream, const char* what) {
    if (int rc = policy_check_inputs(p, io, what)) return rc;
    if (VJP && (!io->g_states || !io->g_raw || !io->g_state0 || !io->scratch))
        return fail(QS_ERR_NULL, what, "NULL g_states / g_raw / g_state0 / scratch");
    int maxw = 0;
    if (int rc = policy_check_shape(io, act_type, n_envs, drones_per_env, substeps, effects, nullptr, what, maxw)) return rc;
    const int A = act_width(act_type), D = drones_per_env;
    PolArgs a;
    memset(&a, 0, sizeof(a));
    a.P = *p; a.io = *io;
    a.E = n_envs; a.D = D; a.A = A; a.substeps = substeps;
    a.N = (long long)n_envs * D;
    a.maxw = maxw;
    a.cw = maxw > io->in_dim ? maxw : io->in_dim;
    // doubles of shared memory per aviary: the observation row, the hidden activations (two buffers forward, every layer
    // backward), the mean action / its cotangent, and backward the two cotangent buffers and the history ring
    // The forward is refused where its VJP would be: a trajectory that cannot be differentiated must not come back with a grad_fn.
    const size_t per = VJP ? policy_vjp_doubles(io, D, A, maxw) : (size_t)io->in_dim + 2 * (size_t)maxw + io->out_dim;
    int M = 0;
    if (int rc = policy_ctas(io, D, A, maxw, per, what, M)) return rc;
    a.M = M;
    const size_t smem = per * M * sizeof(double);
    const unsigned blocks = (unsigned)((n_envs + M - 1) / M);
    return traj_launch(what, effects, [](auto EFF) {
        return VJP ? dyn_policy_traj_vjp_kernel<decltype(EFF)::value> : dyn_policy_traj_kernel<decltype(EFF)::value>;
    }, blocks, kPolTPB, smem, (cudaStream_t)stream, a);
}

}  // namespace
}  // namespace qsi

using namespace qsi;

extern "C" {

int qs_sizeof_dyn_policy_traj_io(void) { return (int)sizeof(QsDynPolicyTrajIO); }

int qs_dyn_policy_traj(const QsParams* p, const QsDynPolicyTrajIO* io, int act_type, int n_envs, int drones_per_env, int substeps,
                       unsigned effects, void* stream) {
    return launch_policy_traj<false>(p, io, act_type, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_policy_traj");
}

int qs_dyn_policy_traj_vjp(const QsParams* p, const QsDynPolicyTrajIO* io, int act_type, int n_envs, int drones_per_env, int substeps,
                           unsigned effects, void* stream) {
    return launch_policy_traj<true>(p, io, act_type, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_policy_traj_vjp");
}

}  // extern "C"
