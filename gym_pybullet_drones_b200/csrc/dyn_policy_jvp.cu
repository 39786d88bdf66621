// dyn_policy_jvp.cu -- qs_dyn_policy_traj_jvp / qs_dyn_policy_tick_jac: forward mode of the policy trajectories of
// qs_dyn_policy_traj (include/quadsim.h, DESIGN.md 4.5) on mlp_tangent.cuh's tick tangent.  Tick k restarts from the forward's
// stored state k-1, saved observation obs[k] and stored raw actions, as qs_dyn_policy_traj_vjp does, so the loop is linearised at
// the forward's bits.  Per tick, the hidden activations are recomputed with the forward's own actor_forward, the observation's
// tangent is pushed through the actor as a GEMM chain on the FP64 tensor cores (actor_tangent: cta_gemm, each layer's activation
// derivative in the epilogue), and one thread per drone runs the clip, the decode and the physics.
//   dyn_policy_traj_jvp_kernel<EFF>: a CTA owns M aviaries for all T ticks, as the forward does; the observation's buffer holds
//     its tangent once the first layer has read it, and the history's tangent is shifted in place.
//   dyn_policy_tick_jac_kernel<EFF>: a CTA owns tick k of 8 aviaries; per aviary, the unit tangents of the columns go through the
//     same actor_tangent in groups of 8 rows (one mma m-tile).  cta_gemm's rows are independent, so each column is the JVP
//     kernel's result for that unit tangent, bit for bit.
#include "policy_actor.cuh"
#include "mlp_tangent.cuh"

namespace qsi {
namespace {

struct PolJvpArgs {
    QsParams P;
    QsDynPolicyTrajJvpIO io;
    long long N;
    int E, D, A, substeps;
    int M;                          // aviaries per CTA (the JVP), or rows of one aviary's tangents (8, the Jacobian)
    int maxw;                       // widest hidden layer: the row stride of the tangent buffers
    int nzd;                        // entries of one drone's loop state: 16 + B A (+ 4 with drag)
};

// t_mean [M][out_dim] = d actor / d obs  t_x for the M tangent rows t_x [M][in_dim]; row r reads the hidden activations of row
// hrow(r) of `act` (actor_forward, keep).  Every thread of the CTA calls it; it ends on a barrier.
template <class HRow>
__device__ void actor_tangent(const PolJvpArgs& a, int M, const double* tx, const double* act, HRow hrow, double* c0, double* c1,
                              double* t_mean) {
    const QsDynPolicyTrajJvpIO& io = a.io;
    const double* src = tx;
    int K = io.in_dim, lds = io.in_dim;
    for (int l = 0; l <= io.depth; ++l) {
        const bool last = l == io.depth;
        const int Nout = last ? io.out_dim : io.width[l];
        double* dst = last ? t_mean : ((l & 1) ? c1 : c0);
        const int ldd = last ? io.out_dim : a.maxw;
        const double* h = act + (size_t)l * a.M * a.maxw;
        const int kind = io.activation, maxw = a.maxw;
        cta_gemm(M, src, lds, io.w[l], Nout, 1, K, Nout, [&](int r, int n, double v) {
            dst[(size_t)r * ldd + n] = last ? v : qs::mlp_act_jvp(kind, h[(size_t)hrow(r) * maxw + n], v);
        });
        __syncthreads();
        src = dst; K = Nout; lds = ldd;
    }
}

// the primal of drone i's tick k: the stored start state and drag's previous applied RPMs
template <int EFF>
__device__ __forceinline__ void tick_start(const PolJvpArgs& a, const qs::PhysRow& c, long long i, int k, qs::Drone& d, double up[4]) {
    const QsDynPolicyTrajJvpIO& io = a.io;
    ld_state(k == 0 ? io.state0 : io.states + (long long)(k - 1) * 13 * a.N, a.N, i, d);
    up[0] = up[1] = up[2] = up[3] = 0.0;
    if (EFF & QS_EFFECT_DRAG) {
        if (k > 0) {
            double ra[4], aa[4], raw[4];
            applied_rpm(a, c, i, k - 1, ra, aa, raw, up);
        } else if (io.last_rpm) {
            ld4(io.last_rpm, i, up);
        }
    }
}

template <int EFF>
__global__ void __launch_bounds__(kPolTPB) dyn_policy_traj_jvp_kernel(const __grid_constant__ PolJvpArgs a) {
    extern __shared__ double pol_sm[];
    const QsDynPolicyTrajJvpIO& io = a.io;
    const int M = a.M, D = a.D, A = a.A, B = io.act_buffer_size, in = io.in_dim, out = io.out_dim, od = 12 + B * A;
    double* obs = pol_sm;                                              // the saved observation, then its tangent
    double* act = obs + (size_t)M * in;
    double* tm = act + (size_t)io.depth * M * a.maxw;                  // the mean action's tangent
    double* c0 = tm + (size_t)M * out;
    double* c1 = c0 + (size_t)M * a.maxw;
    double* ring = c1 + (size_t)M * a.maxw;                            // [M D][B A]: the history's tangent, oldest first
    const int e0 = blockIdx.x * M, Mv = min(M, a.E - e0), tid = threadIdx.x;
    const bool live = tid < Mv * D;
    const long long N = a.N, i = (long long)e0 * D + (live ? tid : 0);
    const int m = tid / D, dd = tid % D;
    for (int j = tid; j < M * in; j += blockDim.x) obs[j] = 0.0;        // the rows of a partial CTA's missing aviaries stay zero
    const qs::PhysRow c = row_of(a, i), tc = t_row_of(a, i);
    double* th = ring + (size_t)tid * B * A;
    qs::Drone td = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    double t_ang[3] = {0, 0, 0}, t_up[4] = {0, 0, 0, 0};
    if (live) {
        if (io.t_state0) ld_state(io.t_state0, N, i, td);
        qs::Drone d0;
        ld_state(io.state0, N, i, d0);
        qs::initial_ang_v_jvp(d0, td, t_ang);
        if ((EFF & QS_EFFECT_DRAG) && io.t_last_rpm) ld4(io.t_last_rpm, i, t_up);
        for (int j = 0; j < B * A; ++j) th[j] = io.t_action_buffer ? io.t_action_buffer[i * B * A + j] : 0.0;
    }
    __syncthreads();
    for (int k = 0; k < io.T; ++k) {
        const double* og = io.obs + ((long long)k * a.E + e0) * in;
        for (int j = tid; j < Mv * in; j += blockDim.x) obs[j] = og[j];
        __syncthreads();
        actor_forward(a, obs, act, true, nullptr);
        qs::Drone d = {0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0};
        double up[4] = {0, 0, 0, 0};
        if (live) {
            tick_start<EFF>(a, c, i, k, d, up);
            double* to = obs + (size_t)tid * od;                         // aviary m's row is D drone rows: m * in + dd * od
            qs::obs_head_jvp(d, td, t_ang, to);
            for (int j = 0; j < B * A; ++j) to[12 + j] = th[j];
        }
        __syncthreads();
        actor_tangent(a, M, obs, act, [](int r) { return r; }, c0, c1, tm);
        if (live) {
            double raw[4] = {0, 0, 0, 0}, t_raw[4] = {0, 0, 0, 0}, t_a[4], t_u[4];
            for (int j = 0; j < A; ++j) {
                const long long o = ((long long)k * N + i) * A + j;
                raw[j] = io.actions[o];
                double t = tm[m * out + dd * A + j];
                if (io.t_raw_in) t = t + io.t_raw_in[o];
                t_raw[j] = t;
                io.t_actions[o] = t;
            }
            qs::policy_tick_jvp<EFF>(a.P, c, tc, A, a.substeps, raw, t_raw, d, td, up, t_up, t_a, t_u, t_ang);
            for (int j = 0; j < (B - 1) * A; ++j) th[j] = th[j + A];
            for (int j = 0; j < A; ++j) th[(B - 1) * A + j] = t_a[j];
#pragma unroll
            for (int j = 0; j < 4; ++j) t_up[j] = t_u[j];
            st_state(io.t_states + (long long)k * 13 * N, N, i, td);
        }
        __syncthreads();
    }
}

template <int EFF>
__global__ void __launch_bounds__(kPolTPB) dyn_policy_tick_jac_kernel(const __grid_constant__ PolJvpArgs a) {
    extern __shared__ double pol_sm[];
    const QsDynPolicyTrajJvpIO& io = a.io;
    const int D = a.D, A = a.A, B = io.act_buffer_size, in = io.in_dim, out = io.out_dim, od = 12 + B * A, BA = B * A;
    const int nzd = a.nzd, nz = D * nzd, R = nz + D * A;
    double* obs = pol_sm;                                              // the 8 aviaries' observations, then 8 seed tangents
    double* act = obs + (size_t)kPolMG * in;
    double* tm = act + (size_t)io.depth * kPolMG * a.maxw;
    double* c0 = tm + (size_t)kPolMG * out;
    double* c1 = c0 + (size_t)kPolMG * a.maxw;
    const long long nb = (a.E + kPolMG - 1) / kPolMG;
    const int k = (int)(blockIdx.x / nb), e0 = (int)(blockIdx.x % nb) * kPolMG, Mv = min(kPolMG, a.E - e0), tid = threadIdx.x;
    const long long N = a.N;
    for (int j = tid; j < kPolMG * in; j += blockDim.x) obs[j] = 0.0;
    __syncthreads();
    const double* og = io.obs + ((long long)k * a.E + e0) * in;
    for (int j = tid; j < Mv * in; j += blockDim.x) obs[j] = og[j];
    __syncthreads();
    actor_forward(a, obs, act, true, nullptr);
    const int r = tid / D, dd = tid % D;                               // seed row (column g + r) and drone of this thread
    const bool live = r < kPolMG;
    for (int m = 0; m < Mv; ++m) {
        const long long i = (long long)(e0 + m) * D + dd;
        const qs::PhysRow c = row_of(a, i), tc = t_row_of(a, i);      // t_phys is NULL: the constants carry no tangent here
        for (int g = 0; g < R; g += kPolMG) {
            const int col = g + r;
            const int cd = col < nz ? col / nzd : -1, cc = col < nz ? col % nzd : -1;
            const bool own = cd == dd;                                 // the column is an entry of this drone's loop state
            auto e = [&](int j) { return own && cc == j ? 1.0 : 0.0; };
            qs::Drone d = {0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0};
            double up[4] = {0, 0, 0, 0};
            qs::Drone td = {e(0), e(1), e(2), e(3), e(4), e(5), e(6), e(7), e(8), e(9), e(10), e(11), e(12)};
            double t_ang[3] = {e(13), e(14), e(15)}, t_up[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) t_up[j] = (EFF & QS_EFFECT_DRAG) ? e(16 + BA + j) : 0.0;
            if (live) {
                tick_start<EFF>(a, c, i, k, d, up);
                double* to = obs + (size_t)r * in + dd * od;
                qs::obs_head_jvp(d, td, t_ang, to);
                for (int j = 0; j < BA; ++j) to[12 + j] = e(16 + j);
            }
            __syncthreads();
            actor_tangent(a, kPolMG, obs, act, [m](int) { return m; }, c0, c1, tm);
            if (live && col < R) {
                double raw[4] = {0, 0, 0, 0}, t_raw[4] = {0, 0, 0, 0}, t_a[4], t_u[4];
                for (int j = 0; j < A; ++j) {
                    raw[j] = io.actions[((long long)k * N + i) * A + j];
                    double t = tm[r * out + dd * A + j];
                    if (col - nz == dd * A + j) t = t + 1.0;
                    t_raw[j] = t;
                }
                qs::policy_tick_jvp<EFF>(a.P, c, tc, A, a.substeps, raw, t_raw, d, td, up, t_up, t_a, t_u, t_ang);
                // column col of the aviary's [R][R] block: drone dd's rows of z_{k+1}, then of raw_k
                double* J = io.jac + ((long long)k * a.E + e0 + m) * R * R + (long long)dd * nzd * R + col;
                const double zs[13] = {td.px, td.py, td.pz, td.qx, td.qy, td.qz, td.qw, td.vx, td.vy, td.vz, td.wx, td.wy, td.wz};
                for (int j = 0; j < 13; ++j) J[(long long)j * R] = zs[j];
                for (int j = 0; j < 3; ++j) J[(long long)(13 + j) * R] = t_ang[j];
                for (int j = 0; j < (B - 1) * A; ++j) J[(long long)(16 + j) * R] = e(16 + j + A);
                for (int j = 0; j < A; ++j) J[(long long)(16 + (B - 1) * A + j) * R] = t_a[j];
                if (EFF & QS_EFFECT_DRAG)
                    for (int j = 0; j < 4; ++j) J[(long long)(16 + BA + j) * R] = t_u[j];
                double* Jr = io.jac + ((long long)k * a.E + e0 + m) * R * R + (long long)(nz + dd * A) * R + col;
                for (int j = 0; j < A; ++j) Jr[(long long)j * R] = t_raw[j];
            }
            __syncthreads();
        }
    }
}

template <bool JAC>
int launch_policy_jvp(const QsParams* p, const QsDynPolicyTrajJvpIO* io, int act_type, int n_envs, int drones_per_env, int substeps,
                      unsigned effects, void* stream, const char* what) {
    if (int rc = policy_check_inputs(p, io, what)) return rc;
    if (JAC ? !io->jac : (!io->t_states || !io->t_actions)) return fail(QS_ERR_NULL, what, JAC ? "NULL jac" : "NULL t_states / t_actions");
    int maxw = 0;
    if (int rc = policy_check_shape(io, act_type, n_envs, drones_per_env, substeps, effects, io->t_phys, what, maxw)) return rc;
    const int A = act_width(act_type), D = drones_per_env, BA = io->act_buffer_size * A;
    // doubles of shared memory per aviary (or per seed row): the observation row (then its tangent), every hidden layer, the mean
    // action's tangent, two tangent buffers of maxw and, in the JVP, the history's tangent: never more than the VJP's
    const size_t per = (size_t)io->in_dim + (size_t)io->depth * maxw + io->out_dim + 2 * (size_t)maxw + (JAC ? 0 : (size_t)D * BA);
    int M = 0;
    if (int rc = policy_ctas(io, D, A, maxw, per, what, M)) return rc;
    if (JAC) M = kPolMG;
    const long long ctas = (n_envs + M - 1) / M, blocks = JAC ? (long long)io->T * ctas : ctas;
    if (blocks > 0x7fffffffLL) return fail(QS_ERR_SIZE, what, "T * ceil(n_envs / 8) exceeds 2^31-1 CTAs");
    PolJvpArgs a;
    memset(&a, 0, sizeof(a));
    a.P = *p; a.io = *io;
    if (JAC) a.io.t_state0 = a.io.t_last_rpm = a.io.t_phys = a.io.t_action_buffer = a.io.t_raw_in = nullptr;
    a.E = n_envs; a.D = D; a.A = A; a.substeps = substeps;
    a.N = (long long)n_envs * D;
    a.M = M;
    a.maxw = maxw;
    a.nzd = 16 + BA + ((effects & QS_EFFECT_DRAG) ? 4 : 0);
    const size_t smem = per * M * sizeof(double);
    return traj_launch(what, effects, [](auto EFF) {
        return JAC ? dyn_policy_tick_jac_kernel<decltype(EFF)::value> : dyn_policy_traj_jvp_kernel<decltype(EFF)::value>;
    }, (unsigned)blocks, kPolTPB, smem, (cudaStream_t)stream, a);
}

}  // namespace
}  // namespace qsi

using namespace qsi;

extern "C" {

int qs_sizeof_dyn_policy_traj_jvp_io(void) { return (int)sizeof(QsDynPolicyTrajJvpIO); }

int qs_dyn_policy_traj_jvp(const QsParams* p, const QsDynPolicyTrajJvpIO* io, int act_type, int n_envs, int drones_per_env,
                           int substeps, unsigned effects, void* stream) {
    return launch_policy_jvp<false>(p, io, act_type, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_policy_traj_jvp");
}

int qs_dyn_policy_tick_jac(const QsParams* p, const QsDynPolicyTrajJvpIO* io, int act_type, int n_envs, int drones_per_env,
                           int substeps, unsigned effects, void* stream) {
    return launch_policy_jvp<true>(p, io, act_type, n_envs, drones_per_env, substeps, effects, stream, "qs_dyn_policy_tick_jac");
}

}  // extern "C"
