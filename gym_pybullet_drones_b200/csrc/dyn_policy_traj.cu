// dyn_policy_traj.cu -- qs_dyn_policy_traj / qs_dyn_policy_traj_vjp: differentiable trajectories of an MLP actor driving
// Physics.DYN through the RPM / ONE_D_RPM decode (include/quadsim.h, DESIGN.md 4.5).  A CTA owns M whole aviaries for all T ticks:
// their observation rows live in shared memory (the action history is shifted in place), the actor runs as a float64 GEMM chain
// over the M rows on the FP64 tensor cores (cta_gemm), and
// one thread per drone runs the decode and the physics.  The backward walks the ticks in reverse: it reloads the tick's
// observation and start state from the forward's outputs, recomputes the hidden activations with the forward's own
// actor_forward, runs mlp_adjoint.cuh's tick adjoint, collects the action's cotangent (physics + the returned action + what later
// observations sent back through the history, a ring of B cotangents per drone in shared memory), and pushes it through the
// transposed actor to the observation's cotangent.
#include "qs_common.cuh"
#include "mlp_adjoint.cuh"
#include "traj_io.cuh"

namespace qsi {
namespace {

constexpr int kPolTPB = 256;
constexpr int kPolMG = 8;            // aviaries per CTA come in m-tiles of 8 rows (mma.m8n8k4)
constexpr int kPolMaxM = 16;         // aviaries per CTA at most
constexpr int kPolNT = 4;            // n-tiles a warp carries per pass: one A fragment per m-tile feeds kPolNT products
constexpr size_t kPolSmemMax = 227 * 1024;

struct PolArgs {
    QsParams P;
    QsDynPolicyTrajIO io;
    long long N;
    int E, D, A, substeps;
    int M;                          // aviaries per CTA, a multiple of kPolMG with M * D <= kPolTPB
    int maxw, cw;                   // widest hidden layer; max(maxw, in_dim): the row stride of the cotangent buffers
};

// C[r][n] = sum_k X[r][k] Bm(k, n) for the CTA's M rows (X in shared memory, row stride ldx) and n < Nn, with
// Bm(k, n) = W[k * sk + n * sn] read from global memory: (sk, sn) = (Nout, 1) is a layer, (1, Nout) its transpose.  epi(r, n, c)
// receives every element once.  Every thread of the CTA calls it; no barrier inside.
//
// The product runs on the FP64 tensor cores (mma.sync.aligned.m8n8k4.row.col.f64): lane 4 g + t holds A[g][t], B[t][g] and
// C[g][2 t], C[g][2 t + 1].  A warp owns kPolNT n-tiles at a time for all M / 8 m-tiles, so each weight is loaded exactly once
// per CTA and layer (no other warp needs it: staging it through shared memory would add a copy and no reuse) and each A fragment
// feeds kPolNT products.  Built with -DQS_POLICY_GEMM_FMA the same interface runs mlp_adjoint.cuh's plain FMA loop (what the
// host build uses), four rows per thread: the A/B partner of DESIGN.md 4.5's measurement, not a run-time option.
template <class Epi>
__device__ __forceinline__ void cta_gemm(int M, const double* X, int ldx, const double* W, int sk, int sn, int K, int Nn, Epi epi) {
#if defined(QS_POLICY_GEMM_FMA)
    for (int it = threadIdx.x; it < Nn * (M / 4); it += blockDim.x) {
        const int n = it % Nn, g = it / Nn;
        double acc[4] = {0.0, 0.0, 0.0, 0.0};
        for (int k = 0; k < K; ++k) {
            const double w = W[(long long)k * sk + (long long)n * sn];
#pragma unroll
            for (int m = 0; m < 4; ++m) acc[m] = qs::fmad(X[(size_t)(g * 4 + m) * ldx + k], w, acc[m]);
        }
#pragma unroll
        for (int m = 0; m < 4; ++m) epi(g * 4 + m, n, acc[m]);
    }
#else
    const int warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int MT = M / kPolMG;                                   // 1 or 2
    for (int nt0 = warp * kPolNT; nt0 * 8 < Nn; nt0 += nwarps * kPolNT) {
        double c[kPolNT][2][2];
#pragma unroll
        for (int j = 0; j < kPolNT; ++j) c[j][0][0] = c[j][0][1] = c[j][1][0] = c[j][1][1] = 0.0;
        for (int k0 = 0; k0 < K; k0 += 4) {
            const int kk = k0 + t;
            const bool kin = kk < K;
            const double a0 = kin ? X[(size_t)g * ldx + kk] : 0.0;
            const double a1 = (kin && MT > 1) ? X[(size_t)(8 + g) * ldx + kk] : 0.0;
            double bfr[kPolNT];
#pragma unroll
            for (int j = 0; j < kPolNT; ++j) {
                const int n = (nt0 + j) * 8 + g;
                bfr[j] = (kin && n < Nn) ? W[(long long)kk * sk + (long long)n * sn] : 0.0;
            }
#pragma unroll
            for (int j = 0; j < kPolNT; ++j) {
                asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                             : "+d"(c[j][0][0]), "+d"(c[j][0][1]) : "d"(a0), "d"(bfr[j]));
                if (MT > 1)
                    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                                 : "+d"(c[j][1][0]), "+d"(c[j][1][1]) : "d"(a1), "d"(bfr[j]));
            }
        }
#pragma unroll
        for (int j = 0; j < kPolNT; ++j)
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int n = (nt0 + j) * 8 + 2 * t + h;
                    if (mt < MT && n < Nn) epi(mt * 8 + g, n, c[j][mt][h]);
                }
    }
#endif
}

// The actor's hidden layers (and, with `mean`, its output layer) over the CTA's M observation rows.  Layer l's activations go
// to act + (keep ? l : l & 1) * M * maxw, row stride maxw.  Every thread of the CTA calls it; it ends on a barrier.
__device__ void actor_forward(const PolArgs& a, const double* obs, double* act, bool keep, double* mean) {
    const QsDynPolicyTrajIO& io = a.io;
    const int layers = io.depth + (mean ? 1 : 0);
    const double* x = obs;
    int K = io.in_dim, ldx = io.in_dim;
    for (int l = 0; l < layers; ++l) {
        const bool last = l == io.depth;
        const int Nout = last ? io.out_dim : io.width[l];
        double* dst = last ? mean : act + (size_t)(keep ? l : (l & 1)) * a.M * a.maxw;
        const int ldd = last ? io.out_dim : a.maxw;
        const double* bias = io.b[l];
        const int kind = io.activation;
        cta_gemm(a.M, x, ldx, io.w[l], Nout, 1, K, Nout, [&](int r, int n, double v) {
            v = v + bias[n];
            dst[(size_t)r * ldd + n] = last ? v : qs::mlp_act(kind, v);
        });
        __syncthreads();
        x = dst; K = Nout; ldx = ldd;
    }
}

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

// the applied RPMs of tick k, from the saved raw action
__device__ __forceinline__ void applied_rpm(const PolArgs& a, const qs::PhysRow& c, long long i, int k, double raw_a[4], double aa[4],
                                            double raw[4], double u[4]) {
    aa[0] = aa[1] = aa[2] = aa[3] = 0.0;
    for (int j = 0; j < a.A; ++j) {
        raw_a[j] = a.io.actions[((long long)k * a.N + i) * a.A + j];
        aa[j] = qs::clampd(raw_a[j], -1.0, 1.0);
    }
    qs::policy_rpm(a.A, c, aa, raw);
    clip_rpm(raw, c.max_rpm, u);
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
    if (!p || !io) return fail(QS_ERR_NULL, what, "NULL params / io");
    if (!io->state0 || !io->action_buffer || !io->log_std || !io->states || !io->actions || !io->obs)
        return fail(QS_ERR_NULL, what, "NULL state0 / action_buffer / log_std / states / actions / obs");
    if (VJP && (!io->g_states || !io->g_raw || !io->g_state0 || !io->scratch))
        return fail(QS_ERR_NULL, what, "NULL g_states / g_raw / g_state0 / scratch");
    if (int rc = traj_check_sizes(what, n_envs, drones_per_env, substeps, io->T)) return rc;
    if (act_type != QS_ACT_RPM && act_type != QS_ACT_ONE_D_RPM)
        return fail(QS_ERR_UNSUPPORTED, what, "only the RPM and ONE_D_RPM actions have an adjoint (PID, VEL and ONE_D_PID run the embedded "
                                              "controller)");
    const int A = act_width(act_type), D = drones_per_env;
    if (io->act_buffer_size <= 0) return fail(QS_ERR_SIZE, what, "act_buffer_size must be > 0");
    if (io->activation != QS_MLP_TANH && io->activation != QS_MLP_RELU) return fail(QS_ERR_ENUM, what, "bad activation");
    if (io->depth < 1 || io->depth > QS_MLP_MAX_HIDDEN) return fail(QS_ERR_SIZE, what, "1 to 4 hidden layers");
    int maxw = 0;
    for (int l = 0; l <= io->depth; ++l) {
        if (!io->w[l] || !io->b[l]) return fail(QS_ERR_NULL, what, "NULL weight / bias");
        if (l < io->depth) {
            if (io->width[l] < 1 || io->width[l] > QS_MLP_MAX_WIDTH) return fail(QS_ERR_SIZE, what, "hidden widths must be 1 .. 256");
            maxw = io->width[l] > maxw ? io->width[l] : maxw;
        }
    }
    if (D * A > 32 || D > kPolTPB / kPolMG) return fail(QS_ERR_UNSUPPORTED, what, "up to 32 action outputs (D * A) and 32 drones per aviary");
    if (io->in_dim != D * (12 + io->act_buffer_size * A) || io->out_dim != D * A)
        return fail(QS_ERR_SIZE, what, "in_dim must be D (12 + B A) and out_dim D A");
    if (int rc = traj_check_effects(what, effects, io->phys, nullptr)) return rc;
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
    const size_t per_vjp = (size_t)io->in_dim + (size_t)io->depth * maxw + io->out_dim + 2 * (size_t)a.cw + (size_t)D * io->act_buffer_size * A;
    const size_t per = VJP ? per_vjp : (size_t)io->in_dim + 2 * (size_t)maxw + io->out_dim;
    int M = (int)(kPolSmemMax / (per * sizeof(double)));
    if (kPolSmemMax / (per_vjp * sizeof(double)) < (size_t)kPolMG) M = 0;
    M = M < kPolTPB / D ? M : kPolTPB / D;
    M = M < kPolMaxM ? M : kPolMaxM;
    M -= M % kPolMG;
    if (M < kPolMG)
        return fail(QS_ERR_UNSUPPORTED, what, "the observation rows, hidden activations and cotangents of 8 aviaries exceed the 227 KB of "
                                              "shared memory of a CTA (shorten the action buffer with a lower ctrl_freq, or use fewer drones "
                                              "per aviary)");
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
