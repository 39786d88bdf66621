// rollout_mlp.cu -- qs_rollout_mlp: the policy rollout with a general network (QsMlpPolicy; DESIGN.md 4.1b): the rollout kernel's
// body with warp_mlp in place of warp_net, in a translation unit of its own so that it compiles in parallel with rollout.cu.
#include "rollout_kernel.cuh"

using namespace qsi;

namespace {

// shared memory of a policy CTA besides the fixed part and the staging: window, means, values, log-prob terms (launch_rollout)
size_t mlp_smem_var(int tpb, int obs_dim, int T, int A, int D, int out_tiles) {
    const int n_av_max = 64 / D;
    return (size_t)tpb * obs_dim * 4 + (size_t)(T + 1) * A * 4 + 32 + (size_t)(n_av_max * 8 * out_tiles + n_av_max * 8 + 64) * 4 + 16;
}
// the two staging buffers of both warps: 2 warps x 2 buffers x (max width / 16) k-steps x 1 KB
size_t mlp_stage_bytes(int max_width) { return (size_t)2 * 2 * (max_width / 16) * 1024; }
constexpr size_t kPolicySmemLimit = 200 * 1024;      // what launch_rollout allows a policy CTA

int net_max_width(const QsMlpNet& n) {
    int w = 0;
    for (int l = 0; l < n.depth && l < QS_MLP_MAX_HIDDEN; ++l) w = n.width[l] > w ? n.width[l] : w;
    return w;
}

int check_net(const QsMlpNet& n, const char* which, bool critic) {
    char msg[200];
    if (n.depth < 1 || n.depth > QS_MLP_MAX_HIDDEN) {
        snprintf(msg, sizeof(msg), "qs_rollout_mlp: %s: 1 to %d hidden layers (depth %d)", which, QS_MLP_MAX_HIDDEN, n.depth);
        return fail(QS_ERR_SIZE, msg);
    }
    for (int l = 0; l < n.depth; ++l)
        if (n.width[l] < 64 || n.width[l] > QS_MLP_MAX_WIDTH || n.width[l] % 64) {
            snprintf(msg, sizeof(msg), "qs_rollout_mlp: %s: padded hidden widths must be multiples of 64 up to %d (layer %d: %d)", which,
                     QS_MLP_MAX_WIDTH, l, n.width[l]);
            return fail(QS_ERR_SIZE, msg);
        }
    if (critic ? n.out_tiles != 1 : (n.out_tiles != 1 && n.out_tiles != 2 && n.out_tiles != 4)) {
        snprintf(msg, sizeof(msg), "qs_rollout_mlp: %s: out_tiles must be %s", which, critic ? "1" : "1, 2 or 4");
        return fail(QS_ERR_SIZE, msg);
    }
    for (int l = 0; l <= n.depth; ++l) {
        if (!n.w[l] || !n.b[l]) {
            snprintf(msg, sizeof(msg), "qs_rollout_mlp: %s: layer %d weights are NULL", which, l);
            return fail(QS_ERR_NULL, msg);
        }
        if (!aligned16(n.w[l])) return fail(QS_ERR_ALIGN, "qs_rollout_mlp: policy weight arrays must be 16-byte aligned");
    }
    return 0;
}

template <int EFF, bool PIDACT, bool PHYS, int MODE>
void launch_mlp(const MlpRolloutArgs& a, int blocks, cudaStream_t s) {
    auto* k = rollout_mlp_kernel<EFF, PIDACT, PHYS, MODE>;
    const size_t sm = (size_t)a.stage_off + mlp_stage_bytes(a.stage_ks * 16);
    if (sm > 48 * 1024) cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
    {   // carve-out: the resident CTAs (as many as the staging leaves room for, at most the register limit), the rest is L1
        int ctas = (int)((228 * 1024) / (sm + 1024));
        if (ctas > policy_ctas(EFF)) ctas = policy_ctas(EFF);
        if (ctas < 1) ctas = 1;
        const size_t need = (size_t)ctas * (sm + 1024);
        int pct = (int)((need * 100 + 228 * 1024 - 1) / (228 * 1024));
        cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, pct > 100 ? 100 : pct);
    }
    k<<<blocks, 64, sm, s>>>(a);
}

template <bool PHYS, int MODE>
int launch_mlp_family(const MlpRolloutArgs& a, bool pid_act, cudaStream_t s) {
    const int blocks = (int)((a.N + a.tpb - 1) / a.tpb);
#define QS_MCASE(E)                                                                                                   \
    case E:                                                                                                           \
        if (pid_act) launch_mlp<E, true, PHYS, MODE>(a, blocks, s);                                                  \
        else launch_mlp<E, false, PHYS, MODE>(a, blocks, s);                                                         \
        break;
    switch (a.effects & 7u) { QS_MCASE(0) QS_MCASE(QS_EFFECT_GND) QS_MCASE(QS_EFFECT_DRAG) QS_MCASE(QS_EFFECT_DW) QS_MCASE(7) }
#undef QS_MCASE
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, "qs_rollout_mlp launch");
}

}  // namespace

extern "C" {

int qs_sizeof_mlp_policy(void) { return (int)sizeof(QsMlpPolicy); }

int qs_rollout_mlp_max_ticks(int act_type, int act_buffer_size, int drones_per_env, int max_width) {
    const int tmax = qs_rollout_max_ticks(act_type, act_buffer_size, drones_per_env);
    if (tmax <= 0 || drones_per_env > 64 || max_width < 1 || max_width > QS_MLP_MAX_WIDTH) return 0;
    const int A = act_width(act_type), D = drones_per_env;
    const int wpad = (max_width + 63) / 64 * 64;
    // the window grows by A floats per tick; everything else is fixed: downwash's fixed part (the larger), the staging, the
    // scratch with the widest action outputs
    const size_t fixed = policy_smem_fixed(QS_EFFECT_DW) + mlp_stage_bytes(wpad) + 15 + mlp_smem_var(block_size_for(D, 64), 12 + act_buffer_size * A, 0, A, D, 4);
    if (fixed + (size_t)A * 4 > kPolicySmemLimit) return 0;
    const int t_smem = (int)((kPolicySmemLimit - fixed) / ((size_t)A * 4));
    return t_smem < tmax ? t_smem : tmax;
}

int qs_rollout_mlp(const QsParams* p, const QsState* st, const QsRolloutIO* io, const QsMlpPolicy* policy, int act_type, int task,
                   int n_envs, int drones_per_env, int substeps, unsigned effects, unsigned flags, void* stream) {
    if (!policy) return fail(QS_ERR_NULL, "qs_rollout_mlp: NULL policy");
    if (io && io->policy) return fail(QS_ERR_UNSUPPORTED, "qs_rollout_mlp: QsRolloutIO.policy must be NULL (the policy is the QsMlpPolicy argument)");
    const QsMlpPolicy& q = *policy;
    MlpRolloutArgs a;
    memset(&a, 0, sizeof(a));
    bool pid_act = false;
    if (int rc = prepare_rollout(p, st, io, act_type, task, n_envs, drones_per_env, substeps, effects, flags, q.critic.depth > 0, a, pid_act))
        return rc;
    if (int rc = check_policy_config(a, io)) return rc;
    if (q.activation != QS_MLP_TANH && q.activation != QS_MLP_RELU) return fail(QS_ERR_ENUM, "qs_rollout_mlp: activation must be QS_MLP_TANH or QS_MLP_RELU");
    if (int rc = check_net(q.actor, "actor", false)) return rc;
    if (q.critic.depth != 0)
        if (int rc = check_net(q.critic, "critic", true)) return rc;
    if (!q.log_std) return fail(QS_ERR_NULL, "qs_rollout_mlp: log_std is NULL");
    if (q.out_dim > 8 * q.actor.out_tiles) return fail(QS_ERR_SIZE, "qs_rollout_mlp: policy out_dim exceeds the padded output width");
    if (q.in_dim != drones_per_env * a.obs_dim || q.out_dim != drones_per_env * a.A) return fail(QS_ERR_SIZE, "qs_rollout_mlp: policy in_dim/out_dim must be D*obs_dim / D*A");
    if (q.values && q.critic.depth == 0) return fail(QS_ERR_NULL, "qs_rollout_mlp: values requested without a critic");
    const int wmax = net_max_width(q.actor) > net_max_width(q.critic) ? net_max_width(q.actor) : net_max_width(q.critic);
    if (io->T > qs_rollout_mlp_max_ticks(act_type, io->act_buffer_size, drones_per_env, wmax))
        return fail(QS_ERR_UNSUPPORTED, "qs_rollout_mlp: T exceeds qs_rollout_mlp_max_ticks (split the rollout)");
    a.mlp = q;
    a.pol.log_std = q.log_std; a.pol.noise = q.noise; a.pol.logprob = q.logprob; a.pol.values = q.values;
    a.pol.in_dim = q.in_dim; a.pol.out_dim = q.out_dim; a.pol.nt3 = q.actor.out_tiles;
    a.pol.vw1 = q.critic.depth ? q.critic.w[0] : nullptr;
    const size_t sm_var = mlp_smem_var(a.tpb, a.obs_dim, io->T, a.A, drones_per_env, q.actor.out_tiles);
    a.stage_off = (int)((policy_smem_fixed(a.effects & 7u) + sm_var + 15) / 16 * 16);
    a.stage_ks = wmax / 16;
    cudaStream_t s = (cudaStream_t)stream;
    const int mode = (flags & QS_FLAG_AUTORESET_NEXT_STEP) ? kRolloutNext : (io->final_obs || io->final_values) ? kRolloutFin : kRolloutNone;
    if (mode == kRolloutNext) return a.st.phys ? launch_mlp_family<true, kRolloutNext>(a, pid_act, s) : launch_mlp_family<false, kRolloutNext>(a, pid_act, s);
    if (mode == kRolloutFin) return a.st.phys ? launch_mlp_family<true, kRolloutFin>(a, pid_act, s) : launch_mlp_family<false, kRolloutFin>(a, pid_act, s);
    return a.st.phys ? launch_mlp_family<true, kRolloutNone>(a, pid_act, s) : launch_mlp_family<false, kRolloutNone>(a, pid_act, s);
}

}  // extern "C"
