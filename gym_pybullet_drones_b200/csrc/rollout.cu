// rollout.cu -- qs_rollout: T fused control ticks per launch (DESIGN.md 4.1b).
#include "rollout_kernel.cuh"

using namespace qsi;

extern "C" {

int qs_sizeof_rollout_io(void) { return (int)sizeof(QsRolloutIO); }

int qs_rollout_max_ticks(int act_type, int act_buffer_size, int drones_per_env) {
    const int A = act_width(act_type);
    if (A < 0 || act_type == QS_ACT_RAW_RPM || act_buffer_size <= 0 || drones_per_env <= 0 || drones_per_env > kMaxTPB) return 0;
    const size_t span = (size_t)block_size_for(drones_per_env) * (12 + act_buffer_size * A) * 4;
    if (span + 2 * (size_t)A * 4 > kStageLimit) return 0;
    return (int)((kStageLimit - span) / ((size_t)A * 4)) - 1;
}

int qs_rollout(const QsParams* p, const QsState* st, const QsRolloutIO* io, int act_type, int task,
               int n_envs, int drones_per_env, int substeps, unsigned effects, unsigned flags, void* stream) {
    RolloutArgs a;
    bool pid_act = false;
    if (int rc = prepare_rollout(p, st, io, act_type, task, n_envs, drones_per_env, substeps, effects, flags,
                                 io && io->policy && io->policy->vw1, a, pid_act))
        return rc;
    if (flags & QS_FLAG_AUTORESET_NEXT_STEP) return launch_rollout_next(a, io, pid_act, stream);
    if (io->final_obs || io->final_values)
        return a.st.phys ? launch_rollout<true, kRolloutFin>(a, io, pid_act, stream) : launch_rollout<false, kRolloutFin>(a, io, pid_act, stream);
    return a.st.phys ? launch_rollout<true, kRolloutNone>(a, io, pid_act, stream) : launch_rollout<false, kRolloutNone>(a, io, pid_act, stream);
}

}  // extern "C"

namespace qsi {

int prepare_rollout(const QsParams* p, const QsState* st, const QsRolloutIO* io, int act_type, int task, int n_envs, int drones_per_env,
                    int substeps, unsigned effects, unsigned flags, bool has_critic, RolloutArgs& a, bool& pid_act) {
    if (!p || !io) return fail(QS_ERR_NULL, "qs_rollout: NULL params/io");
    const bool next_step = flags & QS_FLAG_AUTORESET_NEXT_STEP;
    if (int rc = check_state(st, (flags & (QS_FLAG_AUTORESET_SAME_STEP | QS_FLAG_AUTORESET_NEXT_STEP)) ? 1 : 0)) return rc;
    if (n_envs <= 0 || drones_per_env <= 0 || substeps <= 0 || io->T <= 0) return fail(QS_ERR_SIZE, "qs_rollout: sizes must be > 0");
    const int A = act_width(act_type);
    if (A < 0 || act_type == QS_ACT_RAW_RPM) return fail(QS_ERR_ENUM, "qs_rollout: bad act_type");
    if (task != QS_TASK_NONE && task != QS_TASK_HOVER) return fail(QS_ERR_ENUM, "qs_rollout: bad task");
    if (effects & ~7u) return fail(QS_ERR_ENUM, "qs_rollout: bad effects");
    if ((flags & QS_FLAG_AUTORESET_SAME_STEP) && next_step) return fail(QS_ERR_ENUM, "qs_rollout: two autoreset modes");
    if (flags & (QS_FLAG_SKIP_EPILOGUE | QS_FLAG_RPM_FROM_LAST | QS_FLAG_OBS_STATE20))
        return fail(QS_ERR_UNSUPPORTED, "qs_rollout: SKIP_EPILOGUE, RPM_FROM_LAST and OBS_STATE20 are not supported");
    if (next_step && !st->pending_reset) return fail(QS_ERR_NULL, "qs_rollout: NEXT_STEP autoreset needs pending_reset");
    if (drones_per_env > kMaxTPB) return fail(QS_ERR_UNSUPPORTED, "qs_rollout: drones_per_env <= 128");
    if (!io->obs_init || !io->obs || !io->reward || !io->terminated || !io->truncated) return fail(QS_ERR_NULL, "qs_rollout: NULL buffer");
    if ((io->final_obs || io->final_values) && !(flags & QS_FLAG_AUTORESET_SAME_STEP))
        return fail(QS_ERR_UNSUPPORTED, "qs_rollout: final_obs / final_values need QS_FLAG_AUTORESET_SAME_STEP");
    if (io->final_values && !has_critic) return fail(QS_ERR_NULL, "qs_rollout: final_values requested without a policy critic");
    if (io->act_buffer_size <= 0) return fail(QS_ERR_SIZE, "qs_rollout: act_buffer_size must be > 0");
    if (io->T > qs_rollout_max_ticks(act_type, io->act_buffer_size, drones_per_env)) return fail(QS_ERR_UNSUPPORTED, "qs_rollout: T exceeds qs_rollout_max_ticks (split the rollout)");
    if (task == QS_TASK_HOVER && (!st->target_pos || !aligned32(st->target_pos))) return fail(QS_ERR_NULL, "qs_rollout: target_pos NULL/misaligned");
    pid_act = act_type == QS_ACT_PID || act_type == QS_ACT_VEL || act_type == QS_ACT_ONE_D_PID;
    if (pid_act && !st->pid) return fail(QS_ERR_NULL, "qs_rollout: PID action type needs QsState.pid");
    if ((effects & QS_EFFECT_DRAG) && !st->last_rpm) return fail(QS_ERR_NULL, "qs_rollout: DRAG needs QsState.last_rpm");
    if (A == 4 && ((io->actions && !aligned16(io->actions)) || (io->actions_out && !aligned16(io->actions_out)) || !aligned16(io->obs) || (io->obs_last && !aligned16(io->obs_last))))
        return fail(QS_ERR_ALIGN, "qs_rollout: [N][4]-wide buffers must be 16-byte aligned");
    memset(&a, 0, sizeof(a));
    a.P = *p; a.st = *st; a.io = *io;
    a.act_type = act_type; a.task = task; a.n_envs = n_envs; a.D = drones_per_env; a.substeps = substeps;
    if ((long long)n_envs * drones_per_env > 0x7fffffffLL) return fail(QS_ERR_SIZE, "qs_rollout: n_envs * drones_per_env exceeds 2^31-1");
    a.N = n_envs * drones_per_env; a.A = A; a.obs_dim = 12 + io->act_buffer_size * A;
    a.cap = cta_capacity(a.N, drones_per_env, true);
    a.tpb = block_size_for(drones_per_env, a.cap);
    a.effects = effects; a.flags = flags;
    {
        const size_t row_bytes = (size_t)a.obs_dim * 4, span = row_bytes * a.tpb;
        const bool aligned = aligned16(io->obs_init) && (span % 16 == 0) && ((row_bytes * ((size_t)a.N % a.tpb)) % 16 == 0);
        a.stage_mode = (aligned && A == 4) ? 1 : 2;
    }
    return 0;
}

int check_policy_config(const RolloutArgs& a, const QsRolloutIO* io) {
    const unsigned eff = a.effects & 7u;
    if (eff != 0 && eff != QS_EFFECT_GND && eff != QS_EFFECT_DRAG && eff != QS_EFFECT_DW && eff != 7u)
        return fail(QS_ERR_UNSUPPORTED, "qs_rollout: the on-device policy supports no DYN+ effect, GND, DRAG, DW or all three; not GND|DRAG, GND|DW or DRAG|DW");
    if (a.cap > 64) return fail(QS_ERR_UNSUPPORTED, "qs_rollout: the on-device policy supports drones_per_env <= 64");
    if (io->actions) return fail(QS_ERR_UNSUPPORTED, "qs_rollout: pass either actions or a policy");
    return 0;
}

}  // namespace qsi
