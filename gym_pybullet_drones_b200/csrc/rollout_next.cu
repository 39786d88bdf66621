// rollout_next.cu -- qs_rollout with NEXT_STEP autoreset: the rollout kernel's NEXT instantiations (rollout_kernel.cuh), kept out
// of rollout.cu so that the two translation units compile in parallel.
#include "rollout_kernel.cuh"

namespace qsi {

int launch_rollout_next(RolloutArgs& a, const QsRolloutIO* io, bool pid_act, void* stream) {
    return a.st.phys ? launch_rollout<true, kRolloutNext>(a, io, pid_act, stream) : launch_rollout<false, kRolloutNext>(a, io, pid_act, stream);
}

}  // namespace qsi
