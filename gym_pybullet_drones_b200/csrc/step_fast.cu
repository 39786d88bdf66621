// step_fast.cu -- the fused control tick for the common RL configurations (BaseAviary.step, envs/BaseAviary.py:259-383,
// with BaseRLAviary's RPM / ONE_D_RPM actions, KIN observations and the Hover/MultiHover task): no DYN+ effects, no
// embedded PID, aviaries of 1, 2, 4, ... 32 drones, autoreset SAME_STEP or none.  Everything else takes step_general.cu.
//
// Same arithmetic as the general kernel (the per-drone functions of quad_core.cuh), different skeleton:
//   * a TILE of 32 consecutive drones = one contiguous span of observation rows with its own mbarrier and shared-memory
//     window is the unit of work, run by one warp; each CTA is one warp, no __syncthreads anywhere, the aviary reduction is
//     a warp shuffle (aviaries never straddle tiles)
//   * two kernels run one tile's work (tile_step): step_fast_kernel, one tile per warp, and step_pipe_kernel (A = 4 without
//     the fused gather), four tiles per warp with the next tile's loads issued under the current tile's physics
//   * A, the task, the autoreset mode and the rpy precision are template parameters: the instruction stream of an
//     instantiation contains no mode switches (round 1's kernel: 268 IMAD, 101 BRA per warp)
//   * state in/out as 3 x 32 bytes (two 16-byte vector accesses each) + 1 x 8 bytes per thread (float64 planes, no conversions)
//   * A = 4: the old span is TMA-loaded and TMA-stored shifted by one action (16 bytes); the new heads and actions go into the
//     span in shared memory first (pipelined kernel) or over the stored rows afterwards (classic kernel, whose store starts
//     as soon as the span has landed); A = 1: the span is TMA-loaded, funnel-shifted by one float with 128-bit shared-memory
//     accesses into a second 16-byte-aligned window, patched there and TMA-stored
//   * the observation of a freshly reset drone (SAME_STEP autoreset) comes from a precomputed table (qs_reset_heads),
//     not from two atan2f and an asinf in the epilogue
#include "qs_common.cuh"

#ifdef QS_TIMELINE
// debug build only (tools/timeline.py): per-warp phase timestamps (%globaltimer, ns) of the last launch
__device__ unsigned long long g_timeline[4][8192 * 16];
static int g_dbg_slot = 0;
#define QS_STAMP(k) do { if (lane == 0 && wg < 8192) g_timeline[a.dbg_slot & 3][wg * 16 + (k)] = globaltimer_ns(); } while (0)
#define QS_TSTAMP(t, k) do { if (lane == 0 && (t) < 8192) g_timeline[a.dbg_slot & 3][(t) * 16 + (k)] = globaltimer_ns(); } while (0)
#else
#define QS_STAMP(k) do { } while (0)
#define QS_TSTAMP(t, k) do { } while (0)
#endif

namespace qsi {
namespace {

template <int A>
struct FastSmem {
    // per-warp shared-memory window, in floats
    static __host__ __device__ constexpr int span(int od) { return 32 * od; }
    // A = 4: [span + 4 tail floats (rounded to 16 B)] ; A = 1: [X: span + 4 (the shift reads one float past the span)] [Y: span]
    static __host__ __device__ constexpr int x_floats(int od) { return (span(od) + 4 + 3) / 4 * 4; }
    static __host__ __device__ constexpr int y_floats(int od) { return A == 4 ? 0 : (span(od) + 3) / 4 * 4; }
    static __host__ __device__ constexpr int fin_floats(bool fin) { return fin ? 32 * 12 : 0; }
    static __host__ __device__ constexpr int total_bytes(int od, bool fin) {
        return ((x_floats(od) + y_floats(od) + fin_floats(fin)) * 4 + 16 + 127) / 128 * 128;      // + mbarrier, 128-byte multiple
    }
};

// Dead lanes of a ragged last tile shadow the tile's first drone (il) for their loads and store nothing.
struct TileLane { long long i, il, e, tbl; int dslot; bool live; };
__device__ __forceinline__ TileLane tile_lane(const StepArgs& a, long long N, int D, long long w0, int lane) {
    TileLane t;
    t.i = w0 + lane;
    t.live = t.i < N;
    t.il = t.live ? t.i : w0;
    t.e = t.il >> a.log2D;
    t.dslot = (int)t.il & (D - 1);                                          // D is a power of two <= 32
    t.tbl = a.st.tables_per_env ? t.il : t.dslot;
    return t;
}

// What the kernels still need after tile_step: whether the drone was reset (its terminal head is then in fin_s), and for the
// fused gather its aviary's reward and flags.
struct TileEnd { bool reset_me; float rew; bool term, trunc; };

// One 32-drone tile's work, from the action decode to the state stores: S substeps, the task terms reduced over the aviary, the
// per-aviary outputs, the observation head h (the reset table's head for a drone reset in this step) and the state, last_rpm and
// step-counter stores.  Both fast kernels run it, so they give the same bits.  substep(s) runs between substeps (the classic
// kernel's early store); stamp(p) marks point p of the tile for the timeline build: 0 physics done, 1 derived, 2 task terms
// stored, 3 state stored.
template <int A, bool TASK, bool RESET, bool RPYF, bool PHYS, class Substep, class Stamp>
__device__ __forceinline__ TileEnd tile_step(const StepArgs& a, long long N, int D, const TileLane& t, int lane, qs::Drone& d, const float act[4], int sc,
                                             const qs::PhysRow& ph, const D4& tp, bool want_fin, float* fin_s, float h[12],
                                             Substep substep, Stamp stamp) {
    const QsParams& P = a.P;
    const int dmask = D - 1;

    // ---- action decode (BaseRLAviary.py:192,225) + S substeps ---------------------------------------------------------------
    double rpm[4];
    {
        qs::PidState none = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        if constexpr (PHYS) qs::decode_action_k<false>(P, ph, A == 4 ? QS_ACT_RPM : QS_ACT_ONE_D_RPM, act, d, 0.0, none, rpm);
        else qs::decode_action<false>(P, A == 4 ? QS_ACT_RPM : QS_ACT_ONE_D_RPM, act, d, 0.0, none, rpm);
    }
    double R_last[9];
    if constexpr (PHYS) qs::dyn_tick_k<0>(P, ph, d, rpm, rpm, 0.0, a.substeps, R_last, substep);
    else qs::dyn_tick<0>(P, d, rpm, rpm, 0.0, a.substeps, R_last, substep);
    stamp(0);
    qs::Derived o;
    qs::derive<RPYF>(d, R_last, o);
    stamp(1);

    // ---- task terms, reduced over the D drones of the aviary in index order (MultiHoverAviary.py:75-130) ----------------------
    TileEnd r = {false, -1.0f, false, false};
    bool env_done = false;
    if (TASK) {
        const qs::TaskTerms tt = qs::hover_terms(P, d, o, tp.x, tp.y, tp.z);
        double rew = 0.0, dist = 0.0;
        const int base = lane & ~dmask;
        for (int k = 0; k < D; ++k) {
            rew += __shfl_sync(0xffffffffu, tt.reward, base + k);
            dist += __shfl_sync(0xffffffffu, tt.dist, base + k);
        }
        const unsigned oobs = __ballot_sync(0xffffffffu, tt.out_of_bounds && t.live);
        const unsigned gmask = (D == 32 ? 0xffffffffu : ((1u << D) - 1u)) << base;
        const bool term = dist < P.term_dist;                                     // HoverAviary.py:91
        const bool trunc = (oobs & gmask) != 0u || sc >= a.sc_limit;              // HoverAviary.py:113 (sc/PYB_FREQ > EPISODE_LEN_SEC)
        env_done = term || trunc;
        r.rew = (float)rew; r.term = term; r.trunc = trunc;
        if (t.live && t.dslot == 0) {
            a.io.reward[t.e] = (float)rew;
            a.io.terminated[t.e] = term ? 1 : 0;
            a.io.truncated[t.e] = trunc ? 1 : 0;
            if (a.io.done) a.io.done[t.e] = env_done ? 1 : 0;
        }
    } else if (t.live && t.dslot == 0) {
        a.io.reward[t.e] = -1.0f; a.io.terminated[t.e] = 0; a.io.truncated[t.e] = 0;     // CtrlAviary-style dummy task
        if (a.io.done) a.io.done[t.e] = 0;
    }
    stamp(2);

    // ---- observation head, autoreset, state store ----------------------------------------------------------------------------
    h[0] = (float)d.px; h[1] = (float)d.py; h[2] = (float)d.pz;                    // BaseRLAviary.py:310-315
    h[3] = (float)o.roll; h[4] = (float)o.pitch; h[5] = (float)o.yaw;
    h[6] = (float)d.vx; h[7] = (float)d.vy; h[8] = (float)d.vz;
    h[9] = (float)o.ax; h[10] = (float)o.ay; h[11] = (float)o.az;
    r.reset_me = RESET && env_done;
    if (r.reset_me) {
        if (want_fin) {                                                            // terminal head, for final_obs
            float4* f4 = reinterpret_cast<float4*>(fin_s + 12 * lane);
            f4[0] = make_float4(h[0], h[1], h[2], h[3]); f4[1] = make_float4(h[4], h[5], h[6], h[7]); f4[2] = make_float4(h[8], h[9], h[10], h[11]);
        }
        init_drone(a.st, t.tbl, d);                                                // BaseAviary.py:451-505
        const float4* rh = reinterpret_cast<const float4*>(a.st.reset_head) + 3 * t.tbl;
        const float4 r0 = __ldg(rh), r1 = __ldg(rh + 1), r2 = __ldg(rh + 2);
        h[0] = r0.x; h[1] = r0.y; h[2] = r0.z; h[3] = r0.w; h[4] = r1.x; h[5] = r1.y; h[6] = r1.z; h[7] = r1.w;
        h[8] = r2.x; h[9] = r2.y; h[10] = r2.z; h[11] = r2.w;
        rpm[0] = rpm[1] = rpm[2] = rpm[3] = 0.0;                                   // last_clipped_action = 0
        sc = -a.counter_inc;
    }
    if (t.live) {
        store_drone(a.st, N, t.i, d);
        if (a.st.last_rpm) st256(a.st.last_rpm, t.i, rpm[0], rpm[1], rpm[2], rpm[3]);
        if (t.dslot == 0) a.st.step_counter[t.e] = sc + a.counter_inc;             // BaseAviary.py:382
    }
    stamp(3);
    return r;
}

// A = 4: the drone's new head -> slots [4, 16) of its row of the old span in shared memory, its new action -> the 4 slots after
// the row.  The span read 16 bytes further on (shifted) is then the tile's new span.
__device__ __forceinline__ void patch_row_a4(float* xs, int od, int lane, bool live, const float h[12], const float act[4]) {
    if (live) {
        float* row = xs + (size_t)lane * od;
        float4* r4 = reinterpret_cast<float4*>(row + 4);
        r4[0] = make_float4(h[0], h[1], h[2], h[3]); r4[1] = make_float4(h[4], h[5], h[6], h[7]); r4[2] = make_float4(h[8], h[9], h[10], h[11]);
        *reinterpret_cast<float4*>(row + od) = make_float4(act[0], act[1], act[2], act[3]);
    }
    __syncwarp();
}

// A = 4: the terminal observations (final_obs rows of the tile) of the rows in m: the head from fin_s, the history from the
// shifted span.  The newest action comes from the span when patch_row_a4 has run (PATCHED), else from lane r's act.
template <bool PATCHED>
__device__ __forceinline__ void store_final_rows(float* final_obs, const float* fin_s, const float4* shifted, int od, unsigned m, int lane,
                                                 const float act[4]) {
    const int c4n = od >> 2;
    float4* fin = reinterpret_cast<float4*>(final_obs);
    for (; m; m &= m - 1) {
        const int r = __ffs(m) - 1;
        float4 ar = make_float4(0.f, 0.f, 0.f, 0.f);
        if constexpr (!PATCHED)
            ar = make_float4(__shfl_sync(0xffffffffu, act[0], r), __shfl_sync(0xffffffffu, act[1], r),
                             __shfl_sync(0xffffffffu, act[2], r), __shfl_sync(0xffffffffu, act[3], r));
        for (int c = lane; c < c4n; c += 32)
            fin[r * c4n + c] = c < 3 ? reinterpret_cast<const float4*>(fin_s + 12 * r)[c] : (PATCHED || c < c4n - 1 ? shifted[r * c4n + c] : ar);
    }
}

// ---- the classic kernel: one 32-drone tile per warp, one warp per CTA ------------------------------------------------------------
// A: action width (4 = RPM, 1 = ONE_D_RPM).  TASK: Hover/MultiHover reward + flags (else the CtrlAviary-style dummy task).
// RESET: SAME_STEP autoreset.  RPYF: float32 atan2f/asinf for the reported rpy.
// PHYS: the drone's physical constants come from its aviary's row of QsState.phys (else from QsParams).
template <int A, bool TASK, bool RESET, bool RPYF, bool PHYS>
__global__ void __launch_bounds__(32) step_fast_kernel(const __grid_constant__ StepArgs a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int lane = threadIdx.x;
    const int od = a.obs_dim;
    const long long N = a.N;
    const long long wg = (long long)a.first_warp + (long long)blockIdx.x;  // global warp index (a launch may cover a chunk)
    const long long w0 = wg * 32;                                           // first drone of this warp
    if (w0 >= N) return;
    const int D = a.D;
    const TileLane t = tile_lane(a, N, D, w0, lane);
    const int rows = (int)((N - w0) < 32 ? (N - w0) : 32);
    const bool want_fin = RESET && a.io.final_obs != nullptr;

    float* xs = reinterpret_cast<float*>(smem_raw);
    float* ys = xs + FastSmem<A>::x_floats(od);
    float* fin_s = ys + FastSmem<A>::y_floats(od);
    unsigned long long* bar = reinterpret_cast<unsigned long long*>(fin_s + FastSmem<A>::fin_floats(want_fin));

    const float* span_src = a.io.obs_prev + w0 * od;
    float* span_dst = a.io.obs + w0 * od;
    const unsigned span_bytes = (unsigned)(rows * od * 4);
    QS_STAMP(0);
    if (lane == 0) mbar_init(bar, 1);
    // read-only tables (never written by a kernel): safe ahead of the dependency wait
    D4 tp = {0.0, 0.0, 0.0, 0.0};
    if (TASK) tp = ld256_nc(a.st.target_pos, t.tbl);

    // ---- readiness (DESIGN.md 4.1) ----------------------------------------------------------------------------------------
    // This warp's ticket among the steps on these buffers: taken (the atomic has returned, hence the shuffle) BEFORE the CTA lets
    // the next grid launch, so tickets follow launch order and a warp only ever waits for a warp that is already resident.
    // Then, with grid_wait, the whole previous grid (it was not a fast step); then the previous step's warp of the same 32
    // drones.  Nothing written by an earlier kernel is read above this point.
    const bool ticketed = a.io.warp_ticket != nullptr;
    unsigned ticket = 0;
    if (ticketed) {
        if (lane == 0) ticket = atomicAdd(a.io.warp_ticket + wg, 1u);
        ticket = __shfl_sync(0xffffffffu, ticket, 0);
    }
    if (a.grid_wait) asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");        // let the next grid's CTAs take the free slots now
    if (ticketed && lane == 0) warp_wait_turn(a.io.warp_done + wg, ticket, a.io.ready_err);
    __syncwarp();
    QS_STAMP(1);
    // the end of this warp's work: its bulk stores have COMPLETED, then the next step's warp of these drones may go
    auto publish = [&]() {
        if (!ticketed) return;
        if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
        warp_publish(a.io.warp_done + wg, ticket + 1u);
    };

    // ---- loads: state (3 x 32 B + 8 B), action, step counter; then the bulk copy of the old observation span ------------
    qs::Drone d;
    float act[4] = {0.f, 0.f, 0.f, 0.f};
    int sc = 0;
    load_drone(a.st.planes, N, t.il, d);
    if (A == 4) {
        const float4 v = ldg4(a.io.action, t.il);
        act[0] = v.x; act[1] = v.y; act[2] = v.z; act[3] = v.w;
    } else {
        act[0] = __ldg(a.io.action + t.il);
    }
    sc = a.st.step_counter[t.e];
    qs::PhysRow ph;
    if constexpr (PHYS) ph = load_phys(a.st.phys, t.e);                    // one row per aviary: aviaries never straddle warps
    // The bulk copy of the old span (9 KB per warp) is issued only once the step counter -- and with it the batch of small
    // state loads issued just before it -- has ARRIVED: warps issue in order, so the comparison below stalls until then, and
    // the memory system serves every warp's 120 bytes of state ahead of the 19 MB of history the physics does not need yet.
    // (The comparison is always true for a valid counter; the compiler cannot know.)
    auto load_span = [&]() {
        // the old span is dead once copied (the next launch on these buffers overwrites it): evict-first in L2, so its 19 MB
        // make room for this launch's stores and the next launch's state instead of pushing them out (+3 % per step, DESIGN.md 6)
        if (lane == 0) tma_bulk_g2s_read_once(xs, span_src, span_bytes, bar);
    };
    bool issued = false;
    if (__shfl_sync(0xffffffffu, sc, 0) != (int)0x80000000) {
        load_span();
        issued = true;
    }
    QS_STAMP(2);

    // A = 4: the history part of the new rows does not depend on the physics: as soon as the old span has landed (polled between
    // substeps) the copy engine writes it back shifted by one action; the heads and the new actions follow at the end as
    // ordinary stores.  So the 19 MB of history stores overlap the FP64 loop instead of following it.
    const float4* shifted = reinterpret_cast<const float4*>(xs) + 1;
    bool stored = false;
    auto store_span = [&]() {
        if (lane == 0) {
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(span_dst), "r"(smem_u32(shifted)), "r"(span_bytes) : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
        stored = true;
    };
    auto poll = [&](int s) {
        if (A == 4 && issued && !stored && (s & 1)) {
            int ok = 0;
            if (lane == 0) ok = mbar_test(bar, 0) ? 1 : 0;
            if (__shfl_sync(0xffffffffu, ok, 0)) store_span();
        }
    };
    float h[12];
    const TileEnd te = tile_step<A, TASK, RESET, RPYF, PHYS>(a, N, D, t, lane, d, act, sc, ph, tp, want_fin, fin_s, h, poll,
                                                             [&](int p) { QS_STAMP(3 + p); });

    // ---- observation rows --------------------------------------------------------------------------------------------------------
    if (!issued) load_span();
    const unsigned fin_rows = want_fin ? __ballot_sync(0xffffffffu, te.reset_me && t.live) : 0u;
    // Fused observation gather: the finished rows go a second time, straight from shared memory, to the learner's tensor
    // (peer memory over NVLink), the per-aviary outputs with them; the last warp of the grid raises the learner's flag.
    auto gather = [&](const void* rows_smem) {
        if (lane == 0) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                         ::"l"(a.io.obs_gather + w0 * od), "r"(smem_u32(rows_smem)), "r"(span_bytes) : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
        if (t.live && t.dslot == 0) {
            if (a.io.reward_gather) a.io.reward_gather[t.e] = te.rew;
            if (a.io.terminated_gather) a.io.terminated_gather[t.e] = te.term ? 1 : 0;
            if (a.io.truncated_gather) a.io.truncated_gather[t.e] = te.trunc ? 1 : 0;
        }
        if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");      // rows written (not only read) before the flag
        __syncwarp();
        if (a.io.gather_flag) {
            __threadfence_system();
            if (lane == 0) {
                const unsigned nwarps = (unsigned)((N + 31) / 32);
                if (atomicAdd(a.io.gather_counter, 1u) == nwarps - 1u) {
                    *a.io.gather_counter = 0u;
                    __threadfence_system();
                    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(a.io.gather_flag), "r"(a.io.gather_seq) : "memory");
                }
            }
        }
    };
    if (A == 4) {
        if (!stored) { mbar_wait(bar, 0); store_span(); }
        if (want_fin) {
            __syncwarp();
            store_final_rows<false>(a.io.final_obs + w0 * od, fin_s, shifted, od, fin_rows, lane, act);
        }
        QS_STAMP(7);
        // the bulk store wrote stale values into the head and newest-action slots of every row: wait until it has completed,
        // then overwrite them (same addresses: the generic stores must be ordered after the asynchronous ones)
        if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
        __syncwarp();
        if (t.live) {
            float4* row = reinterpret_cast<float4*>(a.io.obs + t.i * od);
            row[0] = make_float4(h[0], h[1], h[2], h[3]); row[1] = make_float4(h[4], h[5], h[6], h[7]); row[2] = make_float4(h[8], h[9], h[10], h[11]);
            row[(od >> 2) - 1] = make_float4(act[0], act[1], act[2], act[3]);
        }
        QS_STAMP(8);
        if (a.io.obs_gather) { patch_row_a4(xs, od, lane, t.live, h, act); gather(shifted); }      // (the bulk store has completed: shared memory is free)
        publish();
        return;
    }
    // A = 1: funnel shift by one float, ys[j] = xs[j + 1], four floats per thread and iteration (LDS.128 + one shuffle + STS.128)
    mbar_wait(bar, 0);
    QS_STAMP(7);
    const int n4 = (rows * od + 3) >> 2;
    for (int j = lane; j < ((n4 + 31) & ~31); j += 32) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (j <= n4) v = reinterpret_cast<const float4*>(xs)[j];              // j == n4: the float past the span (padding)
        float nx = __shfl_down_sync(0xffffffffu, v.x, 1);
        if (lane == 31 && j + 1 <= n4) nx = xs[4 * (j + 1)];
        if (j < n4) reinterpret_cast<float4*>(ys)[j] = make_float4(v.y, v.z, v.w, nx);
    }
    __syncwarp();
    if (t.live) {
        float* row = ys + (size_t)lane * od;                                  // od = 12 + B: odd word stride for B = 15, conflict-free
#pragma unroll
        for (int k = 0; k < 12; ++k) row[k] = h[k];
        row[od - 1] = act[0];
    }
    __syncwarp();
    if (lane == 0) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(span_dst), "r"(smem_u32(ys)), "r"(span_bytes) : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    if (want_fin) {
        float* fin = a.io.final_obs + w0 * od;
        for (unsigned m = fin_rows; m; m &= m - 1) {
            const int r = __ffs(m) - 1;
            for (int c = lane; c < od; c += 32) fin[r * od + c] = c < 12 ? fin_s[12 * r + c] : ys[r * od + c];
        }
    }
    QS_STAMP(8);
    if (a.io.obs_gather) { gather(ys); publish(); return; }
    if (ticketed) publish();
    else if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // shared memory must outlive the bulk store's reads
    QS_STAMP(9);
}

// ---- the pipelined kernel (A = 4): kPipeTiles consecutive 32-drone tiles per warp, two shared-memory stages -------------------
// A tile is the classic kernel's warp unit (its own span of rows, ticket word and done word).  While tile k runs its physics,
// tile k+1's state and actions are on their way into registers and its old span into the other stage, and tile k-1's bulk
// store is still being written.  A tile is published once its bulk store has completed, which the warp checks only after it has
// committed the next tile's store, so the completion round trip is off the critical path too.  Same tile_step as the classic
// kernel: the output bits are the classic kernel's.
// The state and actions travel through registers, not shared memory: 20 KB per warp (B = 15) fit 10 warps on an SM.
// Four tiles per warp measured faster than two on the bench, at 262 144 and at 1 M drones (DESIGN.md 6).
constexpr int kPipeTiles = 4;
struct PipeSmem {
    static __host__ __device__ constexpr int bar_off(int od) { return FastSmem<4>::x_floats(od) * 4; }
    // [old span + 16-byte tail][its mbarrier], 128-byte multiple
    static __host__ __device__ constexpr int stage_bytes(int od) { return (bar_off(od) + 8 + 127) / 128 * 128; }
    static __host__ __device__ constexpr int total_bytes(int od, bool fin) { return 2 * stage_bytes(od) + (fin ? 32 * 12 * 4 : 0); }
};

template <bool TASK, bool RESET, bool RPYF, bool PHYS>
__global__ void __launch_bounds__(32) step_pipe_kernel(const __grid_constant__ StepArgs a) {
    constexpr int K = kPipeTiles;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int lane = threadIdx.x;
    const int od = a.obs_dim;
    const long long N = a.N;
    const long long tiles = (N + 31) / 32;
    const long long t_end = a.n_warps > 0 && (long long)a.first_warp + a.n_warps < tiles ? (long long)a.first_warp + a.n_warps : tiles;
    const long long t0 = (long long)a.first_warp + (long long)blockIdx.x * K;      // first tile of this warp
    if (t0 >= t_end) return;
    const int nt = (int)(t_end - t0 < K ? t_end - t0 : K);
    const bool want_fin = RESET && a.io.final_obs != nullptr;
    const int SB = PipeSmem::stage_bytes(od);
    float* fin_s = reinterpret_cast<float*>(smem_raw + 2 * SB);
    auto stage = [&](int k) { return smem_raw + (k & 1) * SB; };
    auto bar_of = [&](int k) { return reinterpret_cast<unsigned long long*>(stage(k) + PipeSmem::bar_off(od)); };
    const int D = a.D;
    QS_TSTAMP(t0, 0);
    if (lane == 0) { mbar_init(bar_of(0), 1); mbar_init(bar_of(1), 1); }

    // ---- readiness, per tile (DESIGN.md 4.1): lane j takes the ticket of tile j before the next grid may launch, then tries
    // its tile's done word once; a tile found not ready is waited for when its turn comes
    const bool ticketed = a.io.warp_ticket != nullptr;
    unsigned my_ticket = 0;
    if (ticketed && lane < nt) my_ticket = atomicAdd(a.io.warp_ticket + t0 + lane, 1u);
    const unsigned ticket0 = __shfl_sync(0xffffffffu, my_ticket, 0);           // (every lane's atomic has returned)
    if (a.grid_wait) asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    bool rdy = !ticketed;
    if (ticketed && lane < nt) {
        unsigned v;
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(a.io.warp_done + t0 + lane) : "memory");
        rdy = v == my_ticket;
        if (rdy) asm volatile("fence.proxy.async.global;" ::: "memory");
    }
    const unsigned ready_mask = __ballot_sync(0xffffffffu, rdy);
    auto try_turn = [&](int k) -> bool {
        if ((ready_mask >> k) & 1u) return true;
        const unsigned tk = __shfl_sync(0xffffffffu, my_ticket, k);
        int ok = 0;
        if (lane == 0) {
            unsigned v;
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(a.io.warp_done + t0 + k) : "memory");
            ok = v == tk;
            if (ok) asm volatile("fence.proxy.async.global;" ::: "memory");
        }
        return __shfl_sync(0xffffffffu, ok, 0) != 0;
    };
    auto wait_turn = [&](int k, unsigned tk) {          // blocking: the warp holds no finished, unpublished tile here
        if (!((ready_mask >> k) & 1u) && lane == 0) warp_wait_turn(a.io.warp_done + t0 + k, tk, a.io.ready_err);
    };
    auto publish = [&](int k, bool all_done) {          // tile k's stores have completed: all_done = no later group outstanding
        if (!ticketed) return;
        const unsigned tk = __shfl_sync(0xffffffffu, my_ticket, k);
        if (lane == 0) {
            if (all_done) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
            else asm volatile("cp.async.bulk.wait_group 1;" ::: "memory");
        }
        warp_publish(a.io.warp_done + t0 + k, tk + 1u);
        QS_TSTAMP(t0 + k, 7);
    };
    // tile k's loads, after its readiness: state and action into registers (consumed when tile k starts), the old span into
    // stage k & 1.  Dead lanes of a ragged last tile shadow its first drone, as in the classic kernel.
    qs::Drone dn;
    float4 an;
    auto issue = [&](int k) {
        __syncwarp();
        const long long w0 = (t0 + k) * 32;
        const long long il = w0 + lane < N ? w0 + lane : w0;
        load_drone(a.st.planes, N, il, dn);
        an = ldg4(a.io.action, il);
        if (lane == 0) {
            const int rows = (int)(N - w0 < 32 ? N - w0 : 32);
            asm volatile("fence.proxy.async.global;" ::: "memory");
            tma_bulk_g2s_read_once(stage(k), a.io.obs_prev + w0 * od, (unsigned)(rows * od * 4), bar_of(k));
        }
        QS_TSTAMP(t0 + k, 1);
    };
#ifdef QS_TIMELINE
    for (int k = 1; k < nt; ++k) QS_TSTAMP(t0 + k, 0);
#endif
    __syncwarp();
    wait_turn(0, ticket0);
    issue(0);

    int pend = -1;                                      // finished tile whose publish is outstanding
    for (int k = 0; k < nt; ++k) {
        const long long tg = t0 + k;
        const unsigned par = (unsigned)(k >> 1) & 1u;
        qs::Drone d = dn;
        const float4 av = an;
        bool pre = false;
        if (k + 1 < nt && try_turn(k + 1)) {
            // stage (k + 1) & 1 held tile k-1, whose bulk store must have finished reading it
            if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            issue(k + 1);
            pre = true;
        }
        const long long w0 = tg * 32;
        const TileLane t = tile_lane(a, N, D, w0, lane);
        const int rows = (int)((N - w0) < 32 ? (N - w0) : 32);
        unsigned long long* bar = bar_of(k);
        float* xs = reinterpret_cast<float*>(stage(k));
        D4 tp = {0.0, 0.0, 0.0, 0.0};
        if (TASK) tp = ld256_nc(a.st.target_pos, t.tbl);
        const int sc = a.st.step_counter[t.e];
        qs::PhysRow ph;
        if constexpr (PHYS) ph = load_phys(a.st.phys, t.e);

        QS_TSTAMP(tg, 2);
        const float act[4] = {av.x, av.y, av.z, av.w};
        float h[12];
        const TileEnd te = tile_step<4, TASK, RESET, RPYF, PHYS>(a, N, D, t, lane, d, act, sc, ph, tp, want_fin, fin_s, h, qs::NoHook(),
                                                                 [&](int p) { if (p == 0) QS_TSTAMP(tg, 3); else if (p == 3) QS_TSTAMP(tg, 4); });

        // ---- observation rows: patched in shared memory, one bulk store of the shifted span ----------------------------------
        const unsigned fin_rows = want_fin ? __ballot_sync(0xffffffffu, te.reset_me && t.live) : 0u;
        mbar_wait(bar, par);
        QS_TSTAMP(tg, 5);
        patch_row_a4(xs, od, lane, t.live, h, act);
        const float4* shifted = reinterpret_cast<const float4*>(xs) + 1;
        if (lane == 0) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                         ::"l"(a.io.obs + w0 * od), "r"(smem_u32(shifted)), "r"((unsigned)(rows * od * 4)) : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
        if (want_fin) {
            store_final_rows<true>(a.io.final_obs + w0 * od, fin_s, shifted, od, fin_rows, lane, act);
            __syncwarp();                                                              // fin_s is rewritten by the next tile
        }
        QS_TSTAMP(tg, 6);
        if (pend >= 0) publish(pend, false);            // tile k-1: every group but tile k's has completed
        pend = k;
        if (k + 1 < nt && !pre) {
            // tile k+1 was not ready: never spin while holding an unpublished tile
            publish(k, true);
            pend = -1;
            wait_turn(k + 1, __shfl_sync(0xffffffffu, my_ticket, k + 1));
            issue(k + 1);
        }
    }
    if (ticketed) publish(pend, true);
    else if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // shared memory must outlive the bulk store's reads
}

}  // namespace

// The fast kernels cover: RL observations with an action buffer, act RPM / ONE_D_RPM, no DYN+ effects, D in {1,2,4,...,32},
// autoreset SAME_STEP or none without the opt-in clear flags, a span that is 16-byte aligned and sized for every warp.
bool step_fast_eligible(const StepArgs& a) {
    if (a.act_type != QS_ACT_RPM && a.act_type != QS_ACT_ONE_D_RPM) return false;
    if ((a.effects & 7u) != 0u) return false;
    if (a.flags & ~(unsigned)(QS_FLAG_AUTORESET_SAME_STEP | QS_FLAG_RPY_F32)) return false;
    if (a.D > 32 || (a.D & (a.D - 1)) != 0) return false;
    if (!a.io.obs || !a.io.obs_prev || a.io.act_buffer_size < 1 || a.io.dw_fz) return false;
    if (!aligned16(a.io.obs) || !aligned16(a.io.obs_prev)) return false;
    if (a.io.final_obs && !aligned16(a.io.final_obs)) return false;
    if ((a.N % 32) * (long long)a.obs_dim % 4 != 0) return false;                  // ragged last warp: its span must stay a 16-byte multiple
    if ((a.flags & QS_FLAG_AUTORESET_SAME_STEP) && !a.st.reset_head) return false;
    if ((size_t)FastSmem<4>::total_bytes(a.obs_dim, true) > kStageLimit) return false;      // long action buffers (240 Hz control)
    return true;
}

cudaError_t launch_step_fast(const StepArgs& a_in, cudaStream_t s) {
#ifdef QS_TIMELINE
    StepArgs a = a_in;
    a.dbg_slot = g_dbg_slot;
#else
    const StepArgs& a = a_in;
#endif
    const bool fin = (a.flags & QS_FLAG_AUTORESET_SAME_STEP) && a.io.final_obs != nullptr;
    const long long tiles = a.n_warps > 0 ? a.n_warps : (a.N + 31) / 32;
    return with_bool(a.task == QS_TASK_HOVER, [&](auto TASK) {
        return with_bool((a.flags & QS_FLAG_AUTORESET_SAME_STEP) != 0, [&](auto RESET) {
            return with_bool((a.flags & QS_FLAG_RPY_F32) != 0, [&](auto RPYF) {
                return with_bool(a.st.phys != nullptr, [&](auto PHYS) {
                    constexpr bool T = decltype(TASK)::value, R = decltype(RESET)::value, F = decltype(RPYF)::value, P = decltype(PHYS)::value;
                    if (a.A == 4 && a.pipe && !a.io.obs_gather) {      // the pipelined kernel takes A = 4 without the fused gather
                        const size_t sm = (size_t)PipeSmem::total_bytes(a.obs_dim, fin);
                        return launch_step_kernel(step_pipe_kernel<T, R, F, P>, (int)((tiles + kPipeTiles - 1) / kPipeTiles), 32, sm, sm, pdl_enabled(), s, a);
                    }
                    const size_t sm = (size_t)(a.A == 4 ? FastSmem<4>::total_bytes(a.obs_dim, fin) : FastSmem<1>::total_bytes(a.obs_dim, fin));
                    return launch_step_kernel(a.A == 4 ? step_fast_kernel<4, T, R, F, P> : step_fast_kernel<1, T, R, F, P>, (int)tiles, 32, sm, sm,
                                              pdl_enabled(), s, a);
                });
            });
        });
    });
}

}  // namespace qsi

#ifdef QS_TIMELINE
extern "C" int qs_debug_timeline(unsigned long long* host_out, int n_words, int slot) {
    return (int)cudaMemcpyFromSymbol(host_out, g_timeline, (size_t)n_words * 8, (size_t)(slot & 3) * 8192 * 16 * 8);
}
extern "C" void qs_debug_set_slot(int slot) { g_dbg_slot = slot; }
#endif
