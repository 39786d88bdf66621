// step_general.cu -- the fused control tick for every configuration (all DYN+ effects, CtrlAviary state vectors, embedded
// PID action types, NEXT_STEP autoreset, aviaries up to 128 drones per CTA, unstaged observation rows): see DESIGN.md 4.1.
// The common RL configurations take the leaner kernels of step_fast.cu instead.
#include "qs_common.cuh"

namespace qsi {
namespace {

// ---------------------------------------------------------------------------------------------------------
// Row writer: the CTA's rows [c0, c0+rows) of obs are one contiguous span.  Lane = column (V = float4 when the
// action is 4 wide, so one 18-lane instruction moves a whole 72-float row), warps stride over rows, and U
// independent loads are issued before the first store so the L2 round trip is paid once per U rows.
//   column c <  12/W            : kinematic head staged in shared memory by the owning thread
//   12/W <= c < cols - A/W      : prev_obs column c + A/W   (history shifted by one action)
//   c >= cols - A/W             : this tick's action
// Row modes (autoreset): bit0 keep history unshifted, bit1 mirror the row into final_obs, bit2 zero history in obs.
// ---------------------------------------------------------------------------------------------------------
template <typename V, int W, int U>
__device__ __forceinline__ void write_rows(const StepArgs& a, long long c0, int rows, const float* head_s, const float* act_s,
                                           const unsigned char* mode_s, const float* stage_s) {
    const int cols = a.obs_dim / W, hcols = 12 / W, acols = a.A / W, hist_end = cols - acols;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    // CTA-relative 32-bit offsets (a CTA's span is < 2^31 elements); one 64-bit base per buffer
    const V* prev = reinterpret_cast<const V*>(a.io.obs_prev) + c0 * cols;
    V* out = reinterpret_cast<V*>(a.io.obs) + c0 * cols;
    V* fin = reinterpret_cast<V*>(a.io.final_obs) + c0 * cols;
    const V* head = reinterpret_cast<const V*>(head_s);
    const V* stage = reinterpret_cast<const V*>(stage_s);     // prev rows already in shared memory (TMA) or nullptr
    for (int cb = 0; cb < cols; cb += 32) {                   // column block (one iteration when the row fits 32 lanes)
        const int c = cb + lane;
        const bool col_ok = c < cols;
        for (int r0 = warp; r0 < rows; r0 += nwarps * U) {
            V v[U];
            unsigned char md[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int r = r0 + u * nwarps;
                md[u] = 0x80;                                  // 0x80 = nothing to store
                if (r < rows && col_ok) {
                    const unsigned char mode = mode_s[r];
                    if (c < hcols) {
                        v[u] = head[r * hcols + c];
                        md[u] = 0;
                    } else {
                        md[u] = mode;
                        const bool keep = mode & 1;
                        if (c < hist_end || keep) {
                            const int so = r * cols + c + (keep ? 0 : acols);
                            v[u] = stage ? stage[so] : __ldg(prev + so);
                        }
                        else v[u] = reinterpret_cast<const V*>(act_s + 4 * r)[c - hist_end];
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (!(md[u] & 0x80)) {
                    const int o = (r0 + u * nwarps) * cols + c;
                    if (md[u] & 2) fin[o] = v[u];
                    if (md[u] & 4) memset(&v[u], 0, sizeof(V));
                    out[o] = v[u];
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// Fused control tick.  RAW = CtrlAviary semantics (clip raw rpm, [N][20] state vectors out, no task).
// Block = tpb threads, tpb a multiple of D (drones of one aviary never straddle CTAs) when D <= 128.
// ---------------------------------------------------------------------------------------------------------
// PIDACT = the action type runs the embedded DSLPIDControl (PID / VEL / ONE_D_PID): a separate instantiation keeps
// the controller's registers out of the plain RPM kernels.  PHYS = the physical constants come from the aviary's row of
// QsState.phys (a separate instantiation: without the table the kernels are the ones of ABI 3).
template <int EFF, bool RAW, bool PIDACT, bool PHYS>
__global__ void __launch_bounds__(kMaxTPB, 4) step_kernel(const __grid_constant__ StepArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const QsParams& P = a.P;
    const int tpb = a.tpb, D = a.D, A = a.A;
    const int t = threadIdx.x;
    const long long N = a.N;
    const long long c0 = (long long)blockIdx.x * tpb;          // first drone of this CTA
    const long long i = c0 + t;
    const bool live = (t < tpb) && (i < N);
    const int head = RAW ? 20 : 12;                            // floats staged per row
    // shared layout
    float* head_s = reinterpret_cast<float*>(smem_raw);                  // [tpb][head]
    const int cap = a.cap;
    const size_t fixed = smem_fixed(cap);
    float* act_s = head_s + (size_t)cap * 20;                            // [tpb][4]
    double* red_s = reinterpret_cast<double*>(act_s + (size_t)cap * 4);  // [tpb][2] reward, dist
    double* pos_s = red_s + (size_t)cap * 2;                             // [tpb][3] (in-CTA downwash)
    unsigned char* oob_s = reinterpret_cast<unsigned char*>(pos_s + (size_t)cap * 3);   // [tpb]
    unsigned char* mode_s = oob_s + cap;                                 // [tpb] row mode: 0 shift, 1 keep history, 2 also final_obs
    unsigned char* done_s = mode_s + cap;                                // [tpb] per local env
    unsigned long long* bar_s = reinterpret_cast<unsigned long long*>(smem_raw + fixed - 16);   // mbarrier of the row staging
    float* stage_s = reinterpret_cast<float*>(smem_raw + fixed);                                // [tpb][obs_dim] (+A) when staged

    const long long e = live ? i / D : 0;
    const int le = t / D;                                      // local env (meaningful when D <= tpb)
    const int dslot = (int)(i - e * D);                        // drone index inside its aviary
    const long long tbl = a.st.tables_per_env ? i : dslot;

    // Programmatic dependent launch: when the host launched this grid with programmatic stream serialization its CTAs
    // may already be resident while the previous kernel in the stream drains; nothing written by that kernel is read
    // before this point (no-op for ordinary launches).
    asm volatile("griddepcontrol.wait;" ::: "memory");

    qs::Drone d;
    qs::Derived o;
    qs::PidState pst = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    float act[4] = {0.f, 0.f, 0.f, 0.f};
    double rpm[4] = {0, 0, 0, 0}, rpm_prev[4] = {0, 0, 0, 0};
    double R_last[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    int sc = 0;
    bool pending = false;
    constexpr bool pid_act = PIDACT;
    qs::PhysRow ph;

    // The observation rows of this CTA are one contiguous span, and the new rows are the old ones shifted left by one
    // action: new_flat[j] = old_flat[j + A] once every thread has patched its own row (head -> slots [A, A+12), new
    // action -> the A slots after the row, i.e. the dead head slots of the next row).  So: ONE thread starts a TMA bulk
    // copy of the old span into shared memory now (completion on an mbarrier), the physics below runs while it is in
    // flight, then the span is streamed out with a flat, fully coalesced float4 copy.  Spans too large for shared
    // memory are only pulled into L2 (and written by write_rows).
    const bool want_rows = !RAW && a.io.obs && a.io.obs_prev && a.obs_dim > 12 && !(a.flags & QS_FLAG_SKIP_EPILOGUE);
    const int rows = (int)((N - c0) < tpb ? (N - c0) : tpb);
    if (want_rows && a.stage_rows == 1) {
        if (t == 0) mbar_init(bar_s, 1);
        __syncthreads();
    }

    if (live) {
        load_drone(a.st.planes, N, i, d);
        if (a.io.action == nullptr) {
            // CtrlAviary split substeps: the rpm come from last_rpm (RPM_FROM_LAST)
        } else if (RAW && (a.flags & QS_FLAG_ACTION_F64)) {
            const D4 v = ld256(reinterpret_cast<const double*>(a.io.action), i);      // float64 RPMs
            rpm[0] = v.x; rpm[1] = v.y; rpm[2] = v.z; rpm[3] = v.w;
        } else if (A == 4) {
            const float4 v = ldg4(a.io.action, i);
            act[0] = v.x; act[1] = v.y; act[2] = v.z; act[3] = v.w;
        } else if (A == 3) {
            act[0] = __ldg(a.io.action + i * 3); act[1] = __ldg(a.io.action + i * 3 + 1); act[2] = __ldg(a.io.action + i * 3 + 2);
        } else {
            act[0] = __ldg(a.io.action + i);
        }
        if (((EFF & QS_EFFECT_DRAG) || (a.flags & QS_FLAG_RPM_FROM_LAST)) && a.st.last_rpm) load_rpm(a.st.last_rpm, i, rpm_prev);
        if (pid_act) load_pid(a.st.pid, N, i, pst);
        sc = a.st.step_counter[e];
        if ((a.flags & QS_FLAG_AUTORESET_NEXT_STEP) && a.st.pending_reset) pending = a.st.pending_reset[e] != 0;
    }

    // async copy of the old observation span, issued AFTER this thread's state/action loads so that the small, latency
    // critical loads are ahead of the 36 KB bulk transfer in the memory system
    if (want_rows && a.stage_rows == 1) {
        if (t == 0) tma_bulk_g2s(stage_s, a.io.obs_prev + c0 * a.obs_dim, (unsigned)(rows * a.obs_dim * 4), bar_s);
    } else if (want_rows && a.stage_rows == 2) {
        // spans that are not 16-byte aligned (odd action widths): per-thread 4-byte async copies (LDGSTS), still fire-and-forget
        const float* src = a.io.obs_prev + c0 * a.obs_dim;
        for (int j = t; j < rows * a.obs_dim; j += blockDim.x) cp_async4(stage_s + j, src + j);
    } else if (want_rows && t == 0) {
        const uintptr_t p0 = reinterpret_cast<uintptr_t>(a.io.obs_prev + c0 * a.obs_dim);
        const uintptr_t beg = (p0 + 15) & ~(uintptr_t)15;
        const uintptr_t end = (p0 + (uintptr_t)rows * a.obs_dim * 4) & ~(uintptr_t)15;
        if (end > beg) {
            asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(beg), "r"((unsigned)(end - beg)) : "memory");
        }
    }

    if (live && !pending) {
        double cur_yaw = 0.0;
        if (a.act_type == QS_ACT_VEL) {
            double r_, p_;
            qs::quat_to_euler<false>(d.qx, d.qy, d.qz, d.qw, r_, p_, cur_yaw);
        }
        if (a.flags & QS_FLAG_RPM_FROM_LAST) {
            rpm[0] = rpm_prev[0]; rpm[1] = rpm_prev[1]; rpm[2] = rpm_prev[2]; rpm[3] = rpm_prev[3];
        } else if (RAW && (a.flags & QS_FLAG_ACTION_F64)) {
#pragma unroll
            for (int k = 0; k < 4; ++k) rpm[k] = qs::clampd(rpm[k], 0.0, PHYS ? load_phys_rpm(a.st.phys, e).max_rpm : P.max_rpm);   // CtrlAviary.py:140
        } else if constexpr (PHYS) {
            qs::decode_action_k<PIDACT>(P, load_phys_rpm(a.st.phys, e), a.act_type, act, d, cur_yaw, pst, rpm);
        } else {
            qs::decode_action<PIDACT>(P, a.act_type, act, d, cur_yaw, pst, rpm);
        }
    }
    if constexpr (PHYS) { if (live && !pending) ph = load_phys(a.st.phys, e); }      // after the decode (and its PID controller)

    // ---- physics: S substeps ------------------------------------------------------------------------------
    if ((EFF & QS_EFFECT_DW) && a.io.dw_fz == nullptr) {
        // downwash inside the CTA: all drones of an aviary sit in this CTA (D <= tpb), positions go through smem
        for (int s = 0; s < a.substeps; ++s) {
            if (live) { pos_s[3 * t] = d.px; pos_s[3 * t + 1] = d.py; pos_s[3 * t + 2] = d.pz; }
            __syncthreads();
            double fz = 0.0;
            if (live && !pending) {
                const int b = le * D;
                for (int k = 0; k < D; ++k) {                                   // BaseAviary.py:798-811
                    const double dz = pos_s[3 * (b + k) + 2] - d.pz;
                    const double dx = pos_s[3 * (b + k)] - d.px, dy = pos_s[3 * (b + k) + 1] - d.py;
                    const double dxy2 = dx * dx + dy * dy;
                    if (dz > 0.0 && dxy2 < 100.0) fz += qs::downwash_pair(P, dz, dxy2);
                }
                if constexpr (PHYS) qs::dyn_tick_k<EFF>(P, ph, d, rpm, s == 0 ? rpm_prev : rpm, fz, 1, R_last);
                else qs::dyn_tick<EFF>(P, d, rpm, s == 0 ? rpm_prev : rpm, fz, 1, R_last);
            }
            __syncthreads();
        }
    } else if (live && !pending) {
        const double fz = (EFF & QS_EFFECT_DW) ? (double)__ldg(a.io.dw_fz + i) : 0.0;
        if constexpr (PHYS) qs::dyn_tick_k<EFF>(P, ph, d, rpm, rpm_prev, fz, a.substeps, R_last);
        else qs::dyn_tick<EFF>(P, d, rpm, rpm_prev, fz, a.substeps, R_last);
    }

    // ---- derived outputs, task terms --------------------------------------------------------------------
    bool env_done = false;
    if (live) {
        if (pending) {                       // NEXT_STEP autoreset: this call only resets the env
            init_drone(a.st, tbl, d);
            if (a.flags & QS_FLAG_AUTORESET_CLEARS_PID) pst = {0, 0, 0, 0, 0, 0, 0, 0, 0};
            rpm[0] = rpm[1] = rpm[2] = rpm[3] = 0.0;                               // last_clipped_action = 0 (BaseAviary.py:468)
        }
        // a reset drone's head carries float64 angles in every mode (qs_reset_heads)
        if ((a.flags & QS_FLAG_RPY_F32) && !pending) qs::derive<true>(d, R_last, o); else qs::derive<false>(d, R_last, o);
        if (pending) { o.ax = o.ay = o.az = 0.0; }
    }
    const bool want_epilogue = !(a.flags & QS_FLAG_SKIP_EPILOGUE);
    if (!RAW && a.task == QS_TASK_HOVER && want_epilogue) {
        if (live) {
            const D4 tp = ld256_nc(a.st.target_pos, tbl);
            const qs::TaskTerms tt = qs::hover_terms(P, d, o, tp.x, tp.y, tp.z);
            red_s[2 * t] = tt.reward; red_s[2 * t + 1] = tt.dist; oob_s[t] = tt.out_of_bounds ? 1 : 0;
        }
        __syncthreads();
        if (live && dslot == 0) {
            double rew = 0.0, dist = 0.0; bool oob = false;
            for (int k = 0; k < D; ++k) { rew += red_s[2 * (t + k)]; dist += red_s[2 * (t + k) + 1]; oob |= oob_s[t + k] != 0; }
            bool term = dist < P.term_dist;                                        // HoverAviary.py:91
            bool trunc = oob || ((double)sc / P.pyb_freq > P.episode_len_sec);     // HoverAviary.py:113
            if (pending) { rew = 0.0; term = false; trunc = false; }
            a.io.reward[e] = (float)rew;
            a.io.terminated[e] = term ? 1 : 0;
            a.io.truncated[e] = trunc ? 1 : 0;
            if (a.io.done) a.io.done[e] = (term || trunc) ? 1 : 0;
            done_s[le] = (term || trunc) ? 1 : 0;
        }
        __syncthreads();
        if (live) env_done = done_s[le] != 0;
    } else if (!RAW && want_epilogue && live && dslot == 0) {
        a.io.reward[e] = -1.0f; a.io.terminated[e] = 0; a.io.truncated[e] = 0;     // CtrlAviary-style dummy task
        if (a.io.done) a.io.done[e] = 0;
    }

    // ---- stage this drone's row head, autoreset, store state ---------------------------------------------
    if (live) {
        float* h = head_s + (size_t)t * head;
        // row mode bits: 1 = keep history unshifted, 2 = also copy the row to final_obs, 4 = zero the history in obs
        unsigned char mode = pending ? (unsigned char)(1 | ((a.flags & QS_FLAG_AUTORESET_CLEARS_HISTORY) ? 4 : 0)) : (unsigned char)0;
        if (RAW) {
            // _getDroneStateVector (BaseAviary.py:541-561); quaternion reported normalised
            const double inv = rsqrt(qs::quat_norm2(d.qx, d.qy, d.qz, d.qw));
            h[0] = (float)d.px; h[1] = (float)d.py; h[2] = (float)d.pz;
            h[3] = (float)(d.qx * inv); h[4] = (float)(d.qy * inv); h[5] = (float)(d.qz * inv); h[6] = (float)(d.qw * inv);
            h[7] = (float)o.roll; h[8] = (float)o.pitch; h[9] = (float)o.yaw;
            h[10] = (float)d.vx; h[11] = (float)d.vy; h[12] = (float)d.vz;
            h[13] = (float)o.ax; h[14] = (float)o.ay; h[15] = (float)o.az;
            h[16] = (float)rpm[0]; h[17] = (float)rpm[1]; h[18] = (float)rpm[2]; h[19] = (float)rpm[3];
        } else {
            const bool same_step = (a.flags & QS_FLAG_AUTORESET_SAME_STEP) && env_done;
            if (same_step) {
                // terminal observation head goes straight to final_obs (rare path, strided store is fine)
                if (a.io.final_obs) {
                    float* f = a.io.final_obs + i * a.obs_dim;
                    f[0] = (float)d.px; f[1] = (float)d.py; f[2] = (float)d.pz;
                    f[3] = (float)o.roll; f[4] = (float)o.pitch; f[5] = (float)o.yaw;
                    f[6] = (float)d.vx; f[7] = (float)d.vy; f[8] = (float)d.vz;
                    f[9] = (float)o.ax; f[10] = (float)o.ay; f[11] = (float)o.az;
                    mode |= 2;
                }
                if (a.flags & QS_FLAG_AUTORESET_CLEARS_HISTORY) mode |= 4;
                if (a.flags & QS_FLAG_AUTORESET_CLEARS_PID) pst = {0, 0, 0, 0, 0, 0, 0, 0, 0};
                init_drone(a.st, tbl, d);                                          // BaseAviary.py:451-505
                double Rr[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
                qs::derive<false>(d, Rr, o);                                       // float64 angles, as qs_reset_heads
                rpm[0] = rpm[1] = rpm[2] = rpm[3] = 0.0;                           // last_clipped_action = 0
                sc = -a.counter_inc;                                               // -> 0 after the increment below
            }
            // KIN observation head: pos3 rpy3 vel3 ang_v3 (BaseRLAviary.py:310-315)
            h[0] = (float)d.px; h[1] = (float)d.py; h[2] = (float)d.pz;
            h[3] = (float)o.roll; h[4] = (float)o.pitch; h[5] = (float)o.yaw;
            h[6] = (float)d.vx; h[7] = (float)d.vy; h[8] = (float)d.vz;
            h[9] = (float)o.ax; h[10] = (float)o.ay; h[11] = (float)o.az;
            act_s[4 * t] = act[0]; act_s[4 * t + 1] = act[1]; act_s[4 * t + 2] = act[2]; act_s[4 * t + 3] = act[3];
        }
        mode_s[t] = mode;
        store_drone(a.st, N, i, d);
        if (a.st.last_rpm) st256(a.st.last_rpm, i, rpm[0], rpm[1], rpm[2], rpm[3]);
        if (pid_act) store_pid(a.st.pid, N, i, pst);
        if (dslot == 0 && want_epilogue) {
            if (pending) {
                a.st.step_counter[e] = 0;
                a.st.pending_reset[e] = 0;
            } else {
                a.st.step_counter[e] = sc + a.counter_inc;                         // BaseAviary.py:382
                if ((a.flags & QS_FLAG_AUTORESET_NEXT_STEP) && a.st.pending_reset && env_done) a.st.pending_reset[e] = 1;
            }
        }
    }
    // all the FP64 work of this CTA is done: let the next grid in the stream start moving in behind the stores
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if (a.pub_world > 0) {
        // sharded formation (qs_dyn_substeps_pub): the new positions go straight into every rank's gathered array, with the boxes of
        // their chunks and this rank's flag -- the exchange for the NEXT substep's downwash costs no launch of its own
        publish_positions(make_float4((float)d.px, (float)d.py, (float)d.pz, 0.f), live, i, (int)N, a.pub_dst, a.pub_flags, a.pub_counter,
                          a.pub_world, a.pub_rank, a.pub_offset, a.pub_n_total, a.pub_seq);
    }
    if (a.io.obs == nullptr || !want_epilogue) return;
    const int od = a.obs_dim;
    if (want_rows && a.stage_rows) {
        // ---- staged rows: wait for the async copy, patch my row in shared memory, stream the span out ----------
        if (a.stage_rows == 1) mbar_wait(bar_s, 0); else cp_async_commit_wait_all();
        __syncthreads();
        if (live) {
            float* row = stage_s + (size_t)t * od;
            const float* h = head_s + (size_t)t * 12;
            const unsigned char mode = mode_s[t];
            if (mode & 1) {                                   // NEXT_STEP reset tick: history is NOT shifted (or is cleared)
                for (int k = od - 1; k >= 12; --k) row[k + A] = (mode & 4) ? 0.f : row[k];
            } else if (A == 4) {
                *reinterpret_cast<float4*>(row + od) = make_float4(act[0], act[1], act[2], act[3]);
            } else if (A == 3) {
                row[od] = act[0]; row[od + 1] = act[1]; row[od + 2] = act[2];
            } else {
                row[od] = act[0];
            }
            if (A == 4) {
                float4* r4 = reinterpret_cast<float4*>(row + 4);
                r4[0] = make_float4(h[0], h[1], h[2], h[3]); r4[1] = make_float4(h[4], h[5], h[6], h[7]); r4[2] = make_float4(h[8], h[9], h[10], h[11]);
            } else {
                for (int k = 0; k < 12; ++k) row[A + k] = h[k];
            }
        }
        __syncthreads();
        const bool clear_hist = a.flags & QS_FLAG_AUTORESET_CLEARS_HISTORY;
        const int lane = t & 31;
        if (A == 4) {
            const float4* src = reinterpret_cast<const float4*>(stage_s) + 1;
            float4* out = reinterpret_cast<float4*>(a.io.obs + c0 * od);
            const int c4n = od >> 2, n4 = rows * c4n;
            if (a.stage_rows == 1) {
                // TMA bulk store: one thread hands the whole patched span (shared memory, shifted by one action) to the
                // copy engine; the other threads go on to the terminal-observation rows.  The async proxy must see the
                // generic-proxy patches (fence), and shared memory must stay alive until it has been read (wait_group.read).
                if (t == 0) {
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                                 ::"l"(out), "r"(smem_u32(src)), "r"((unsigned)(n4 * 16)) : "memory");
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
            } else {
                const int nt = blockDim.x;
                int j = t;
                for (; j + 5 * nt < n4; j += 6 * nt) {        // 6 independent LDS.128 in flight, then 6 coalesced STG.128
                    const float4 v0 = src[j], v1 = src[j + nt], v2 = src[j + 2 * nt], v3 = src[j + 3 * nt], v4 = src[j + 4 * nt], v5 = src[j + 5 * nt];
                    out[j] = v0; out[j + nt] = v1; out[j + 2 * nt] = v2; out[j + 3 * nt] = v3; out[j + 4 * nt] = v4; out[j + 5 * nt] = v5;
                }
                for (; j < n4; j += nt) out[j] = src[j];
            }
            // SAME_STEP autoreset: the history part of the terminal observation of finished rows.  Each warp ballots the
            // flags of its own 32 rows and copies only the flagged ones, a whole row per instruction.
            if (a.io.final_obs && (a.flags & QS_FLAG_AUTORESET_SAME_STEP)) {
                float4* fin = reinterpret_cast<float4*>(a.io.final_obs + c0 * od);
                unsigned m = __ballot_sync(0xffffffffu, live && (mode_s[t] & 2));
                const int r0 = t & ~31;
                for (; m; m &= m - 1) {
                    const int r = r0 + __ffs(m) - 1;
                    for (int c = 3 + lane; c < c4n; c += 32) fin[r * c4n + c] = src[r * c4n + c];
                }
            }
        } else {
            const float* src = stage_s + A;
            float* out = a.io.obs + c0 * od;
            for (int j = t; j < rows * od; j += blockDim.x) out[j] = src[j];
            if (a.io.final_obs && (a.flags & QS_FLAG_AUTORESET_SAME_STEP)) {
                float* fin = a.io.final_obs + c0 * od;
                unsigned m = __ballot_sync(0xffffffffu, live && (mode_s[t] & 2));
                const int r0 = t & ~31;
                for (; m; m &= m - 1) {
                    const int r = r0 + __ffs(m) - 1;
                    for (int c = 12 + lane; c < od; c += 32) fin[r * od + c] = src[r * od + c];
                }
            }
        }
        if (A == 4 && a.stage_rows == 1 && t == 0) {
            if (clear_hist) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");       // stores complete (ordering vs the zeroing below)
            else asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");             // shared memory has been read
        }
        if (clear_hist) {                                     // optional: the observation after a reset carries an empty action buffer
            __syncthreads();
            if (live && (mode_s[t] & 4) && !(mode_s[t] & 1)) {
                float* orow = a.io.obs + i * od;
                for (int k = 12; k < od; ++k) orow[k] = 0.f;
            }
        }
        return;
    }
    __syncthreads();

    // ---- cooperative, coalesced write of this CTA's observation rows (unstaged paths) -----------------------------
    if (RAW) {
        float* out = a.io.obs + c0 * 20;
        for (int j = t; j < rows * 20; j += blockDim.x) out[j] = head_s[j];
    } else if (A == 4) {
        write_rows<float4, 4, 8>(a, c0, rows, head_s, act_s, mode_s, nullptr);
    } else {
        write_rows<float, 1, 8>(a, c0, rows, head_s, act_s, mode_s, nullptr);
    }
}

size_t step_smem_bytes(const StepArgs& a) {
    return smem_fixed(a.cap) + (a.stage_rows ? (size_t)a.tpb * a.obs_dim * 4 + 32 : 0);
}

}  // namespace

cudaError_t launch_step_general(const StepArgs& a, bool raw, bool pid_act, bool pdl_ok, cudaStream_t s) {
    const int blocks = (int)((a.N + a.tpb - 1) / a.tpb);
    const int threads = ((a.tpb + 31) / 32) * 32;
    const size_t sm = step_smem_bytes(a);
    const bool pdl = pdl_enabled() && pdl_ok;
    cudaError_t err = cudaSuccess;
    with_int(AllEffects{}, (int)(a.effects & 7u), [&](auto EFF) {
        err = with_bool(raw, [&](auto RAW) {
            return with_bool(pid_act, [&](auto PIDACT) {
                return with_bool(a.st.phys != nullptr, [&](auto PHYS) {
                    // the shared-memory limit is the largest step_smem_bytes, the same for every launch of a kernel
                    return launch_step_kernel(step_kernel<decltype(EFF)::value, decltype(RAW)::value, decltype(PIDACT)::value, decltype(PHYS)::value>,
                                              blocks, threads, sm, kStepSmemFixed + kStageLimit + 32, pdl, s, a);
                });
            });
        });
    });
    return err;
}

}  // namespace qsi
