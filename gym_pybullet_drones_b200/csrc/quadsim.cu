// quadsim.cu -- C ABI (include/quadsim.h) of the vectorised quadrotor simulator: argument checking and launch of
// the fused control tick (step_fast.cu / step_general.cu), the host-buffer tick, the stand-alone PID and reset kernels.
// The other entry points live next to their kernels: rollout.cu (qs_rollout), formation.cu (downwash, adjacency).
//
// Layout in HBM (DESIGN.md 3):
//   state   : float64 planes [pos|w.x] [quat] [vel|w.y] of [N][4] + w.z [N]: three 32-byte accesses + one 8-byte per thread
//   obs     : float32 row-major [N][12+B*A]; a warp owns 32 consecutive rows = one contiguous span that is staged in
//             shared memory by one TMA bulk copy, patched (new head, new action) and written back by one TMA bulk store
//   consts  : QsParams travels in the kernel parameter (constant bank, uniform operands -- no load instruction)
// No tensor cores: the path is element-wise; the roofline that bounds it is HBM bandwidth (DESIGN.md).
#include "qs_common.cuh"

#include <map>
#include <mutex>
#include <utility>

namespace qsi {
thread_local char g_err[256] = "";

// Per (device, stream): the last early-triggering library launch (PdlPrev).  Unknown streams read kPdlNone: nothing of the
// library that triggers early ran on them.  The per-thread default stream is tracked per host thread.
constexpr int kPdlDevices = 32;
static std::mutex g_pdl_mu;
static std::map<std::pair<int, cudaStream_t>, PdlPrev>* g_pdl = new std::map<std::pair<int, cudaStream_t>, PdlPrev>();   // never freed
static thread_local PdlPrev t_pdl_per_thread[kPdlDevices] = {};

PdlPrev pdl_prev(cudaStream_t s) {
    int dev = -1;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kPdlDevices) { (void)cudaGetLastError(); return kPdlOther; }
    if (s == cudaStreamPerThread) return t_pdl_per_thread[dev];
    std::lock_guard<std::mutex> lk(g_pdl_mu);
    const auto it = g_pdl->find(std::make_pair(dev, s));
    return it == g_pdl->end() ? kPdlNone : it->second;
}

void pdl_note(cudaStream_t s, PdlPrev what) {
    int dev = -1;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kPdlDevices) { (void)cudaGetLastError(); return; }
    if (s == cudaStreamPerThread) { t_pdl_per_thread[dev] = what; return; }
    std::lock_guard<std::mutex> lk(g_pdl_mu);
    (*g_pdl)[std::make_pair(dev, s)] = what;
}
}  // namespace qsi
using namespace qsi;

namespace {
// Launches one step kernel and records it for the ordering of the next one (include/quadsim.h, qs_step; DESIGN.md 4.1).
// A fast step skips the whole-grid wait when its stream predecessor that may have triggered early is a fast step: a
// fast step only touches the drones of its own warps, and the per-warp tickets order it after the previous step on the
// same buffers.  The wait stays when that predecessor is another early-triggering kernel, without the readiness words,
// and with obs_gather (the learner's flag counts the warps of one grid at a time).  A general step directly after a
// fast step is launched as an ordinary dependent (full stream order): the fast step may finish before ITS predecessor.
cudaError_t launch_step_tracked(StepArgs& a, bool fast, bool state20, bool pid_act, cudaStream_t s) {
    const PdlPrev prev = pdl_prev(s);
    if (fast) {
        a.grid_wait = (prev == kPdlOther || !a.io.warp_ticket || a.io.obs_gather) ? 1 : 0;
        const cudaError_t e = launch_step_fast(a, s);
        if (e == cudaSuccess) pdl_note(s, kPdlFast);
        return e;
    }
    const cudaError_t e = launch_step_general(a, state20, pid_act, prev != kPdlFast, s);
    pdl_note(s, kPdlOther);
    return e;
}
}  // namespace

namespace {

// ---------------------------------------------------------------------------------------------------------
// DSLPIDControl.computeControl for n drones (stand-alone entry).
// ---------------------------------------------------------------------------------------------------------
struct PidArgs {
    QsParams P;
    double* pid;
    double dt;
    const float *pos, *quat, *vel, *tpos, *trpy, *tvel, *trr;
    int pos_stride, quat_stride, vel_stride, n;
    float *rpm_out, *pos_e_out, *yaw_e_out;
};

// pos / quat / vel from the float64 state planes, float64 targets, float64 RPMs out (qs_pid_control_state)
struct PidStateArgs {
    QsParams P;
    double* pid;
    double dt;
    const double* planes;
    const double *tpos, *trpy, *tvel, *trr;
    long long n;
    double* rpm_out;
    float *pos_e_out, *yaw_e_out;
};

__global__ void __launch_bounds__(128) pid_state_kernel(const __grid_constant__ PidStateArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long N = a.n;
    if (i >= N) return;
    const D4 p0 = ld256(a.planes, i), p1 = ld256(a.planes, N + i), p2 = ld256(a.planes, 2 * N + i);
    qs::PidState st;
    load_pid(a.pid, N, i, st);
    const double tyaw = a.trpy ? a.trpy[3 * i + 2] : 0.0;
    double tv[3] = {0, 0, 0}, tr[3] = {0, 0, 0};
    if (a.tvel) { tv[0] = a.tvel[3 * i]; tv[1] = a.tvel[3 * i + 1]; tv[2] = a.tvel[3 * i + 2]; }
    if (a.trr) { tr[0] = a.trr[3 * i]; tr[1] = a.trr[3 * i + 1]; tr[2] = a.trr[3 * i + 2]; }
    double rpm[4], pe[3], ye;
    qs::pid_control(a.P, st, a.dt, p0.x, p0.y, p0.z, p1.x, p1.y, p1.z, p1.w, p2.x, p2.y, p2.z,
                    a.tpos[3 * i], a.tpos[3 * i + 1], a.tpos[3 * i + 2], tyaw, tv[0], tv[1], tv[2], tr[0], tr[1], tr[2], rpm, pe, ye);
    store_pid(a.pid, N, i, st);
    st256(a.rpm_out, i, qs::clampd(rpm[0], 0.0, a.P.max_rpm), qs::clampd(rpm[1], 0.0, a.P.max_rpm),
          qs::clampd(rpm[2], 0.0, a.P.max_rpm), qs::clampd(rpm[3], 0.0, a.P.max_rpm));            // CtrlAviary.py:140
    if (a.pos_e_out) { a.pos_e_out[3 * i] = (float)pe[0]; a.pos_e_out[3 * i + 1] = (float)pe[1]; a.pos_e_out[3 * i + 2] = (float)pe[2]; }
    if (a.yaw_e_out) a.yaw_e_out[i] = (float)ye;
}

__global__ void __launch_bounds__(128) pid_kernel(const __grid_constant__ PidArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long N = a.n;
    if (i >= N) return;
    const float* p = a.pos + i * a.pos_stride;
    const float* q = a.quat + i * a.quat_stride;
    const float* v = a.vel + i * a.vel_stride;
    qs::PidState st;
    load_pid(a.pid, N, i, st);
    const double tyaw = a.trpy ? (double)a.trpy[3 * i + 2] : 0.0;
    double tv[3] = {0, 0, 0}, tr[3] = {0, 0, 0};
    if (a.tvel) { tv[0] = a.tvel[3 * i]; tv[1] = a.tvel[3 * i + 1]; tv[2] = a.tvel[3 * i + 2]; }
    if (a.trr) { tr[0] = a.trr[3 * i]; tr[1] = a.trr[3 * i + 1]; tr[2] = a.trr[3 * i + 2]; }
    double rpm[4], pe[3], ye;
    qs::pid_control(a.P, st, a.dt, p[0], p[1], p[2], q[0], q[1], q[2], q[3], v[0], v[1], v[2],
                    a.tpos[3 * i], a.tpos[3 * i + 1], a.tpos[3 * i + 2], tyaw, tv[0], tv[1], tv[2], tr[0], tr[1], tr[2],
                    rpm, pe, ye);
    store_pid(a.pid, N, i, st);
    reinterpret_cast<float4*>(a.rpm_out)[i] = make_float4((float)rpm[0], (float)rpm[1], (float)rpm[2], (float)rpm[3]);
    if (a.pos_e_out) { a.pos_e_out[3 * i] = (float)pe[0]; a.pos_e_out[3 * i + 1] = (float)pe[1]; a.pos_e_out[3 * i + 2] = (float)pe[2]; }
    if (a.yaw_e_out) a.yaw_e_out[i] = (float)ye;
}

// ---------------------------------------------------------------------------------------------------------
// Masked reset (BaseAviary.reset / _housekeeping).
// ---------------------------------------------------------------------------------------------------------
struct ResetArgs {
    QsState st;
    const unsigned char* mask;
    int D, reset_pid, obs_dim, raw20;
    long long N;
    float* obs;
};

__global__ void __launch_bounds__(128) reset_kernel(const __grid_constant__ ResetArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.N) return;
    const long long e = i / a.D;
    if (a.mask && !a.mask[e]) return;
    const int dslot = (int)(i - e * a.D);
    const long long tbl = a.st.tables_per_env ? i : dslot;
    qs::Drone d;
    init_drone(a.st, tbl, d);
    qs::Derived o;
    const double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    qs::derive<false>(d, R, o);
    store_drone(a.st, a.N, i, d);
    if (a.st.last_rpm) st256(a.st.last_rpm, i, 0.0, 0.0, 0.0, 0.0);
    if (a.reset_pid && a.st.pid)
        for (int k = 0; k < 9; ++k) a.st.pid[k * a.N + i] = 0.0;
    if (dslot == 0) {
        a.st.step_counter[e] = 0;
        if (a.st.pending_reset) a.st.pending_reset[e] = 0;
    }
    if (a.obs) {
        if (a.raw20) {
            float* h = a.obs + i * 20;
            h[0] = (float)d.px; h[1] = (float)d.py; h[2] = (float)d.pz;
            h[3] = (float)d.qx; h[4] = (float)d.qy; h[5] = (float)d.qz; h[6] = (float)d.qw;
            h[7] = (float)o.roll; h[8] = (float)o.pitch; h[9] = (float)o.yaw;
            for (int k = 10; k < 20; ++k) h[k] = 0.f;
        } else {
            float* h = a.obs + i * a.obs_dim;
            h[0] = (float)d.px; h[1] = (float)d.py; h[2] = (float)d.pz;
            h[3] = (float)o.roll; h[4] = (float)o.pitch; h[5] = (float)o.yaw;
            for (int k = 6; k < 12; ++k) h[k] = 0.f;
        }
    }
}

// learner side of the fused observation gather: wait until every rank's flag carries the sequence number
__global__ void wait_flags_kernel(const unsigned* flags, unsigned seq, int world, unsigned* err) {
    if ((int)threadIdx.x < world) {
        const long long t0 = clock64();
        unsigned v;
        do {
            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + threadIdx.x) : "memory");
            if (clock64() - t0 > 4000000000LL) { if (err) atomicExch(err, 1u); break; }
        } while ((int)(v - seq) < 0);
    }
}

// one Logger entry per logged drone (utils/Logger.py:83-119), appended to the device ring
__global__ void log_append_kernel(QsParams P, QsState st, const float* __restrict__ obs, int obs_dim, const float* __restrict__ controls,
                                  QsLogRing rg, long long N, int D) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    const long long head = *rg.head;
    if (j < rg.n_drones) {
        const long long i = rg.first_drone + j;
        qs::Drone d;
        load_drone(st.planes, N, i, d);
        double roll, pitch, yaw;
        qs::quat_to_euler<false>(d.qx, d.qy, d.qz, d.qw, roll, pitch, yaw);
        const float* row = obs + i * obs_dim;
        const int av = (obs_dim == 20 && !rg.kin_rows) ? 13 : 9;                // ang_v in a state vector / in a KIN row
        double* o = rg.ring + ((head % rg.capacity) * rg.n_drones + j) * 32;
        o[0] = d.px; o[1] = d.py; o[2] = d.pz; o[3] = d.vx; o[4] = d.vy; o[5] = d.vz;          // Logger.py:117
        o[6] = roll; o[7] = pitch; o[8] = yaw;
        o[9] = row[av]; o[10] = row[av + 1]; o[11] = row[av + 2];
        double rpm[4] = {0, 0, 0, 0};
        if (st.last_rpm) load_rpm(st.last_rpm, i, rpm);
        o[12] = rpm[0]; o[13] = rpm[1]; o[14] = rpm[2]; o[15] = rpm[3];
        for (int k = 0; k < 12; ++k) o[16 + k] = controls ? (double)controls[12 * j + k] : 0.0;
        o[28] = (double)st.step_counter[i / D] * P.dt;                          // simulation time after the tick
        o[29] = o[30] = o[31] = 0.0;
    }
}
__global__ void log_advance_kernel(long long* head) { *head += 1; }      // after every CTA of the append has read it (stream order)

// the head of a freshly reset drone carries float64 angles whatever QS_FLAG_RPY_F32 is: the same bits as reset_kernel writes, so an
// aviary's first observation does not depend on whether reset() or an autoreset produced it
__global__ void reset_heads_kernel(QsState st, int rows, float* __restrict__ out) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    qs::Drone d;
    init_drone(st, r, d);
    qs::Derived o;
    const double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    qs::derive<false>(d, R, o);
    float* h = out + 12 * (long long)r;
    h[0] = (float)d.px; h[1] = (float)d.py; h[2] = (float)d.pz;
    h[3] = (float)o.roll; h[4] = (float)o.pitch; h[5] = (float)o.yaw;
    h[6] = (float)d.vx; h[7] = (float)d.vy; h[8] = (float)d.vz;
    h[9] = (float)o.ax; h[10] = (float)o.ay; h[11] = (float)o.az;
}

// Ascending indices of the finished aviaries (stream compaction of the done flags): one CTA of 1024 threads, a thread takes
// 32 consecutive flags, block-wide exclusive scan of the counts, chunks of 32 768 flags in sequence.
__global__ void __launch_bounds__(1024) compact_done_kernel(const unsigned char* __restrict__ done, int E, long long* __restrict__ idx, int* __restrict__ count) {
    __shared__ int warp_tot[32];
    __shared__ int chunk_tot;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    int base = 0;
    for (int c0 = 0; c0 < E; c0 += 1024 * 32) {
        const int b = c0 + 32 * t;
        unsigned mask = 0u;
        if (b + 32 <= E && ((reinterpret_cast<uintptr_t>(done) + b) & 15u) == 0) {
            const uint4 v0 = *reinterpret_cast<const uint4*>(done + b), v1 = *reinterpret_cast<const uint4*>(done + b + 16);
            const unsigned w[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
            for (int q = 0; q < 8; ++q)
#pragma unroll
                for (int r = 0; r < 4; ++r) if ((w[q] >> (8 * r)) & 0xffu) mask |= 1u << (4 * q + r);
        } else {
            for (int q = 0; q < 32; ++q) if (b + q < E && done[b + q]) mask |= 1u << q;
        }
        const int cnt = __popc(mask);
        int incl = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            int w = warp_tot[lane], wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += v; }
            warp_tot[lane] = wi - w;                                  // exclusive prefix of the warp totals
            if (lane == 31) chunk_tot = wi;
        }
        __syncthreads();
        int off = base + warp_tot[warp] + incl - cnt;
        for (unsigned m = mask; m; m &= m - 1) idx[off++] = b + __ffs(m) - 1;
        base += chunk_tot;
        __syncthreads();
    }
    if (t == 0) *count = base;
}

// per-aviary outputs -> mapped host arrays (229 KB for 32 768 aviaries): one kernel next to the observation copy instead of four
// small cudaMemcpyAsync in front of it
__global__ void __launch_bounds__(256) small_outputs_kernel(const float* __restrict__ rew, const unsigned char* __restrict__ te,
                                                            const unsigned char* __restrict__ tr, const unsigned char* __restrict__ dn,
                                                            float* __restrict__ rew_h, unsigned char* __restrict__ te_h,
                                                            unsigned char* __restrict__ tr_h, unsigned char* __restrict__ dn_h, int E) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int e4 = i * 4;
    if (e4 + 3 < E && ((reinterpret_cast<uintptr_t>(rew) | reinterpret_cast<uintptr_t>(rew_h)) & 15u) == 0 &&
        ((reinterpret_cast<uintptr_t>(te) | reinterpret_cast<uintptr_t>(tr) | reinterpret_cast<uintptr_t>(te_h) | reinterpret_cast<uintptr_t>(tr_h)) & 3u) == 0 &&
        (!dn_h || ((reinterpret_cast<uintptr_t>(dn) | reinterpret_cast<uintptr_t>(dn_h)) & 3u) == 0)) {
        reinterpret_cast<float4*>(rew_h)[i] = reinterpret_cast<const float4*>(rew)[i];
        reinterpret_cast<unsigned*>(te_h)[i] = reinterpret_cast<const unsigned*>(te)[i];
        reinterpret_cast<unsigned*>(tr_h)[i] = reinterpret_cast<const unsigned*>(tr)[i];
        if (dn_h) reinterpret_cast<unsigned*>(dn_h)[i] = reinterpret_cast<const unsigned*>(dn)[i];
    } else {
        for (int e = e4; e < E && e < e4 + 4; ++e) { rew_h[e] = rew[e]; te_h[e] = te[e]; tr_h[e] = tr[e]; if (dn_h) dn_h[e] = dn[e]; }
    }
}

// kinematic heads of the observation rows -> packed [N][12] array (mapped host memory): head-only transfer mode of qs_step_host
__global__ void __launch_bounds__(256) pack_heads_kernel(const float* __restrict__ obs, int od, long long N, float* __restrict__ dst) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;      // one float4 of a head per thread (rows are 16-byte multiples)
    if (j >= 3 * N) return;
    const long long r = j / 3;
    const int c = (int)(j - 3 * r);
    if ((od & 3) == 0) reinterpret_cast<float4*>(dst)[j] = *reinterpret_cast<const float4*>(obs + r * od + 4 * c);
    else { const float* s = obs + r * od + 4 * c; float* d = dst + 4 * j; d[0] = s[0]; d[1] = s[1]; d[2] = s[2]; d[3] = s[3]; }
}

// rows of the k finished aviaries (one aviary = D*obs_dim contiguous floats) -> compact array, indices and k alongside;
// dst / idx_out / k_out may be mapped host memory (the stores then travel over PCIe next to the observation copy)
__global__ void __launch_bounds__(128) gather_rows_kernel(const float* __restrict__ src, const long long* __restrict__ idx, const int* __restrict__ count,
                                                          float* __restrict__ dst, long long* __restrict__ idx_out, int* __restrict__ k_out, int row_floats) {
    const int k = *count;
    if (blockIdx.x == 0 && threadIdx.x == 0) *k_out = k;
    const bool vec = (row_floats & 3) == 0 && ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15u) == 0;
    for (int r = blockIdx.x; r < k; r += gridDim.x) {
        const long long ev = idx[r];
        if (threadIdx.x == 0) idx_out[r] = ev;
        const float* s = src + ev * (long long)row_floats;
        float* d = dst + (long long)r * row_floats;
        if (vec) for (int j = threadIdx.x; j < (row_floats >> 2); j += blockDim.x) reinterpret_cast<float4*>(d)[j] = reinterpret_cast<const float4*>(s)[j];
        else for (int j = threadIdx.x; j < row_floats; j += blockDim.x) d[j] = s[j];
    }
}

}  // namespace

namespace qsi {

int check_state(const QsState* st, int need_tables) {
    if (!st || !st->planes || !st->step_counter) return fail(QS_ERR_NULL, "QsState: planes/step_counter is NULL");
    if (!aligned32(st->planes)) return fail(QS_ERR_ALIGN, "QsState.planes must be 32-byte aligned");
    if (st->last_rpm && !aligned32(st->last_rpm)) return fail(QS_ERR_ALIGN, "QsState.last_rpm must be 32-byte aligned");
    if (st->pos_f32 && !aligned16(st->pos_f32)) return fail(QS_ERR_ALIGN, "QsState.pos_f32 must be 16-byte aligned");
    if (st->phys && !aligned32(st->phys)) return fail(QS_ERR_ALIGN, "QsState.phys must be 32-byte aligned");
    if (need_tables) {
        if (!st->init_pos || !st->init_quat) return fail(QS_ERR_NULL, "QsState: init_pos/init_quat is NULL");
        if (!aligned32(st->init_pos) || !aligned32(st->init_quat)) return fail(QS_ERR_ALIGN, "init tables must be 32-byte aligned");
    }
    return 0;
}

// CTA capacity in drones.  32-drone CTAs (one warp) for the single-tick kernels (tools/ab.py compares 32 / 64 / 128 via
// QS_CTA_CAP): more, smaller CTAs per SM sit at different phases (load / FP64 / store) at any instant, and 65 536 drones
// spread 15-16 CTAs per SM over the H100's 132 SMs instead of 3-4.
// The multi-tick rollout keeps its window in shared memory for many ticks and prefers 64.
int cta_capacity(long long N, int D, bool rollout) {
    static const int forced = getenv("QS_CTA_CAP") ? atoi(getenv("QS_CTA_CAP")) : 0;      // experiments only
    if (forced == 32 || forced == 64 || forced == 128) return D <= forced ? forced : kMaxTPB;
    (void)N;
    if (D <= 32 && !rollout) return 32;
    return D <= 64 ? 64 : kMaxTPB;
}

}  // namespace qsi

// =============================================================================================================
extern "C" {

int qs_abi_version(void) { return QS_ABI_VERSION; }
const char* qs_last_error(void) { return g_err; }
int qs_sizeof_params(void) { return (int)sizeof(QsParams); }
int qs_sizeof_state(void) { return (int)sizeof(QsState); }
int qs_sizeof_step_io(void) { return (int)sizeof(QsStepIO); }

// Validates the arguments of one control tick and fills the kernel argument block; nothing is launched.
// fast = the configuration is one of step_fast.cu's (else step_general.cu takes it).
static int prepare_step(const QsParams* p, const QsState* st, const QsStepIO* io, int act_type, int task,
                        int n_envs, int drones_per_env, int substeps, unsigned effects, unsigned flags,
                        StepArgs& a, bool& state20_out, bool& pid_act_out, bool& fast) {
    if (!p || !io) return fail(QS_ERR_NULL, "qs_step: NULL params/io");
    const bool autoreset = flags & (QS_FLAG_AUTORESET_SAME_STEP | QS_FLAG_AUTORESET_NEXT_STEP);
    if (int rc = check_state(st, autoreset ? 1 : 0)) return rc;
    if (n_envs <= 0 || drones_per_env <= 0 || substeps <= 0) return fail(QS_ERR_SIZE, "qs_step: n_envs, drones_per_env, substeps must be > 0");
    const int A = act_width(act_type);
    const bool state20 = flags & QS_FLAG_OBS_STATE20;
    if (A < 0 || (act_type == QS_ACT_RAW_RPM && !state20)) return fail(QS_ERR_ENUM, "qs_step: bad act_type (use qs_dyn_substeps for raw rpm)");
    if (state20 && (task != QS_TASK_NONE || autoreset)) return fail(QS_ERR_UNSUPPORTED, "qs_step: OBS_STATE20 needs QS_TASK_NONE and no autoreset");
    if (task != QS_TASK_NONE && task != QS_TASK_HOVER) return fail(QS_ERR_ENUM, "qs_step: bad task");
    if (effects & ~7u) return fail(QS_ERR_ENUM, "qs_step: bad effects");
    if ((flags & QS_FLAG_AUTORESET_SAME_STEP) && (flags & QS_FLAG_AUTORESET_NEXT_STEP)) return fail(QS_ERR_ENUM, "qs_step: two autoreset modes");
    if (!io->action) return fail(QS_ERR_NULL, "qs_step: action is NULL");
    if (A == 4 && !aligned16(io->action)) return fail(QS_ERR_ALIGN, "qs_step: [N][4] action must be 16-byte aligned");
    const bool skip = flags & QS_FLAG_SKIP_EPILOGUE;
    if ((flags & QS_FLAG_RPM_FROM_LAST) && !st->last_rpm) return fail(QS_ERR_NULL, "qs_step: RPM_FROM_LAST needs QsState.last_rpm");
    if (!skip && !state20 && (!io->reward || !io->terminated || !io->truncated)) return fail(QS_ERR_NULL, "qs_step: reward/terminated/truncated is NULL");
    if (io->act_buffer_size < 0) return fail(QS_ERR_SIZE, "qs_step: act_buffer_size < 0");
    if (io->obs && io->act_buffer_size > 0 && !state20 && !io->obs_prev) return fail(QS_ERR_NULL, "qs_step: obs_prev is NULL");
    if (io->obs && io->obs == io->obs_prev) return fail(QS_ERR_UNSUPPORTED, "qs_step: obs and obs_prev must be distinct buffers");
    if (task == QS_TASK_HOVER && !st->target_pos) return fail(QS_ERR_NULL, "qs_step: target_pos is NULL");
    if (task == QS_TASK_HOVER && !aligned32(st->target_pos)) return fail(QS_ERR_ALIGN, "qs_step: target_pos must be 32-byte aligned");
    if (task == QS_TASK_HOVER && drones_per_env > kMaxTPB) return fail(QS_ERR_UNSUPPORTED, "qs_step: task reduction supports drones_per_env <= 128");
    const bool pid_act = act_type == QS_ACT_PID || act_type == QS_ACT_VEL || act_type == QS_ACT_ONE_D_PID;
    if (pid_act && !st->pid) return fail(QS_ERR_NULL, "qs_step: PID action type needs QsState.pid");
    if ((effects & QS_EFFECT_DRAG) && !st->last_rpm) return fail(QS_ERR_NULL, "qs_step: DRAG needs QsState.last_rpm");
    if ((effects & QS_EFFECT_DW) && !io->dw_fz && drones_per_env > kMaxTPB)
        return fail(QS_ERR_UNSUPPORTED, "qs_step: in-CTA downwash needs drones_per_env <= 128 (else pass dw_fz from qs_downwash, substeps = 1)");
    if ((effects & QS_EFFECT_DW) && io->dw_fz && substeps != 1) return fail(QS_ERR_UNSUPPORTED, "qs_step: external dw_fz requires substeps == 1");
    if (st->phys && io->dw_fz) return fail(QS_ERR_UNSUPPORTED, "qs_step: per-aviary physical constants (QsState.phys) are not supported with external downwash (dw_fz)");
    if ((flags & QS_FLAG_AUTORESET_NEXT_STEP) && !st->pending_reset) return fail(QS_ERR_NULL, "qs_step: NEXT_STEP autoreset needs pending_reset");
    memset(&a, 0, sizeof(a));
    a.P = *p; a.st = *st; a.io = *io;
    a.act_type = act_type; a.task = task; a.n_envs = n_envs; a.D = drones_per_env; a.substeps = substeps;
    if ((long long)n_envs * drones_per_env > 0x7fffffffLL) return fail(QS_ERR_SIZE, "qs_step: n_envs * drones_per_env exceeds 2^31-1");
    a.N = n_envs * drones_per_env; a.A = A; a.obs_dim = state20 ? 20 : 12 + io->act_buffer_size * A;
    a.cap = cta_capacity(a.N, drones_per_env);
    a.tpb = block_size_for(drones_per_env, a.cap);
    a.counter_inc = io->tick_substeps > 0 ? io->tick_substeps : substeps;
    a.effects = effects; a.flags = flags;
    {
        static const int late = getenv("QS_LATE_TMA") ? atoi(getenv("QS_LATE_TMA")) : 1;
        static const int early = getenv("QS_EARLY_STORE") ? atoi(getenv("QS_EARLY_STORE")) : 1;
        static const int rowl = getenv("QS_ROW_LOADS") ? atoi(getenv("QS_ROW_LOADS")) : 0;
        a.flags_late_tma = late; a.early_store = early; a.row_loads = rowl;
        a.grid_wait = 1;
    }
    if ((io->warp_ticket == nullptr) != (io->warp_done == nullptr)) return fail(QS_ERR_NULL, "qs_step: warp_ticket and warp_done go together");
    if ((reinterpret_cast<uintptr_t>(io->warp_ticket) | reinterpret_cast<uintptr_t>(io->warp_done) | reinterpret_cast<uintptr_t>(io->ready_err)) & 3u)
        return fail(QS_ERR_ALIGN, "qs_step: warp_ticket / warp_done / ready_err must be 4-byte aligned");
    a.log2D = -1;
    for (int k = 0; k < 6; ++k) if ((1 << k) == drones_per_env) a.log2D = k;
    {   // time-out threshold on the integer step counter, evaluated with the reference's float64 division
        long long s = (long long)(p->episode_len_sec * p->pyb_freq) - 2;
        if (s < 0) s = 0;
        while (!((double)s / p->pyb_freq > p->episode_len_sec) && s < 0x7fffffffLL) ++s;
        a.sc_limit = (int)s;
    }
    if (st->reset_head && !aligned16(st->reset_head)) return fail(QS_ERR_ALIGN, "qs_step: reset_head must be 16-byte aligned");
    // staging of the CTA's prev_obs rows in shared memory: TMA bulk copy when every CTA's span is 16-byte aligned and sized,
    // per-thread LDGSTS otherwise; none when the span does not fit (e.g. 240 Hz control: 120-action buffers)
    {
        const size_t row_bytes = (size_t)a.obs_dim * 4, span = row_bytes * a.tpb;
        const bool aligned = aligned16(io->obs_prev) && aligned16(io->obs) && (span % 16 == 0) && ((row_bytes * ((size_t)a.N % a.tpb)) % 16 == 0);
        a.stage_rows = 0;
        if (io->obs && io->act_buffer_size > 0 && !state20 && span <= kStageLimit) a.stage_rows = (aligned && A == 4) ? 1 : 2;
    }
    const bool fast_off = getenv("QS_FAST") && atoi(getenv("QS_FAST")) == 0;      // A/B and bit-identity tests: force the general kernel
    {   // A/B and bit-identity tests: QS_FAST_PIPE=0 forces the classic fast kernel, 2 or 4 the tiles per warp of the pipelined one
        const int v = getenv("QS_FAST_PIPE") ? atoi(getenv("QS_FAST_PIPE")) : kPipeTilesDefault;
        a.pipe_tiles = v <= 1 ? 0 : (v < 4 ? 2 : 4);
    }
    if (io->obs_gather) {
        if (fast_off || !step_fast_eligible(a)) return fail(QS_ERR_UNSUPPORTED, "qs_step: obs_gather needs a configuration of step_fast.cu (RPM / ONE_D_RPM, no effects, D | 32)");
        if (!aligned16(io->obs_gather)) return fail(QS_ERR_ALIGN, "qs_step: obs_gather must be 16-byte aligned");
        if (io->gather_flag && !io->gather_counter) return fail(QS_ERR_NULL, "qs_step: gather_flag needs gather_counter");
    }
    fast = !fast_off && step_fast_eligible(a);
    state20_out = state20; pid_act_out = pid_act;
    return 0;
}

int qs_step(const QsParams* p, const QsState* st, const QsStepIO* io, int act_type, int task,
            int n_envs, int drones_per_env, int substeps, unsigned effects, unsigned flags, void* stream) {
    StepArgs a;
    bool state20 = false, pid_act = false, fast = false;
    if (int rc = prepare_step(p, st, io, act_type, task, n_envs, drones_per_env, substeps, effects, flags, a, state20, pid_act, fast)) return rc;
    const cudaError_t e = launch_step_tracked(a, fast, state20, pid_act, (cudaStream_t)stream);
    return e == cudaSuccess ? 0 : cuda_fail(e, "qs_step launch");
}

int qs_sizeof_host_io(void) { return (int)sizeof(QsHostIO); }

int qs_step_call(const QsStepCall* c, void* stream) {
    if (!c) return fail(QS_ERR_NULL, "qs_step_call: NULL call");
    return qs_step(c->p, c->st, c->io, c->act_type, c->task, c->n_envs, c->drones_per_env, c->substeps, c->effects, c->flags, stream);
}

int qs_host_is_pinned(const void* p) {
    if (!p) return 0;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { (void)cudaGetLastError(); return 0; }
    return at.type == cudaMemoryTypeHost ? 1 : 0;
}

constexpr int kMaxHostChunks = 8, kMaxHostDevices = 32;
#ifndef QS_HOST_CHUNKS_DEFAULT
#define QS_HOST_CHUNKS_DEFAULT 4
#endif
// events (timing disabled) that order chunk c's observation copy after chunk c's kernel: one set per host thread and device,
// created on first use, never destroyed (a handful of driver objects for the life of the process)
static cudaEvent_t* host_chunk_events() {
    static thread_local cudaEvent_t ev[kMaxHostDevices][kMaxHostChunks];
    static thread_local bool made[kMaxHostDevices] = {};
    int dev = -1;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxHostDevices) { (void)cudaGetLastError(); return nullptr; }
    if (!made[dev]) {
        for (int c = 0; c < kMaxHostChunks; ++c)
            if (cudaEventCreateWithFlags(&ev[dev][c], cudaEventDisableTiming) != cudaSuccess) { (void)cudaGetLastError(); return nullptr; }
        made[dev] = true;
    }
    return ev[dev];
}

int qs_step_host(const QsParams* p, const QsState* st, const QsStepIO* io, const QsHostIO* h, int act_type, int task,
                 int n_envs, int drones_per_env, int substeps, unsigned effects, unsigned flags, void* stream) {
    if (!io || !h) return fail(QS_ERR_NULL, "qs_step_host: NULL io");
    if (!h->action_host || !h->obs_host || !h->reward_host || !h->terminated_host || !h->truncated_host || !h->action_dev)
        return fail(QS_ERR_NULL, "qs_step_host: NULL host buffer / action_dev");
    if (!io->obs || !io->reward || !io->terminated || !io->truncated) return fail(QS_ERR_NULL, "qs_step_host: NULL device buffer");
    const int A = act_width(act_type);
    if (A < 0) return fail(QS_ERR_ENUM, "qs_step_host: bad act_type");
    const bool state20 = flags & QS_FLAG_OBS_STATE20;
    const long long N = (long long)n_envs * drones_per_env;
    const int od = state20 ? 20 : 12 + io->act_buffer_size * A;
    const bool want_final = (flags & QS_FLAG_AUTORESET_SAME_STEP) && io->final_obs && h->final_obs_host;
    if (want_final && (!io->done || !h->done_host || !h->final_env_host || !h->n_final_host || !h->final_env_dev || !h->n_final_dev))
        return fail(QS_ERR_NULL, "qs_step_host: final_obs transfer needs done / final_env / n_final buffers");
    if ((h->ev_fork == nullptr) != (h->ev_join == nullptr) || (h->side_stream && !h->ev_fork))
        return fail(QS_ERR_NULL, "qs_step_host: side_stream needs ev_fork and ev_join");
    cudaStream_t s = (cudaStream_t)stream;
    static const bool trace = getenv("QS_TRACE") != nullptr;
    static int trace_n = 0;
    auto now = []() { timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec * 1e6 + ts.tv_nsec * 1e-3; };
    const double t0 = trace ? now() : 0.0;
    QsStepIO dio = *io;
    dio.action = h->action_dev;
    StepArgs sa;
    bool sa_state20 = false, sa_pid = false, sa_fast = false;
    if (int rc = prepare_step(p, st, &dio, act_type, task, n_envs, drones_per_env, substeps, effects, flags, sa, sa_state20, sa_pid, sa_fast)) return rc;
    cudaError_t e = cudaSuccess;
    // Chunked pipeline (fast kernels, full-observation transfer): the batch is cut into `chunks` ranges of whole warps; chunk c's
    // actions go up, its tick runs, and its observation rows come down on the side stream while chunk c+1's actions go up and its
    // tick runs -- the 19 MB device->host copy, which bounds the call, starts after 1/chunks of the H2D + kernel time instead of
    // after all of it, and the launch / copy-issue gaps between dependent operations hide behind it.
    // QS_HOST_CHUNKS=n forces n (1 = off); default 4 from 16 384 drones up.
    int chunks = 1;
    cudaEvent_t* cev = nullptr;
    const long long warps_total = (N + 31) / 32;
    if (sa_fast && h->side_stream && h->ev_join && !(h->obs_head_host && !state20) && !io->obs_gather) {
        const char* ce = getenv("QS_HOST_CHUNKS");
        chunks = ce ? atoi(ce) : (N >= 16384 ? QS_HOST_CHUNKS_DEFAULT : 1);
        if (chunks > kMaxHostChunks) chunks = kMaxHostChunks;
        if (chunks > warps_total) chunks = (int)warps_total;
        if (chunks > 1 && !(cev = host_chunk_events())) chunks = 1;
    }
    bool forked = false, small_done = false;
    const bool chunked = chunks > 1;
    if (chunked) {
        cudaStream_t cs = (cudaStream_t)h->side_stream;
        for (int c = 0; c < chunks; ++c) {
            const long long w0 = warps_total * c / chunks, w1 = warps_total * (c + 1) / chunks;
            const long long d0 = w0 * 32, d1 = (w1 * 32 < N) ? w1 * 32 : N;
            e = cudaMemcpyAsync(h->action_dev + d0 * A, h->action_host + d0 * A, (size_t)(d1 - d0) * A * 4, cudaMemcpyHostToDevice, s);
            if (e != cudaSuccess) return cuda_fail(e, "qs_step_host H2D action");
            sa.first_warp = (int)w0; sa.n_warps = (int)(w1 - w0);
            e = launch_step_tracked(sa, true, sa_state20, sa_pid, s);
            if (e != cudaSuccess) return cuda_fail(e, "qs_step_host launch");
            cudaEventRecord(cev[c], s);
            cudaStreamWaitEvent(cs, cev[c], 0);
            cudaMemcpyAsync(h->obs_host + d0 * od, io->obs + d0 * od, (size_t)(d1 - d0) * od * 4, cudaMemcpyDeviceToHost, cs);
        }
        cudaEventRecord((cudaEvent_t)h->ev_join, cs);
        forked = true;                                                   // joined below, after the small outputs have been queued on s
    } else {
        e = cudaMemcpyAsync(h->action_dev, h->action_host, (size_t)N * A * 4, cudaMemcpyHostToDevice, s);
        if (e != cudaSuccess) return cuda_fail(e, "qs_step_host H2D action");
        e = launch_step_tracked(sa, sa_fast, sa_state20, sa_pid, s);
        if (e != cudaSuccess) return cuda_fail(e, "qs_step_host launch");
    }
    if (want_final) {
        // terminal observations: device-side compaction of the done flags (ascending), then the gather kernel writes the rows,
        // their indices and the count into the mapped host arrays.  On a side stream this overlaps the copies below.
        float* rows_h = nullptr; long long* idx_h = nullptr; int* k_h = nullptr;
        if ((e = cudaHostGetDevicePointer(reinterpret_cast<void**>(&rows_h), h->final_obs_host, 0)) != cudaSuccess ||
            (e = cudaHostGetDevicePointer(reinterpret_cast<void**>(&idx_h), h->final_env_host, 0)) != cudaSuccess ||
            (e = cudaHostGetDevicePointer(reinterpret_cast<void**>(&k_h), h->n_final_host, 0)) != cudaSuccess)
            return cuda_fail(e, "qs_step_host: final_obs_host / final_env_host / n_final_host must be pinned, mapped host memory");
        cudaStream_t fs = s;
        if (h->side_stream && h->ev_fork) {
            if (!chunked) {
                fs = (cudaStream_t)h->side_stream;
                cudaEventRecord((cudaEvent_t)h->ev_fork, s);
                cudaStreamWaitEvent(fs, (cudaEvent_t)h->ev_fork, 0);
                forked = true;
            }
            // the per-aviary outputs travel by kernel stores into the (mapped) host arrays on the side stream as well
            float* rew_h = nullptr; unsigned char *te_h = nullptr, *tr_h = nullptr, *dn_h = nullptr;
            static const bool small_kernel = !(getenv("QS_SMALL_OUT") && atoi(getenv("QS_SMALL_OUT")) == 0);
            if (small_kernel && cudaHostGetDevicePointer(reinterpret_cast<void**>(&rew_h), h->reward_host, 0) == cudaSuccess &&
                cudaHostGetDevicePointer(reinterpret_cast<void**>(&te_h), h->terminated_host, 0) == cudaSuccess &&
                cudaHostGetDevicePointer(reinterpret_cast<void**>(&tr_h), h->truncated_host, 0) == cudaSuccess &&
                cudaHostGetDevicePointer(reinterpret_cast<void**>(&dn_h), h->done_host, 0) == cudaSuccess) {
                small_outputs_kernel<<<(n_envs / 4 + 256) / 256, 256, 0, fs>>>(io->reward, io->terminated, io->truncated, io->done,
                                                                                  rew_h, te_h, tr_h, dn_h, n_envs);
                small_done = true;
            } else {
                (void)cudaGetLastError();
            }
        }
        compact_done_kernel<<<1, 1024, 0, fs>>>(io->done, n_envs, h->final_env_dev, h->n_final_dev);
        const int row_floats = drones_per_env * od;
        const int blocks = n_envs < 1056 ? n_envs : 1056;                                  // 132 SMs x 8, grid-stride over the k rows
        gather_rows_kernel<<<blocks, 128, 0, fs>>>(io->final_obs, h->final_env_dev, h->n_final_dev, rows_h, idx_h, k_h, row_floats);
        if (forked && !chunked) cudaEventRecord((cudaEvent_t)h->ev_join, fs);
    } else if (h->n_final_host) {
        *h->n_final_host = 0;
    }
    if (!small_done) {
        cudaMemcpyAsync(h->reward_host, io->reward, (size_t)n_envs * 4, cudaMemcpyDeviceToHost, s);
        cudaMemcpyAsync(h->terminated_host, io->terminated, (size_t)n_envs, cudaMemcpyDeviceToHost, s);
        cudaMemcpyAsync(h->truncated_host, io->truncated, (size_t)n_envs, cudaMemcpyDeviceToHost, s);
        if (io->done && h->done_host) cudaMemcpyAsync(h->done_host, io->done, (size_t)n_envs, cudaMemcpyDeviceToHost, s);
    }
    if (h->obs_head_host && !state20) {
        float* heads_h = nullptr;
        if ((e = cudaHostGetDevicePointer(reinterpret_cast<void**>(&heads_h), h->obs_head_host, 0)) != cudaSuccess)
            return cuda_fail(e, "qs_step_host: obs_head_host must be pinned, mapped host memory");
        pack_heads_kernel<<<(unsigned)((3 * N + 255) / 256), 256, 0, s>>>(io->obs, od, N, heads_h);
    } else if (!chunked) {
        cudaMemcpyAsync(h->obs_host, io->obs, (size_t)N * od * 4, cudaMemcpyDeviceToHost, s);
    }
    if (forked) cudaStreamWaitEvent(s, (cudaEvent_t)h->ev_join, 0);
    const double t1 = trace ? now() : 0.0;
    e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) return cuda_fail(e, "qs_step_host sync");
    if (trace && (++trace_n % 50) == 0)
        fprintf(stderr, "[qs_step_host] enqueue %.0f us, sync %.0f us, n_final %d\n", t1 - t0, now() - t1, h->n_final_host ? *h->n_final_host : -1);
    e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, "qs_step_host");
}

int qs_dyn_substeps(const QsParams* p, const QsState* st, const float* rpm, float* state20_out, const float* dw_fz,
                    int n_envs, int drones_per_env, int substeps, unsigned effects, unsigned flags, void* stream) {
    return qs_dyn_substeps_pub(p, st, rpm, state20_out, dw_fz, n_envs, drones_per_env, substeps, effects, flags, nullptr, stream);
}

int qs_dyn_substeps_pub(const QsParams* p, const QsState* st, const float* rpm, float* state20_out, const float* dw_fz,
                        int n_envs, int drones_per_env, int substeps, unsigned effects, unsigned flags, const QsDwPublish* pub, void* stream) {
    if (!p || (!rpm && !(flags & QS_FLAG_RPM_FROM_LAST))) return fail(QS_ERR_NULL, "qs_dyn_substeps: NULL params/rpm");
    if ((flags & QS_FLAG_RPM_FROM_LAST) && (!st || !st->last_rpm)) return fail(QS_ERR_NULL, "qs_dyn_substeps: RPM_FROM_LAST needs QsState.last_rpm");
    if (int rc = check_state(st, 0)) return rc;
    if (n_envs <= 0 || drones_per_env <= 0 || substeps <= 0) return fail(QS_ERR_SIZE, "qs_dyn_substeps: sizes must be > 0");
    if (rpm && !aligned16(rpm)) return fail(QS_ERR_ALIGN, "qs_dyn_substeps: rpm must be 16-byte aligned");
    if (rpm && (flags & QS_FLAG_ACTION_F64) && !aligned32(rpm)) return fail(QS_ERR_ALIGN, "qs_dyn_substeps: float64 rpm must be 32-byte aligned");
    if (effects & ~7u) return fail(QS_ERR_ENUM, "qs_dyn_substeps: bad effects");
    if ((effects & QS_EFFECT_DRAG) && !st->last_rpm) return fail(QS_ERR_NULL, "qs_dyn_substeps: DRAG needs QsState.last_rpm");
    if ((effects & QS_EFFECT_DW) && !dw_fz && drones_per_env > kMaxTPB)
        return fail(QS_ERR_UNSUPPORTED, "qs_dyn_substeps: in-CTA downwash needs drones_per_env <= 128 (else pass dw_fz, substeps = 1)");
    if ((effects & QS_EFFECT_DW) && dw_fz && substeps != 1) return fail(QS_ERR_UNSUPPORTED, "qs_dyn_substeps: external dw_fz requires substeps == 1");
    if (st->phys && (dw_fz || pub))
        return fail(QS_ERR_UNSUPPORTED, "qs_dyn_substeps: per-aviary physical constants (QsState.phys) are not supported with external downwash or a formation publish");
    StepArgs a;
    memset(&a, 0, sizeof(a));
    a.P = *p; a.st = *st;
    a.io.action = rpm; a.io.obs = state20_out; a.io.dw_fz = dw_fz;
    a.act_type = QS_ACT_RAW_RPM; a.task = QS_TASK_NONE; a.n_envs = n_envs; a.D = drones_per_env; a.substeps = substeps;
    if ((long long)n_envs * drones_per_env > 0x7fffffffLL) return fail(QS_ERR_SIZE, "qs_dyn_substeps: n_envs * drones_per_env exceeds 2^31-1");
    a.N = n_envs * drones_per_env; a.A = 4; a.obs_dim = 20;
    a.cap = cta_capacity(a.N, drones_per_env);
    a.tpb = block_size_for(drones_per_env, a.cap);
    a.counter_inc = substeps;
    a.effects = effects; a.flags = flags & (QS_FLAG_RPY_F32 | QS_FLAG_RPM_FROM_LAST | QS_FLAG_ACTION_F64);
    if (pub) {
        if (!pub->gathered || !pub->flags || !pub->counter) return fail(QS_ERR_NULL, "qs_dyn_substeps_pub: NULL publish pointer");
        if (pub->world <= 0 || pub->world > QS_MAX_PEERS || pub->rank < 0 || pub->rank >= pub->world) return fail(QS_ERR_SIZE, "qs_dyn_substeps_pub: bad world/rank");
        if (n_envs != 1) return fail(QS_ERR_UNSUPPORTED, "qs_dyn_substeps_pub: one formation = one aviary (n_envs == 1)");
        if (pub->offset < 0 || pub->n_total < pub->offset + a.N) return fail(QS_ERR_SIZE, "qs_dyn_substeps_pub: bad offset/n_total");
        if (pub->offset % 32 != 0 || (a.N % 32 != 0 && pub->offset + a.N != pub->n_total) || a.tpb % 32 != 0)
            return fail(QS_ERR_ALIGN, "qs_dyn_substeps_pub: slices must start on a multiple of 32 drones (a chunk never straddles ranks)");
        for (int r = 0; r < pub->world; ++r) {
            if (!pub->gathered[r] || !pub->flags[r]) return fail(QS_ERR_NULL, "qs_dyn_substeps_pub: NULL peer pointer");
            if (!aligned16(pub->gathered[r])) return fail(QS_ERR_ALIGN, "qs_dyn_substeps_pub: gathered arrays must be 16-byte aligned");
            a.pub_dst[r] = pub->gathered[r]; a.pub_flags[r] = pub->flags[r];
        }
        a.pub_counter = pub->counter; a.pub_world = pub->world; a.pub_rank = pub->rank; a.pub_offset = pub->offset;
        a.pub_n_total = pub->n_total; a.pub_seq = pub->seq;
    }
    const cudaError_t e = launch_step_tracked(a, false, true, false, (cudaStream_t)stream);
    return e == cudaSuccess ? 0 : cuda_fail(e, "qs_dyn_substeps launch");
}

int qs_pid_control(const QsParams* p, double* pid_state, double control_timestep,
                   const float* cur_pos, int pos_stride, const float* cur_quat, int quat_stride,
                   const float* cur_vel, int vel_stride,
                   const float* target_pos, const float* target_rpy, const float* target_vel, const float* target_rpy_rates,
                   int n, float* rpm_out, float* pos_e_out, float* yaw_e_out, void* stream) {
    if (!p || !pid_state || !cur_pos || !cur_quat || !cur_vel || !target_pos || !rpm_out) return fail(QS_ERR_NULL, "qs_pid_control: NULL argument");
    if (n <= 0 || pos_stride < 3 || quat_stride < 4 || vel_stride < 3) return fail(QS_ERR_SIZE, "qs_pid_control: bad n/stride");
    if (!(control_timestep > 0.0)) return fail(QS_ERR_SIZE, "qs_pid_control: control_timestep must be > 0");
    if (!aligned16(rpm_out)) return fail(QS_ERR_ALIGN, "qs_pid_control: rpm_out must be 16-byte aligned");
    PidArgs a;
    a.P = *p; a.pid = pid_state; a.dt = control_timestep;
    a.pos = cur_pos; a.quat = cur_quat; a.vel = cur_vel; a.tpos = target_pos; a.trpy = target_rpy; a.tvel = target_vel; a.trr = target_rpy_rates;
    a.pos_stride = pos_stride; a.quat_stride = quat_stride; a.vel_stride = vel_stride; a.n = n;
    a.rpm_out = rpm_out; a.pos_e_out = pos_e_out; a.yaw_e_out = yaw_e_out;
    pid_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, "qs_pid_control launch");
}

int qs_pid_control_state(const QsParams* p, double* pid_state, double control_timestep, const QsState* st, int n,
                         const double* target_pos, const double* target_rpy, const double* target_vel, const double* target_rpy_rates,
                         double* rpm_out, float* pos_e_out, float* yaw_e_out, void* stream) {
    if (!p || !pid_state || !st || !st->planes || !target_pos || !rpm_out) return fail(QS_ERR_NULL, "qs_pid_control_state: NULL argument");
    if (n <= 0) return fail(QS_ERR_SIZE, "qs_pid_control_state: n must be > 0");
    if (!(control_timestep > 0.0)) return fail(QS_ERR_SIZE, "qs_pid_control_state: control_timestep must be > 0");
    if (!aligned32(st->planes) || !aligned32(rpm_out)) return fail(QS_ERR_ALIGN, "qs_pid_control_state: planes / rpm_out must be 32-byte aligned");
    PidStateArgs a;
    a.P = *p; a.pid = pid_state; a.dt = control_timestep; a.planes = st->planes;
    a.tpos = target_pos; a.trpy = target_rpy; a.tvel = target_vel; a.trr = target_rpy_rates; a.n = n;
    a.rpm_out = rpm_out; a.pos_e_out = pos_e_out; a.yaw_e_out = yaw_e_out;
    pid_state_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, "qs_pid_control_state launch");
}

int qs_wait_flags(const unsigned* flags, unsigned seq, int world, unsigned* err_flag, void* stream) {
    if (!flags) return fail(QS_ERR_NULL, "qs_wait_flags: NULL flags");
    if (world <= 0 || world > QS_MAX_PEERS) return fail(QS_ERR_SIZE, "qs_wait_flags: world must be in [1, QS_MAX_PEERS]");
    wait_flags_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(flags, seq, world, err_flag);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, "qs_wait_flags launch");
}

int qs_sizeof_log_ring(void) { return (int)sizeof(QsLogRing); }

int qs_log_append(const QsParams* p, const QsState* st, const float* obs, int obs_dim, const float* controls,
                  const QsLogRing* ring, int n_envs, int drones_per_env, void* stream) {
    if (!p || !ring || !ring->ring || !ring->head || !obs) return fail(QS_ERR_NULL, "qs_log_append: NULL argument");
    if (int rc = check_state(st, 0)) return rc;
    if (n_envs <= 0 || drones_per_env <= 0 || ring->capacity <= 0 || ring->n_drones <= 0 || ring->first_drone < 0 ||
        (long long)ring->first_drone + ring->n_drones > (long long)n_envs * drones_per_env)
        return fail(QS_ERR_SIZE, "qs_log_append: bad ring geometry");
    if (obs_dim < 12) return fail(QS_ERR_SIZE, "qs_log_append: obs_dim < 12");
    const int blocks = (ring->n_drones + 127) / 128;
    log_append_kernel<<<blocks, 128, 0, (cudaStream_t)stream>>>(*p, *st, obs, obs_dim, controls, *ring, (long long)n_envs * drones_per_env, drones_per_env);
    log_advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(ring->head);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, "qs_log_append launch");
}

int qs_reset_heads(const QsState* st, int rows, unsigned flags, float* out, void* stream) {
    if (!st || !st->init_pos || !st->init_quat || !out) return fail(QS_ERR_NULL, "qs_reset_heads: NULL argument");
    if (!aligned32(st->init_pos) || !aligned32(st->init_quat) || !aligned16(out)) return fail(QS_ERR_ALIGN, "qs_reset_heads: misaligned table");
    if (rows <= 0) return fail(QS_ERR_SIZE, "qs_reset_heads: rows must be > 0");
    (void)flags;
    reset_heads_kernel<<<(rows + 127) / 128, 128, 0, (cudaStream_t)stream>>>(*st, rows, out);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, "qs_reset_heads launch");
}

int qs_reset(const QsParams* p, const QsState* st, const unsigned char* mask, int n_envs, int drones_per_env,
             int reset_pid, float* obs, int obs_dim, int raw_state20, void* stream) {
    (void)p;
    if (int rc = check_state(st, 1)) return rc;
    if (n_envs <= 0 || drones_per_env <= 0) return fail(QS_ERR_SIZE, "qs_reset: sizes must be > 0");
    if (obs && !raw_state20 && obs_dim < 12) return fail(QS_ERR_SIZE, "qs_reset: obs_dim < 12");
    ResetArgs a;
    a.st = *st; a.mask = mask; a.D = drones_per_env; a.reset_pid = reset_pid; a.obs_dim = obs_dim; a.raw20 = raw_state20;
    a.N = (long long)n_envs * drones_per_env; a.obs = obs;
    reset_kernel<<<(int)((a.N + 127) / 128), 128, 0, (cudaStream_t)stream>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, "qs_reset launch");
}

}  // extern "C"
