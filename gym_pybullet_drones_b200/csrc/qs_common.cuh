// qs_common.cuh -- shared by the translation units of libquadsim.so: error convention, argument structs, the state
// load/store helpers (float64 planes, 32-byte accesses), TMA bulk-copy / mbarrier wrappers, launch geometry, the dispatch from
// run-time options to kernel instantiations.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <time.h>
#include <type_traits>

#include "quad_core.cuh"

namespace qsi {

extern thread_local char g_err[256];          // defined in quadsim.cu (qs_last_error)

inline int fail(int code, const char* msg) {
    snprintf(g_err, sizeof(g_err), "%s", msg);
    return code;
}
inline int fail(int code, const char* what, const char* msg) {
    snprintf(g_err, sizeof(g_err), "%s: %s", what, msg);
    return code;
}

inline int cuda_fail(cudaError_t e, const char* where) {
    snprintf(g_err, sizeof(g_err), "%s: %s", where, cudaGetErrorString(e));
    return (int)e;
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
inline bool aligned32(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 31u) == 0; }

constexpr int kMaxTPB = 128;          // threads (= drones) per CTA upper bound
// fixed part of the step kernel's dynamic shared memory (heads, actions, reductions, in-CTA downwash positions, flags,
// mbarrier), rounded so that the staged rows that follow are 128-byte aligned
__host__ __device__ constexpr size_t smem_fixed(int cap) {
    return ((size_t)cap * 20 * 4 + (size_t)cap * 4 * 4 + (size_t)cap * 2 * 8 + (size_t)cap * 3 * 8 + 3 * (size_t)cap + 16 + 127) / 128 * 128;
}
constexpr size_t kStepSmemFixed = smem_fixed(kMaxTPB);      // upper bound (cap = 128)

struct StepArgs {
    QsParams P;
    QsState st;
    QsStepIO io;
    int act_type, task, n_envs, D, substeps, N, A, obs_dim, tpb, counter_inc;
    unsigned effects, flags;
    int stage_rows;      // 1: the CTA's prev_obs rows are staged in shared memory by one TMA bulk copy
    int cap;             // CTA capacity in drones (64 or 128): sizes the shared-memory arrays
    int log2D;           // log2(D) when D is a power of two, else -1
    int sc_limit;        // smallest step counter with (double)sc / pyb_freq > episode_len_sec (HoverAviary.py:113)
    int grid_wait;       // fast kernels: 1 = griddepcontrol.wait for the whole previous grid (quadsim.cu launch_step_tracked, DESIGN.md 4.1)
    int dbg_slot;        // QS_TIMELINE builds: which timeline buffer this launch stamps
    int pipe;            // fast kernels, A = 4: 1 = step_pipe_kernel, 0 = the classic kernel (QS_FAST_PIPE=0)
    int first_warp, n_warps;   // fast kernels: launch over 32-drone tiles [first_warp, first_warp + n_warps) of the batch only (n_warps = 0:
                         // all); qs_step_host pipelines chunks of the batch against their host copies
    // formation exchange fused into the dynamics kernel (qs_dyn_substeps_pub; general kernel only): pub_world > 0 = on
    float* pub_dst[QS_MAX_PEERS];
    unsigned* pub_flags[QS_MAX_PEERS];
    unsigned* pub_counter;
    int pub_world, pub_rank, pub_offset, pub_n_total;
    unsigned pub_seq;
};

// order-preserving float <-> int keys for warp-wide min / max (redux.sync)
__device__ __forceinline__ int f2key(float x) { const int i = __float_as_int(x); return i ^ ((i >> 31) & 0x7fffffff); }
__device__ __forceinline__ float key2f(int k) { return __int_as_float(k ^ ((k >> 31) & 0x7fffffff)); }
__device__ __forceinline__ float warp_min(float x) { return key2f(__reduce_min_sync(0xffffffffu, f2key(x))); }
__device__ __forceinline__ float warp_max(float x) { return key2f(__reduce_max_sync(0xffffffffu, f2key(x))); }
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Formation exchange, producer side (used by dw_publish_kernel and by the dynamics kernel's epilogue): every thread pushes the
// position v of drone `idx` of this rank's slice (ok = the drone exists) into every rank's gathered array, lane 0 of a warp the box
// of its chunk of 32; then the last CTA of the grid to arrive raises this rank's flag on every rank with release semantics.
// Must be reached by every thread of the CTA; a warp = 32 consecutive drones starting on a multiple of 32.
__device__ __forceinline__ void publish_positions(float4 v, bool ok, long long idx, int n, float* const* dst, unsigned* const* flags,
                                                  unsigned* counter, int world, int rank, int offset, int n_total, unsigned seq) {
    constexpr float BIG = 3e30f;
    const int lane = threadIdx.x & 31;
    const float x0 = warp_min(ok ? v.x : BIG), x1 = warp_max(ok ? v.x : -BIG);
    const float y0 = warp_min(ok ? v.y : BIG), y1 = warp_max(ok ? v.y : -BIG);
    const float z0 = warp_min(ok ? v.z : BIG), z1 = warp_max(ok ? v.z : -BIG);
    const long long first = idx - lane;                                   // warp-uniform
    if (first < n) {
        const long long chunk = (offset + first) >> 5;
        for (int r = 0; r < world; ++r) {
            float4* d = reinterpret_cast<float4*>(dst[r]);
            if (ok) d[offset + idx] = v;
            if (lane == 0) {
                float4* b = d + n_total + 2 * chunk;
                b[0] = make_float4(x0, y0, z0, 0.f);
                b[1] = make_float4(x1, y1, z1, 0.f);
            }
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence_system();                                           // cumulative over the CTA's stores (barrier above)
        const unsigned t = atomicAdd(counter, 1u);
        if (t == gridDim.x - 1) {
            *counter = 0u;
            __threadfence_system();
            for (int r = 0; r < world; ++r) st_release_sys(flags[r] + rank, seq);
        }
    }
}

__device__ __forceinline__ float4 ldg4(const float* base, long long idx4) {
    return __ldg(reinterpret_cast<const float4*>(base) + idx4);
}
__device__ __forceinline__ void st4(float* base, long long idx4, float4 v) {
    reinterpret_cast<float4*>(base)[idx4] = v;
}

// 32-byte global accesses: one drone's double4 as two adjacent 16-byte vector accesses (sm_90's widest global load / store
// is 128 bits); both halves fall into the same 32-byte sector, so a warp still touches whole sectors only
struct D4 { double x, y, z, w; };
__device__ __forceinline__ D4 ld256(const double* base, long long idx4) {
    D4 v;
    const double* p = base + 4 * idx4;
    asm volatile("ld.global.v2.f64 {%0,%1}, [%4];\n\tld.global.v2.f64 {%2,%3}, [%4+16];"
                 : "=d"(v.x), "=d"(v.y), "=d"(v.z), "=d"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ D4 ld256_nc(const double* base, long long idx4) {       // read-only tables
    D4 v;
    const double* p = base + 4 * idx4;
    asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%4];\n\tld.global.nc.v2.f64 {%2,%3}, [%4+16];"
                 : "=d"(v.x), "=d"(v.y), "=d"(v.z), "=d"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ void st256(double* base, long long idx4, double x, double y, double z, double w) {
    asm volatile("st.global.v2.f64 [%0], {%1,%2};\n\tst.global.v2.f64 [%0+16], {%3,%4};"
                 ::"l"(base + 4 * idx4), "d"(x), "d"(y), "d"(z), "d"(w) : "memory");
}

// ---- TMA bulk copy (cp.async.bulk, SASS UBLKCP) + mbarrier: one thread moves a whole contiguous span global -> shared
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* bar) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// the same copy for data read once and dead afterwards: its L2 lines are marked evict-first, so they leave the cache ahead of
// lines that will still be read (what this launch stores, what the next launch prefetches)
__device__ __forceinline__ void tma_bulk_g2s_read_once(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* bar) {
    unsigned long long pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(pol) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
    unsigned ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    } while (!ok);
}

__device__ __forceinline__ bool mbar_test(unsigned long long* bar, unsigned parity) {      // non-blocking
    unsigned ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

// ---- per-warp readiness between consecutive fast steps on the same buffers (QsStepIO.warp_ticket / warp_done, DESIGN.md 4.1)
// One thread per warp.  Spins until *done == ticket (acquire, gpu scope), backing off with __nanosleep; after ~1 s of
// %globaltimer it raises *err and proceeds, so a protocol bug shows up as a wrong result and a non-zero error word, never as
// a hung GPU.  The fence orders the acquire before the warp's later bulk copies, which read through the async proxy.
__device__ __forceinline__ void warp_wait_turn(const unsigned* done, unsigned ticket, unsigned* err) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(done) : "memory");
    if (v != ticket) {
        const unsigned long long t0 = globaltimer_ns();
        unsigned ns = 32;
        do {
            __nanosleep(ns);
            if (ns < 1024) ns <<= 1;
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(done) : "memory");
            if (v != ticket && globaltimer_ns() - t0 > 1000000000ull) { if (err) atomicOr(err, 1u); break; }
        } while (v != ticket);
    }
    asm volatile("fence.proxy.async.global;" ::: "memory");
}
// All 32 lanes.  Every generic store of the warp (state, counters, rewards, observation patches, terminal rows) and its bulk
// stores, which must have COMPLETED (cp.async.bulk.wait_group 0, not .read), come before the release of the next ticket.
__device__ __forceinline__ void warp_publish(unsigned* done, unsigned next) {
    __threadfence();
    __syncwarp();
    if ((threadIdx.x & 31) == 0) {
        asm volatile("fence.proxy.async.global;" ::: "memory");
        asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(done), "r"(next) : "memory");
    }
}

__device__ __forceinline__ void cp_async4(float* dst_smem, const float* src_gmem) {      // LDGSTS, 4-byte granule
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit_wait_all() {
    asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
}

__device__ __forceinline__ void load_drone(const double* planes, long long N, long long i, qs::Drone& d) {
    const D4 p0 = ld256(planes, i), p1 = ld256(planes, N + i), p2 = ld256(planes, 2 * N + i);
    const double wz = planes[12 * N + i];
    d.px = p0.x; d.py = p0.y; d.pz = p0.z;
    d.qx = p1.x; d.qy = p1.y; d.qz = p1.z; d.qw = p1.w;
    d.vx = p2.x; d.vy = p2.y; d.vz = p2.z;
    d.wx = p0.w; d.wy = p2.w; d.wz = wz;
}

// normalises the quaternion (the north-star's "quaternion renormalise"; Bullet's own read-back goes through a
// rotation matrix and renormalises too) and stores the planes (+ the optional float32 position mirror)
__device__ __forceinline__ void store_drone(const QsState& st, long long N, long long i, qs::Drone& d) {
    const double inv = rsqrt(qs::quat_norm2(d.qx, d.qy, d.qz, d.qw));
    d.qx = __dmul_rn(d.qx, inv); d.qy = __dmul_rn(d.qy, inv); d.qz = __dmul_rn(d.qz, inv); d.qw = __dmul_rn(d.qw, inv);
    double* planes = st.planes;
    st256(planes, i, d.px, d.py, d.pz, d.wx);
    st256(planes, N + i, d.qx, d.qy, d.qz, d.qw);
    st256(planes, 2 * N + i, d.vx, d.vy, d.vz, d.wy);
    planes[12 * N + i] = d.wz;
    if (st.pos_f32) st4(st.pos_f32, i, make_float4((float)d.px, (float)d.py, (float)d.pz, 0.f));
}

// what store_drone + load_drone do to the state between two ticks of a multi-tick kernel: the quaternion is renormalised, nothing
// is rounded (the planes are float64), so T fused ticks equal T single-tick calls bit for bit
__device__ __forceinline__ void round_to_planes(qs::Drone& d) {
    const double inv = rsqrt(qs::quat_norm2(d.qx, d.qy, d.qz, d.qw));
    d.qx = __dmul_rn(d.qx, inv); d.qy = __dmul_rn(d.qy, inv); d.qz = __dmul_rn(d.qz, inv); d.qw = __dmul_rn(d.qw, inv);
}

__device__ __forceinline__ void init_drone(const QsState& st, long long tbl, qs::Drone& d) {
    const D4 ip = ld256_nc(st.init_pos, tbl), iq = ld256_nc(st.init_quat, tbl);
    d.px = ip.x; d.py = ip.y; d.pz = ip.z;
    d.qx = iq.x; d.qy = iq.y; d.qz = iq.z; d.qw = iq.w;
    d.vx = d.vy = d.vz = 0.0;
    d.wx = d.wy = d.wz = 0.0;
}

// row e of QsState.phys (include/quadsim.h): 7 x 16 bytes of the 128-byte row through the read-only path.  The drones of one
// aviary read the same row, so within a warp the loads are broadcasts; the padding is never read.
__device__ __forceinline__ qs::PhysRow load_phys(const double* phys, long long e) {
    const double2* r = reinterpret_cast<const double2*>(phys + 16 * e);
    const double2 v0 = __ldg(r), v1 = __ldg(r + 1), v2 = __ldg(r + 2), v3 = __ldg(r + 3), v4 = __ldg(r + 4), v5 = __ldg(r + 5), v6 = __ldg(r + 6);
    qs::PhysRow c;
    c.inv_m = v0.x; c.gravity = v0.y; c.kf = v1.x; c.km = v1.y; c.kx = v2.x; c.ky = v2.y;
    c.j[0] = v3.x; c.j[1] = v3.y; c.j[2] = v4.x; c.j_inv[0] = v4.y; c.j_inv[1] = v5.x; c.j_inv[2] = v5.y;
    c.hover_rpm = v6.x; c.max_rpm = v6.y;
    return c;
}
// only the two columns the action decode reads (HOVER_RPM, MAX_RPM): the embedded PID controller runs between the decode and the
// physics, and the full row live across it would spill
__device__ __forceinline__ qs::PhysRow load_phys_rpm(const double* phys, long long e) {
    const double2 v6 = __ldg(reinterpret_cast<const double2*>(phys + 16 * e) + 6);
    qs::PhysRow c;
    c.hover_rpm = v6.x; c.max_rpm = v6.y;
    return c;
}

__device__ __forceinline__ void load_rpm(const double* last_rpm, long long i, double rpm[4]) {
    const D4 v = ld256(last_rpm, i);
    rpm[0] = v.x; rpm[1] = v.y; rpm[2] = v.z; rpm[3] = v.w;
}
__device__ __forceinline__ void load_pid(const double* ps, long long N, long long i, qs::PidState& pst) {
    pst.ipx = ps[i]; pst.ipy = ps[N + i]; pst.ipz = ps[2 * N + i];
    pst.lr = ps[3 * N + i]; pst.lp = ps[4 * N + i]; pst.ly = ps[5 * N + i];
    pst.irx = ps[6 * N + i]; pst.iry = ps[7 * N + i]; pst.irz = ps[8 * N + i];
}
__device__ __forceinline__ void store_pid(double* ps, long long N, long long i, const qs::PidState& pst) {
    ps[i] = pst.ipx; ps[N + i] = pst.ipy; ps[2 * N + i] = pst.ipz;
    ps[3 * N + i] = pst.lr; ps[4 * N + i] = pst.lp; ps[5 * N + i] = pst.ly;
    ps[6 * N + i] = pst.irx; ps[7 * N + i] = pst.iry; ps[8 * N + i] = pst.irz;
}


constexpr size_t kStageLimit = 40 * 1024;      // bytes of staged rows per CTA (4 CTAs/SM must fit in 227 KB)

inline int act_width(int act_type) {
    switch (act_type) {
        case QS_ACT_RPM: case QS_ACT_VEL: case QS_ACT_RAW_RPM: return 4;
        case QS_ACT_PID: return 3;
        case QS_ACT_ONE_D_RPM: case QS_ACT_ONE_D_PID: return 1;
        default: return -1;
    }
}

// ---- from run-time options to a kernel instantiation (host code).  Every launcher picks its template arguments through these
// two: the generic lambda f receives the value as a type and names the kernel once.
template <int... Vs> struct IntList {};
// f(std::integral_constant<int, V>{}) for the V of the list that equals v; false, and no call, when none does
template <int... Vs, class F>
bool with_int(IntList<Vs...>, int v, F&& f) {
    return ((v == Vs && (f(std::integral_constant<int, Vs>{}), true)) || ...);
}
// f(std::true_type{}) or f(std::false_type{}); returns what f returns
template <class F>
auto with_bool(bool b, F&& f) { return b ? f(std::true_type{}) : f(std::false_type{}); }

// the DYN+ effect sets that have kernels, written here only
using AllEffects = IntList<0, 1, 2, 3, 4, 5, 6, 7>;                                                  // general step, action rollout
using PolicyEffects = IntList<0, QS_EFFECT_GND, QS_EFFECT_DRAG, QS_EFFECT_DW, 7>;                    // policy and control rollouts
using TrajEffects = IntList<0, QS_EFFECT_GND, QS_EFFECT_DRAG, QS_EFFECT_GND | QS_EFFECT_DRAG>;       // differentiable trajectories
using PlanEffects = IntList<0, QS_EFFECT_GND, QS_EFFECT_DRAG, QS_EFFECT_GND | QS_EFFECT_DRAG, QS_EFFECT_DW, 7>;   // mppi
using DwTrajEffects = IntList<QS_EFFECT_DW, 7>;                                                      // downwash trajectories
inline bool policy_effects_supported(unsigned eff) { return with_int(PolicyEffects{}, (int)eff, [](auto) {}); }

int check_state(const QsState* st, int need_tables);                      // quadsim.cu
int cta_capacity(long long N, int D, bool rollout = false);               // quadsim.cu
inline int block_size_for(int D, int cap = kMaxTPB) { return D <= cap ? D * (cap / D) : cap; }

// launchers of the kernel families (one translation unit each)
// pdl_ok = false: an ordinary stream-ordered launch (not a programmatic dependent of the previous kernel)
cudaError_t launch_step_general(const StepArgs& a, bool raw, bool pid_act, bool pdl_ok, cudaStream_t s);      // step_general.cu
bool step_fast_eligible(const StepArgs& a);                                                       // step_fast.cu
cudaError_t launch_step_fast(const StepArgs& a, cudaStream_t s);                                  // step_fast.cu

// QS_PDL=0 (a debugging switch for the ordering protocol): the step kernels are ordinary stream-ordered launches
inline bool pdl_enabled() {
    static const bool on = !(getenv("QS_PDL") && atoi(getenv("QS_PDL")) == 0);
    return on;
}
// kernel<<<blocks, threads, smem, s>>>(a), a programmatic dependent of the previous kernel on s when pdl is set (the kernel's
// griddepcontrol instructions then decide what overlaps).  Above 48 KB, the kernel's dynamic shared-memory limit is first
// raised to smem_limit.
inline cudaError_t launch_step_kernel(void (*kernel)(StepArgs), int blocks, int threads, size_t smem, size_t smem_limit, bool pdl,
                                      cudaStream_t s, const StepArgs& a) {
    if (smem > 48 * 1024) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_limit);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(blocks); cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, a);
}

// What the last library launch on a stream that lets its successor start early (griddepcontrol.launch_dependents) was:
// nothing yet, a fast step, or another kernel (general step, formation publish).  Only the library's own early-triggering
// launches are recorded; every other kernel or copy releases its successor at completion.  quadsim.cu.
enum PdlPrev { kPdlNone = 0, kPdlFast = 1, kPdlOther = 2 };
PdlPrev pdl_prev(cudaStream_t s);
void pdl_note(cudaStream_t s, PdlPrev what);

}  // namespace qsi
