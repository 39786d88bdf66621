// rollout_kernel.cuh -- the fused multi-tick rollout kernel and its launchers (DESIGN.md 4.1b), shared by rollout.cu (no autoreset,
// SAME_STEP), rollout_next.cu (NEXT_STEP) and rollout_mlp.cu (the general network): one kernel, each translation unit
// instantiates its own networks and modes.
#pragma once
#include "qs_common.cuh"
#include <cuda_fp16.h>

namespace qsi {

// ---------------------------------------------------------------------------------------------------------
// Multi-tick rollout: the fused control tick in a loop.  Drone state lives in registers, the CTA's observation rows in a
// shared-memory window that slides by one action per tick (new_flat[j] = old_flat[j + A], so "shifting the history" is
// `base += A`); per tick the kernel reads the action and writes the rows, reward and flags.  Bit-identical to T calls of
// qs_step: the state is rounded to its float32 plane representation at every tick boundary exactly like store/load.
// ---------------------------------------------------------------------------------------------------------
struct RolloutArgs {
    QsParams P;
    QsState st;
    QsRolloutIO io;
    QsPolicy pol;        // copy of *io.policy (device pointers inside) when POLICY
    int act_type, task, n_envs, D, substeps, N, A, obs_dim, tpb;
    unsigned effects, flags;
    int stage_mode, cap;
};

// qs_rollout_mlp (rollout_mlp.cu): the rollout arguments plus the general network.  `pol` carries what the kernel body shares
// with the classic policy: log_std, noise, logprob, values, in_dim, out_dim, nt3 = actor.out_tiles, vw1 != NULL iff a critic.
struct MlpRolloutArgs : RolloutArgs {
    QsMlpPolicy mlp;
    int stage_off, stage_ks;   // per-warp activation staging: byte offset in dynamic shared memory, k-steps per buffer
};

// Who chooses the actions: the caller or the seeded generator (none), the classic [64, 64] Tanh network of qs_rollout (QsPolicy),
// or the general network of qs_rollout_mlp (QsMlpPolicy).  NET picks the kernel's argument type.
enum RolloutNet { kNetNone, kNetClassic, kNetMlp };
template <int NET> struct RolloutArgsOf { using type = RolloutArgs; };
template <> struct RolloutArgsOf<kNetMlp> { using type = MlpRolloutArgs; };

// What a rollout produces besides the per-tick outputs: nothing more (none), the terminal observations and their critic values
// of SAME_STEP autoreset (FIN), or the NEXT_STEP autoreset ticks (NEXT).  FIN and NEXT never combine.
enum RolloutMode { kRolloutNone = 0, kRolloutFin = 1, kRolloutNext = 2 };
inline int rollout_mode(const QsRolloutIO* io, unsigned flags) {
    return (flags & QS_FLAG_AUTORESET_NEXT_STEP) ? kRolloutNext : (io->final_obs || io->final_values) ? kRolloutFin : kRolloutNone;
}

// the NEXT_STEP rollouts of qs_rollout (rollout_next.cu: a translation unit of their own, compiled in parallel with rollout.cu)
int launch_rollout_next(RolloutArgs& a, const QsRolloutIO* io, bool pid_act, void* stream);
// The argument checks of both entry points and the RolloutArgs they give (rollout.cu); has_critic: the policy, if any, has a
// critic.  `what`, here and below, is the name of the entry point that was called.
int prepare_rollout(const char* what, const QsParams* p, const QsState* st, const QsRolloutIO* io, int act_type, int task, int n_envs,
                    int drones_per_env, int substeps, unsigned effects, unsigned flags, bool has_critic, RolloutArgs& a, bool& pid_act);
// the checks every on-device policy shares: effect set, drones per aviary, no caller actions
int check_policy_config(const char* what, const RolloutArgs& a, const QsRolloutIO* io);
// check_policy_config, then the checks of the classic network io->policy (rollout.cu)
int check_classic_policy(const RolloutArgs& a, const QsRolloutIO* io);

namespace {

// ---- on-device policy: SB3-MlpPolicy-shaped MLP on the tensor cores, fp32-accurate ------------------------------------------------
// One warp takes 16 aviaries (one m-tile) through the whole network: Y[16][64] = X[16][K] W[K][64] per layer as mma.sync.m16n8k16
// F16 tiles with a two-term split of both operands: x = x_hi + x_lo, w = w_hi + w_lo with x_hi = fp16(x) and
// x_lo' = fp16(2^11 (x - x_hi)) (the scaling keeps the remainder out of the fp16 subnormals), and
//     x w ~ x_hi w_hi + 2^-11 (x_hi w_lo' + x_lo' w_hi)
// with fp32 accumulation in two accumulator sets -- relative error ~2^-21 per product, i.e. fp32-level (a plain F16/TF32/BF16 mma has
// 2^-11 / 2^-8 and fails the 1e-5 parity with the fp32 torch network).  FP16 and TF32 carry the same 11 significant bits, but one
// m16n8k16 F16 instruction does twice the work of an m16n8k8 TF32 one at the same issue rate (8 cycles per SM sub-partition,
// tools/mma_rate.cu): 3 instead of 6 mma per 16x8x16 block.
//  * Weights: split once on the host (MlpPolicy) and stored in FRAGMENT ORDER, [k-step][n-tile][lane] x 16 bytes = the lane's
//    {b0 hi, b1 hi, b0 lo', b1 lo'} registers, so a B fragment is one fully coalesced 128-bit load (L1-resident: the CTAs use
//    ~160 KB of the SM's 256 KB as shared memory, the actor's 55 KB of weights stay in the rest).
//  * First layer: the observation rows are read from the shared-memory window as 128-bit loads -- lane t supplies elements
//    4t .. 4t+3 of each 16-wide k-step instead of the canonical {2t, 2t+1, 2t+8, 2t+9}; W1 is packed with the same permutation of
//    k, so the product is unchanged -- and split per fragment (both conversions saturate to +-65504, so an observation acts
//    like one clipped to +-(65504 + 65504 / 2048) = +-65535.984375).
//  * Hidden layers never leave the registers: the accumulator fragment of n-tiles (2j, 2j+1) IS the A fragment of k-step j of the
//    next layer (tanh, split, pack) -- no shared-memory round trip, no barrier between layers.
// K = 144 / 64 and M = 32 rows per CTA are below a wgmma tile (M = 64 per warpgroup, B operand through shared-memory descriptors)
// and the weights would have to be staged in shared memory next to the observation window -- see DESIGN.md 4.1b.
constexpr float kLoScale = 2048.f, kLoInv = 1.f / 2048.f;

__device__ __forceinline__ unsigned pack_f16x2_sat(float lo_elem, float hi_elem) {
    unsigned r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi_elem), "f"(lo_elem));
    return r;
}
// (x0, x1) -> packed halves of the leading parts and of the scaled remainders
__device__ __forceinline__ void f16_split2(float x0, float x1, unsigned& hi, unsigned& lo) {
    hi = pack_f16x2_sat(x0, x1);
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hi));
    lo = pack_f16x2_sat((x0 - f.x) * kLoScale, (x1 - f.y) * kLoScale);
}
__device__ __forceinline__ void mma_f16(float c[4], const unsigned a[4], unsigned b0, unsigned b1) {
    asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// tanh(x) = 1 - 2 / (exp(2x) + 1) on the special-function unit: absolute error ~2e-7 (the libm tanhf costs ~4x the instructions)
__device__ __forceinline__ float tanh_fast(float x) { return 1.f - __fdividef(2.f, __expf(2.f * x) + 1.f); }

// G n-tiles from n0 against one A fragment: three sweeps, so that no mma waits for the one issued just before it
template <int G>
__device__ __forceinline__ void mma_group(float (*c)[4], float (*cx)[4], const unsigned (&ah)[4], const unsigned (&al)[4], const uint4 (&b)[G]) {
#pragma unroll
    for (int n = 0; n < G; ++n) mma_f16(cx[n], al, b[n].x, b[n].y);          // x_lo' w_hi
#pragma unroll
    for (int n = 0; n < G; ++n) mma_f16(c[n], ah, b[n].x, b[n].y);           // x_hi  w_hi
#pragma unroll
    for (int n = 0; n < G; ++n) mma_f16(cx[n], ah, b[n].z, b[n].w);          // x_hi  w_lo'
}
template <int G>
__device__ __forceinline__ void load_bfrag(uint4 (&b)[G], const uint4* __restrict__ W) {
#pragma unroll
    for (int n = 0; n < G; ++n) b[n] = __ldg(W + 32 * n);
}
template <int NT>
__device__ __forceinline__ void init_acc(float (&c)[NT][4], float (&cx)[NT][4], const float* __restrict__ bias, int t) {
#pragma unroll
    for (int n = 0; n < NT; ++n) {
        const float2 b = __ldg(reinterpret_cast<const float2*>(bias + 8 * n + 2 * t));
        c[n][0] = b.x; c[n][1] = b.y; c[n][2] = b.x; c[n][3] = b.y;
        cx[n][0] = 0.f; cx[n][1] = 0.f; cx[n][2] = 0.f; cx[n][3] = 0.f;
    }
}
// accumulators of a 64-unit hidden layer -> tanh -> the 4 k-steps of A fragments of the next layer
__device__ __forceinline__ void hidden_to_afrag(const float (&c)[8][4], const float (&cx)[8][4], unsigned (&hh)[4][4], unsigned (&hl)[4][4]) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int n = 2 * j + h;
            const float v0 = tanh_fast(fmaf(cx[n][0], kLoInv, c[n][0])), v1 = tanh_fast(fmaf(cx[n][1], kLoInv, c[n][1]));
            const float v2 = tanh_fast(fmaf(cx[n][2], kLoInv, c[n][2])), v3 = tanh_fast(fmaf(cx[n][3], kLoInv, c[n][3]));
            f16_split2(v0, v1, hh[j][2 * h], hl[j][2 * h]);                  // row g
            f16_split2(v2, v3, hh[j][2 * h + 1], hl[j][2 * h + 1]);          // row g + 8
        }
}

// One network (in -> 64 tanh -> 64 tanh -> 8 nt3 outputs) for 16 aviaries, by one warp.  x_s: rows of in_dim fp32 values in shared
// memory (rows past n_rows repeat the last row; their outputs are not stored); W1/W2/W3: fragment-ordered weights (see above; W1 with
// the 4t permutation); out_s rows have stride 8 nt3 floats (padded outputs).
__device__ __forceinline__ void warp_net(const float* x_s, int in_dim, const uint4* __restrict__ W1, const uint4* __restrict__ W2,
                                         const uint4* __restrict__ W3, const float* b1, const float* b2, const float* b3, int nt3, float* out_s,
                                         int n_rows, int lane) {
    const int g = lane >> 2, t = lane & 3;
    unsigned hh[4][4], hl[4][4];
    {   // ---- layer 1: K = in_dim from shared memory ----
        float c[8][4], cx[8][4];
        init_acc<8>(c, cx, b1, t);
        const int last = n_rows - 1;
        const float* p0 = x_s + (size_t)(g < last ? g : last) * in_dim + 4 * t;
        const float* p1 = x_s + (size_t)(g + 8 < last ? g + 8 : last) * in_dim + 4 * t;
        const bool vec4 = ((reinterpret_cast<size_t>(x_s) & 15) == 0) && ((in_dim & 3) == 0);
        // four rotating B buffers of 2 n-tiles: each is refilled with the next k-step's tiles right after its mma group, i.e. three
        // groups (18 mma) plus the next fragment split ahead of its use
        const uint4* w = W1 + lane;
        uint4 b0[2], b1[2], b2[2], b3[2];
        load_bfrag<2>(b0, w); load_bfrag<2>(b1, w + 2 * 32); load_bfrag<2>(b2, w + 4 * 32); load_bfrag<2>(b3, w + 6 * 32);
#pragma unroll 1
        for (int k0 = 0; k0 < in_dim; k0 += 16, w += 8 * 32) {
            unsigned ah[4], al[4];
            if (vec4 && k0 + 16 <= in_dim) {
                const float4 u = *reinterpret_cast<const float4*>(p0 + k0), v = *reinterpret_cast<const float4*>(p1 + k0);
                f16_split2(u.x, u.y, ah[0], al[0]); f16_split2(v.x, v.y, ah[1], al[1]);
                f16_split2(u.z, u.w, ah[2], al[2]); f16_split2(v.z, v.w, ah[3], al[3]);
            } else {                                         // unaligned rows (odd action width) or the ragged last k-step: elements past
                const int ka = k0 + 4 * t;                   // in_dim are zeros (their weights are zero rows)
                const float* q0 = p0 + k0; const float* q1 = p1 + k0;
                f16_split2(ka < in_dim ? q0[0] : 0.f, ka + 1 < in_dim ? q0[1] : 0.f, ah[0], al[0]);
                f16_split2(ka < in_dim ? q1[0] : 0.f, ka + 1 < in_dim ? q1[1] : 0.f, ah[1], al[1]);
                f16_split2(ka + 2 < in_dim ? q0[2] : 0.f, ka + 3 < in_dim ? q0[3] : 0.f, ah[2], al[2]);
                f16_split2(ka + 2 < in_dim ? q1[2] : 0.f, ka + 3 < in_dim ? q1[3] : 0.f, ah[3], al[3]);
            }
            const bool more = k0 + 16 < in_dim;
            mma_group<2>(c, cx, ah, al, b0);         if (more) load_bfrag<2>(b0, w + 8 * 32);
            mma_group<2>(c + 2, cx + 2, ah, al, b1); if (more) load_bfrag<2>(b1, w + 10 * 32);
            mma_group<2>(c + 4, cx + 4, ah, al, b2); if (more) load_bfrag<2>(b2, w + 12 * 32);
            mma_group<2>(c + 6, cx + 6, ah, al, b3); if (more) load_bfrag<2>(b3, w + 14 * 32);
        }
        hidden_to_afrag(c, cx, hh, hl);
    }
    {   // ---- layer 2: K = 64 from registers ----
        float c[8][4], cx[8][4];
        init_acc<8>(c, cx, b2, t);
        const uint4* w = W2 + lane;
        uint4 ba[2], bb[2];
        load_bfrag<2>(ba, w);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
#pragma unroll
            for (int n = 0; n < 8; n += 4) {
                load_bfrag<2>(bb, w + (8 * j + n + 2) * 32);
                mma_group<2>(c + n, cx + n, hh[j], hl[j], ba);
                if (8 * j + n + 4 < 32) load_bfrag<2>(ba, w + (8 * j + n + 4) * 32);
                mma_group<2>(c + n + 2, cx + n + 2, hh[j], hl[j], bb);
            }
        }
        hidden_to_afrag(c, cx, hh, hl);
    }
    // ---- layer 3: K = 64 from registers, one n-tile of 8 outputs at a time ----
    const int ost = 8 * nt3;
    for (int n = 0; n < nt3; ++n) {
        float c[1][4], cx[1][4];
        init_acc<1>(c, cx, b3 + 8 * n, t);
        uint4 b[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) b[j] = __ldg(W3 + ((size_t)j * nt3 + n) * 32 + lane);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            mma_f16(cx[0], hl[j], b[j].x, b[j].y); mma_f16(c[0], hh[j], b[j].x, b[j].y); mma_f16(cx[0], hh[j], b[j].z, b[j].w);
        }
        float* o0 = out_s + (size_t)g * ost + 8 * n + 2 * t;
        if (g < n_rows) *reinterpret_cast<float2*>(o0) = make_float2(fmaf(cx[0][0], kLoInv, c[0][0]), fmaf(cx[0][1], kLoInv, c[0][1]));
        if (g + 8 < n_rows) *reinterpret_cast<float2*>(o0 + 8 * ost) = make_float2(fmaf(cx[0][2], kLoInv, c[0][2]), fmaf(cx[0][3], kLoInv, c[0][3]));
    }
}

// ---- general network (qs_rollout_mlp): any depth 1..4, hidden widths up to 256, tanh or ReLU ----------------------------------
// warp_net's arithmetic, layer by layer in chunks of 64 output columns (one 8 n-tile register tile each).  A hidden layer's split
// activations do not fit the registers, so they go through shared memory in A-fragment order: [k-step][hi, lo'][lane] x uint4.  A
// lane writes exactly the words it reads back as the next layer's A fragment (the accumulator of n-tiles 2j, 2j+1 IS k-step j's A
// fragment), so the staging needs no barrier; two buffers per warp alternate between layers, because every output chunk reads
// all k-steps of the layer's input.  Per accumulator the mma order is warp_net's (k-steps ascending; lo'.hi, hi.hi, hi.lo'), so a
// [64, 64] tanh network gives warp_net's bits.
__device__ __forceinline__ float mlp_act(float x, bool relu) { return relu ? fmaxf(x, 0.f) : tanh_fast(x); }

// one 64-unit chunk: accumulators -> activation -> split -> its 4 k-steps of A fragments at `st` (the chunk's first k-step)
__device__ __forceinline__ void chunk_to_stage(const float (&c)[8][4], const float (&cx)[8][4], bool relu, uint4* st, int lane) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        unsigned hh[4], hl[4];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int n = 2 * j + h;
            const float v0 = mlp_act(fmaf(cx[n][0], kLoInv, c[n][0]), relu), v1 = mlp_act(fmaf(cx[n][1], kLoInv, c[n][1]), relu);
            const float v2 = mlp_act(fmaf(cx[n][2], kLoInv, c[n][2]), relu), v3 = mlp_act(fmaf(cx[n][3], kLoInv, c[n][3]), relu);
            f16_split2(v0, v1, hh[2 * h], hl[2 * h]);
            f16_split2(v2, v3, hh[2 * h + 1], hl[2 * h + 1]);
        }
        st[(2 * j) * 32 + lane] = make_uint4(hh[0], hh[1], hh[2], hh[3]);
        st[(2 * j + 1) * 32 + lane] = make_uint4(hl[0], hl[1], hl[2], hl[3]);
    }
}

// One network of a QsMlpNet for 16 aviaries, by one warp (x_s, n_rows, out_s as warp_net; out_s rows have stride 8 out_tiles).
// stage: the warp's two buffers of stage_ks k-steps each.
__device__ __forceinline__ void warp_mlp(const float* x_s, int in_dim, const QsMlpNet& net, bool relu, float* out_s, int n_rows, int lane,
                                         uint4* stage, int stage_ks) {
    const int g = lane >> 2, t = lane & 3;
    {   // ---- layer 0: K = in_dim from the observation window, chunk by chunk ----
        const int last = n_rows - 1;
        const float* p0 = x_s + (size_t)(g < last ? g : last) * in_dim + 4 * t;
        const float* p1 = x_s + (size_t)(g + 8 < last ? g + 8 : last) * in_dim + 4 * t;
        const bool vec4 = ((reinterpret_cast<size_t>(x_s) & 15) == 0) && ((in_dim & 3) == 0);
        const int ntot = net.width[0] >> 3, kstride = ntot * 32;
#pragma unroll 1
        for (int ch = 0; ch < (net.width[0] >> 6); ++ch) {
            float c[8][4], cx[8][4];
            init_acc<8>(c, cx, net.b[0] + 64 * ch, t);
            const uint4* w = reinterpret_cast<const uint4*>(net.w[0]) + 8 * ch * 32 + lane;
            uint4 b0[2], b1[2], b2[2], b3[2];
            load_bfrag<2>(b0, w); load_bfrag<2>(b1, w + 2 * 32); load_bfrag<2>(b2, w + 4 * 32); load_bfrag<2>(b3, w + 6 * 32);
#pragma unroll 1
            for (int k0 = 0; k0 < in_dim; k0 += 16, w += kstride) {
                unsigned ah[4], al[4];
                if (vec4 && k0 + 16 <= in_dim) {
                    const float4 u = *reinterpret_cast<const float4*>(p0 + k0), v = *reinterpret_cast<const float4*>(p1 + k0);
                    f16_split2(u.x, u.y, ah[0], al[0]); f16_split2(v.x, v.y, ah[1], al[1]);
                    f16_split2(u.z, u.w, ah[2], al[2]); f16_split2(v.z, v.w, ah[3], al[3]);
                } else {
                    const int ka = k0 + 4 * t;
                    const float* q0 = p0 + k0; const float* q1 = p1 + k0;
                    f16_split2(ka < in_dim ? q0[0] : 0.f, ka + 1 < in_dim ? q0[1] : 0.f, ah[0], al[0]);
                    f16_split2(ka < in_dim ? q1[0] : 0.f, ka + 1 < in_dim ? q1[1] : 0.f, ah[1], al[1]);
                    f16_split2(ka + 2 < in_dim ? q0[2] : 0.f, ka + 3 < in_dim ? q0[3] : 0.f, ah[2], al[2]);
                    f16_split2(ka + 2 < in_dim ? q1[2] : 0.f, ka + 3 < in_dim ? q1[3] : 0.f, ah[3], al[3]);
                }
                const bool more = k0 + 16 < in_dim;
                mma_group<2>(c, cx, ah, al, b0);         if (more) load_bfrag<2>(b0, w + kstride);
                mma_group<2>(c + 2, cx + 2, ah, al, b1); if (more) load_bfrag<2>(b1, w + kstride + 2 * 32);
                mma_group<2>(c + 4, cx + 4, ah, al, b2); if (more) load_bfrag<2>(b2, w + kstride + 4 * 32);
                mma_group<2>(c + 6, cx + 6, ah, al, b3); if (more) load_bfrag<2>(b3, w + kstride + 6 * 32);
            }
            chunk_to_stage(c, cx, relu, stage + (size_t)(4 * ch) * 64, lane);
        }
    }
    // ---- hidden layers 1 .. depth-1: K = width[l-1] from one staging buffer into the other ----
#pragma unroll 1
    for (int l = 1; l < net.depth; ++l) {
        const uint4* in = stage + (size_t)((l - 1) & 1) * stage_ks * 64;
        uint4* outb = stage + (size_t)(l & 1) * stage_ks * 64;
        const int ks_in = net.width[l - 1] >> 4, ntot = net.width[l] >> 3, kstride = ntot * 32;
#pragma unroll 1
        for (int ch = 0; ch < (net.width[l] >> 6); ++ch) {
            float c[8][4], cx[8][4];
            init_acc<8>(c, cx, net.b[l] + 64 * ch, t);
            const uint4* w = reinterpret_cast<const uint4*>(net.w[l]) + 8 * ch * 32 + lane;
            uint4 b0[2], b1[2], b2[2], b3[2];
            load_bfrag<2>(b0, w); load_bfrag<2>(b1, w + 2 * 32); load_bfrag<2>(b2, w + 4 * 32); load_bfrag<2>(b3, w + 6 * 32);
#pragma unroll 1
            for (int j = 0; j < ks_in; ++j, w += kstride) {
                const uint4 h = in[(2 * j) * 32 + lane], lo = in[(2 * j + 1) * 32 + lane];
                const unsigned ah[4] = {h.x, h.y, h.z, h.w}, al[4] = {lo.x, lo.y, lo.z, lo.w};
                const bool more = j + 1 < ks_in;
                mma_group<2>(c, cx, ah, al, b0);         if (more) load_bfrag<2>(b0, w + kstride);
                mma_group<2>(c + 2, cx + 2, ah, al, b1); if (more) load_bfrag<2>(b1, w + kstride + 2 * 32);
                mma_group<2>(c + 4, cx + 4, ah, al, b2); if (more) load_bfrag<2>(b2, w + kstride + 4 * 32);
                mma_group<2>(c + 6, cx + 6, ah, al, b3); if (more) load_bfrag<2>(b3, w + kstride + 6 * 32);
            }
            chunk_to_stage(c, cx, relu, outb + (size_t)(4 * ch) * 64, lane);
        }
    }
    // ---- output layer: K = width[depth-1] from staging, one n-tile of 8 outputs at a time, 4 k-steps per round ----
    const uint4* in = stage + (size_t)((net.depth - 1) & 1) * stage_ks * 64;
    const int ks_in = net.width[net.depth - 1] >> 4, nto = net.out_tiles, ost = 8 * nto;
    const uint4* W = reinterpret_cast<const uint4*>(net.w[net.depth]);
    for (int n = 0; n < nto; ++n) {
        float c[1][4], cx[1][4];
        init_acc<1>(c, cx, net.b[net.depth] + 8 * n, t);
#pragma unroll 1
        for (int j0 = 0; j0 < ks_in; j0 += 4) {
            uint4 b[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) b[j] = __ldg(W + ((size_t)(j0 + j) * nto + n) * 32 + lane);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint4 h = in[(2 * (j0 + j)) * 32 + lane], lo = in[(2 * (j0 + j) + 1) * 32 + lane];
                const unsigned ah[4] = {h.x, h.y, h.z, h.w}, al[4] = {lo.x, lo.y, lo.z, lo.w};
                mma_f16(cx[0], al, b[j].x, b[j].y); mma_f16(c[0], ah, b[j].x, b[j].y); mma_f16(cx[0], ah, b[j].z, b[j].w);
            }
        }
        float* o0 = out_s + (size_t)g * ost + 8 * n + 2 * t;
        if (g < n_rows) *reinterpret_cast<float2*>(o0) = make_float2(fmaf(cx[0][0], kLoInv, c[0][0]), fmaf(cx[0][1], kLoInv, c[0][1]));
        if (g + 8 < n_rows) *reinterpret_cast<float2*>(o0 + 8 * ost) = make_float2(fmaf(cx[0][2], kLoInv, c[0][2]), fmaf(cx[0][3], kLoInv, c[0][3]));
    }
}

// What a policy rollout hands over across policy_forward besides the drone: the embedded controller's state (PIDACT) and the
// previous tick's RPMs (drag).  Members a variant does not carry are neither written nor read.
struct ParkedCtl {
    qs::Drone d;
    qs::PidState pst;
    double rpm_prev[4];
};
__device__ __forceinline__ qs::Drone& parked_drone(qs::Drone* p) { return *p; }
__device__ __forceinline__ qs::Drone& parked_drone(ParkedCtl* p) { return p->d; }

__device__ __forceinline__ bool has_critic(const RolloutArgs& a) { return a.pol.vw1 != nullptr; }
__device__ __forceinline__ bool has_critic(const MlpRolloutArgs& a) { return a.mlp.critic.depth != 0; }

// The policy part of one tick for the whole CTA: actor (and critic) over the CTA's aviaries in tiles of 16; work item i = net x tile
// goes to warp i & 1.  Deliberately NOT inlined: inside the tick loop its ~120 live registers made the compiler spill the drone state
// in the middle of the physics substeps; as a call, the state is saved once per tick around it.  `parked` is not touched: the caller
// hands over the address of its drone state (Park = qs::Drone, or ParkedCtl with the controller state and previous RPMs) so that
// the state demonstrably lives in local memory across the call (one store + load per tick) instead of being spilled piecemeal
// inside the substep loop.  CRITIC_ONLY: the critic alone (on the terminal rows of a same-step autoreset, for final_values).
// Args: RolloutArgs runs warp_net on the classic network, MlpRolloutArgs warp_mlp on the general one.
template <bool CRITIC_ONLY, class Args, class Park>
__device__ __noinline__ void policy_forward(const Args& a, const float* base, float* mean_s, float* val_s, int n_av, int t, Park* parked) {
    constexpr bool MLP = std::is_same<Args, MlpRolloutArgs>::value;
    if (n_av < 0) parked_drone(parked).px = 0.0;             // never taken; keeps the hand-over opaque to the optimiser
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = t >> 5, lane = t & 31, ost = 8 * a.pol.nt3;
    uint4* stage = nullptr;                                  // the general network: the warp's staging buffers, its activation
    bool relu = false;
    if constexpr (MLP) {
        stage = reinterpret_cast<uint4*>(smem_raw + a.stage_off) + (size_t)warp * 2 * a.stage_ks * 64;
        relu = a.mlp.activation == QS_MLP_RELU;
    }
    const int tiles = (n_av + 15) >> 4, items = has_critic(a) ? 2 * tiles : tiles;
    for (int i = (CRITIC_ONLY ? tiles : 0) + warp; i < items; i += 2) {
        const bool critic = CRITIC_ONLY || i >= tiles;
        const int r0 = 16 * (critic ? i - tiles : i);
        const float* x0 = base + (size_t)r0 * a.pol.in_dim;
        if constexpr (MLP) {
            if (!critic) warp_mlp(x0, a.pol.in_dim, a.mlp.actor, relu, mean_s + (size_t)r0 * ost, n_av - r0, lane, stage, a.stage_ks);
            else warp_mlp(x0, a.pol.in_dim, a.mlp.critic, relu, val_s + (size_t)r0 * 8, n_av - r0, lane, stage, a.stage_ks);
        } else if (!critic) {
            warp_net(x0, a.pol.in_dim, reinterpret_cast<const uint4*>(a.pol.w1), reinterpret_cast<const uint4*>(a.pol.w2), reinterpret_cast<const uint4*>(a.pol.w3),
                     a.pol.b1, a.pol.b2, a.pol.b3, a.pol.nt3, mean_s + (size_t)r0 * ost, n_av - r0, lane);
        } else {
            warp_net(x0, a.pol.in_dim, reinterpret_cast<const uint4*>(a.pol.vw1), reinterpret_cast<const uint4*>(a.pol.vw2), reinterpret_cast<const uint4*>(a.pol.vw3),
                     a.pol.vb1, a.pol.vb2, a.pol.vb3, 1, val_s + (size_t)r0 * 8, n_av - r0, lane);
        }
    }
    __syncthreads();                                         // means / values of every aviary of the CTA are in shared memory
}

// policy_forward with the live state parked across the call: the drone, with PIDACT the controller state, with drag `rp` (the RPMs
// the next tick's drag reads)
template <int EFF, bool PIDACT, bool CRITIC_ONLY, class Args>
__device__ __forceinline__ void parked_policy_forward(const Args& a, const float* base, float* mean_s, float* val_s, int n_av, int t,
                                                      qs::Drone& d, qs::PidState& pst, double (&rp)[4]) {
    if constexpr (PIDACT || (EFF & QS_EFFECT_DRAG)) {
        ParkedCtl parked;
        parked.d = d;
        if constexpr (PIDACT) parked.pst = pst;
        if constexpr ((EFF & QS_EFFECT_DRAG) != 0) for (int j = 0; j < 4; ++j) parked.rpm_prev[j] = rp[j];
        policy_forward<CRITIC_ONLY>(a, base, mean_s, val_s, n_av, t, &parked);
        d = parked.d;
        if constexpr (PIDACT) pst = parked.pst;
        if constexpr ((EFF & QS_EFFECT_DRAG) != 0) for (int j = 0; j < 4; ++j) rp[j] = parked.rpm_prev[j];
    } else {
        qs::Drone parked = d;
        policy_forward<CRITIC_ONLY>(a, base, mean_s, val_s, n_av, t, &parked);
        d = parked;
    }
}

// the kinematic head of an observation row: pos3 rpy3 vel3 ang_v3 (BaseRLAviary.py:310-315)
__device__ __forceinline__ void store_head(float* row, const qs::Drone& d, const qs::Derived& o) {
    row[0] = (float)d.px; row[1] = (float)d.py; row[2] = (float)d.pz;
    row[3] = (float)o.roll; row[4] = (float)o.pitch; row[5] = (float)o.yaw;
    row[6] = (float)d.vx; row[7] = (float)d.vy; row[8] = (float)d.vz;
    row[9] = (float)o.ax; row[10] = (float)o.ay; row[11] = (float)o.az;
}

__device__ __forceinline__ unsigned long long splitmix64(unsigned long long x) {
    x += 0x9E3779B97F4A7C15ull;
    unsigned long long z = x;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ float u32_to_pm1(unsigned u) { return (float)(u >> 8) * (1.0f / 8388608.0f) - 1.0f; }   // [-1, 1)

// Fixed part of a POLICY CTA's dynamic shared memory: red_s [64][2] doubles, oob [64], done [64], and with in-CTA downwash the
// positions pos_s [64][3] doubles; the mbarrier sits in the last 16 bytes.  1280 bytes without downwash, 2816 with it.
__host__ __device__ constexpr size_t policy_smem_fixed(int eff) {
    return (eff & QS_EFFECT_DW) ? (size_t)(64 * 2 * 8 + 64 + 64 + 64 * 3 * 8 + 16 + 127) / 128 * 128 : (size_t)(64 * 2 * 8 + 64 + 64 + 16 + 112);
}
constexpr size_t kPolicyPosOffset = 64 * 2 * 8 + 64 + 64;       // pos_s of the downwash variants (8-byte aligned)
// resident CTAs per SM a POLICY variant is compiled for (__launch_bounds__) and its shared-memory carve-out is sized for: 7 give
// 128 registers; the in-CTA downwash substep loop (positions of the aviary's drones, barriers, all three effects) spills the drone
// state at 128, so those variants get 6 CTAs and 168 registers (DESIGN.md 4.1b)
__host__ __device__ constexpr int policy_ctas(int eff) { return (eff & QS_EFFECT_DW) ? 6 : 7; }
// the rest of a policy CTA's dynamic shared memory (the general network adds its staging): window, means, values, log-prob terms
inline size_t policy_smem_var(int tpb, int obs_dim, int T, int A, int D, int out_tiles) {
    const int n_av_max = 64 / D;
    return (size_t)tpb * obs_dim * 4 + (size_t)(T + 1) * A * 4 + 32 + (size_t)(n_av_max * 8 * out_tiles + n_av_max * 8 + 64) * 4 + 16;
}
constexpr size_t kPolicySmemLimit = 200 * 1024;      // what a policy CTA may use
// shared-memory carve-out of a policy kernel: just enough for `ctas` resident CTAs of `sm` bytes, so that the weights find the
// rest of the 256 KB as L1
template <class K>
void set_policy_carveout(K* kernel, int ctas, size_t sm) {
    const size_t need = (size_t)ctas * (sm + 1024);
    const int pct = (int)((need * 100 + 228 * 1024 - 1) / (228 * 1024));
    cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, pct > 100 ? 100 : pct);
}

// PHYS: the physical constants come from the aviary's row of QsState.phys, re-read (L1) every tick rather than held in 28
// registers for the whole rollout -- the POLICY variants have none to spare (128 registers, 7 CTAs per SM, DESIGN.md 4.1b).
// POLICY takes every EFF x PIDACT combination the envs produce (EFF = 0, GND, DRAG, DW, all three): the physics and the embedded
// controller are the action rollout's code, so a policy rollout gives the bits of the action rollout fed its clipped actions.
// MODE (RolloutMode) FIN: the terminal observations (io.final_obs) and with POLICY their critic values (io.final_values) are
// produced.  NEXT: NEXT_STEP autoreset -- an aviary whose latch is set at the start of a tick is only reset by it (its action is
// ignored, its history is not shifted); the latch is carried in a register from tick to tick.  Template values rather than
// run-time branches: the new code moved the registers and spills of every entry that does not need it.  NET (RolloutNet) picks
// the type of `a`, which stays the kernel's own __grid_constant__ parameter: a shared body taking `a` by reference moved the
// registers and spills of existing entries (DESIGN.md 4.1b).
template <int EFF, bool PIDACT, int NET, bool PHYS, int MODE>
__global__ void __launch_bounds__(NET != kNetNone ? 64 : kMaxTPB, NET != kNetNone ? policy_ctas(EFF) : 4)
rollout_kernel(const __grid_constant__ typename RolloutArgsOf<NET>::type a) {
    constexpr bool POLICY = NET != kNetNone;
    constexpr bool FIN = MODE == kRolloutFin, NEXT = MODE == kRolloutNext;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const QsParams& P = a.P;
    const int tpb = a.tpb, D = a.D, A = a.A, od = a.obs_dim, T = a.io.T;
    const int t = threadIdx.x;
    const long long N = a.N, E = a.n_envs;
    const long long c0 = (long long)blockIdx.x * tpb;
    const long long i = c0 + t;
    const bool live = (t < tpb) && (i < N);
    const int rows = (int)((N - c0) < tpb ? (N - c0) : tpb);
    double* red_s = reinterpret_cast<double*>(smem_raw);                               // [tpb][2]
    const int cap = a.cap;
    // POLICY (CTA of 64 drones): a compact fixed part -- red_s [64][2] doubles, oob [64], done [64], with downwash pos_s [64][3]
    // doubles, mbarrier -- so that 7 CTAs per SM (924 on the H100's 132 SMs) fit into shared memory next to the window and the
    // MLP scratch
    const size_t fixed = POLICY ? policy_smem_fixed(EFF) : smem_fixed(cap);           // 1280 for POLICY, 2816 with downwash
    double* pos_s = (POLICY && (EFF & QS_EFFECT_DW)) ? reinterpret_cast<double*>(smem_raw + kPolicyPosOffset)
                                                     : red_s + (size_t)cap * 2;         // [tpb][3] (in-CTA downwash only)
    unsigned char* oob_s = POLICY ? reinterpret_cast<unsigned char*>(red_s + 128) : reinterpret_cast<unsigned char*>(pos_s + (size_t)cap * 3);
    unsigned char* done_s = oob_s + (POLICY ? 64 : cap);
    unsigned long long* bar_s = reinterpret_cast<unsigned long long*>(smem_raw + fixed - 16);
    float* stage_s = reinterpret_cast<float*>(smem_raw + fixed);                       // [tpb*od + (T+1)*A] sliding window
    // POLICY scratch after the window: padded action means [n_av][8 nt3]; padded values [n_av][8]; log-prob terms [64]
    float* pol_s = stage_s + ((((size_t)tpb * od + (size_t)(T + 1) * A) + 3) & ~(size_t)3);
    float* mean_s = pol_s;
    float* val_s = mean_s + (size_t)(64 / (D < 1 ? 1 : D)) * 8 * a.pol.nt3;
    float* lp_s = val_s + (size_t)(64 / (D < 1 ? 1 : D)) * 8;

    const long long e = live ? i / D : 0;
    const int le = t / D;
    const int dslot = (int)(i - e * D);
    const long long tbl = a.st.tables_per_env ? i : dslot;

    if (a.stage_mode == 1) {
        if (t == 0) mbar_init(bar_s, 1);
        __syncthreads();
    }
    qs::Drone d;
    qs::PidState pst = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    double rpm_prev[4] = {0, 0, 0, 0};
    int sc = 0;
    bool pend = false;                         // NEXT: this tick only resets my aviary (its pending_reset latch)
    if (live) {
        load_drone(a.st.planes, N, i, d);
        if ((EFF & QS_EFFECT_DRAG) && a.st.last_rpm) load_rpm(a.st.last_rpm, i, rpm_prev);
        if (PIDACT) load_pid(a.st.pid, N, i, pst);
        sc = a.st.step_counter[e];
        if constexpr (NEXT) pend = a.st.pending_reset[e] != 0;
    }
    if (a.stage_mode == 1) {
        if (t == 0) tma_bulk_g2s(stage_s, a.io.obs_init + c0 * od, (unsigned)(rows * od * 4), bar_s);
        mbar_wait(bar_s, 0);
    } else {
        const float* src = a.io.obs_init + c0 * od;
        for (int j = t; j < rows * od; j += blockDim.x) cp_async4(stage_s + j, src + j);
        cp_async_commit_wait_all();
    }
    __syncthreads();

    float* base = stage_s;                     // window start: rows of the observation BEFORE the current tick
    double rpm[4] = {0, 0, 0, 0};
    for (int k = 0; k < T; ++k) {
        // ---- this tick's action: caller-provided or generated on the device --------------------------------------
        float act[4] = {0.f, 0.f, 0.f, 0.f};
        float raw_act[4] = {0.f, 0.f, 0.f, 0.f};
        if (POLICY) {
            // the aviaries of this CTA: rows [le D, le D + D) of the window = one flattened observation of in_dim floats each
            const int n_av = rows / D;
            const int ost = 8 * a.pol.nt3;                        // padded width of the output rows in mean_s
            // the controller state and the previous RPMs are live across the call too: handed over the same way
            parked_policy_forward<EFF, PIDACT, false>(a, base, mean_s, val_s, n_av, t, d, pst, rpm_prev);
            float lp = 0.f;
            if (live) {
                const int od_out = a.pol.out_dim;
                for (int j = 0; j < A; ++j) {
                    const int idx = dslot * A + j;
                    const float ls = __ldg(a.pol.log_std + idx);
                    const float eps = a.pol.noise ? __ldg(a.pol.noise + ((long long)k * E + e) * od_out + idx) : 0.f;
                    const float r = fmaf(expf(ls), eps, mean_s[le * ost + idx]);
                    raw_act[j] = r;
                    act[j] = fminf(fmaxf(r, -1.f), 1.f);                             // the env clips to its action space
                    lp += -0.5f * eps * eps - ls - 0.91893853320467274f;            // log N(r; mean, std)
                }
                lp_s[t] = lp;
            }
            __syncthreads();
            if (live && dslot == 0) {
                float s_lp = 0.f;
                for (int q = 0; q < D; ++q) s_lp += lp_s[t + q];
                const long long oe = (long long)k * E + e;
                if (a.pol.logprob) a.pol.logprob[oe] = s_lp;
                if (a.pol.values && a.pol.vw1) a.pol.values[oe] = val_s[le * 8];
            }
        }
        if (live) {
            if (POLICY) {
                // (act / raw_act set above)
            } else if (a.io.actions) {
                const float* ap = a.io.actions + ((long long)k * N + i) * A;
                if (A == 4) { const float4 v = __ldg(reinterpret_cast<const float4*>(ap)); act[0] = v.x; act[1] = v.y; act[2] = v.z; act[3] = v.w; }
                else if (A == 3) { act[0] = __ldg(ap); act[1] = __ldg(ap + 1); act[2] = __ldg(ap + 2); }
                else act[0] = __ldg(ap);
            } else {
                const unsigned long long key = a.io.seed + 2ull * (unsigned long long)((a.io.tick0 + k) * N + i);
                const unsigned long long r0 = splitmix64(key), r1 = splitmix64(key + 1);
                act[0] = u32_to_pm1((unsigned)r0); act[1] = u32_to_pm1((unsigned)(r0 >> 32));
                act[2] = u32_to_pm1((unsigned)r1); act[3] = u32_to_pm1((unsigned)(r1 >> 32));
                if (A < 4) act[3] = 0.f;
                if (A < 3) { act[1] = 0.f; act[2] = 0.f; }
            }
            float* tail = base + (size_t)t * od + od;        // new action -> the A slots after my row (dead head of the next row)
            if (NEXT && pend) {
                // reset tick: my row enters the next window UNSHIFTED (or with CLEARS_HISTORY empty), no action appended:
                // new_row[q] = old_row[q] for q >= 12, descending because new_row = old_row + A.  The window has been read (the
                // policy pass ends with a barrier) and store_head has not yet overwritten [A, A+12) of the old row; the copy's
                // spill past my row reaches only the next row's dead head [0, A), where the tail would have gone.
                float* row = base + (size_t)t * od;
                const bool clear = a.flags & QS_FLAG_AUTORESET_CLEARS_HISTORY;
                for (int q = od - 1; q >= 12; --q) row[q + A] = clear ? 0.f : row[q];
            } else if (A == 4) *reinterpret_cast<float4*>(tail) = make_float4(act[0], act[1], act[2], act[3]);
            else if (A == 3) { tail[0] = act[0]; tail[1] = act[1]; tail[2] = act[2]; }
            else tail[0] = act[0];
            if (a.io.actions_out) {
                float* ao = a.io.actions_out + ((long long)k * N + i) * A;
                const float* av = POLICY ? raw_act : act;                        // PPO stores the unclipped sample
                if (A == 4) *reinterpret_cast<float4*>(ao) = make_float4(av[0], av[1], av[2], av[3]);
                else if (A == 3) { ao[0] = av[0]; ao[1] = av[1]; ao[2] = av[2]; }
                else ao[0] = av[0];
            }
        }
        // ---- physics ---------------------------------------------------------------------------------------------
        double R_last[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
        qs::PhysRow ph;
        if (live && !pend) {                                   // (a reset tick decodes nothing and runs no physics)
            double cur_yaw = 0.0;
            if (a.act_type == QS_ACT_VEL) { double r_, p_; qs::quat_to_euler<false>(d.qx, d.qy, d.qz, d.qw, r_, p_, cur_yaw); }
            if constexpr (PHYS) {
                qs::decode_action_k<PIDACT>(P, load_phys_rpm(a.st.phys, e), a.act_type, act, d, cur_yaw, pst, rpm);
                ph = load_phys(a.st.phys, e);                 // after the decode (and its PID controller)
            } else {
                qs::decode_action<PIDACT>(P, a.act_type, act, d, cur_yaw, pst, rpm);
            }
        }
        if (EFF & QS_EFFECT_DW) {
            for (int s = 0; s < a.substeps; ++s) {
                if (live) { pos_s[3 * t] = d.px; pos_s[3 * t + 1] = d.py; pos_s[3 * t + 2] = d.pz; }
                __syncthreads();
                if (live && !pend) {                           // all drones of an aviary are pending together
                    const double fz = qs::downwash_fz(P, pos_s, le * D, D, d.px, d.py, d.pz);
                    if constexpr (POLICY) {
                        // the same values selected element by element: a pointer chosen at run time between the two arrays
                        // puts both in local memory, inside the substep loop (the policy variants have no registers to spare);
                        // for the same reason the row of constants is re-read (L1) every substep, not held across the barriers
                        double rp[4];
                        for (int j = 0; j < 4; ++j) rp[j] = s == 0 ? rpm_prev[j] : rpm[j];
                        if constexpr (PHYS) qs::dyn_tick_k<EFF>(P, load_phys(a.st.phys, e), d, rpm, rp, fz, 1, R_last);
                        else qs::dyn_tick<EFF>(P, d, rpm, rp, fz, 1, R_last);
                    } else if constexpr (PHYS) {
                        qs::dyn_tick_k<EFF>(P, ph, d, rpm, s == 0 ? rpm_prev : rpm, fz, 1, R_last);
                    } else {
                        qs::dyn_tick<EFF>(P, d, rpm, s == 0 ? rpm_prev : rpm, fz, 1, R_last);
                    }
                }
                __syncthreads();
            }
        } else if (live && !pend) {
            if constexpr (PHYS) qs::dyn_tick_k<EFF>(P, ph, d, rpm, rpm_prev, 0.0, a.substeps, R_last);
            else qs::dyn_tick<EFF>(P, d, rpm, rpm_prev, 0.0, a.substeps, R_last);
        }
        qs::Derived o;
        if constexpr (NEXT) {
            if (live && pend) {                                // the reset of qs_step's NEXT_STEP tick: init pose, rates and ang_v zero
                init_drone(a.st, tbl, d);
                if (a.flags & QS_FLAG_AUTORESET_CLEARS_PID) pst = {0, 0, 0, 0, 0, 0, 0, 0, 0};
                rpm[0] = rpm[1] = rpm[2] = rpm[3] = 0.0;       // last_clipped_action = 0 (the next tick's drag reads it)
                sc = -a.substeps;                              // -> 0 after the increment below
            }
        }
        // a reset drone's head carries float64 angles in every mode (qs_reset_heads)
        if (live) { if ((a.flags & QS_FLAG_RPY_F32) && !(NEXT && pend)) qs::derive<true>(d, R_last, o); else qs::derive<false>(d, R_last, o); }
        if (NEXT && live && pend) { o.ax = o.ay = o.az = 0.0; }
        // ---- task ------------------------------------------------------------------------------------------------
        bool env_done = false;
        if (a.task == QS_TASK_HOVER) {
            if (live) {
                const D4 tp = ld256_nc(a.st.target_pos, tbl);
                const qs::TaskTerms tt = qs::hover_terms(P, d, o, tp.x, tp.y, tp.z);
                red_s[2 * t] = tt.reward; red_s[2 * t + 1] = tt.dist; oob_s[t] = tt.out_of_bounds ? 1 : 0;
            }
            __syncthreads();
            if (live && dslot == 0) {
                double rew = 0.0, dist = 0.0; bool oob = false;
                for (int q = 0; q < D; ++q) { rew += red_s[2 * (t + q)]; dist += red_s[2 * (t + q) + 1]; oob |= oob_s[t + q] != 0; }
                bool term = dist < P.term_dist;
                bool trunc = oob || ((double)sc / P.pyb_freq > P.episode_len_sec);
                if (NEXT && pend) { rew = 0.0; term = false; trunc = false; }
                const long long oe = (long long)k * E + e;
                a.io.reward[oe] = (float)rew; a.io.terminated[oe] = term ? 1 : 0; a.io.truncated[oe] = trunc ? 1 : 0;
                if (a.io.done) a.io.done[oe] = (term || trunc) ? 1 : 0;
                done_s[le] = (term || trunc) ? 1 : 0;
            }
            __syncthreads();
            if (live) env_done = done_s[le] != 0;
        } else if (live && dslot == 0) {
            const long long oe = (long long)k * E + e;
            a.io.reward[oe] = -1.0f; a.io.terminated[oe] = 0; a.io.truncated[oe] = 0;
            if (a.io.done) a.io.done[oe] = 0;
        }
        // ---- autoreset, head, bookkeeping ----------------------------------------------------------------------------
        if constexpr (FIN) {
            const bool fin = live && (a.flags & QS_FLAG_AUTORESET_SAME_STEP) && env_done;
            if (fin) {
                // the terminal observation in my row of the next window: the head of the state before the reset, the history before
                // CLEARS_HISTORY zeroes it -- the row qs_step writes to final_obs (rare path: strided stores are fine)
                float* row = base + A + (size_t)t * od;
                store_head(row, d, o);
                if (a.io.final_obs) {
                    float* f = a.io.final_obs + ((long long)k * N + i) * od;
                    for (int q = 0; q < od; ++q) f[q] = row[q];
                }
            }
            if constexpr (POLICY) {
                // the critic on the terminal rows, which exist only between the task and the reset: one pass of the critic alone,
                // on the ticks where an aviary of this CTA finished (CTA-uniform branch); the other aviaries' rows are evaluated
                // too and dropped.  The pass ends with a barrier, so the reset below overwrites rows nobody reads any more.
                if (a.io.final_values && __syncthreads_or(fin)) {
                    parked_policy_forward<EFF, PIDACT, true>(a, base + A, mean_s, val_s, rows / D, t, d, pst, rpm);
                    if (fin && dslot == 0) a.io.final_values[(long long)k * E + e] = val_s[le * 8];
                }
            }
        }
        if (live) {
            float* row = base + A + (size_t)t * od;              // my row in the NEXT window
            if ((a.flags & QS_FLAG_AUTORESET_SAME_STEP) && env_done) {
                if (a.flags & QS_FLAG_AUTORESET_CLEARS_HISTORY) for (int q = 12; q < od; ++q) row[q] = 0.f;
                if (a.flags & QS_FLAG_AUTORESET_CLEARS_PID) pst = {0, 0, 0, 0, 0, 0, 0, 0, 0};
                init_drone(a.st, tbl, d);
                const double Rr[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
                qs::derive<false>(d, Rr, o);                   // float64 angles, as qs_reset_heads
                rpm[0] = rpm[1] = rpm[2] = rpm[3] = 0.0;
                sc = -a.substeps;
            }
            store_head(row, d, o);
            sc += a.substeps;
            if (k < T - 1) round_to_planes(d);                // (the final store_drone applies the same rounding once)
            rpm_prev[0] = rpm[0]; rpm_prev[1] = rpm[1]; rpm_prev[2] = rpm[2]; rpm_prev[3] = rpm[3];
        }
        if constexpr (NEXT) pend = env_done;                   // the latch of the next tick (false on a reset tick)
        __syncthreads();
        // ---- stream the CTA's rows out: obs[k][c0 .. c0+rows) = window shifted by one action ----------------------------
        base += A;
        {
            float* outp = a.io.obs + ((long long)k * N + c0) * od;
            float* lastp = (k == T - 1 && a.io.obs_last) ? a.io.obs_last + c0 * od : nullptr;
            if (A == 4 && a.stage_mode == 1) {
                // TMA bulk store of the window (see step_kernel); the window is rewritten next tick, so wait until the
                // copy engine has read it
                if (t == 0) {
                    const unsigned bytes = (unsigned)(rows * od * 4);
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(outp), "r"(smem_u32(base)), "r"(bytes) : "memory");
                    if (lastp) asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(lastp), "r"(smem_u32(base)), "r"(bytes) : "memory");
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                }
            } else if (A == 4) {
                const float4* src = reinterpret_cast<const float4*>(base);
                float4* out = reinterpret_cast<float4*>(outp);
                float4* last = reinterpret_cast<float4*>(lastp);
                const int n4 = rows * (od >> 2), nt = blockDim.x;
                int j = t;
                for (; j + 5 * nt < n4; j += 6 * nt) {
                    const float4 v0 = src[j], v1 = src[j + nt], v2 = src[j + 2 * nt], v3 = src[j + 3 * nt], v4 = src[j + 4 * nt], v5 = src[j + 5 * nt];
                    out[j] = v0; out[j + nt] = v1; out[j + 2 * nt] = v2; out[j + 3 * nt] = v3; out[j + 4 * nt] = v4; out[j + 5 * nt] = v5;
                    if (last) { last[j] = v0; last[j + nt] = v1; last[j + 2 * nt] = v2; last[j + 3 * nt] = v3; last[j + 4 * nt] = v4; last[j + 5 * nt] = v5; }
                }
                for (; j < n4; j += nt) { const float4 v = src[j]; out[j] = v; if (last) last[j] = v; }
            } else {
                for (int j = t; j < rows * od; j += blockDim.x) { const float v = base[j]; outp[j] = v; if (lastp) lastp[j] = v; }
            }
        }
        __syncthreads();
    }
    if (live) {
        store_drone(a.st, N, i, d);
        if (a.st.last_rpm) st256(a.st.last_rpm, i, rpm[0], rpm[1], rpm[2], rpm[3]);
        if (PIDACT) store_pid(a.st.pid, N, i, pst);
        if (dslot == 0) a.st.step_counter[e] = sc;
        if (NEXT && dslot == 0) a.st.pending_reset[e] = pend ? 1 : 0;
    }
}

// Launches the policy rollout with network NET for the effect set and action type of `a`, 64 threads per CTA (two warps: 64
// drones, 32 hidden units each in the MLP); `sm`: the CTA's dynamic shared memory.  check_policy_config has rejected every effect
// set outside PolicyEffects.
template <int NET, bool PHYS, int MODE>
int launch_policy(const typename RolloutArgsOf<NET>::type& a, size_t sm, bool pid_act, cudaStream_t s) {
    const int blocks = (int)((a.N + a.tpb - 1) / a.tpb);
    with_int(PolicyEffects{}, (int)(a.effects & 7u), [&](auto EFF) {
        with_bool(pid_act, [&](auto PIDACT) {
            auto* k = rollout_kernel<decltype(EFF)::value, decltype(PIDACT)::value, NET, PHYS, MODE>;
            if (sm > 48 * 1024) cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
            // the resident CTAs the carve-out is sized for: the register limit, and for the general network at most as many as
            // its staging leaves room for
            int ctas = policy_ctas(EFF);
            if (NET == kNetMlp) {
                const int fit = (int)((228 * 1024) / (sm + 1024));
                ctas = fit < 1 ? 1 : fit < ctas ? fit : ctas;
            }
            set_policy_carveout(k, ctas, sm);
            k<<<blocks, 64, sm, s>>>(a);
        });
    });
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, NET == kNetMlp ? "qs_rollout_mlp launch" : "qs_rollout (policy) launch");
}

// qs_rollout: validates the classic policy (if any) and launches the rollout kernel family of `a` (PHYS: with the per-aviary
// table; MODE: see rollout_kernel)
template <bool PHYS, int MODE>
int launch_rollout(RolloutArgs& a, const QsRolloutIO* io, bool pid_act, void* stream) {
    const int eff = (int)(a.effects & 7u);
    cudaStream_t s = (cudaStream_t)stream;
    if (io->policy) {
        if (int rc = check_classic_policy(a, io)) return rc;
        a.pol = *io->policy;
        const size_t sm = policy_smem_fixed(eff) + policy_smem_var(a.tpb, a.obs_dim, io->T, a.A, a.D, a.pol.nt3);
        if (sm > kPolicySmemLimit) return fail(QS_ERR_UNSUPPORTED, "qs_rollout: policy + window exceed shared memory");
        return launch_policy<kNetClassic, PHYS, MODE>(a, sm, pid_act, s);
    }
    const int blocks = (int)((a.N + a.tpb - 1) / a.tpb);
    const int threads = ((a.tpb + 31) / 32) * 32;
    const size_t sm = smem_fixed(a.cap) + (size_t)a.tpb * a.obs_dim * 4 + (size_t)(io->T + 1) * a.A * 4 + 32;
    with_int(AllEffects{}, eff, [&](auto EFF) {
        with_bool(pid_act, [&](auto PIDACT) {
            auto* k = rollout_kernel<decltype(EFF)::value, decltype(PIDACT)::value, kNetNone, PHYS, MODE>;
            if (sm > 48 * 1024) cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kStepSmemFixed + kStageLimit + 32));
            k<<<blocks, threads, sm, s>>>(a);
        });
    });
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, "qs_rollout launch");
}

}  // namespace
}  // namespace qsi
