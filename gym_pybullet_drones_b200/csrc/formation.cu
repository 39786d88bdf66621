// formation.cu -- pairwise downwash for large aviaries / sharded formations and the neighbourhood query (DESIGN.md 4.3).
#include "qs_common.cuh"

using namespace qsi;

namespace {

// ---------------------------------------------------------------------------------------------------------
// Pairwise downwash for large aviaries: tiled all-pairs with exact bounding-box culling.  A CTA owns 128 drones
// ("rows") of ONE aviary and runs 1024 threads: thread (slice s, row n) evaluates the tile entries k = s (mod 8), so a
// 16 384-drone formation fills 128 SMs with 32 warps each instead of 64 SMs with 8.  The sources stream through shared
// memory in tiles of 1024 = 32 chunks of 32 (next tile prefetched into registers); every chunk carries its bounding box (warp redux on order-preserving
// integer keys), every warp knows the box of its 32 rows, and a warp skips a chunk when NO pair of the two boxes can
// contribute: all dz <= 0, or every dxy^2 >= 100 (BaseAviary.py:800), or every pair takes dw_pair's underflow early-out
// (dxy^2 > 220 beta_max^2: skipping changes no bit of the result).  Index-coherent
// formations (grids, Morton order) therefore cost O(N k) instead of O(N^2).  The pair term is float32 (predicate
// first, expf only for pairs in range), partial sums are float64 and are combined in a fixed order (deterministic).
// (qs_downwash: no workspace.  qs_downwash_boxed / qs_downwash_rows below use a precomputed box table instead of tiles.)
// ---------------------------------------------------------------------------------------------------------
struct DwArgs {
    float prop_radius, dw1, dw2, dw3;
    const float* rows;
    float* fz;
    int D, tiles_per_env, cull;
};

constexpr int kDwDrones = 128, kDwSlices = 8, kDwTile = 1024, kDwChunks = kDwTile / 32;
constexpr long long kDwSpinLimit = 4000000000LL;   // ~2 s of SM clock

// One pair of BaseAviary._downwash (BaseAviary.py:798-806) in float32: alpha exp(-.5 (dxy/beta)^2), 0 when the pair fails
// the reference's predicate (dz > 0, dxy < 10) or when the Gaussian is below float32 range anyway (dxy^2 > 220 beta^2:
// exp2(-158) flushes to 0, so the early-out changes no bit).  Reciprocals and exp2 are the SFU approximations (1-2 ulp):
// the kernel is SFU/ALU bound, and the oracle tolerance (1e-5) is three orders above that.
__device__ __forceinline__ float dw_pair(float prop_radius, float dw1, float dw2, float dw3, float dz, float dxy2) {
    const float beta = dw2 * dz + dw3;
    const float b2 = beta * beta;
    if (!(dz > 0.f && dxy2 < 100.f) || dxy2 > 220.f * b2) return 0.f;
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(dz * b2));                  // one SFU reciprocal for 1/dz and 1/beta^2
    const float rr = (0.25f * prop_radius) * (b2 * r);
    const float u2 = dxy2 * (dz * r);
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-0.72134752f * u2));      // exp(-u2/2) = 2^(-u2 log2(e)/2)
    return dw1 * (rr * rr) * e;
}

__global__ void __launch_bounds__(kDwDrones * kDwSlices) downwash_kernel(const __grid_constant__ DwArgs a) {
    __shared__ float4 tile[kDwTile];
    __shared__ float cbox[kDwChunks][6];                  // xmin xmax ymin ymax zmin zmax per chunk
    __shared__ double part[kDwSlices][kDwDrones];
    constexpr float BIG = 3e30f;
    const int env = blockIdx.x / a.tiles_per_env;
    const int tb = blockIdx.x - env * a.tiles_per_env;
    const long long base = (long long)env * a.D;
    const int ln = threadIdx.x % kDwDrones, sl = threadIdx.x / kDwDrones;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int n = tb * kDwDrones + ln;                    // my row inside the aviary
    const bool live = n < a.D;
    float4 me = make_float4(0.f, 0.f, BIG, 0.f);
    if (live) me = ldg4(a.rows, base + n);
    // box of this warp's 32 rows (warp-uniform)
    const float rx0 = warp_min(live ? me.x : BIG), rx1 = warp_max(live ? me.x : -BIG);
    const float ry0 = warp_min(live ? me.y : BIG), ry1 = warp_max(live ? me.y : -BIG);
    const float rz0 = warp_min(live ? me.z : BIG), rz1 = warp_max(live ? me.z : -BIG);
    const float* src = a.rows + base * 4;
    const int n_src = a.D;
    double acc = 0.0;
    const float4 dead = make_float4(0.f, 0.f, -BIG, 0.f);
    auto load_src = [&](int j) { return j < n_src ? ldg4(src, j) : dead; };
    float4 nxt = load_src(threadIdx.x);
    for (int j0 = 0; j0 < n_src; j0 += kDwTile) {
        {
            const float4 o = nxt;
            const bool ok = j0 + (int)threadIdx.x < n_src;
            tile[threadIdx.x] = o;
            const float x0 = warp_min(ok ? o.x : BIG), x1 = warp_max(ok ? o.x : -BIG);
            const float y0 = warp_min(ok ? o.y : BIG), y1 = warp_max(ok ? o.y : -BIG);
            const float z0 = warp_min(ok ? o.z : BIG), z1 = warp_max(ok ? o.z : -BIG);
            if (lane == 0) { float* c = cbox[warp]; c[0] = x0; c[1] = x1; c[2] = y0; c[3] = y1; c[4] = z0; c[5] = z1; }
        }
        __syncthreads();
        if (j0 + kDwTile < n_src) nxt = load_src(j0 + kDwTile + threadIdx.x);        // in flight during the evaluation
        bool act;
        {
            const float* c = cbox[lane];
            const float dzhi = c[5] - rz0, dzlo = fmaxf(c[4] - rz1, 0.f);
            const float gx = fmaxf(fmaxf(c[0] - rx1, rx0 - c[1]), 0.f), gy = fmaxf(fmaxf(c[2] - ry1, ry0 - c[3]), 0.f);
            const float g2 = gx * gx + gy * gy;
            const float b0 = fabsf(a.dw2 * dzlo + a.dw3), b1 = fabsf(a.dw2 * dzhi + a.dw3);
            const float bm = fmaxf(b0, b1);
            act = (dzhi > 0.f) && !(g2 > 100.001f) && !(g2 > 220.f * bm * bm);
            if (!a.cull) act = true;
        }
        unsigned m = __ballot_sync(0xffffffffu, act);
        float part_f = 0.f;
        while (m) {
            const int c = __ffs(m) - 1;
            m &= m - 1;
#pragma unroll
            for (int q = 0; q < 32 / kDwSlices; ++q) {
                const float4 o = tile[c * 32 + sl + kDwSlices * q];
                const float dz = o.z - me.z;
                const float dx = o.x - me.x, dy = o.y - me.y;
                const float dxy2 = dx * dx + dy * dy;
                part_f -= dw_pair(a.prop_radius, a.dw1, a.dw2, a.dw3, dz, dxy2);
            }
        }
        acc += (double)part_f;
        __syncthreads();
    }
    part[sl][ln] = acc;
    __syncthreads();
    if (sl == 0 && live) {
        double t = 0.0;
#pragma unroll
        for (int k = 0; k < kDwSlices; ++k) t += part[k][ln];
        a.fz[base + n] = (float)t;
    }
}

// ---------------------------------------------------------------------------------------------------------
// Boxed downwash (formations): the sources carry a table of bounding boxes, one per chunk of 32 consecutive positions
// ({min x,y,z,-}{max x,y,z,-}).  A CTA = 32 rows x 8 slices (256 threads, no position tile in shared memory): per batch
// of 256 chunks each warp tests 32 boxes against the box of the 32 rows (same exact predicate as above), the eight
// ballot words go through shared memory, then every warp walks the active chunks in index order and evaluates its 4
// entries of each (uniform 16-byte loads).  Cost: O(N/32) box tests + the pairs that can contribute, per row group;
// the small CTAs (N/32 of them) keep every SM busy when a formation is split over several GPUs.
// ---------------------------------------------------------------------------------------------------------
struct DwbArgs {
    float prop_radius, dw1, dw2, dw3;
    const float* rows;
    float* fz;
    const float* src;          // nullptr: sources of an aviary are its own rows
    const float* boxes;        // [chunks][8], per aviary when src == nullptr
    int n_src, D, groups_per_env, chunks, cull;
    const unsigned* ready;
    unsigned seq;
    int world;
    unsigned* err;
};

__global__ void __launch_bounds__(256, 4) downwash_boxed_kernel(const __grid_constant__ DwbArgs a) {
    __shared__ unsigned masks[8];
    __shared__ double part[8][32];
    constexpr float BIG = 3e30f;
    const int env = blockIdx.x / a.groups_per_env;
    const int g = blockIdx.x - env * a.groups_per_env;
    const long long base = (long long)env * a.D;
    const int lane = threadIdx.x & 31, sl = threadIdx.x >> 5;
    const int n = g * 32 + lane;
    const bool live = n < a.D;
    if (a.ready) {
        if ((int)threadIdx.x < a.world) {
            const long long t0 = clock64();
            while ((int)(ld_acquire_sys(a.ready + threadIdx.x) - a.seq) < 0) {
                if (clock64() - t0 > kDwSpinLimit) { if (a.err) atomicExch(a.err, 1u); break; }
            }
        }
        __syncthreads();
    }
    const bool shared_src = a.src != nullptr;            // exchange buffers are written by peers: L2-coherent loads
    float4 me = make_float4(0.f, 0.f, BIG, 0.f);
    // with flags this kernel may have been resident while the producer of `rows` (the dynamics kernel with the fused publish) was
    // still storing: read them past L1, after the flag wait above
    if (live) me = a.ready ? __ldcg(reinterpret_cast<const float4*>(a.rows) + base + n) : ldg4(a.rows, base + n);
    const float rx0 = warp_min(live ? me.x : BIG), rx1 = warp_max(live ? me.x : -BIG);
    const float ry0 = warp_min(live ? me.y : BIG), ry1 = warp_max(live ? me.y : -BIG);
    const float rz0 = warp_min(live ? me.z : BIG), rz1 = warp_max(live ? me.z : -BIG);
    const float4* src = reinterpret_cast<const float4*>(shared_src ? a.src : a.rows + base * 4);
    const float4* boxes = reinterpret_cast<const float4*>(a.boxes) + (shared_src ? 0 : (long long)env * a.chunks * 2);
    const int n_src = shared_src ? a.n_src : a.D;
    const float4 dead = make_float4(0.f, 0.f, -BIG, 0.f);
    double acc = 0.0;
    for (int cb = 0; cb < a.chunks; cb += 256) {
        {
            const int c = cb + sl * 32 + lane;
            bool act = false;
            if (c < a.chunks) {
                const float4 lo = shared_src ? __ldcg(boxes + 2 * c) : __ldg(boxes + 2 * c);
                const float4 hi = shared_src ? __ldcg(boxes + 2 * c + 1) : __ldg(boxes + 2 * c + 1);
                const float dzhi = hi.z - rz0, dzlo = fmaxf(lo.z - rz1, 0.f);
                const float gx = fmaxf(fmaxf(lo.x - rx1, rx0 - hi.x), 0.f), gy = fmaxf(fmaxf(lo.y - ry1, ry0 - hi.y), 0.f);
                const float g2 = gx * gx + gy * gy;
                const float b0 = fabsf(a.dw2 * dzlo + a.dw3), b1 = fabsf(a.dw2 * dzhi + a.dw3);
                const float bm = fmaxf(b0, b1);
                act = (dzhi > 0.f) && !(g2 > 100.001f) && !(g2 > 220.f * bm * bm);
                if (!a.cull) act = true;
            }
            const unsigned m = __ballot_sync(0xffffffffu, act);
            if (lane == 0) masks[sl] = m;
        }
        __syncthreads();
#pragma unroll 1
        for (int w = 0; w < 8; ++w) {
            unsigned m = masks[w];
            float part_f = 0.f;
            while (m) {
                const int c = cb + w * 32 + __ffs(m) - 1;
                m &= m - 1;
                float4 o[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int j = c * 32 + sl + 8 * q;
                    o[q] = dead;
                    if (j < n_src) o[q] = shared_src ? __ldcg(src + j) : __ldg(src + j);
                }
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float dz = o[q].z - me.z;
                    const float dx = o[q].x - me.x, dy = o[q].y - me.y;
                    const float dxy2 = dx * dx + dy * dy;
                    part_f -= dw_pair(a.prop_radius, a.dw1, a.dw2, a.dw3, dz, dxy2);
                }
            }
            acc += (double)part_f;
        }
        __syncthreads();
    }
    part[sl][lane] = acc;
    __syncthreads();
    if (sl == 0 && live) {
        double t = 0.0;
#pragma unroll
        for (int k = 0; k < 8; ++k) t += part[k][lane];
        a.fz[base + n] = (float)t;
    }
}

// boxes of the chunks of 32 consecutive positions, per aviary: one warp per chunk
__global__ void __launch_bounds__(256) dw_boxes_kernel(const float* __restrict__ pos, float* __restrict__ boxes, int D, int chunks, long long total_chunks) {
    constexpr float BIG = 3e30f;
    const long long wc = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (wc >= total_chunks) return;
    const int lane = threadIdx.x & 31;
    const long long env = wc / chunks;
    const int c = (int)(wc - env * chunks);
    const int i = c * 32 + lane;
    const bool ok = i < D;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ok) v = ldg4(pos, env * D + i);
    const float x0 = warp_min(ok ? v.x : BIG), x1 = warp_max(ok ? v.x : -BIG);
    const float y0 = warp_min(ok ? v.y : BIG), y1 = warp_max(ok ? v.y : -BIG);
    const float z0 = warp_min(ok ? v.z : BIG), z1 = warp_max(ok ? v.z : -BIG);
    if (lane == 0) {
        float4* b = reinterpret_cast<float4*>(boxes) + 2 * wc;
        b[0] = make_float4(x0, y0, z0, 0.f);
        b[1] = make_float4(x1, y1, z1, 0.f);
    }
}

// Push this GPU's slice of a formation's positions AND the boxes of its chunks into every rank's gathered array (own +
// NVLink peers), then raise this rank's sequence flag on every rank: remote stores are fire-and-forget, the last CTA to
// finish (fence + counter) publishes the flags with release semantics.  offset is a multiple of 32, so a warp = a chunk.
struct PubArgs {
    const float* pos;
    float* dst[QS_MAX_PEERS];
    unsigned* flags[QS_MAX_PEERS];
    unsigned* counter;
    int n, offset, n_total, world, rank;
    unsigned seq;
};

__global__ void __launch_bounds__(128) dw_publish_kernel(const __grid_constant__ PubArgs a) {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");      // the consumer synchronises on the flags
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool ok = i < a.n;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ok) v = ldg4(a.pos, i);
    publish_positions(v, ok, i, a.n, a.dst, a.flags, a.counter, a.world, a.rank, a.offset, a.n_total, a.seq);
}

// ---------------------------------------------------------------------------------------------------------
// Neighbourhood query (BaseAviary._getAdjacencyMatrix, BaseAviary.py:658-675): out[e][i][j] = (i == j) or
// |pos_i - pos_j| < radius.  HBM-write bound by nature (D^2 bytes per aviary), instruction-issue bound in practice
// (>= 8 instructions per pair: 3 subtractions, 3 multiply-adds, compare, pack), so the work per pair is kept minimal:
// a lane keeps the positions of its 16 consecutive COLUMNS in registers for the whole row tile (256 rows), the row
// position is a warp-uniform load, the 16 results are packed into one 16-byte store (a warp writes 512 contiguous bytes
// of a row).  The comparison is float32; pairs within 2e-4 (relative) of the threshold are re-evaluated with the
// reference's float64 arithmetic on the float64 positions (rare, warp-voted branch).
// ---------------------------------------------------------------------------------------------------------
struct AdjArgs {
    const double* planes;
    unsigned char* out;
    double radius;
    int D, col_tiles, row_tiles;
};

constexpr int kAdjCols = 512, kAdjRows = 256;
// ---- adjacency kernel: column pairs, sign-bit decisions --------------------------------------------------------------------
// A lane's 16 columns are 8 register PAIRS per coordinate; one pair operation handles two columns: 3 x add2 (differences:
// the row is stored NEGATED and duplicated in shared memory, so it arrives as paired operands by LDS.128 + LDS.64), mul2 +
// 2 x fma2 (squared distance), add2 s = d2 - r2lo and add2 u = s - (r2hi - r2lo).  The SIGN BITS carry the decisions:
// sign(s) = "near", ~sign(s) & sign(u) = "inside the float32 band" (accumulated over the 16 pairs with one LOP3 per pair,
// tested once per row); the 16 result bytes are built from the sign bits by PRMT with sign replication (3 PRMT + 1 LOP3 per
// 4 pairs) -- no FSETP, no SEL.  Rows whose band bit came up are re-evaluated pair by pair (float32 band per pair, then the
// reference's float64 arithmetic on the float64 positions).  The tile's 512 column positions are converted to float32 once
// per CTA through shared memory.  Registers are capped for 3 CTAs per SM.
// sm_90 has no packed float32 instructions: each pair operation is two scalar round-to-nearest operations (explicit
// intrinsics, so the compiler cannot contract a multiply and an add into an FFMA), which gives the packed forms' bits.
typedef unsigned long long u64;
__device__ __forceinline__ u64 pack2(float lo, float hi) { u64 r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi)); return r; }
__device__ __forceinline__ void unpack2(u64 v, unsigned& lo, unsigned& hi) { asm("mov.b64 {%0, %1}, %2;" : "=r"(lo), "=r"(hi) : "l"(v)); }
__device__ __forceinline__ float lo2(u64 v) { return __uint_as_float((unsigned)v); }
__device__ __forceinline__ float hi2(u64 v) { return __uint_as_float((unsigned)(v >> 32)); }
__device__ __forceinline__ u64 add2(u64 a, u64 b) { return pack2(__fadd_rn(lo2(a), lo2(b)), __fadd_rn(hi2(a), hi2(b))); }
__device__ __forceinline__ u64 mul2(u64 a, u64 b) { return pack2(__fmul_rn(lo2(a), lo2(b)), __fmul_rn(hi2(a), hi2(b))); }
__device__ __forceinline__ u64 fma2(u64 a, u64 b, u64 c) { return pack2(__fmaf_rn(lo2(a), lo2(b), lo2(c)), __fmaf_rn(hi2(a), hi2(b), hi2(c))); }
__device__ __forceinline__ unsigned prmt(unsigned a, unsigned b, unsigned c) { unsigned r; asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }

__global__ void __launch_bounds__(256, 3) adjacency_kernel(const __grid_constant__ AdjArgs a) {
    __shared__ __align__(16) float4 rows_a[kAdjRows];          // {-x, -x, -y, -y} of the tile's rows
    __shared__ __align__(16) float2 rows_b[kAdjRows];          // {-z, -z}
    __shared__ __align__(16) float cols_s[3][kAdjCols];        // x[], y[], z[] of the tile's columns (float32)
    int b = blockIdx.x;
    const int ct = b % a.col_tiles; b /= a.col_tiles;
    const int rt = b % a.row_tiles;
    const int env = b / a.row_tiles;
    const long long base = (long long)env * a.D;
    const int c0 = ct * kAdjCols, r0 = rt * kAdjRows;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int k = threadIdx.x; k < kAdjRows; k += blockDim.x) {
        float x = 0.f, y = 0.f, z = 0.f;
        if (r0 + k < a.D) { const D4 p = ld256(a.planes, base + r0 + k); x = (float)p.x; y = (float)p.y; z = (float)p.z; }
        rows_a[k] = make_float4(-x, -x, -y, -y);
        rows_b[k] = make_float2(-z, -z);
    }
    for (int k = threadIdx.x; k < kAdjCols; k += blockDim.x) {
        float x = 3e30f, y = 3e30f, z = 3e30f;                  // columns past the aviary: infinitely far
        if (c0 + k < a.D) { const D4 p = ld256(a.planes, base + c0 + k); x = (float)p.x; y = (float)p.y; z = (float)p.z; }
        cols_s[0][k] = x; cols_s[1][k] = y; cols_s[2][k] = z;
    }
    __syncthreads();
    const int j0 = c0 + 16 * lane;                             // my 16 columns = 8 packed pairs per coordinate
    u64 cx[8], cy[8], cz[8];
#pragma unroll
    for (int v = 0; v < 4; ++v) {
        const float4 fx = reinterpret_cast<const float4*>(cols_s[0])[4 * lane + v];
        const float4 fy = reinterpret_cast<const float4*>(cols_s[1])[4 * lane + v];
        const float4 fz = reinterpret_cast<const float4*>(cols_s[2])[4 * lane + v];
        cx[2 * v] = pack2(fx.x, fx.y); cx[2 * v + 1] = pack2(fx.z, fx.w);
        cy[2 * v] = pack2(fy.x, fy.y); cy[2 * v + 1] = pack2(fy.z, fy.w);
        cz[2 * v] = pack2(fz.x, fz.y); cz[2 * v + 1] = pack2(fz.z, fz.w);
    }
    const float r2f = (float)(a.radius * a.radius);
    float r2lo = r2f * (1.f - 2e-4f), r2hi = r2f * (1.f + 2e-4f);           // outside [lo, hi] float32 decides
    if (a.radius < 0.0) r2lo = r2hi = -1.f;                                 // |d| < negative radius: never
    const u64 nlo2 = pack2(-r2lo, -r2lo);
    const float nbw = -(r2hi - r2lo);
    const u64 nbw2 = pack2(nbw, nbw);
    const bool vec = (a.D % 16) == 0;
    for (int rr = warp; rr < kAdjRows; rr += 8) {
        const int i = r0 + rr;
        if (i >= a.D) break;
        const float4 ma = rows_a[rr];                                       // warp-uniform (broadcast)
        const float2 mb = rows_b[rr];
        const u64 mx = pack2(ma.x, ma.y), my = pack2(ma.z, ma.w), mz = pack2(mb.x, mb.y);
        unsigned w[4];
        unsigned band = 0u;                                                 // sign bit: some pair of mine is inside the float32 band
#pragma unroll
        for (int g = 0; g < 4; ++g) {                                       // 4 pairs of columns -> one word of 4 result bytes
            unsigned sg[4];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int q = 2 * g + h;
                const u64 dx = add2(cx[q], mx), dy = add2(cy[q], my), dz = add2(cz[q], mz);
                const u64 d2 = fma2(dz, dz, fma2(dy, dy, mul2(dx, dx)));
                const u64 s = add2(d2, nlo2);                               // < 0: nearer than the lower band edge
                const u64 u = add2(s, nbw2);                                // < 0: nearer than the upper band edge
                unsigned s0, s1, u0, u1;
                unpack2(s, s0, s1); unpack2(u, u0, u1);
                band |= ~s0 & u0;
                band |= ~s1 & u1;
                sg[2 * h] = s0; sg[2 * h + 1] = s1;
            }
            // byte k of the word = sign of sg[k] replicated (PRMT selector nibble: 8 = replicate the sign of the chosen byte)
            const unsigned t01 = prmt(sg[0], sg[1], 0x00FBu);               // byte0 <- sign(sg0.byte3), byte1 <- sign(sg1.byte3)
            const unsigned t23 = prmt(sg[2], sg[3], 0x00FBu);
            w[g] = prmt(t01, t23, 0x5410u) & 0x01010101u;
        }
        if (__any_sync(0xffffffffu, (int)band < 0)) {                       // rare: the reference's float64 arithmetic decides
            if ((int)band < 0) {
                const float mxs = -ma.x, mys = -ma.z, mzs = -mb.x;
                const D4 md = ld256(a.planes, base + i);
#pragma unroll 1
                for (int q = 0; q < 16; ++q) {
                    if (j0 + q >= a.D) break;
                    const float dx = cols_s[0][16 * lane + q] - mxs, dy = cols_s[1][16 * lane + q] - mys, dz = cols_s[2][16 * lane + q] - mzs;
                    const float d2 = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
                    if (d2 < r2lo || d2 > r2hi) continue;                   // float32 decided this one
                    const D4 od = ld256(a.planes, base + j0 + q);           // BaseAviary.py:670
                    const double ex = md.x - od.x, ey = md.y - od.y, ez = md.z - od.z;
                    const bool near = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)), __dmul_rn(ez, ez))) < a.radius;
                    const unsigned bit = 1u << (8 * (q & 3));
                    const unsigned keep = ~bit, set = near ? bit : 0u;
                    if ((q >> 2) == 0) w[0] = (w[0] & keep) | set; else if ((q >> 2) == 1) w[1] = (w[1] & keep) | set;
                    else if ((q >> 2) == 2) w[2] = (w[2] & keep) | set; else w[3] = (w[3] & keep) | set;
                }
            }
        }
        const int dj = i - j0;                                              // identity (BaseAviary.py:666)
        if ((unsigned)dj < 16u) {
            const unsigned bit = 1u << (8 * (dj & 3));
            if ((dj >> 2) == 0) w[0] |= bit; else if ((dj >> 2) == 1) w[1] |= bit; else if ((dj >> 2) == 2) w[2] |= bit; else w[3] |= bit;
        }
        unsigned char* dst = a.out + ((size_t)(base + i)) * a.D + j0;
        if (vec) {
            if (j0 < a.D) *reinterpret_cast<uint4*>(dst) = make_uint4(w[0], w[1], w[2], w[3]);
        } else {
            for (int q = 0; q < 16 && j0 + q < a.D; ++q) dst[q] = (unsigned char)((w[q >> 2] >> (8 * (q & 3))) & 0xffu);
        }
    }
}

}  // namespace

extern "C" {

static int launch_downwash(const QsParams* p, const float* rows, int n_envs, int D, float* fz_out, void* stream, const char* what) {
    const char* cull_env = getenv("QS_DW_CULL");              // QS_DW_CULL=0: evaluate every chunk (test / measurement switch)
    DwArgs a;
    a.prop_radius = (float)p->prop_radius; a.dw1 = (float)p->dw_coeff[0]; a.dw2 = (float)p->dw_coeff[1]; a.dw3 = (float)p->dw_coeff[2];
    a.rows = rows; a.fz = fz_out; a.D = D; a.tiles_per_env = (D + kDwDrones - 1) / kDwDrones;
    a.cull = (cull_env && cull_env[0] == '0') ? 0 : 1;
    downwash_kernel<<<n_envs * a.tiles_per_env, kDwDrones * kDwSlices, 0, (cudaStream_t)stream>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, what);
}

int qs_downwash(const QsParams* p, const QsState* st, int n_envs, int drones_per_env, float* fz_out, void* stream) {
    if (!p || !st || !st->pos_f32 || !fz_out) return fail(QS_ERR_NULL, "qs_downwash: NULL argument (QsState.pos_f32 is required)");
    if (!aligned16(st->pos_f32)) return fail(QS_ERR_ALIGN, "qs_downwash: pos_f32 must be 16-byte aligned");
    if (n_envs <= 0 || drones_per_env <= 0) return fail(QS_ERR_SIZE, "qs_downwash: sizes must be > 0");
    return launch_downwash(p, st->pos_f32, n_envs, drones_per_env, fz_out, stream, "qs_downwash launch");
}

static int launch_downwash_boxed(const QsParams* p, const float* rows, int n_envs, int D, const float* src, int n_src, const float* boxes,
                                 const unsigned* ready, unsigned seq, int world, unsigned* err, float* fz_out, void* stream, const char* what) {
    const char* cull_env = getenv("QS_DW_CULL");
    DwbArgs a;
    a.prop_radius = (float)p->prop_radius; a.dw1 = (float)p->dw_coeff[0]; a.dw2 = (float)p->dw_coeff[1]; a.dw3 = (float)p->dw_coeff[2];
    a.rows = rows; a.fz = fz_out; a.src = src; a.boxes = boxes; a.n_src = n_src; a.D = D; a.groups_per_env = (D + 31) / 32;
    a.chunks = ((src ? n_src : D) + 31) / 32;
    a.cull = (cull_env && cull_env[0] == '0') ? 0 : 1; a.ready = ready; a.seq = seq; a.world = world; a.err = err;
    const long long blocks = (long long)n_envs * a.groups_per_env;
    if (blocks > 0x7fffffffLL) return fail(QS_ERR_SIZE, "downwash: too many row groups");
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)blocks); cfg.blockDim = dim3(256); cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[1];
    // with flags: programmatic dependent of the publish kernel (which triggers at its first instruction): the launch
    // latency and the row loads overlap the push; the data dependency is carried by the flags, own rank's included
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = ready ? 1 : 0;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, downwash_boxed_kernel, a);
    return e == cudaSuccess ? 0 : cuda_fail(e, what);
}

static int launch_boxes(const float* pos, float* boxes, int n_envs, int D, void* stream, const char* what) {
    const int chunks = (D + 31) / 32;
    const long long total = (long long)n_envs * chunks;
    dw_boxes_kernel<<<(unsigned)((total + 7) / 8), 256, 0, (cudaStream_t)stream>>>(pos, boxes, D, chunks, total);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, what);
}

int qs_downwash_boxed(const QsParams* p, const QsState* st, int n_envs, int drones_per_env, float* boxes_ws, float* fz_out, void* stream) {
    if (!p || !st || !st->pos_f32 || !fz_out || !boxes_ws) return fail(QS_ERR_NULL, "qs_downwash_boxed: NULL argument (QsState.pos_f32 is required)");
    if (!aligned16(st->pos_f32) || !aligned16(boxes_ws)) return fail(QS_ERR_ALIGN, "qs_downwash_boxed: pos_f32 / boxes_ws must be 16-byte aligned");
    if (n_envs <= 0 || drones_per_env <= 0) return fail(QS_ERR_SIZE, "qs_downwash_boxed: sizes must be > 0");
    if (int rc = launch_boxes(st->pos_f32, boxes_ws, n_envs, drones_per_env, stream, "qs_downwash_boxed: boxes launch")) return rc;
    return launch_downwash_boxed(p, st->pos_f32, n_envs, drones_per_env, nullptr, 0, boxes_ws, nullptr, 0u, 0, nullptr, fz_out, stream,
                                 "qs_downwash_boxed launch");
}

long long qs_dw_gathered_floats(int n_total) { return n_total > 0 ? 4LL * n_total + 8LL * ((n_total + 31) / 32) : 0; }

int qs_dw_boxes(float* gathered, int n_total, void* stream) {
    if (!gathered) return fail(QS_ERR_NULL, "qs_dw_boxes: NULL argument");
    if (!aligned16(gathered)) return fail(QS_ERR_ALIGN, "qs_dw_boxes: gathered must be 16-byte aligned");
    if (n_total <= 0) return fail(QS_ERR_SIZE, "qs_dw_boxes: n_total must be > 0");
    return launch_boxes(gathered, gathered + 4LL * n_total, 1, n_total, stream, "qs_dw_boxes launch");
}

int qs_downwash_rows(const QsParams* p, const float* rows_pos, int n_rows, const float* gathered, int n_total,
                     const unsigned* ready_flags, unsigned seq, int world, unsigned* err_flag, float* fz_out, void* stream) {
    if (!p || !rows_pos || !gathered || !fz_out) return fail(QS_ERR_NULL, "qs_downwash_rows: NULL argument");
    if (!aligned16(rows_pos) || !aligned16(gathered)) return fail(QS_ERR_ALIGN, "qs_downwash_rows: position arrays must be 16-byte aligned");
    if (n_rows <= 0 || n_total <= 0) return fail(QS_ERR_SIZE, "qs_downwash_rows: sizes must be > 0");
    if (ready_flags && (world <= 0 || world > QS_MAX_PEERS)) return fail(QS_ERR_SIZE, "qs_downwash_rows: world must be in [1, QS_MAX_PEERS]");
    return launch_downwash_boxed(p, rows_pos, 1, n_rows, gathered, n_total, gathered + 4LL * n_total, ready_flags, seq,
                                 ready_flags ? world : 0, err_flag, fz_out, stream, "qs_downwash_rows launch");
}

int qs_dw_publish(const float* pos, int n, int offset, float* const* gathered, int n_total, unsigned* const* flags, int world, int rank,
                  unsigned seq, unsigned* counter, void* stream) {
    if (!pos || !gathered || !flags || !counter) return fail(QS_ERR_NULL, "qs_dw_publish: NULL argument");
    if (world <= 0 || world > QS_MAX_PEERS || rank < 0 || rank >= world) return fail(QS_ERR_SIZE, "qs_dw_publish: bad world/rank");
    if (n <= 0 || offset < 0 || n_total < offset + n) return fail(QS_ERR_SIZE, "qs_dw_publish: bad n/offset/n_total");
    if (offset % 32 != 0 || (n % 32 != 0 && offset + n != n_total))
        return fail(QS_ERR_ALIGN, "qs_dw_publish: slices must start on a multiple of 32 drones (a chunk never straddles ranks)");
    if (!aligned16(pos)) return fail(QS_ERR_ALIGN, "qs_dw_publish: pos must be 16-byte aligned");
    PubArgs a;
    for (int r = 0; r < world; ++r) {
        if (!gathered[r] || !flags[r]) return fail(QS_ERR_NULL, "qs_dw_publish: NULL peer pointer");
        if (!aligned16(gathered[r])) return fail(QS_ERR_ALIGN, "qs_dw_publish: gathered arrays must be 16-byte aligned");
        a.dst[r] = gathered[r]; a.flags[r] = flags[r];
    }
    a.pos = pos; a.counter = counter; a.n = n; a.offset = offset; a.n_total = n_total; a.world = world; a.rank = rank; a.seq = seq;
    dw_publish_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(a);
    pdl_note((cudaStream_t)stream, kPdlOther);                          // triggers its successor at its first instruction
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, "qs_dw_publish launch");
}

int qs_enable_peer_access(int peer_device) {
    const cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
    if (e == cudaErrorPeerAccessAlreadyEnabled) { (void)cudaGetLastError(); return 0; }
    return e == cudaSuccess ? 0 : cuda_fail(e, "qs_enable_peer_access");
}

// CUDA IPC of a (possibly sub-allocated) device buffer: handle of the enclosing allocation + byte offset.
int qs_ipc_export(const void* ptr, void* handle64, unsigned long long* offset) {
    if (!ptr || !handle64 || !offset) return fail(QS_ERR_NULL, "qs_ipc_export: NULL argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    typedef int (*range_fn)(unsigned long long*, size_t*, unsigned long long);
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qr;
    cudaError_t e = cudaGetDriverEntryPoint("cuMemGetAddressRange", &f, cudaEnableDefault, &qr);
    if (e != cudaSuccess || !f) return e != cudaSuccess ? cuda_fail(e, "qs_ipc_export: cuMemGetAddressRange lookup") : fail(QS_ERR_UNSUPPORTED, "qs_ipc_export: no cuMemGetAddressRange");
    unsigned long long base = 0;
    size_t size = 0;
    if (reinterpret_cast<range_fn>(f)(&base, &size, (unsigned long long)(uintptr_t)ptr) != 0) return fail(QS_ERR_UNSUPPORTED, "qs_ipc_export: cuMemGetAddressRange failed");
    e = cudaIpcGetMemHandle(reinterpret_cast<cudaIpcMemHandle_t*>(handle64), reinterpret_cast<void*>((uintptr_t)base));
    if (e != cudaSuccess) return cuda_fail(e, "qs_ipc_export: cudaIpcGetMemHandle");
    *offset = (unsigned long long)(uintptr_t)ptr - base;
    return 0;
}

int qs_ipc_import(const void* handle64, unsigned long long offset, void** ptr_out) {
    if (!handle64 || !ptr_out) return fail(QS_ERR_NULL, "qs_ipc_import: NULL argument");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, sizeof(h));
    void* base = nullptr;
    const cudaError_t e = cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) return cuda_fail(e, "qs_ipc_import: cudaIpcOpenMemHandle");
    *ptr_out = static_cast<char*>(base) + offset;
    return 0;
}

int qs_adjacency(const QsState* st, int n_envs, int drones_per_env, double radius, unsigned char* out, void* stream) {
    if (!st || !st->planes || !out) return fail(QS_ERR_NULL, "qs_adjacency: NULL argument");
    if (!aligned32(st->planes)) return fail(QS_ERR_ALIGN, "qs_adjacency: planes must be 32-byte aligned");
    if (n_envs <= 0 || drones_per_env <= 0) return fail(QS_ERR_SIZE, "qs_adjacency: sizes must be > 0");
    if (drones_per_env % 16 == 0 && !aligned16(out)) return fail(QS_ERR_ALIGN, "qs_adjacency: out must be 16-byte aligned");
    AdjArgs a;
    a.planes = st->planes; a.out = out; a.radius = radius; a.D = drones_per_env;
    a.col_tiles = (drones_per_env + kAdjCols - 1) / kAdjCols; a.row_tiles = (drones_per_env + kAdjRows - 1) / kAdjRows;
    const long long blocks = (long long)n_envs * a.col_tiles * a.row_tiles;
    if (blocks > 0x7fffffffLL) return fail(QS_ERR_SIZE, "qs_adjacency: too many tiles");
    adjacency_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, "qs_adjacency launch");
}

}  // extern "C"
