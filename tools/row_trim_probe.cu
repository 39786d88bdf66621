// row_trim_probe.cu -- copy-only model of step_pipe_kernel's memory traffic (no physics), built and run by row_trim_probe.py.
// Question: does fetching only the 224 history bytes of each 288-byte observation row (B = 15, A = 4) save DRAM time, or do
// the skipped 64 bytes (the old head and the oldest action, sectors 0-1 of the row) come in anyway with the needed sectors?
//
// Per 32-row tile, like the step kernel: the state-sized streams (3 x 32 B + 8 B float64 read and written, a 16-byte action
// read) go through registers, the old rows through one of two shared-memory stages, and one bulk store writes the new rows.
// One warp per CTA, four tiles per warp, the next tile's loads issued before the current tile's store.
//   bulk      one 1-D cp.async.bulk of the whole span (rows x 288 B), L2 evict-first: what the kernel does today
//   tensor    one cp.async.bulk.tensor.2d per tile over the obs buffer seen as [N][od/2] 8-byte elements, box {od/2, 32} at
//             (8, w0): columns 16 .. od-1 of each row, the box's last 16 floats per row out of bounds (zero-filled, not read);
//             L2 evict-first, with the tensor map's L2 promotion NONE / 64B / 128B / 256B
//   tensor_full  the same tensor load at (0, w0): the whole rows, nothing skipped, promotion NONE.  Against `tensor` it prices
//             the skipped bytes alone; against `bulk` the 2-D tensor path alone.
// All write the same bytes (checked first, at the smallest, the bench's and the largest row width, ragged N).
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); exit(1); } } while (0)

constexpr int K = 4;                 // tiles per warp
constexpr int kFinBytes = 32 * 12 * 4;      // the step kernel's terminal-head buffer: allocated, so occupancy matches

struct Args { const float* prev; float* next; const double* sin; double* sout; const float* act; long long N; int od; };

// MODE 0: bulk, 1: tensor (trimmed box), 2: tensor_full.  Stage: [128-byte prefix, tensor modes][rows][16-byte tail][mbarrier]
__host__ __device__ constexpr int box_off(int mode) { return mode ? 128 : 0; }
__host__ __device__ constexpr int bar_off(int mode, int od) { return box_off(mode) + 32 * od * 4 + 16; }
__host__ __device__ constexpr int stage_bytes(int mode, int od) { return (bar_off(mode, od) + 8 + 127) / 128 * 128; }

__device__ __forceinline__ unsigned s32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

template <int MODE>
__global__ void __launch_bounds__(32) probe_kernel(const __grid_constant__ CUtensorMap tm, const __grid_constant__ Args a) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int lane = threadIdx.x, od = a.od;
    const long long N = a.N, tiles = (N + 31) / 32, t0 = (long long)blockIdx.x * K;
    if (t0 >= tiles) return;
    const int nt = (int)(tiles - t0 < K ? tiles - t0 : K);
    constexpr bool TENSOR = MODE > 0, TRIM = MODE == 1;
    const int SB = stage_bytes(MODE, od);
    auto stage = [&](int k) { return smem + (k & 1) * SB; };
    auto bar = [&](int k) { return reinterpret_cast<unsigned long long*>(stage(k) + bar_off(MODE, od)); };
    if (lane == 0) {
        for (int s = 0; s < 2; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(s32(bar(s))) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    double4 s0, s1, s2; double s3; float4 av;
    auto issue = [&](int k) {
        const long long w0 = (t0 + k) * 32, il = w0 + lane < N ? w0 + lane : w0;
        const double4* p = reinterpret_cast<const double4*>(a.sin);
        s0 = p[il]; s1 = p[N + il]; s2 = p[2 * N + il]; s3 = a.sin[12 * N + il];
        av = reinterpret_cast<const float4*>(a.act)[il];
        if (lane == 0) {
            unsigned long long pol;
            asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
            const int rows = (int)(N - w0 < 32 ? N - w0 : 32);
            const unsigned tx = TENSOR ? 32u * od * 4u : (unsigned)(rows * od * 4);
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(bar(k))), "r"(tx) : "memory");
            if (TENSOR)
                asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3}], [%4], %5;"
                             ::"r"(s32(stage(k) + box_off(MODE))), "l"(&tm), "r"(TRIM ? 8 : 0), "r"((int)w0), "r"(s32(bar(k))), "l"(pol) : "memory");
            else
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                             ::"r"(s32(stage(k))), "l"(a.prev + w0 * od), "r"(tx), "r"(s32(bar(k))), "l"(pol) : "memory");
        }
    };
    issue(0);
    for (int k = 0; k < nt; ++k) {
        const double4 d0 = s0, d1 = s1, d2 = s2; const double d3 = s3; const float4 act = av;
        if (k + 1 < nt) {
            if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");      // stage (k+1)&1 was tile k-1's store source
            __syncwarp();
            issue(k + 1);
        }
        const long long w0 = (t0 + k) * 32, i = w0 + lane;
        const bool live = i < N;
        const int rows = (int)(N - w0 < 32 ? N - w0 : 32);
        if (live) {
            double4* q = reinterpret_cast<double4*>(a.sout);
            q[i] = d0; q[N + i] = d1; q[2 * N + i] = d2; a.sout[12 * N + i] = d3;
        }
        const float h[12] = {(float)d0.x, (float)d0.y, (float)d0.z, (float)d0.w, (float)d1.x, (float)d1.y,
                             (float)d1.z, (float)d1.w, (float)d2.x, (float)d2.y, (float)d2.z, (float)d3};
        unsigned ok;
        do {
            asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                         : "=r"(ok) : "r"(s32(bar(k))), "r"((unsigned)(k >> 1) & 1u) : "memory");
        } while (!ok);
        float* xs = reinterpret_cast<float*>(stage(k));
        // new row r = [head_r | old columns 16 .. od-1 | act_r]: bulk: the span read from +4 floats, head_r over old columns
        // 0..11 of row r (slots 4..15), act_r over the first 4 floats of row r+1; tensor: the span read from 12 floats before
        // the box, head_r in the 12 floats before row r's slot, act_r over the first 4 of its 16 zero-filled floats
        float* rows_s = xs + box_off(MODE) / 4;
        float* hd = TRIM ? rows_s + lane * od - 12 : rows_s + lane * od + 4;
        float* ad = TRIM ? rows_s + lane * od + od - 16 : rows_s + lane * od + od;
        const float* src = TRIM ? rows_s - 12 : rows_s + 4;
        if (live) {
            float4* h4 = reinterpret_cast<float4*>(hd);
            h4[0] = make_float4(h[0], h[1], h[2], h[3]); h4[1] = make_float4(h[4], h[5], h[6], h[7]); h4[2] = make_float4(h[8], h[9], h[10], h[11]);
            *reinterpret_cast<float4*>(ad) = act;
        }
        __syncwarp();
        if (lane == 0) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(a.next + w0 * od), "r"(s32(src)), "r"((unsigned)(rows * od * 4)) : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
    }
    if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

static PFN_cuTensorMapEncodeTiled_v12000 encode_fn() {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qr;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qr));
    if (!f) { fprintf(stderr, "no cuTensorMapEncodeTiled\n"); exit(1); }
    return reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(f);
}

static CUtensorMap make_map(const float* base, long long N, int od, CUtensorMapL2promotion prom) {
    CUtensorMap m;
    const cuuint64_t dims[2] = {(cuuint64_t)(od / 2), (cuuint64_t)N};
    const cuuint64_t strides[1] = {(cuuint64_t)od * 4};
    const cuuint32_t box[2] = {(cuuint32_t)(od / 2), 32}, es[2] = {1, 1};
    const CUresult r = encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, const_cast<float*>(base), dims, strides, box, es,
                                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, prom, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { fprintf(stderr, "cuTensorMapEncodeTiled failed: %d\n", (int)r); exit(1); }
    return m;
}

struct Pair { float *prev, *next, *act; double *sin, *sout; };

static Pair make_pair(long long N, int od, unsigned seed) {
    Pair p;
    CK(cudaMalloc(&p.prev, N * od * 4)); CK(cudaMalloc(&p.next, N * od * 4)); CK(cudaMalloc(&p.act, N * 16));
    CK(cudaMalloc(&p.sin, 13 * N * 8)); CK(cudaMalloc(&p.sout, 13 * N * 8));
    std::vector<float> f((size_t)N * od);
    for (size_t j = 0; j < f.size(); ++j) f[j] = (float)((j * 2654435761u + seed) % 100003) * 1e-3f;
    CK(cudaMemcpy(p.prev, f.data(), f.size() * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(p.act, f.data(), N * 16, cudaMemcpyHostToDevice));
    std::vector<double> s((size_t)13 * N);
    for (size_t j = 0; j < s.size(); ++j) s[j] = (double)((j * 40503u + seed) % 9973) * 0.25;
    CK(cudaMemcpy(p.sin, s.data(), s.size() * 8, cudaMemcpyHostToDevice));
    CK(cudaMemset(p.next, 0xff, N * od * 4)); CK(cudaMemset(p.sout, 0, 13 * N * 8));
    return p;
}
static void free_pair(Pair& p) { cudaFree(p.prev); cudaFree(p.next); cudaFree(p.act); cudaFree(p.sin); cudaFree(p.sout); }

static void launch(int variant, const Pair& p, const CUtensorMap& m, long long N, int od, cudaStream_t s) {
    const Args a = {p.prev, p.next, p.sin, p.sout, p.act, N, od};
    const long long tiles = (N + 31) / 32;
    const int grid = (int)((tiles + K - 1) / K);
    const int mode = variant == 0 ? 0 : variant < 5 ? 1 : 2;
    const int smem = 2 * stage_bytes(mode, od) + kFinBytes;
    if (mode == 0) probe_kernel<0><<<grid, 32, smem, s>>>(m, a);
    else if (mode == 1) probe_kernel<1><<<grid, 32, smem, s>>>(m, a);
    else probe_kernel<2><<<grid, 32, smem, s>>>(m, a);
}

constexpr int kVariants = 6;
static const CUtensorMapL2promotion kProm[kVariants] = {CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_64B,
                                                        CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_L2_PROMOTION_NONE};
static const char* kName[kVariants] = {"bulk", "tensor_none", "tensor_64b", "tensor_128b", "tensor_256b", "tensor_full"};

int main(int argc, char** argv) {
    const int runs = argc > 1 ? atoi(argv[1]) : 3;
    const int reps = argc > 2 ? atoi(argv[2]) : 2000;
    const int smax = 2 * stage_bytes(1, 304) + kFinBytes;
    CK(cudaFuncSetAttribute(probe_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, smax));
    CK(cudaFuncSetAttribute(probe_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smax));
    CK(cudaFuncSetAttribute(probe_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, smax));
    // 1. all variants write the same bytes: B = 1 (box wholly out of bounds), B = 15, B = 73 (od/2 = 152 elements), ragged N
    for (int od : {16, 72, 304}) {
        const long long N = 32 * 37 + 1;
        Pair p = make_pair(N, od, 7);
        std::vector<float> ref((size_t)N * od), got((size_t)N * od);
        std::vector<double> sref((size_t)13 * N), sgot((size_t)13 * N);
        for (int v = 0; v < kVariants; ++v) {
            CK(cudaMemset(p.next, 0xff, N * od * 4));
            launch(v, p, make_map(p.prev, N, od, kProm[v]), N, od, 0);
            CK(cudaDeviceSynchronize());
            CK(cudaMemcpy(v ? got.data() : ref.data(), p.next, N * od * 4, cudaMemcpyDeviceToHost));
            CK(cudaMemcpy(v ? sgot.data() : sref.data(), p.sout, 13 * N * 8, cudaMemcpyDeviceToHost));
            if (v && (memcmp(ref.data(), got.data(), ref.size() * 4) || memcmp(sref.data(), sgot.data(), sref.size() * 8))) {
                printf("{\"check\": \"%s\", \"od\": %d, \"N\": %lld, \"equal\": false}\n", kName[v], od, N);
                return 1;
            }
        }
        // the expected rows, from the inputs on the host: [state head | old columns 16.. | action]
        std::vector<float> prev((size_t)N * od), act((size_t)N * 4);
        CK(cudaMemcpy(prev.data(), p.prev, N * od * 4, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(act.data(), p.act, N * 16, cudaMemcpyDeviceToHost));
        for (long long i = 0; i < N; ++i)
            for (int c = 12; c < od; ++c) {
                const float want = c < od - 4 ? prev[i * od + c + 4] : act[i * 4 + c - (od - 4)];
                if (memcmp(&want, &ref[i * od + c], 4)) {
                    printf("{\"check\": \"layout\", \"od\": %d, \"row\": %lld, \"col\": %d, \"equal\": false}\n", od, i, c);
                    return 1;
                }
            }
        printf("{\"check\": \"all variants\", \"od\": %d, \"N\": %lld, \"equal\": true}\n", od, N);
        free_pair(p);
    }
    // 2. time: 65 536 rows over 8 rotating buffer sets (the bench), 1 048 576 rows over 2; variants alternate, `runs` rounds
    const int od = 72;
    for (long long N : {65536LL, 1048576LL}) {
        const int rot = N == 65536 ? 8 : 2;
        const int n = N == 65536 ? reps : reps / 8;
        std::vector<Pair> ps;
        std::vector<CUtensorMap> maps[kVariants];
        for (int r = 0; r < rot; ++r) ps.push_back(make_pair(N, od, r));
        for (int v = 0; v < kVariants; ++v)
            for (int r = 0; r < rot; ++r) maps[v].push_back(make_map(ps[r].prev, N, od, kProm[v]));
        cudaEvent_t e0, e1;
        CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
        for (int run = 0; run < runs; ++run)
            for (int v = 0; v < kVariants; ++v) {
                for (int k = 0; k < 4 * rot; ++k) launch(v, ps[k % rot], maps[v][k % rot], N, od, 0);
                CK(cudaEventRecord(e0));
                for (int k = 0; k < n; ++k) launch(v, ps[k % rot], maps[v][k % rot], N, od, 0);
                CK(cudaEventRecord(e1));
                CK(cudaEventSynchronize(e1));
                float ms;
                CK(cudaEventElapsedTime(&ms, e0, e1));
                printf("{\"N\": %lld, \"variant\": \"%s\", \"run\": %d, \"us_per_launch\": %.3f}\n", N, kName[v], run, ms * 1e3 / n);
                fflush(stdout);
            }
        CK(cudaGetLastError());
        for (auto& p : ps) free_pair(p);
    }
    return 0;
}
