// tma_probe.cu -- how fast can the demod kernel's access pattern be streamed at all?
// Every warp walks work tiles of 32 rows (row pitch = PITCH bytes) in boxes of [32 rows][BOXB bytes] with S boxes in
// flight, exactly like demod_fast_kernel, but does nothing with the data.  MODE 1 streams the same bytes as contiguous
// 1-D bulk copies (the friendliest pattern) for comparison.
// Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tma_probe tma_probe.cu -lcuda
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstdint>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect(uint32_t bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile("{\n.reg .pred p;\nW_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra D_%=;\nbra W_%=;\nD_%=:\n}\n" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma2d(uint32_t dst, const CUtensorMap* map, int x, int y, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst), "l"(map), "r"(x), "r"(y), "r"(bar) : "memory");
}
__device__ __forceinline__ void bulk1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

template <int MODE>
__global__ void probe(const __grid_constant__ CUtensorMap map, const uint8_t* base, long long nrows, int pitch, int boxb, int stages, int warps,
                      unsigned long long* counter, uint32_t* sink) {
    extern __shared__ __align__(128) uint8_t sm[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t sbase = smem_u32(sm);
    const uint32_t bar0 = sbase + warp * 64;
    const uint32_t stagebytes = 32u * boxb;
    const uint32_t stage0 = sbase + 1024 + warp * stages * stagebytes;
    if (lane == 0) for (int s = 0; s < stages; s++) mbar_init(bar0 + s * 8, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    const long long ntiles = nrows / 32;
    const int nbox = pitch / boxb;
    uint32_t phases = 0, acc = 0;
    int st = 0;
    for (;;) {
        unsigned long long tile = 0;
        if (lane == 0) tile = atomicAdd(counter, 1ull);
        tile = __shfl_sync(0xFFFFFFFFu, tile, 0);
        if ((long long)tile >= ntiles) break;
        auto issue = [&](int t, int stage) {
            if (t >= nbox) return;
            if (lane == 0) {
                mbar_expect(bar0 + stage * 8, stagebytes);
                if (MODE == 0) tma2d(stage0 + stage * stagebytes, &map, t * boxb, (int)(tile * 32), bar0 + stage * 8);
                else bulk1d(stage0 + stage * stagebytes, base + (tile * nbox + t) * (long long)stagebytes, stagebytes, bar0 + stage * 8);
            }
        };
        for (int s = 0; s < stages; s++) issue(s, (st + s) % stages);
        for (int t = 0; t < nbox; t++) {
            mbar_wait(bar0 + st * 8, (phases >> st) & 1u);
            phases ^= 1u << st;
            uint32_t v;
            asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(stage0 + st * stagebytes + lane * 4));
            acc ^= v;
            __syncwarp();
            issue(t + stages, st);
            st = (st + 1 == stages) ? 0 : st + 1;
        }
    }
    if (acc == 0x12345678u) sink[0] = acc;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int main(int argc, char** argv) {
    const long long bytes = (argc > 1 ? atoll(argv[1]) : 4ll) << 30;
    const int pitch = 8192;
    const long long nrows = bytes / pitch;
    uint8_t* d; cudaMalloc(&d, bytes); cudaMemset(d, 1, bytes);
    unsigned long long* counter; cudaMalloc(&counter, 8);
    uint32_t* sink; cudaMalloc(&sink, 4);
    void* fp = nullptr; cudaDriverEntryPointQueryResult q;
    cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q);
    EncodeTiledFn enc = (EncodeTiledFn)fp;
    int sms = 132; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    cudaFuncSetAttribute(probe<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(probe<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    struct Cfg { int mode, boxb, stages, warps, promo; };
    const Cfg cfgs[] = {
        {0, 176, 2, 8, 2}, {0, 176, 2, 12, 2}, {0, 176, 2, 12, 3}, {0, 176, 3, 12, 3}, {0, 176, 4, 12, 3}, {0, 176, 2, 16, 3},
        {0, 256, 2, 12, 3}, {0, 256, 3, 12, 3}, {0, 128, 4, 12, 3}, {0, 512, 2, 8, 3}, {0, 512, 2, 12, 3}, {0, 1024, 2, 6, 3}, {0, 64, 8, 12, 3},
        {1, 176, 2, 12, 2}, {1, 176, 4, 12, 2}, {1, 512, 2, 12, 2},
    };
    for (const Cfg& c : cfgs) {
        if (pitch % c.boxb) { /* 176 does not divide 8192: walk 46 boxes = 8096 B of each row */ }
        CUtensorMap map;
        const cuuint64_t gdim[2] = {(cuuint64_t)pitch, (cuuint64_t)nrows};
        const cuuint64_t gstride[1] = {(cuuint64_t)pitch};
        const cuuint32_t box[2] = {(cuuint32_t)c.boxb, 32u};
        const cuuint32_t estr[2] = {1u, 1u};
        const CUtensorMapL2promotion pr = c.promo == 3 ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : c.promo == 2 ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B : CU_TENSOR_MAP_L2_PROMOTION_NONE;
        CUresult r = enc(&map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, d, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, pr, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { printf("encode failed %d\n", (int)r); continue; }
        const int smem = 1024 + c.warps * c.stages * 32 * c.boxb;
        if (smem > 227 * 1024) { printf("skip (smem)\n"); continue; }
        float best = 1e9f;
        for (int rep = 0; rep < 4; rep++) {
            cudaMemset(counter, 0, 8);
            cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
            cudaEventRecord(e0);
            if (c.mode == 0) probe<0><<<sms, c.warps * 32, smem>>>(map, d, nrows, pitch, c.boxb, c.stages, c.warps, counter, sink);
            else probe<1><<<sms, c.warps * 32, smem>>>(map, d, nrows, pitch, c.boxb, c.stages, c.warps, counter, sink);
            cudaEventRecord(e1);
            cudaError_t e = cudaDeviceSynchronize();
            if (e != cudaSuccess) { printf("error %s\n", cudaGetErrorString(e)); return 1; }
            float ms; cudaEventElapsedTime(&ms, e0, e1);
            if (ms < best) best = ms;
        }
        const double moved = (double)(nrows / 32) * (pitch / c.boxb) * 32.0 * c.boxb;
        printf("mode %d box %4d B x 32 rows, %d stages, %2d warps, promo %d: %.3f ms  %.0f GB/s\n", c.mode, c.boxb, c.stages, c.warps, c.promo, best, moved / best / 1e6);
    }
    return 0;
}
