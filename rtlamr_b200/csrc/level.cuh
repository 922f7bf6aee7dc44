// level.cuh -- the level of an input capture: a histogram of the exponents e = floor(log2 |x|) of its components x, the
// values convert.cuh's fmt_x defines.  include/ertgpu_level.h turns the histogram into a gain (ertgpu_measure_input).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "convert.cuh"

namespace ert {

constexpr int kLvThreads = 256;
constexpr int kLvZero = 256, kLvNan = 257, kLvCounters = 258;  // after the 256 exponent bins
constexpr int kLvNone = kLvCounters;                             // a lane with no component

__device__ __forceinline__ int lv_bin(int e) { return min(max(e, -128), 127) + 128; }

// The counter of one component: bin e + 128 (e clamped to [-128, 127]; infinities in the top bin), kLvZero or kLvNan.
// e comes from the bits alone: 31 - clz(|x|) for integers, the exponent field for floats (a subnormal's from its leading
// mantissa bit).
__device__ __forceinline__ int lv_classify(int32_t x) {  // int8, int16, int32: |-2^31| = 2^31 as uint32
    if (x == 0) return kLvZero;
    const uint32_t a = x < 0 ? 0u - (uint32_t)x : (uint32_t)x;
    return lv_bin(31 - __clz(a));
}
__device__ __forceinline__ int lv_classify(float x) {
    const uint32_t u = __float_as_uint(x), ex = (u >> 23) & 0xffu, m = u & 0x7fffffu;
    if (ex == 0xffu) return m ? kLvNan : 255;
    if (ex == 0) return m ? lv_bin(31 - __clz(m) - 149) : kLvZero;  // m * 2^-149
    return lv_bin((int)ex - 127);
}
__device__ __forceinline__ int lv_classify(double x) {
    const uint64_t u = (uint64_t)__double_as_longlong(x), m = u & 0xfffffffffffffull;
    const uint32_t ex = (uint32_t)(u >> 52) & 0x7ffu;
    if (ex == 0x7ffu) return m ? kLvNan : 255;
    if (ex == 0) return m ? lv_bin(63 - __clzll((long long)m) - 1074) : kLvZero;  // m * 2^-1074
    return lv_bin((int)ex - 1023);
}
__device__ __forceinline__ int lv_classify(int8_t x) { return lv_classify((int32_t)x); }
__device__ __forceinline__ int lv_classify(int16_t x) { return lv_classify((int32_t)x); }

// Count one component per lane in the CTA's counters: lanes with the same counter add once, together.  All 32 lanes of
// the warp take part.
__device__ __forceinline__ void lv_count(unsigned int* s, int bin) {
    const unsigned peers = __match_any_sync(0xffffffffu, bin);
    if (bin != kLvNone && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&s[bin], (unsigned)__popc(peers));
}

// The histogram of the nbytes bytes (whole IQ samples of format F != cu8) at in (16-byte aligned), added to
// counters[0..257]: the 256 exponent bins, then zeros, then NaNs.  Each thread classifies the components of one 16-byte
// group per step; the last nbytes % 16 bytes are one more group, read byte by byte.  Integer counts: the result does not
// depend on the grid.  Per launch at most 2^32 - 1 components reach one CTA.
template <int F>
__global__ void __launch_bounds__(kLvThreads) level_kernel(const uint8_t* __restrict__ in, long long nbytes,
                                                           unsigned long long* __restrict__ counters) {
    constexpr int S = ertfmt_bytes(F), kComps = 32 / S;  // components per 16 bytes
    __shared__ unsigned int s[kLvCounters];
    for (int i = threadIdx.x; i < kLvCounters; i += kLvThreads) s[i] = 0;
    __syncthreads();
    const long long groups = nbytes / 16, tail = nbytes % 16;
    const long long ngroups = groups + (tail != 0);
    const long long stride = (long long)gridDim.x * kLvThreads;
    for (long long base = (long long)blockIdx.x * kLvThreads; base < ngroups; base += stride) {  // uniform per CTA
        const long long grp = base + threadIdx.x;
        uint32_t x[4] = {0, 0, 0, 0};
        int n = 0;  // components of this lane's group
        if (grp < groups) {
            const uint4 v = __ldcs(reinterpret_cast<const uint4*>(in) + grp);
            x[0] = v.x;
            x[1] = v.y;
            x[2] = v.z;
            x[3] = v.w;
            n = kComps;
        } else if (grp == groups && tail) {
            const uint8_t* p = in + 16 * groups;
            for (int b = 0; b < tail; b++) x[b >> 2] |= (uint32_t)p[b] << (8 * (b & 3));
            n = (int)(2 * tail / S);
        }
#pragma unroll
        for (int c = 0; c < kComps; c++) lv_count(s, c < n ? lv_classify(fmt_x<F>(x, c)) : kLvNone);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kLvCounters; i += kLvThreads)
        if (s[i]) atomicAdd(counters + i, (unsigned long long)s[i]);
}

}  // namespace ert
