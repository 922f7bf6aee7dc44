// Input-format conversion: signed 8-bit, signed 16-bit and float32 IQ (ertgpu_set_input_format) -> the uint8 IQ the
// decoder reads.  One formula for every format: u = clamp(rint(fl32(x * g)), -128, 127) + 128, NaN -> 128.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ertgpu.h"

namespace ert {

// bytes per IQ sample of a format
__host__ __device__ constexpr int fmt_sample_bytes(int f) {
    return f == ERTGPU_FORMAT_CS16 ? 4 : f == ERTGPU_FORMAT_CF32 ? 8 : 2;
}

// One IQ component x (int8, int16 or float32, exact in float32) times g as the decoder's byte.  The product is one
// float32 multiply rounded to nearest even (__fmul_rn: never contracted).  NaN is decided here, before fmaxf (which
// would return -128) and cvt.rni (which has its own NaN rule) see it; infinities clamp.
__device__ __forceinline__ uint32_t fmt_byte(float x, float g) {
    const float p = __fmul_rn(x, g);
    if (p != p) return 128u;
    return (uint32_t)(__float2int_rn(fminf(fmaxf(p, -128.0f), 127.0f)) + 128);
}

// The bytes of IQ sample j of format F (F != cu8) at src: I in the low byte, Q in the high byte.
template <int F>
__device__ __forceinline__ uchar2 fmt_sample(const uint8_t* src, long long j, float g) {
    float i, q;
    if constexpr (F == ERTGPU_FORMAT_CS8) {
        const char2 v = *reinterpret_cast<const char2*>(src + 2 * j);
        i = (float)v.x;
        q = (float)v.y;
    } else if constexpr (F == ERTGPU_FORMAT_CS16) {
        const short2 v = *reinterpret_cast<const short2*>(src + 4 * j);
        i = (float)v.x;
        q = (float)v.y;
    } else {
        const float2 v = *reinterpret_cast<const float2*>(src + 8 * j);
        i = v.x;
        q = v.y;
    }
    return make_uchar2((unsigned char)fmt_byte(i, g), (unsigned char)fmt_byte(q, g));
}

constexpr int kCvtThreads = 256;

// Native-rate conversion of ngroups groups of 8 IQ samples (16 output bytes each) from `in` (16-byte aligned, format
// F) to `out` (16-byte aligned).  Grid-stride loop; each group is one, two or four 16-byte loads and one 16-byte store.
template <int F>
__global__ void __launch_bounds__(kCvtThreads) convert_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                                                              long long ngroups, float g) {
    constexpr int kLoads = fmt_sample_bytes(F) * 8 / 16;
    for (long long grp = (long long)blockIdx.x * blockDim.x + threadIdx.x; grp < ngroups;
         grp += (long long)gridDim.x * blockDim.x) {
        const uint4* src = reinterpret_cast<const uint4*>(in) + grp * kLoads;
        uint4 v[kLoads];
#pragma unroll
        for (int k = 0; k < kLoads; k++) v[k] = __ldcs(src + k);   // read once: do not keep it in L2
        uint32_t w[4];
        if constexpr (F == ERTGPU_FORMAT_CS8) {
            const uint32_t x[4] = {v[0].x, v[0].y, v[0].z, v[0].w};
#pragma unroll
            for (int k = 0; k < 4; k++) {
                uint32_t o = 0;
#pragma unroll
                for (int b = 0; b < 4; b++) o |= fmt_byte((float)(int8_t)(x[k] >> (8 * b)), g) << (8 * b);
                w[k] = o;
            }
        } else if constexpr (F == ERTGPU_FORMAT_CS16) {
            const uint32_t x[8] = {v[0].x, v[0].y, v[0].z, v[0].w, v[1].x, v[1].y, v[1].z, v[1].w};
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const uint32_t a = x[2 * k], b = x[2 * k + 1];
                w[k] = fmt_byte((float)(int16_t)(a & 0xffffu), g) | fmt_byte((float)(int16_t)(a >> 16), g) << 8 |
                       fmt_byte((float)(int16_t)(b & 0xffffu), g) << 16 | fmt_byte((float)(int16_t)(b >> 16), g) << 24;
            }
        } else {
#pragma unroll
            for (int k = 0; k < 4; k++)
                w[k] = fmt_byte(__uint_as_float(v[k].x), g) | fmt_byte(__uint_as_float(v[k].y), g) << 8 |
                       fmt_byte(__uint_as_float(v[k].z), g) << 16 | fmt_byte(__uint_as_float(v[k].w), g) << 24;
        }
        reinterpret_cast<uint4*>(out)[grp] = make_uint4(w[0], w[1], w[2], w[3]);
    }
}

}  // namespace ert
