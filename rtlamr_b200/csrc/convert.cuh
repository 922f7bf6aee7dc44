// Input-format conversion: every complex SigMF datatype (ertgpu_set_input_format) -> the uint8 IQ the decoder reads.
// One formula for every format: u = clamp(rint(p), -128, 127) + 128, NaN -> 128, with p = fl32(x * g) where the
// component x is exact in float32 (8- and 16-bit integers, float32) and p = fl64(x * (double)g) where it is not (32-bit
// integers, float64).  x is the stored value, less 2^15 or 2^31 for the unsigned formats; a big-endian value is byte
// permuted first.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>
#include <utility>

#include "../../include/ertgpu.h"

namespace ert {

// bytes per IQ sample of a format
__host__ __device__ constexpr int fmt_sample_bytes(int f) {
    return f == ERTGPU_FORMAT_CS16 || f == ERTGPU_FORMAT_CS16BE || f == ERTGPU_FORMAT_CU16 || f == ERTGPU_FORMAT_CU16BE ? 4
           : f == ERTGPU_FORMAT_CF64 || f == ERTGPU_FORMAT_CF64BE                                                      ? 16
           : f == ERTGPU_FORMAT_CF32 || f >= ERTGPU_FORMAT_CF32BE                                                      ? 8
                                                                                                                      : 2;
}

// Every input format, and f(std::integral_constant<int, F>{}) for the one equal to `format`; false when none is.
using AllFormats = std::integer_sequence<int, ERTGPU_FORMAT_CU8, ERTGPU_FORMAT_CS8, ERTGPU_FORMAT_CS16, ERTGPU_FORMAT_CF32,
                                         ERTGPU_FORMAT_CS16BE, ERTGPU_FORMAT_CF32BE, ERTGPU_FORMAT_CU16, ERTGPU_FORMAT_CU16BE,
                                         ERTGPU_FORMAT_CS32, ERTGPU_FORMAT_CS32BE, ERTGPU_FORMAT_CU32, ERTGPU_FORMAT_CU32BE,
                                         ERTGPU_FORMAT_CF64, ERTGPU_FORMAT_CF64BE>;
template <typename Fn, int... Fs>
bool fmt_visit_in(int format, Fn&& f, std::integer_sequence<int, Fs...>) {
    return ((format == Fs ? (f(std::integral_constant<int, Fs>{}), true) : false) || ...);
}
template <typename Fn>
bool fmt_visit(int format, Fn&& f) { return fmt_visit_in(format, f, AllFormats{}); }

// The name of a format: its SigMF datatype, or cu8 / cs8 / cs16 / cf32 for the first four.
inline const char* fmt_name(int f) {
    switch (f) {
        case ERTGPU_FORMAT_CU8: return "cu8";
        case ERTGPU_FORMAT_CS8: return "cs8";
        case ERTGPU_FORMAT_CS16: return "cs16";
        case ERTGPU_FORMAT_CF32: return "cf32";
        case ERTGPU_FORMAT_CS16BE: return "ci16_be";
        case ERTGPU_FORMAT_CF32BE: return "cf32_be";
        case ERTGPU_FORMAT_CU16: return "cu16_le";
        case ERTGPU_FORMAT_CU16BE: return "cu16_be";
        case ERTGPU_FORMAT_CS32: return "ci32_le";
        case ERTGPU_FORMAT_CS32BE: return "ci32_be";
        case ERTGPU_FORMAT_CU32: return "cu32_le";
        case ERTGPU_FORMAT_CU32BE: return "cu32_be";
        case ERTGPU_FORMAT_CF64: return "cf64_le";
        case ERTGPU_FORMAT_CF64BE: return "cf64_be";
        default: return nullptr;
    }
}

// The default gain of a format, which maps full scale to full scale (0 for cu8, which is not scaled).
inline float fmt_default_scale(int f) {
    switch (f) {
        case ERTGPU_FORMAT_CU8: return 0.0f;
        case ERTGPU_FORMAT_CS8: return 1.0f;
        case ERTGPU_FORMAT_CS16: case ERTGPU_FORMAT_CS16BE: case ERTGPU_FORMAT_CU16: case ERTGPU_FORMAT_CU16BE: return 1.0f / 256.0f;
        case ERTGPU_FORMAT_CS32: case ERTGPU_FORMAT_CS32BE: case ERTGPU_FORMAT_CU32: case ERTGPU_FORMAT_CU32BE: return 1.0f / 16777216.0f;
        default: return 128.0f;   // float32 and float64
    }
}

// One IQ component x (int8, int16 or float32, exact in float32) times g as the decoder's byte.  The product is one
// float32 multiply rounded to nearest even (__fmul_rn: never contracted).  NaN is decided here, before fmaxf (which
// would return -128) and cvt.rni (which has its own NaN rule) see it; infinities clamp.
__device__ __forceinline__ uint32_t fmt_byte(float x, float g) {
    const float p = __fmul_rn(x, g);
    if (p != p) return 128u;
    return (uint32_t)(__float2int_rn(fminf(fmaxf(p, -128.0f), 127.0f)) + 128);
}

// The same in double for the components float32 cannot hold: p = fl64(x * (double)g), one multiply rounded to nearest
// even, then clamped and rounded half to even in double.
__device__ __forceinline__ uint32_t fmt_byte_d(double x, float g) {
    const double p = __dmul_rn(x, (double)g);
    if (p != p) return 128u;
    return (uint32_t)(__double2int_rn(fmin(fmax(p, -128.0), 127.0)) + 128);
}

// Component c (0: I of the first sample, 1: its Q, 2: I of the next, ...) of format F (F != cu8) from the little-endian
// 32-bit words x of the samples' bytes: the value x the gain multiplies, as the type that holds it exactly (int8_t,
// int16_t, int32_t, float or double).  It is the stored value, byte permuted first for a big-endian format, less 2^15 or
// 2^31 for an unsigned one.  convert_kernel, resample_kernel and level_kernel read every component through this.
template <int F>
__device__ __forceinline__ auto fmt_x(const uint32_t* x, int c) {
    constexpr bool be = F == ERTGPU_FORMAT_CS16BE || F == ERTGPU_FORMAT_CF32BE || F == ERTGPU_FORMAT_CU16BE ||
                        F == ERTGPU_FORMAT_CS32BE || F == ERTGPU_FORMAT_CU32BE || F == ERTGPU_FORMAT_CF64BE;
    constexpr bool un = F == ERTGPU_FORMAT_CU16 || F == ERTGPU_FORMAT_CU16BE || F == ERTGPU_FORMAT_CU32 || F == ERTGPU_FORMAT_CU32BE;
    constexpr int S = fmt_sample_bytes(F);
    static_assert(F != ERTGPU_FORMAT_CU8, "cu8 is not converted");
    if constexpr (S == 2) {         // cs8: four components per word
        return (int8_t)(x[c >> 2] >> (8 * (c & 3)));
    } else if constexpr (S == 4) {  // 16-bit: one word per sample, I in the low half
        uint32_t w = x[c >> 1];
        if constexpr (be) w = __byte_perm(w, 0, 0x2301);
        if constexpr (un) w ^= 0x80008000u;   // v - 2^15 as int16
        return (int16_t)((c & 1) ? w >> 16 : w & 0xffffu);
    } else if constexpr (S == 8) {  // 32-bit: one word per component
        uint32_t w = x[c];
        if constexpr (be) w = __byte_perm(w, 0, 0x0123);
        if constexpr (F == ERTGPU_FORMAT_CF32 || F == ERTGPU_FORMAT_CF32BE) {
            return __uint_as_float(w);
        } else {
            if constexpr (un) w ^= 0x80000000u;   // v - 2^31 as int32
            return (int32_t)w;
        }
    } else {                        // float64: two words per component
        uint32_t lo = x[2 * c], hi = x[2 * c + 1];
        if constexpr (be) {
            const uint32_t t = __byte_perm(lo, 0, 0x0123);
            lo = __byte_perm(hi, 0, 0x0123);
            hi = t;
        }
        return __hiloint2double((int)hi, (int)lo);
    }
}

// A component as the decoder's byte: float32 arithmetic for the types float32 holds exactly, double for the others.
__device__ __forceinline__ uint32_t fmt_byte_x(int8_t x, float g) { return fmt_byte((float)x, g); }
__device__ __forceinline__ uint32_t fmt_byte_x(int16_t x, float g) { return fmt_byte((float)x, g); }
__device__ __forceinline__ uint32_t fmt_byte_x(float x, float g) { return fmt_byte(x, g); }
__device__ __forceinline__ uint32_t fmt_byte_x(int32_t x, float g) { return fmt_byte_d((double)x, g); }
__device__ __forceinline__ uint32_t fmt_byte_x(double x, float g) { return fmt_byte_d(x, g); }

template <int F>
__device__ __forceinline__ uint32_t fmt_comp(const uint32_t* x, int c, float g) { return fmt_byte_x(fmt_x<F>(x, c), g); }

// The bytes of IQ sample j of format F (F != cu8) at src: I in the low byte, Q in the high byte.
template <int F>
__device__ __forceinline__ uchar2 fmt_sample(const uint8_t* src, long long j, float g) {
    constexpr int S = fmt_sample_bytes(F);
    uint32_t x[(S + 3) / 4];
    // cs8, cs16 and cf32 are loaded as the vector of their components, which the compiler reads in place
    if constexpr (F == ERTGPU_FORMAT_CS8) {
        const char2 v = *reinterpret_cast<const char2*>(src + 2 * j);
        x[0] = (uint32_t)(uint8_t)v.x | (uint32_t)(uint8_t)v.y << 8;
    } else if constexpr (F == ERTGPU_FORMAT_CS16) {
        const short2 v = *reinterpret_cast<const short2*>(src + 4 * j);
        x[0] = (uint32_t)(uint16_t)v.x | (uint32_t)(uint16_t)v.y << 16;
    } else if constexpr (F == ERTGPU_FORMAT_CF32) {
        const float2 v = *reinterpret_cast<const float2*>(src + 8 * j);
        x[0] = __float_as_uint(v.x);
        x[1] = __float_as_uint(v.y);
    } else if constexpr (S == 4) {
        x[0] = *reinterpret_cast<const uint32_t*>(src + 4 * j);
    } else if constexpr (S == 8) {
        const uint2 v = *reinterpret_cast<const uint2*>(src + 8 * j);
        x[0] = v.x;
        x[1] = v.y;
    } else {
        const uint4 v = *reinterpret_cast<const uint4*>(src + 16 * j);
        x[0] = v.x;
        x[1] = v.y;
        x[2] = v.z;
        x[3] = v.w;
    }
    return make_uchar2((unsigned char)fmt_comp<F>(x, 0, g), (unsigned char)fmt_comp<F>(x, 1, g));
}

// The wide component of the channel path (include/ertgpu_resample.h): s_w = clamp(rint(p * 2^7), +-16383), NaN -> 0,
// with p the product fmt_byte / fmt_byte_d form.  The * 2^7 is exact, and the clamp comes first, as in fmt_byte.
__device__ __forceinline__ int fmt_wide(float x, float g) {
    const float p = __fmul_rn(__fmul_rn(x, g), 128.0f);
    if (p != p) return 0;
    return __float2int_rn(fminf(fmaxf(p, -16383.0f), 16383.0f));
}
__device__ __forceinline__ int fmt_wide_d(double x, float g) {
    const double p = __dmul_rn(__dmul_rn(x, (double)g), 128.0);
    if (p != p) return 0;
    return __double2int_rn(fmin(fmax(p, -16383.0), 16383.0));
}
__device__ __forceinline__ int fmt_wide_x(int8_t x, float g) { return fmt_wide((float)x, g); }
__device__ __forceinline__ int fmt_wide_x(int16_t x, float g) { return fmt_wide((float)x, g); }
__device__ __forceinline__ int fmt_wide_x(float x, float g) { return fmt_wide(x, g); }
__device__ __forceinline__ int fmt_wide_x(int32_t x, float g) { return fmt_wide_d((double)x, g); }
__device__ __forceinline__ int fmt_wide_x(double x, float g) { return fmt_wide_d(x, g); }

// IQ sample j of format F at src as one word of int16 s_w,I | s_w,Q << 16.
template <int F>
__device__ __forceinline__ uint32_t fmt_wide_sample(const uint8_t* src, long long j, float g) {
    if constexpr (F == ERTGPU_FORMAT_CU8) {
        const uchar2 u = *reinterpret_cast<const uchar2*>(src + 2 * j);
        return ((uint32_t)(64 * (2 * (int)u.x - 255)) & 0xffffu) | ((uint32_t)(64 * (2 * (int)u.y - 255)) << 16);
    } else {
        constexpr int S = fmt_sample_bytes(F);
        uint32_t x[(S + 3) / 4];
        if constexpr (S == 2) {
            x[0] = *reinterpret_cast<const uint16_t*>(src + 2 * j);
        } else if constexpr (S == 4) {
            x[0] = *reinterpret_cast<const uint32_t*>(src + 4 * j);
        } else if constexpr (S == 8) {
            const uint2 v = *reinterpret_cast<const uint2*>(src + 8 * j);
            x[0] = v.x;
            x[1] = v.y;
        } else {
            const uint4 v = *reinterpret_cast<const uint4*>(src + 16 * j);
            x[0] = v.x;
            x[1] = v.y;
            x[2] = v.z;
            x[3] = v.w;
        }
        return ((uint32_t)fmt_wide_x(fmt_x<F>(x, 0), g) & 0xffffu) | ((uint32_t)fmt_wide_x(fmt_x<F>(x, 1), g) << 16);
    }
}

constexpr int kCvtThreads = 256;

// Native-rate conversion of ngroups groups of 8 IQ samples (16 output bytes each) from `in` (16-byte aligned, format
// F) to `out` (16-byte aligned).  Grid-stride loop; each group is one, two, four or eight 16-byte loads and one 16-byte
// store.
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
        uint32_t x[4 * kLoads];
#pragma unroll
        for (int k = 0; k < kLoads; k++) {
            x[4 * k] = v[k].x;
            x[4 * k + 1] = v[k].y;
            x[4 * k + 2] = v[k].z;
            x[4 * k + 3] = v[k].w;
        }
        uint32_t w[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if constexpr (F == ERTGPU_FORMAT_CS8) {
                uint32_t o = 0;
#pragma unroll
                for (int b = 0; b < 4; b++) o |= fmt_comp<F>(x, 4 * k + b, g) << (8 * b);
                w[k] = o;
            } else {
                w[k] = fmt_comp<F>(x, 4 * k, g) | fmt_comp<F>(x, 4 * k + 1, g) << 8 | fmt_comp<F>(x, 4 * k + 2, g) << 16 |
                       fmt_comp<F>(x, 4 * k + 3, g) << 24;
            }
        }
        reinterpret_cast<uint4*>(out)[grp] = make_uint4(w[0], w[1], w[2], w[3]);
    }
}

}  // namespace ert
