// demod_generic.cuh -- magnitude + Manchester matched filter + quantize + pack for ANY chip
// length, one thread per reference block ("chain").
//
// Replaces, fused into one pass: MagLUT.Execute (protocol/decode.go:219-225), Filter
// (decode.go:229-245) and the bit packing of Search (decode.go:259-265).
//
// Why one thread per block: Filter restarts its float32 running sum at every block and adds
// strictly left to right (decode.go:232-236); any re-association changes ~1e-5..6e-4 of the sign
// bits (SURVEY.md section 2.2), so the only exact parallelism is ACROSS blocks.  Each thread
// therefore walks one block's BS+SL samples in order; a warp owns 32 consecutive blocks.
//
// Algebra used (bit-identical to the reference expression at decode.go:242):
//   A[j] = fl(c[j+CL] - c[j])                       one subtraction per sample
//   f[i] = fl(A[i] - A[i+CL]) = fl((c[i+CL]-c[i]) - (c[i+SL]-c[i+CL]))
// so a ring of CL running sums and a ring of CL chip sums replace the csum array.
//
// This variant keeps both rings in shared memory laid out [ring slot][lane] (conflict free)
// and takes CL at run time.  It is the correctness baseline and the path for chip lengths
// without a specialised kernel (demod_fast.cuh).
#pragma once

#include "ert_common.cuh"

namespace ert {

// One IQ sample's magnitude, sample index j relative to the first sample of the call.
// j < 0 reaches into the IQ history kept from the previous call; before the start of the
// stream the reference's Signal buffer holds zeros (decode.go:144).
__device__ __forceinline__ float mag_at(const uint8_t* __restrict__ iq, const uint8_t* __restrict__ hist,
                                        int hist_samples, int hist_valid, long long j,
                                        const float* __restrict__ lut) {
    const uint8_t* p;
    if (j >= 0) {
        p = iq + 2 * j;
    } else {
        if (-j > hist_valid) return 0.0f;
        p = hist + 2 * ((long long)hist_samples + j);
    }
    const uint32_t iq16 = *reinterpret_cast<const uint16_t*>(p);  // I in the low byte, Q in the high byte (2-byte aligned)
    return __fadd_rn(lut[iq16 & 0xFFu], lut[iq16 >> 8]);
}

// grid: ceil(nblocks / blockDim.x) CTAs; dynamic smem: (256 + 2*CL*blockDim.x) floats
__global__ void demod_generic_kernel(const uint8_t* __restrict__ iq, const uint8_t* __restrict__ hist,
                                     int hist_samples, int hist_valid, const float* __restrict__ lut_g,
                                     uint32_t* __restrict__ plane_out,  // word 0 = first bit of block 0 of the call
                                     long long nblocks, int BS, int CL) {
    extern __shared__ float gen_smem[];
    float* lut = gen_smem;                       // 256
    float* cring = gen_smem + 256;                 // [CL][blockDim.x]
    float* aring = cring + CL * blockDim.x;    // [CL][blockDim.x]
    const int tid = threadIdx.x, nthr = blockDim.x;
    for (int i = tid; i < 256; i += nthr) lut[i] = lut_g[i];
    for (int r = 0; r < CL; r++) {
        cring[r * nthr + tid] = 0.0f;
        aring[r * nthr + tid] = 0.0f;
    }
    __syncthreads();

    const long long b = (long long)blockIdx.x * nthr + tid;
    if (b >= nblocks) return;
    const int SL = 2 * CL;
    const long long first = b * BS - SL;  // first sample of Signal[0] for this block
    uint32_t* out = plane_out + b * (BS >> 5);

    float c = 0.0f;
    int r = 0;
    uint32_t word = 0;
    int nbits = 0, wi = 0;
    const int steps = BS + SL - 1;  // csum[BS+SL] is never read by Filter
    for (int t = 0; t < steps; t++) {
        const long long j = first + t;
        float m;
        if (j >= 0) {
            const uint8_t* p = iq + 2 * j;
            m = __fadd_rn(lut[p[0]], lut[p[1]]);
        } else {
            m = mag_at(iq, hist, hist_samples, hist_valid, j, lut);
        }
        c = __fadd_rn(c, m);                         // csum[t+1]
        const float c_old = cring[r * nthr + tid];   // csum[t+1-CL]
        cring[r * nthr + tid] = c;
        const float a = __fsub_rn(c, c_old);         // A[t+1-CL]
        const float a_old = aring[r * nthr + tid];   // A[t+1-SL]
        aring[r * nthr + tid] = a;
        if (t >= SL - 1) {
            const float f = __fsub_rn(a_old, a);     // f[t+1-SL]
            word = (word << 1) | (1u - (__float_as_uint(f) >> 31));  // decode.go:243
            if (++nbits == 32) {
                out[wi++] = word;
                nbits = 0;
                word = 0;
            }
        }
        r = (r + 1 == CL) ? 0 : r + 1;
    }
}

// ---- parity taps -----------------------------------------------------------------------

// Decoder.Signal and Decoder.csum exactly as after the Decode of block b (relative to call).
__global__ void tap_signal_csum_kernel(const uint8_t* __restrict__ iq, const uint8_t* __restrict__ hist,
                                       int hist_samples, int hist_valid, const float* __restrict__ lut,
                                       long long b, int BS, int SL, float* __restrict__ signal,
                                       float* __restrict__ csum) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    const long long first = b * BS - SL;
    float c = 0.0f;
    csum[0] = 0.0f;
    for (int t = 0; t < BS + SL; t++) {
        const float m = mag_at(iq, hist, hist_samples, hist_valid, first + t, lut);
        signal[t] = m;
        c = __fadd_rn(c, m);
        csum[t + 1] = c;
    }
}

// r900 Parser.quantized after the Parse of block b (r900/r900.go:96-149): chain over BUF
// magnitudes starting at sample (b+1)*BS - BUF, then the three 4-chip correlators.
__global__ void tap_r900_csum_kernel(const uint8_t* __restrict__ iq, const uint8_t* __restrict__ hist,
                                     int hist_samples, int hist_valid, const float* __restrict__ lut,
                                     long long b, int BS, int BUF, float* __restrict__ csum) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    const long long first = (b + 1) * BS - BUF;
    float c = 0.0f;
    csum[0] = 0.0f;
    for (int t = 0; t < BUF; t++) {
        c = __fadd_rn(c, mag_at(iq, hist, hist_samples, hist_valid, first + t, lut));
        csum[t + 1] = c;
    }
}

// one r900 digit from five running sums (r900/r900.go:119-149)
__device__ __forceinline__ uint8_t r900_digit(float s0, float s1, float s2, float s3, float s4) {
    const float c0 = s0;
    const float c1 = __fadd_rn(s1, s1);
    const float c2 = __fadd_rn(s2, s2);
    const float c3 = __fadd_rn(s3, s3);
    const float c4 = s4;
    const float a0 = __fsub_rn(__fsub_rn(c2, c4), c0);                                        // 1100
    const float a1 = __fsub_rn(__fsub_rn(__fadd_rn(__fsub_rn(c1, c2), c3), c4), c0);          // 1010
    const float a2 = __fsub_rn(__fadd_rn(__fsub_rn(c1, c3), c4), c0);                         // 1001
    float best = fabsf(a0), win = a0;
    int arg = 0;
    if (fabsf(a1) > best) { best = fabsf(a1); arg = 1; win = a1; }
    if (fabsf(a2) > best) { best = fabsf(a2); arg = 2; win = a2; }
    if (win > 0.0f) arg += 3;
    return (uint8_t)arg;
}

__global__ void tap_r900_digits_kernel(const float* __restrict__ csum, int BUF, int CL,
                                       uint8_t* __restrict__ quantized) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= BUF) return;
    const int limit = BUF - 4 * CL;
    uint8_t d = 0;
    if (i < limit) d = r900_digit(csum[i], csum[i + CL], csum[i + 2 * CL], csum[i + 3 * CL], csum[i + 4 * CL]);
    quantized[i] = d;
}

}  // namespace ert
