// Stage 1 of a decimating tuned input (ertgpu_allow_input_decimation): IQ at R_in -> uint8 IQ at R_mid = R_in / D,
// the channel mixed to 0 Hz and lowpassed on the way, as include/ertgpu_resample.h states it (all integer).  The
// untuned uint8 resample_kernel (resample.cuh) then takes R_mid to R_out.  Input of another format (convert.cuh) is
// converted to uint8 as it is staged, exactly as resample_kernel does.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ertgpu.h"
#include "../../include/ertgpu_resample.h"
#include "convert.cuh"
#include "resample.cuh"  // wide_input, rs_mix

namespace ert {

constexpr int kDcThreads = 256;
constexpr int kDcSpanWords = 20480;  // most input samples one tile stages (80 KiB, so that two CTAs fit an SM)
constexpr int kDcMaxPer = 16;        // most outputs per thread and tile
constexpr int kDcChannelsSpanWords = kDcSpanWords * 2 / 3;  // decimate_channels_kernel's: X and U in the same 80 KiB

struct DcArgs {
    // input samples [hist_first, hist_first + hist_n) are in hist (uint8), the next cur_n ones in cur (the handle's format)
    const uint8_t* hist;
    const uint8_t* cur;
    long long hist_first, hist_n, cur_n;
    // outputs [n0, n0 + count): output n0 + i goes to out[2i..2i+1]
    long long n0, count;
    uint8_t* out;
    // input samples [carry_first, carry_first + carry_n) are copied to carry_dst (the next call's history)
    uint8_t* carry_dst;
    long long carry_first, carry_n;
    int D, T1;
    int per;      // outputs of a thread per tile: a tile is kDcThreads * per outputs
    float scale;  // g of the input format (not read for uint8 input)
    const uint32_t* E;  // the mixer table (ertrs_nco_table) and its step W at R_in
    uint32_t W;
};

// Outputs a thread computes per tile, so that a tile's input span, (kDcThreads * per - 1) * D + T1 samples, fits
// span_words (for every D <= ERTRS_MAX_D).
// decimate_channels_kernel passes a smaller span_words, so that its uint8 copy of the span fits beside it.
inline int dc_per_thread(int D, int T1, int span_words = kDcSpanWords) {
    const int per = (span_words - T1) / (kDcThreads * D);
    return per < 1 ? 1 : per > kDcMaxPer ? kDcMaxPer : per;
}

// Staged word i sits at i + i / 32: lanes that read words D apart then hit different banks for every D <= 32.
__device__ __forceinline__ int dc_skew(int i) { return i + (i >> 5); }

// Shared memory of one CTA: E, the taps h_0 .. h_{T1/2-1} as int32 and the skewed span of the largest tile.
inline size_t dc_smem_bytes(int D, int T1, int per) {
    const long long span = ((long long)kDcThreads * per - 1) * D + T1;
    return ((size_t)ERTRS_NCO_N + (size_t)(T1 / 2) + (size_t)(span + (span >> 5) + 1)) * 4;
}

// Input sample g as uint8 IQ: from the history as it is, from cur converted from format F.
template <int F>
__device__ __forceinline__ uchar2 dc_input(const DcArgs& a, long long g) {  // g >= 0
    const long long e = a.hist_first + a.hist_n;
    if (g < e) return *reinterpret_cast<const uchar2*>(a.hist + 2 * (g - a.hist_first));
    if constexpr (F == ERTGPU_FORMAT_CU8) return *reinterpret_cast<const uchar2*>(a.cur + 2 * (g - e));
    else return fmt_sample<F>(a.cur, g - e, a.scale);
}

// The mixer: uint8 IQ u times E[ph >> (32 - NCO_BITS)], as one word of int16 s'_I | s'_Q << 16.
__device__ __forceinline__ uint32_t dc_mix(uchar2 u, const uint32_t* tabE, uint32_t ph) {
    const uint32_t e = tabE[ph >> (32 - ERTRS_NCO_BITS)];
    const int ce = (int)(short)(e & 0xffffu), se = (int)e >> 16;
    const int si = 2 * (int)u.x - 255, sq = 2 * (int)u.y - 255;
    const int mi = (si * ce + sq * se + (1 << (ERTRS_E_S - 1))) >> ERTRS_E_S;
    const int mq = (sq * ce - si * se + (1 << (ERTRS_E_S - 1))) >> ERTRS_E_S;
    return ((uint32_t)mi & 0xffffu) | ((uint32_t)mq << 16);
}

// The nloc outputs of a tile from its staged span X (skewed), output m to out[2m..2m+1]: the symmetric taps are
// folded, so an output takes T1/2 - 1 pair sums and the centre tap, two multiply-adds per pair.  WIDE: output m is the
// word of int16 ertrs_wide_mid(acc_I) | ertrs_wide_mid(acc_Q) << 16 at out[4m..4m+3].
template <bool WIDE = false>
__device__ __forceinline__ void dc_filter(const uint32_t* X, const int* taps, int T1, int D, int nloc, uint8_t* out) {
    const int c = T1 / 2 - 1;
    for (int m = threadIdx.x; m < nloc; m += kDcThreads) {
        const int o = m * D;  // the output's first tap reads staged word o
        int ai = 0, aq = 0;
#pragma unroll 4
        for (int t = 0; t < c; t++) {
            const uint32_t x0 = X[dc_skew(o + t)], x1 = X[dc_skew(o + T1 - 2 - t)];
            const int h = taps[t];
            ai += h * ((int)(short)(x0 & 0xffffu) + (int)(short)(x1 & 0xffffu));
            aq += h * (((int)x0 >> 16) + ((int)x1 >> 16));
        }
        const uint32_t xc = X[dc_skew(o + c)];
        ai += taps[c] * (int)(short)(xc & 0xffffu);
        aq += taps[c] * ((int)xc >> 16);
        if constexpr (WIDE) {
            const int wi = min(ERTRS_WIDE_MAX, max(-ERTRS_WIDE_MAX, (ai + (1 << (ERTRS_S - 1))) >> ERTRS_S));
            const int wq = min(ERTRS_WIDE_MAX, max(-ERTRS_WIDE_MAX, (aq + (1 << (ERTRS_S - 1))) >> ERTRS_S));
            reinterpret_cast<uint32_t*>(out)[m] = ((uint32_t)wi & 0xffffu) | ((uint32_t)wq << 16);
            continue;
        }
        const int ui = min(255, max(0, (ai + (1 << (ERTRS_S + 8))) >> (ERTRS_S + 1)));
        const int uq = min(255, max(0, (aq + (1 << (ERTRS_S + 8))) >> (ERTRS_S + 1)));
        *reinterpret_cast<uchar2*>(out + 2 * m) = make_uchar2((unsigned char)ui, (unsigned char)uq);
    }
}

// Persistent grid over tiles of kDcThreads * per outputs.  Each CTA keeps E and the taps in shared memory and stages a
// tile's input span once, each sample mixed by E[k_g] into one word of int16 s'_I | s'_Q << 16 (s' = 0 before the
// stream start).  Thread t computes outputs t, t + 256, ... of the tile, each whole (dc_filter).
// WIDE: the first stage of the wide channel path (include/ertgpu_resample.h): the staged, carried and written samples
// are s_w words (wide_input), written by dc_filter<true>.
template <int F, bool WIDE>
__device__ __forceinline__ void dc_stage(const int16_t* __restrict__ g_taps, const DcArgs& a, uint32_t* dc_smem) {
    const int T1 = a.T1, c = a.T1 / 2 - 1, D = a.D;
    uint32_t* tabE = dc_smem;
    int* taps = reinterpret_cast<int*>(dc_smem + ERTRS_NCO_N);
    uint32_t* X = dc_smem + ERTRS_NCO_N + T1 / 2;
    for (int i = threadIdx.x; i < ERTRS_NCO_N; i += kDcThreads) tabE[i] = a.E[i];
    for (int i = threadIdx.x; i <= c; i += kDcThreads) taps[i] = g_taps[i];
    if (blockIdx.x == 0)
        for (long long i = threadIdx.x; i < a.carry_n; i += kDcThreads) {
            if constexpr (WIDE) reinterpret_cast<uint32_t*>(a.carry_dst)[i] = wide_input<F>(a, a.carry_first + i);
            else *reinterpret_cast<uchar2*>(a.carry_dst + 2 * i) = dc_input<F>(a, a.carry_first + i);  // carry_first >= 0
        }
    const long long tile_n = (long long)kDcThreads * a.per;
    const long long ntiles = (a.count + tile_n - 1) / tile_n;
    const uint32_t dph = (uint32_t)kDcThreads * a.W;  // phase accumulator step between a thread's staged samples
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long nb = a.n0 + tile * tile_n;
        const long long ne = min(nb + tile_n, a.n0 + a.count);
        const long long j_lo = nb * D - T1 / 2 + 1;
        const int nspan = (int)((ne - 1 - nb) * D + T1);
        __syncthreads();  // the previous tile's span is no longer read (and E and the taps are in place)
        // (uint32)g * W + 2^19 for g = j_lo + i, exact mod 2^32 whatever the sign of j_lo
        uint32_t ph = (uint32_t)(j_lo + threadIdx.x) * a.W + (1u << (31 - ERTRS_NCO_BITS));
        for (int i = threadIdx.x; i < nspan; i += kDcThreads, ph += dph) {
            const long long g = j_lo + i;
            if constexpr (WIDE) {
                uint32_t x = 0;
                if (g >= 0) {
                    const uint32_t w = wide_input<F>(a, g);
                    x = rs_mix((int)(short)(w & 0xffffu), (int)w >> 16, tabE, ph);
                }
                X[dc_skew(i)] = x;
            } else {
                X[dc_skew(i)] = g >= 0 ? dc_mix(dc_input<F>(a, g), tabE, ph) : 0u;
            }
        }
        __syncthreads();
        if constexpr (WIDE) dc_filter<true>(X, taps, T1, D, (int)(ne - nb), a.out + 4 * (nb - a.n0));
        else dc_filter(X, taps, T1, D, (int)(ne - nb), a.out + 2 * (nb - a.n0));
    }
}

template <int F>
__global__ void __launch_bounds__(kDcThreads) decimate_kernel(const int16_t* __restrict__ g_taps, DcArgs a) {
    extern __shared__ __align__(16) uint32_t dc_smem[];
    dc_stage<F, false>(g_taps, a, dc_smem);
}

// The first stage of a wide decimating handle: s_w words in, s_w words (ertrs_wide_mid) out, into resample_wide_kernel<
// kFmtMid>.  Same shared memory and tiles as decimate_kernel.
template <int F>
__global__ void __launch_bounds__(kDcThreads) decimate_wide_kernel(const int16_t* __restrict__ g_taps, DcArgs a) {
    extern __shared__ __align__(16) uint32_t dc_smem[];
    dc_stage<F, true>(g_taps, a, dc_smem);
}

// The channels of one capture that decimate_channels_kernel serves: channel c mixes with step W[c], writes its outputs
// to out[c] and its copy of the input history to carry_dst[c].
struct DcChannels {
    uint32_t W[ERTGPU_MAX_CHANNELS];
    uint8_t* out[ERTGPU_MAX_CHANNELS];
    uint8_t* carry_dst[ERTGPU_MAX_CHANNELS];
    int n;
};

// Shared memory of one CTA of decimate_channels_kernel: decimate_kernel's, and the tile's span as uint8 IQ.
inline size_t dc_channels_smem_bytes(int D, int T1, int per) {
    const long long span = ((long long)kDcThreads * per - 1) * D + T1;
    return dc_smem_bytes(D, T1, per) + (size_t)((span + 1) / 2) * 4;
}

// decimate_kernel for ch.n channels of one capture at once.  The channels share everything of a's but W, out and
// carry_dst (a's are not read).  A tile's input span is read and converted to uint8 IQ once, into U; then, channel by
// channel, U is mixed with that channel's step into X and filtered into its outputs, with decimate_kernel's integer
// formulas, so channel c's bytes are those of decimate_kernel at W[c].  The history carry is converted once and stored
// for every channel, so that each handle keeps a history of its own.
template <int F>
__global__ void __launch_bounds__(kDcThreads) decimate_channels_kernel(const int16_t* __restrict__ g_taps, DcArgs a,
                                                                       const __grid_constant__ DcChannels ch) {
    extern __shared__ __align__(16) uint32_t dc_smem[];
    const int T1 = a.T1, c = a.T1 / 2 - 1, D = a.D;
    const long long tile_n = (long long)kDcThreads * a.per;
    const long long span_max = (tile_n - 1) * D + T1;
    uint32_t* tabE = dc_smem;
    int* taps = reinterpret_cast<int*>(dc_smem + ERTRS_NCO_N);
    uint32_t* X = dc_smem + ERTRS_NCO_N + T1 / 2;
    uchar2* U = reinterpret_cast<uchar2*>(X + span_max + (span_max >> 5) + 1);
    for (int i = threadIdx.x; i < ERTRS_NCO_N; i += kDcThreads) tabE[i] = a.E[i];
    for (int i = threadIdx.x; i <= c; i += kDcThreads) taps[i] = g_taps[i];
    if (blockIdx.x == 0)
        for (long long i = threadIdx.x; i < a.carry_n; i += kDcThreads) {
            const uchar2 u = dc_input<F>(a, a.carry_first + i);  // carry_first >= 0
            for (int k = 0; k < ch.n; k++) *reinterpret_cast<uchar2*>(ch.carry_dst[k] + 2 * i) = u;
        }
    const long long ntiles = (a.count + tile_n - 1) / tile_n;
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long nb = a.n0 + tile * tile_n;
        const long long ne = min(nb + tile_n, a.n0 + a.count);
        const long long j_lo = nb * D - T1 / 2 + 1;
        const int nspan = (int)((ne - 1 - nb) * D + T1);
        __syncthreads();  // the previous tile's U and X are no longer read (and E and the taps are in place)
        for (int i = threadIdx.x; i < nspan; i += kDcThreads) {
            const long long g = j_lo + i;
            U[i] = g >= 0 ? dc_input<F>(a, g) : make_uchar2(0, 0);  // g < 0 is mixed to 0 below, whatever U holds
        }
        for (int k = 0; k < ch.n; k++) {
            const uint32_t W = ch.W[k], dph = (uint32_t)kDcThreads * W;
            __syncthreads();  // U is staged, and the previous channel's X is no longer read
            uint32_t ph = (uint32_t)(j_lo + threadIdx.x) * W + (1u << (31 - ERTRS_NCO_BITS));
            for (int i = threadIdx.x; i < nspan; i += kDcThreads, ph += dph)
                X[dc_skew(i)] = j_lo + i >= 0 ? dc_mix(U[i], tabE, ph) : 0u;
            __syncthreads();
            dc_filter(X, taps, T1, D, (int)(ne - nb), ch.out[k] + 2 * (nb - a.n0));
        }
    }
}

}  // namespace ert
