// signal.cuh -- per-packet signal reports (include/ertgpu_signal.h has the definitions): one warp per emitted candidate
// sums the powers of its high and low chips and the lag-1 correlation of its high chips over the decoder's own bytes.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ertgpu_signal.h"
#include "ert_common.cuh"

namespace ert {

constexpr int kSignalWarps = 8;

// Sample j of the call (j < 0: the history in front of it), as mag_at reads it; false before the stream's first sample.
__device__ __forceinline__ bool signal_sample(const uint8_t* __restrict__ iq, const uint8_t* __restrict__ hist,
                                              int hist_samples, int hist_valid, long long j, int* si, int* sq) {
    const uint8_t* p;
    if (j >= 0) {
        p = iq + 2 * j;
    } else {
        if (-j > hist_valid) return false;
        p = hist + 2 * ((long long)hist_samples + j);
    }
    const uint32_t v = *reinterpret_cast<const uint16_t*>(p);  // I in the low byte, Q in the high byte
    *si = 2 * (int)(v & 0xFFu) - 255;
    *sq = 2 * (int)(v >> 8) - 255;
    return true;
}

__device__ __forceinline__ long long warp_sum(long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    return v;
}

// Records of the counters[kCntOut] candidates of the pipeline (at most cap) whose bytes are at iq (call sample 0 =
// block first_block's first sample) behind the history hist.
__global__ void __launch_bounds__(kSignalWarps * 32)
packet_signal_kernel(const uint8_t* __restrict__ iq, const uint8_t* __restrict__ hist, int hist_samples, int hist_valid,
                     const __grid_constant__ ertsig_geometry geo, long long first_block,
                     const ertgpu_candidate* __restrict__ cands, unsigned long long cap,
                     const unsigned long long* __restrict__ counters, ertgpu_signal* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    unsigned long long n = counters[kCntOut];
    if (n > cap) n = cap;
    const int g = geo.CL >> 2, m = geo.CL - 2 * g;  // inner samples per chip
    for (unsigned long long w = (unsigned long long)blockIdx.x * kSignalWarps + (threadIdx.x >> 5); w < n;
         w += (unsigned long long)gridDim.x * kSignalWarps) {
        const ertgpu_candidate& c = cands[w];
        const int proto = ertsig_protocol(&geo, c.preamble_id, c.check_mask);
        const int symbols = proto < 0 ? 0 : geo.span[proto] - 1;
        const long long a0 = ertsig_first_sample(&geo, c.block - first_block, c.idx);
        long long n_on = 0, e_on = 0, n_off = 0, e_off = 0, r_re = 0, r_im = 0, n_pairs = 0;
        // one symbol at a time: its bit is read once, lanes stride over its 2m inner samples (first chip, then second)
        for (int k = 1; k <= symbols; k++) {
            const bool first_high = ertsig_bit(c.bytes, k, geo.PK) != 0;
            const long long s0 = a0 + (long long)k * geo.SL;
            for (int t = lane; t < 2 * m; t += 32) {
                const int chip = t >= m, q = g + t - chip * m;
                const long long j = s0 + chip * geo.CL + q;
                int si, sq;
                if (!signal_sample(iq, hist, hist_samples, hist_valid, j, &si, &sq)) continue;
                const long long e = si * si + sq * sq;
                if ((chip == 0) != first_high) {
                    n_off++;
                    e_off += e;
                    continue;
                }
                n_on++;
                e_on += e;
                int pi, pq;
                if (q > g && signal_sample(iq, hist, hist_samples, hist_valid, j - 1, &pi, &pq)) {
                    r_re += si * pi + sq * pq;  // s[n] conj(s[n-1])
                    r_im += sq * pi - si * pq;
                    n_pairs++;
                }
            }
        }
        n_on = warp_sum(n_on); e_on = warp_sum(e_on); n_off = warp_sum(n_off); e_off = warp_sum(e_off);
        r_re = warp_sum(r_re); r_im = warp_sum(r_im); n_pairs = warp_sum(n_pairs);
        if (lane == 0) {
            ertgpu_signal s;
            s.n_on = n_on; s.e_on = e_on; s.n_off = n_off; s.e_off = e_off;
            s.r_re = r_re; s.r_im = r_im; s.n_pairs = n_pairs;
            s.protocol = proto;
            s.symbols = symbols;
            out[w] = s;
        }
    }
}

}  // namespace ert
