// Input-rate resampler: IQ at R_in -> uint8 IQ at R_out = DataRate * ChipLength, in front of the demod.
// The arithmetic is include/ertgpu_resample.h's, all of it integer, so the bytes do not depend on the order
// in which anything is summed.  Input of another format (convert.cuh) is converted to uint8 as it is staged.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ertgpu_resample.h"
#include "convert.cuh"

namespace ert {

constexpr int kRsThreads = 256;
constexpr int kRsPerThread = 8;
constexpr long long kRsTile = (long long)kRsThreads * kRsPerThread;  // outputs per tile

struct RsArgs {
    // input samples [hist_first, hist_first + hist_n) are in hist (uint8), the next cur_n ones in cur (the handle's format)
    const uint8_t* hist;
    const uint8_t* cur;
    long long hist_first, hist_n, cur_n;
    // outputs [n0, n0 + count): output n0 + i goes to out[2i..2i+1] and, when i >= split, also to out2[2(i - split)]
    long long n0, count, split;
    // n0 - base_n < L + count keeps (n - base_n) * M in 64 bits: k_n = base_k + floor((n - base_n) * M / L)
    long long base_n, base_k;
    uint8_t* out;
    uint8_t* out2;
    // input samples [carry_first, carry_first + carry_n) are copied to carry_dst (the next call's history)
    uint8_t* carry_dst;
    long long carry_first, carry_n;
    long long L, M;
    // stepping kRsThreads outputs: phase + step_phi (wrapping at L), k + step_k, q + step_q remainder step_r
    long long step_k, step_phi, step_q, step_r;
    int T;
    float scale;  // g of the input format (not read for uint8 input)
    // tuned instances only: the mixer table E (ertrs_nco_table), the NCO step W and the table's sub-phases P
    const uint32_t* E;
    uint32_t W;
    int P;
    // wide instances only (resample_wide_kernel): the channel gain k, and the histogram that replaces the output bytes
    // when not null (ertgpu_measure_channel)
    int gain;
    unsigned long long* level;
};

// The input format of a wide cascade's second stage: the first stage's s_w pairs (ertrs_wide_mid), already mixed.
constexpr int kFmtMid = -1;

// The table as the kernel reads it: A[p][t] = h0 * 2^F + 2^(F-1) (int32), D[p][m] = the int16 pair
// (h1 - h0 of taps 2m, 2m+1), so that c_t = (A + d * w) >> F.  P rows each.
inline void rs_pack_table(const int16_t* table, int P, int T, int32_t* A, uint32_t* D) {
    for (int p = 0; p < P; p++)
        for (int t = 0; t < T; t++) {
            const int32_t h0 = table[p * T + t], d = (int32_t)table[(p + 1) * T + t] - h0;
            A[p * T + t] = h0 * (1 << ERTRS_F) + (1 << (ERTRS_F - 1));
            if (t & 1) D[p * (T / 2) + t / 2] |= (uint32_t)d << 16;
            else D[p * (T / 2) + t / 2] = (uint32_t)d & 0xffffu;
        }
}

// Input sample g as uint8 IQ: from the history as it is, from cur converted from format F.
template <int F>
__device__ __forceinline__ uchar2 rs_input(const RsArgs& a, long long g) {  // g >= 0
    const long long e = a.hist_first + a.hist_n;
    if constexpr (F == ERTGPU_FORMAT_CU8) {
        const uint8_t* src = g < e ? a.hist + 2 * (g - a.hist_first) : a.cur + 2 * (g - e);
        return *reinterpret_cast<const uchar2*>(src);
    } else {
        if (g < e) return *reinterpret_cast<const uchar2*>(a.hist + 2 * (g - a.hist_first));
        return fmt_sample<F>(a.cur, g - e, a.scale);
    }
}

// Input sample g of a wide instance as one word of int16 s_w,I | s_w,Q << 16 (include/ertgpu_resample.h): the history
// and the first stage's output hold such words, cur is converted from format F.
template <int F, class Args>
__device__ __forceinline__ uint32_t wide_input(const Args& a, long long g) {  // g >= 0
    const long long e = a.hist_first + a.hist_n;
    if (g < e) return reinterpret_cast<const uint32_t*>(a.hist)[g - a.hist_first];
    if constexpr (F == kFmtMid) return reinterpret_cast<const uint32_t*>(a.cur)[g - e];
    else return fmt_wide_sample<F>(a.cur, g - e, a.scale);
}

// s' = s * conj(E[ph >> (32 - NCO_BITS)]) for the int16 pair s, as one word of int16 s'_I | s'_Q << 16 (ertrs_mix).
__device__ __forceinline__ uint32_t rs_mix(int si, int sq, const uint32_t* tabE, uint32_t ph) {
    const uint32_t e = tabE[ph >> (32 - ERTRS_NCO_BITS)];
    const int c = (int)(short)(e & 0xffffu), s = (int)e >> 16;
    const int mi = (si * c + sq * s + (1 << (ERTRS_E_S - 1))) >> ERTRS_E_S;
    const int mq = (sq * c - si * s + (1 << (ERTRS_E_S - 1))) >> ERTRS_E_S;
    return ((uint32_t)mi & 0xffffu) | ((uint32_t)mq << 16);
}

// The tuned resampler (ertrs_plan_tuned): as below, but every staged sample is mixed by E[k_g] first, so X[j] holds
// the int16 pair (s'_I[j], s'_Q[j]) with s' = 0 before the stream start, and the taps are plain multiply-adds (dp2a
// takes only 8-bit samples).  One path serves every output.  P is the plan's (a.P).
// WIDE: the channel path of include/ertgpu_resample.h.  The staged and carried samples are s_w words (wide_input), the
// byte is ertrs_wide_byte at k = a.gain, or, with a.level, floor(log2 |acc|) is counted there instead.  F = kFmtMid
// reads a first stage's output at W = 0 without mixing (E[0] = (2^14, 0) mixes s to s) and keeps no E.
template <int F, bool WIDE = false>
__device__ __forceinline__ void resample_tuned(const int32_t* __restrict__ g_A, const uint32_t* __restrict__ g_D,
                                               const RsArgs& a, int32_t* smem) {
    const int T = a.T, T2 = a.T / 2, P = a.P;
    unsigned int* lv = reinterpret_cast<unsigned int*>(smem);  // WIDE: the CTA's level counters, in front of the table
    int32_t* tabA = WIDE ? smem + ERTRS_GAIN_BINS : smem;
    uint32_t* tabD = reinterpret_cast<uint32_t*>(tabA + P * T);
    uint32_t* tabE = tabD + P * T2;
    uint32_t* X = F == kFmtMid ? tabE : tabE + ERTRS_NCO_N;
    for (int i = threadIdx.x; i < P * T; i += kRsThreads) tabA[i] = g_A[i];
    for (int i = threadIdx.x; i < P * T2; i += kRsThreads) tabD[i] = g_D[i];
    if constexpr (F != kFmtMid)
        for (int i = threadIdx.x; i < ERTRS_NCO_N; i += kRsThreads) tabE[i] = a.E[i];
    if constexpr (WIDE) {
        if (threadIdx.x < ERTRS_GAIN_BINS) lv[threadIdx.x] = 0;
        if (blockIdx.x == 0)
            for (long long i = threadIdx.x; i < a.carry_n; i += kRsThreads)
                reinterpret_cast<uint32_t*>(a.carry_dst)[i] = wide_input<F>(a, a.carry_first + i);
    } else if (blockIdx.x == 0) {
        for (long long i = threadIdx.x; i < a.carry_n; i += kRsThreads)
            *reinterpret_cast<uchar2*>(a.carry_dst + 2 * i) = rs_input<F>(a, a.carry_first + i);  // carry_first >= 0
    }
    const long long Q = (long long)P << ERTRS_F;
    const long long ntiles = (a.count + kRsTile - 1) / kRsTile;
    const uint32_t dph = (uint32_t)kRsThreads * a.W;  // phase accumulator step between a thread's staged samples
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long nb = a.n0 + tile * kRsTile;
        const long long ne = min(nb + kRsTile, a.n0 + a.count);
        const long long j_lo = a.base_k + ((nb - a.base_n) * a.M) / a.L - T / 2 + 1;
        const long long j_hi = a.base_k + ((ne - 1 - a.base_n) * a.M) / a.L + T / 2;
        const int nspan = (int)(j_hi - j_lo + 1);
        __syncthreads();  // the previous tile's span is no longer read (and the tables are in place)
        // (uint32)g * W + 2^19 for g = j_lo + i, exact mod 2^32 whatever the sign of j_lo
        uint32_t ph = (uint32_t)(j_lo + threadIdx.x) * a.W + (1u << (31 - ERTRS_NCO_BITS));
        for (int i = threadIdx.x; i < nspan; i += kRsThreads, ph += dph) {
            const long long g = j_lo + i;
            uint32_t xw = 0;
            if constexpr (WIDE) {
                if (g >= 0) {
                    const uint32_t w = wide_input<F>(a, g);
                    xw = F == kFmtMid ? w : rs_mix((int)(short)(w & 0xffffu), (int)w >> 16, tabE, ph);
                }
            } else if (g >= 0) {
                const uchar2 u = rs_input<F>(a, g);
                const uint32_t e = tabE[ph >> (32 - ERTRS_NCO_BITS)];
                const int c = (int)(short)(e & 0xffffu), s = (int)e >> 16;
                const int si = 2 * (int)u.x - 255, sq = 2 * (int)u.y - 255;
                const int mi = (si * c + sq * s + (1 << (ERTRS_E_S - 1))) >> ERTRS_E_S;
                const int mq = (sq * c - si * s + (1 << (ERTRS_E_S - 1))) >> ERTRS_E_S;
                xw = ((uint32_t)mi & 0xffffu) | ((uint32_t)mq << 16);
            }
            X[i] = xw;
        }
        __syncthreads();

        long long n = nb + threadIdx.x;
        if (n < ne) {
            const long long nr = n - a.base_n;
            long long k = (nr * a.M) / a.L;
            long long phi = nr * a.M - k * a.L;
            k += a.base_k;
            long long q = (phi * Q) / a.L;
            long long r = phi * Q - q * a.L;
            for (int it = 0; it < kRsPerThread && n < ne; it++) {
                const int p = (int)(q >> ERTRS_F), w = (int)(q & ((1 << ERTRS_F) - 1));
                const int32_t* A = tabA + p * T;
                const uint32_t* D = tabD + p * T2;
                const long long j0 = k - T / 2 + 1;
                const uint32_t* x = X + (int)(j0 - j_lo);
                const int tc = T / 2 - 1 + (p >= P / 2 ? 1 : 0);
                int csum = 0, ai = 0, aq = 0;
#pragma unroll 4
                for (int m = 0; m < T2; m++) {
                    const int2 a01 = *reinterpret_cast<const int2*>(A + 2 * m);
                    const uint32_t dp = D[m];
                    const int c0 = (a01.x + ((int)(dp << 16) >> 16) * w) >> ERTRS_F;
                    const int c1 = (a01.y + ((int)dp >> 16) * w) >> ERTRS_F;
                    const uint32_t x0 = x[2 * m], x1 = x[2 * m + 1];
                    csum += c0 + c1;
                    ai += c0 * (int)(short)(x0 & 0xffffu) + c1 * (int)(short)(x1 & 0xffffu);
                    aq += c0 * ((int)x0 >> 16) + c1 * ((int)x1 >> 16);
                }
                const int delta = (1 << ERTRS_S) - csum;
                const uint32_t xc = x[tc];
                ai += delta * (int)(short)(xc & 0xffffu);
                aq += delta * ((int)xc >> 16);
                if constexpr (WIDE) {
                    if (a.level) {
                        if (ai) atomicAdd(&lv[31 - __clz(abs(ai))], 1u);
                        if (aq) atomicAdd(&lv[31 - __clz(abs(aq))], 1u);
                    } else {
                        const int sh = ERTRS_S + ERTRS_WIDE_BITS - a.gain;
                        const int ui = min(255, max(0, ((ai + (1 << (sh - 1)) - 1) >> sh) + 128));
                        const int uq = min(255, max(0, ((aq + (1 << (sh - 1)) - 1) >> sh) + 128));
                        const uchar2 o = make_uchar2((unsigned char)ui, (unsigned char)uq);
                        const long long i = n - a.n0;
                        *reinterpret_cast<uchar2*>(a.out + 2 * i) = o;
                        if (i >= a.split) *reinterpret_cast<uchar2*>(a.out2 + 2 * (i - a.split)) = o;
                    }
                } else {
                    const int ui = min(255, max(0, (ai + (1 << (ERTRS_S + 8))) >> (ERTRS_S + 1)));
                    const int uq = min(255, max(0, (aq + (1 << (ERTRS_S + 8))) >> (ERTRS_S + 1)));
                    const uchar2 o = make_uchar2((unsigned char)ui, (unsigned char)uq);
                    const long long i = n - a.n0;
                    *reinterpret_cast<uchar2*>(a.out + 2 * i) = o;
                    if (i >= a.split) *reinterpret_cast<uchar2*>(a.out2 + 2 * (i - a.split)) = o;
                }
                n += kRsThreads;
                k += a.step_k;
                phi += a.step_phi;
                q += a.step_q;
                r += a.step_r;
                if (r >= a.L) { r -= a.L; q++; }
                if (phi >= a.L) { phi -= a.L; k++; q -= Q; }
            }
        }
    }
    if constexpr (WIDE) {
        if (a.level) {
            __syncthreads();
            if (threadIdx.x < ERTRS_GAIN_BINS && lv[threadIdx.x]) atomicAdd(a.level + threadIdx.x, (unsigned long long)lv[threadIdx.x]);
        }
    }
}

// Persistent grid over tiles of kRsTile outputs.  Each CTA keeps the table in shared memory and stages the input
// span of a tile as words X[j] = int8 bytes (v_I[j], v_I[j+1], v_Q[j], v_Q[j+1]), v = u - 128, so that one dp2a
// per component applies two taps: with s = 2v + 1 and sum_t c_t = 2^S, acc = 2 * sum_t c_t * v_t + 2^S.  Thread t
// computes outputs t, t + 256, ... of the tile.  Outputs whose window reaches before the stream start (s = 0 there)
// take a per-tap path.  F: the input format; the history and the carried samples are uint8 after conversion.
// TUNED: the mixing instance (resample_tuned).
template <int F, bool TUNED>
__global__ void __launch_bounds__(kRsThreads) resample_kernel(const int32_t* __restrict__ g_A,
                                                              const uint32_t* __restrict__ g_D, RsArgs a) {
    extern __shared__ __align__(16) int32_t rs_smem[];
    if constexpr (TUNED) {
        resample_tuned<F>(g_A, g_D, a, rs_smem);
        return;
    }
    const int T = a.T, T2 = a.T / 2;
    int32_t* tabA = rs_smem;
    uint32_t* tabD = reinterpret_cast<uint32_t*>(rs_smem + ERTRS_P * T);
    uint32_t* X = tabD + ERTRS_P * T2;
    for (int i = threadIdx.x; i < ERTRS_P * T; i += blockDim.x) tabA[i] = g_A[i];
    for (int i = threadIdx.x; i < ERTRS_P * T2; i += blockDim.x) tabD[i] = g_D[i];
    if (blockIdx.x == 0)
        for (long long i = threadIdx.x; i < a.carry_n; i += blockDim.x)
            *reinterpret_cast<uchar2*>(a.carry_dst + 2 * i) = rs_input<F>(a, a.carry_first + i);  // carry_first >= 0
    const long long Q = (long long)ERTRS_P << ERTRS_F;
    const long long ntiles = (a.count + kRsTile - 1) / kRsTile;
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long nb = a.n0 + tile * kRsTile;
        const long long ne = min(nb + kRsTile, a.n0 + a.count);
        const long long j_lo = a.base_k + ((nb - a.base_n) * a.M) / a.L - T / 2 + 1;
        const long long j_hi = a.base_k + ((ne - 1 - a.base_n) * a.M) / a.L + T / 2;
        const int nspan = (int)(j_hi - j_lo + 1);
        __syncthreads();  // the previous tile's span is no longer read (and the table is in place)
        for (int i = threadIdx.x; i < nspan; i += blockDim.x) {
            const long long g = j_lo + i;
            const uchar2 u0 = g >= 0 ? rs_input<F>(a, g) : make_uchar2(128, 128);
            const uchar2 u1 = (i + 1 < nspan && g + 1 >= 0) ? rs_input<F>(a, g + 1) : make_uchar2(128, 128);
            X[i] = ((uint32_t)u0.x | ((uint32_t)u1.x << 8) | ((uint32_t)u0.y << 16) | ((uint32_t)u1.y << 24)) ^ 0x80808080u;
        }
        __syncthreads();

        long long n = nb + threadIdx.x;
        if (n < ne) {
            const long long nr = n - a.base_n;
            long long k = (nr * a.M) / a.L;
            long long phi = nr * a.M - k * a.L;
            k += a.base_k;
            long long q = (phi * Q) / a.L;
            long long r = phi * Q - q * a.L;
            for (int it = 0; it < kRsPerThread && n < ne; it++) {
                const int p = (int)(q >> ERTRS_F), w = (int)(q & ((1 << ERTRS_F) - 1));
                const int32_t* A = tabA + p * T;
                const uint32_t* D = tabD + p * T2;
                const long long j0 = k - T / 2 + 1;
                const uint32_t* x = X + (int)(j0 - j_lo);
                const int tc = T / 2 - 1 + (p >= ERTRS_P / 2 ? 1 : 0);
                int ai, aq;
                if (j0 >= 0) {
                    int csum = 0, vi = 0, vq = 0;
#pragma unroll 4
                    for (int m = 0; m < T2; m++) {
                        const int2 a01 = *reinterpret_cast<const int2*>(A + 2 * m);
                        const uint32_t dp = D[m];
                        const int c0 = (a01.x + ((int)(dp << 16) >> 16) * w) >> ERTRS_F;
                        const int c1 = (a01.y + ((int)dp >> 16) * w) >> ERTRS_F;
                        const int cp = (int)__byte_perm((uint32_t)c0, (uint32_t)c1, 0x5410);
                        const int xv = (int)x[2 * m];
                        csum = __dp2a_lo(cp, 0x0101, csum);
                        vi = __dp2a_lo(cp, xv, vi);
                        vq = __dp2a_hi(cp, xv, vq);
                    }
                    const int delta = (1 << ERTRS_S) - csum;
                    const uint32_t xc = x[tc];
                    vi += delta * (int)(signed char)(xc & 0xffu);
                    vq += delta * (int)(signed char)((xc >> 16) & 0xffu);
                    ai = 2 * vi + (1 << ERTRS_S);
                    aq = 2 * vq + (1 << ERTRS_S);
                } else {  // the window reaches before the stream start: s = 0 there
                    int csum = 0;
                    ai = aq = 0;
                    int ci_c = 0, cq_c = 0;
                    for (int t = 0; t < T; t++) {
                        const uint32_t dp = D[t >> 1];
                        const int d = (t & 1) ? ((int)dp >> 16) : ((int)(dp << 16) >> 16);
                        const int c = (A[t] + d * w) >> ERTRS_F;
                        csum += c;
                        if (j0 + t < 0) continue;
                        const uint32_t xt = x[t];
                        const int si = 2 * (int)(signed char)(xt & 0xffu) + 1, sq = 2 * (int)(signed char)((xt >> 16) & 0xffu) + 1;
                        ai += c * si;
                        aq += c * sq;
                        if (t == tc) { ci_c = si; cq_c = sq; }
                    }
                    const int delta = (1 << ERTRS_S) - csum;
                    ai += delta * ci_c;
                    aq += delta * cq_c;
                }
                const int ui = min(255, max(0, (ai + (1 << (ERTRS_S + 8))) >> (ERTRS_S + 1)));
                const int uq = min(255, max(0, (aq + (1 << (ERTRS_S + 8))) >> (ERTRS_S + 1)));
                const uchar2 o = make_uchar2((unsigned char)ui, (unsigned char)uq);
                const long long i = n - a.n0;
                *reinterpret_cast<uchar2*>(a.out + 2 * i) = o;
                if (i >= a.split) *reinterpret_cast<uchar2*>(a.out2 + 2 * (i - a.split)) = o;
                // next output of this thread: n + kRsThreads
                n += kRsThreads;
                k += a.step_k;
                phi += a.step_phi;
                q += a.step_q;
                r += a.step_r;
                if (r >= a.L) { r -= a.L; q++; }
                if (phi >= a.L) { phi -= a.L; k++; q -= Q; }
            }
        }
    }
}

// Shared memory of one CTA: the table (A and D) of P sub-phases, the words of the largest input span of a tile and,
// for a tuned instance, the mixer table E.
inline size_t rs_smem_bytes(int P, int T, long long L, long long M, bool tuned) {
    const long long span = ((kRsTile - 1) * M + L - 1) / L + 1 + T + 1;
    return (size_t)P * T * 6 + (size_t)span * 4 + (tuned ? (size_t)ERTRS_NCO_N * 4 : 0);
}

// The wide channel path's resampler (include/ertgpu_resample.h): resample_tuned<F, true>, the one stage of a wide tuned
// handle or, with F = kFmtMid, the second stage of a wide decimating one.
template <int F>
__global__ void __launch_bounds__(kRsThreads) resample_wide_kernel(const int32_t* __restrict__ g_A,
                                                                   const uint32_t* __restrict__ g_D, RsArgs a) {
    extern __shared__ __align__(16) int32_t rs_smem[];
    resample_tuned<F, true>(g_A, g_D, a, rs_smem);
}

// Its shared memory: rs_smem_bytes of a tuned instance (without E for kFmtMid), and the level counters.
inline size_t rs_wide_smem_bytes(int P, int T, long long L, long long M, bool mid) {
    return rs_smem_bytes(P, T, L, M, !mid) + ERTRS_GAIN_BINS * 4;
}

}  // namespace ert
