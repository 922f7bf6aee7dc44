/*
 * ertgpu_resample.h -- the prototype lowpass of the input-rate resampler, as one header shared by
 * libertgpu.so (rtlamr_b200/csrc/resample.cuh) and by the CPU restatement the tests check it
 * against, so both use the same integer table.  Not part of the reference API: rtlamr decodes only
 * at DataRate * ChipLength samples per second (protocol/decode.go:132-133).
 *
 * Resampling R_in -> R_out = L/M * R_in (L/M reduced, 1/4 <= L/M <= 4).  Output n sits at input
 * time n*M/L: k_n = floor(n*M/L), phase phi_n = n*M mod L.  It reads the T input samples
 * k_n - T/2 + 1 ... k_n + T/2 (samples before the stream start count as s = 0).
 *
 * The table holds the windowed-sinc prototype h(d) (d in input samples, h(-d) = h(d)) at P
 * sub-phases per input sample:  table[p*T + t] = round(2^S * h(t - T/2 + 1 - p/P)) for p = 0..P
 * (row P is the extra row for interpolation).  Every row sums to exactly 2^S, and
 * table[p][t] == table[P-p][T-1-t].  The design is a Kaiser window (70 dB) on a sinc cut off at
 * half of min(R_in, R_out), with the transition band 0.40 ... 0.60 * min(R_in, R_out).
 *
 * Per output, with q = floor(phi_n * P * 2^F / L), p = q >> F, w = q & (2^F - 1):
 *   c_t = table[p][t] + (((table[p+1][t] - table[p][t]) * w + 2^(F-1)) >> F)
 *   c_{T/2-1+(p >= P/2)} += 2^S - sum_t c_t        (the tap nearest the output time; DC gain exactly 2^S)
 *   acc = sum_t c_t * s_t,   s = 2u - 255
 *   u_out = clamp((acc + 2^(S+8)) >> (S+1), 0, 255)
 * so a constant input u comes out as exactly u.  All of that is integer arithmetic; only the table
 * design below uses floating point, once, on the host.
 */
#ifndef ERTGPU_RESAMPLE_H
#define ERTGPU_RESAMPLE_H

#include <stdint.h>

#include "ertgpu.h"

#define ERTRS_P 256      /* sub-phases per input sample                   */
#define ERTRS_S 14       /* DC gain 2^S (peak tap <= 2^S fits int16)      */
#define ERTRS_F 16       /* bits of the interpolation weight              */
#define ERTRS_MAX_T 224  /* taps per output (untuned plans stay <= 88)    */
#define ERTRS_ATTEN_DB 70.0
#define ERTRS_NCO_BITS 12 /* log2 of the entries of the mixer table E     */
#define ERTRS_NCO_N (1 << ERTRS_NCO_BITS)
#define ERTRS_E_S 14      /* |E[k]| ~ 2^E_S                                */
#define ERTRS_MAX_D 64    /* largest stage-1 decimation (R_in <= 256 R_out) */

static inline int64_t ertrs_gcd(int64_t a, int64_t b) {
    while (b) {
        int64_t t = a % b;
        a = b;
        b = t;
    }
    return a;
}

/* sin(pi*x) from IEEE adds and multiplies only (no libm), so every build computes the same table */
static inline double ertrs_sinpi(double x) {
    double n = (double)(int64_t)(x >= 0 ? x + 0.5 : x - 0.5); /* nearest integer */
    double r = x - n;                                           /* |r| <= 0.5 */
    const double pr = 3.14159265358979323846 * r, p2 = pr * pr;
    double term = pr, sum = pr;
    for (int k = 1; k < 14; k++) {
        term *= -p2 / (double)((2 * k) * (2 * k + 1));
        sum += term;
    }
    return ((int64_t)n & 1) ? -sum : sum;
}

/* modified Bessel function I0 by its power series */
static inline double ertrs_i0(double x) {
    double term = 1.0, sum = 1.0;
    const double q = x * x / 4.0;
    for (int k = 1; k < 200; k++) {
        term *= q / ((double)k * (double)k);
        sum += term;
        if (term < sum * 1e-18) break;
    }
    return sum;
}

/* Fill *info for R_in -> R_out at P = ERTRS_P (rates positive, checked by the caller). */
static inline void ertrs_fill_plan(int64_t rate_in, int64_t rate_out, ertgpu_resampler_info* info) {
    const int64_t g = ertrs_gcd(rate_out, rate_in);
    info->rate_in = rate_in;
    info->rate_out = rate_out;
    info->L = rate_out / g;
    info->M = rate_in / g;
    /* cut-off scale: min(R_in, R_out) in cycles per input sample */
    const double nu = rate_out < rate_in ? (double)rate_out / (double)rate_in : 1.0;
    const double width = 0.2 * nu; /* 0.40 ... 0.60 * nu */
    const double n = (ERTRS_ATTEN_DB - 7.95) / (14.36 * width);
    int32_t T = 2 * (int32_t)((n + 1.999999) / 2.0);
    if (T < 8) T = 8;
    if (T > ERTRS_MAX_T) T = ERTRS_MAX_T;
    info->T = T;
    info->P = ERTRS_P;
    info->S = ERTRS_S;
    info->F = ERTRS_F;
}

/* Fill *info for R_in -> R_out.  Returns 0, or -1 when a rate is not positive or the ratio is outside
 * [1/4, 4]. */
static inline int ertrs_plan(int64_t rate_in, int64_t rate_out, ertgpu_resampler_info* info) {
    if (rate_in <= 0 || rate_out <= 0) return -1;
    if (rate_out * 4 < rate_in || rate_out > rate_in * 4) return -1;
    ertrs_fill_plan(rate_in, rate_out, info);
    return 0;
}

/* Number of outputs whose window lies inside the first x input samples (k_n + T/2 <= x - 1). */
static inline int64_t ertrs_out_end(const ertgpu_resampler_info* info, int64_t x) {
    const int64_t a = x - info->T / 2;
    if (a <= 0) return 0;
    return (int64_t)(((__int128)a * info->L + info->M - 1) / info->M);
}

/*
 * Tuned input (ertgpu_set_input_tuning): the channel at offset D = center - capture_center Hz from the
 * capture's centre is mixed to 0 Hz as the resampler stages its input, so the same lowpass is the channel
 * filter.  All integer:
 *   W   = round(D * 2^32 / R_in) (half away from zero) mod 2^32        (ertrs_nco_step)
 *   k_g = ((uint32)g * W + 2^19) >> 20,  g = input index since the stream start
 *   E[k] = (round(2^14 cos 2 pi k/4096), round(2^14 sin 2 pi k/4096))  (ertrs_nco_table)
 *   s'_I = (s_I C + s_Q S + 2^13) >> 14,  s'_Q = (s_Q C - s_I S + 2^13) >> 14  (floor; ertrs_mix)
 * i.e. s * e^(-j 2 pi D g / R_in), and the outputs are the untuned formula with s' for s.  |s'| <= 361.
 */

/* The plan of a tuned handle: R_out / R_in in [1/10, 4] and the channel inside the capture,
 * |D| + 0.4 * min(R_in, R_out) <= 0.5 * R_in.  T as ertrs_plan (at most ERTRS_MAX_T); P = 256 for T <= 96,
 * 128 for T <= 160 and 64 above, so that the table, one tile's input span and E fit one CTA's shared
 * memory.  Inside [1/4, 4] every plan is ertrs_plan's (T <= 88).  Returns 0 or -1. */
static inline int ertrs_plan_tuned(int64_t rate_in, int64_t rate_out, int64_t offset_hz, ertgpu_resampler_info* info) {
    if (rate_in <= 0 || rate_out <= 0) return -1;
    if (rate_out * 10 < rate_in || rate_out > rate_in * 4) return -1;
    const int64_t lo = rate_out < rate_in ? rate_out : rate_in;
    const int64_t ad = offset_hz < 0 ? -offset_hz : offset_hz;
    if (ad > rate_in || 10 * ad + 4 * lo > 5 * rate_in) return -1;
    ertrs_fill_plan(rate_in, rate_out, info);
    info->P = info->T <= 96 ? 256 : info->T <= 160 ? 128 : 64;
    return 0;
}

/*
 * Decimating tuned input (ertgpu_allow_input_decimation): above 10:1 the channel goes through two stages.
 *   Stage 1 mixes and decimates by D: the tuned formula above with L = 1, M = D and a single table row, so every output
 *     has phase 0 and no coefficient is interpolated.  Output n reads the T1 mixed samples s' at nD - T1/2 + 1 ...
 *     nD + T1/2 (s' = 0 before the stream start):  u_mid = clamp((sum_t h_t s'_t + 2^(S+8)) >> (S+1), 0, 255).
 *     h is a Kaiser-windowed (70 dB) sinc with its passband edge at 0.4 R_out, its stopband edge at R_mid - 0.6 R_out
 *     and the cut-off midway, R_mid = R_in / D; T1 (even) is the Kaiser estimate for that transition band.  The int16
 *     taps are symmetric about tap T1/2 - 1 (h_t = h_{T1-2-t}, h_{T1-1} = 0) and sum to exactly 2^S (the residual goes
 *     to the centre tap).
 *   Stage 2 is the untuned uint8 resampler of ertrs_fill_plan(R_in, D * R_out): the same L/M, T and table as
 *     R_mid -> R_out, fed with the stage-1 bytes.
 */

/* The plan of a handle that allows decimation.  R_in <= 10 R_out: D = 1, T1 = 0 and *info is ertrs_plan_tuned's.
 * 10 R_out < R_in <= 256 R_out: D = ceil(R_in / (4 R_out)) (so 3 R_out < R_mid <= 4 R_out), the channel inside the
 * capture (|offset| + 0.4 R_out <= 0.5 R_in), and *info the second stage's plan.  Returns 0 or -1. */
static inline int ertrs_plan_decimated(int64_t rate_in, int64_t rate_out, int64_t offset_hz, ertgpu_decimator_info* dec,
                                       ertgpu_resampler_info* info) {
    if (rate_in <= 0 || rate_out <= 0) return -1;
    dec->rate_in = rate_in;
    dec->rate_out = rate_out;
    dec->S = ERTRS_S;
    dec->reserved = 0;
    if (rate_in <= 10 * rate_out) {
        dec->D = 1;
        dec->T1 = 0;
        return ertrs_plan_tuned(rate_in, rate_out, offset_hz, info);
    }
    if (rate_in > ERTRS_MAX_D * 4 * rate_out) return -1;
    const int64_t ad = offset_hz < 0 ? -offset_hz : offset_hz;
    if (10 * ad + 4 * rate_out > 5 * rate_in) return -1;
    const int64_t D = (rate_in + 4 * rate_out - 1) / (4 * rate_out);
    const double width = ((double)rate_in / (double)D - (double)rate_out) / (double)rate_in; /* cycles per input sample */
    const double n = (ERTRS_ATTEN_DB - 7.95) / (14.36 * width);
    int32_t T1 = 2 * (int32_t)((n + 1.999999) / 2.0);
    if (T1 < 8) T1 = 8;
    dec->D = (int32_t)D;
    dec->T1 = T1;
    ertrs_fill_plan(rate_in, D * rate_out, info);
    return 0;
}

/* The stage-1 taps h_0 .. h_{T1-1} of a plan with D >= 2.  Returns 0, or -1 if a tap does not fit int16. */
static inline int ertrs_build_decimator(const ertgpu_decimator_info* dec, int16_t* taps) {
    const int32_t T1 = dec->T1, c = T1 / 2 - 1;
    const double half = 0.5 * (double)T1;
    const double mid = (double)dec->rate_in / (double)dec->D;
    const double fc = 0.5 * (mid - 0.2 * (double)dec->rate_out) / (double)dec->rate_in; /* cycles per input sample */
    const double beta = 0.1102 * (ERTRS_ATTEN_DB - 8.7);
    int64_t sum = 0;
    for (int32_t t = 0; t <= c; t++) { /* d = t - c <= 0; the other half mirrors it */
        const double d = (double)(t - c), z = d / half;
        const double w = ertrs_i0(beta * __builtin_sqrt(1.0 - z * z)) / ertrs_i0(beta);
        const double x = 2.0 * fc * d;
        const double sinc = x == 0.0 ? 1.0 : ertrs_sinpi(x) / (3.14159265358979323846 * x);
        const double v = (double)(1 << dec->S) * 2.0 * fc * sinc * w;
        const double r = v >= 0 ? (double)(int64_t)(v + 0.5) : -(double)(int64_t)(-v + 0.5);
        if (r > 32767.0 || r < -32768.0) return -1;
        taps[t] = taps[T1 - 2 - t] = (int16_t)r;
        sum += t == c ? (int64_t)taps[t] : 2 * (int64_t)taps[t];
    }
    taps[T1 - 1] = 0;
    const int64_t cc = taps[c] + ((1 << dec->S) - sum);
    if (cc > 32767 || cc < -32768) return -1;
    taps[c] = (int16_t)cc;
    return 0;
}

/* W = round(D * 2^32 / R_in), rounded half away from zero, modulo 2^32 (|D| <= R_in) */
static inline uint32_t ertrs_nco_step(int64_t offset_hz, int64_t rate_in) {
    const int64_t ad = offset_hz < 0 ? -offset_hz : offset_hz;
    const int64_t w = (int64_t)((((__int128)ad << 33) + rate_in) / ((__int128)2 * rate_in));
    return (uint32_t)(offset_hz < 0 ? -w : w);
}

/* E[k] = C | S << 16 (int16 each), k = 0 .. ERTRS_NCO_N - 1; sin and cos from ertrs_sinpi, no libm */
static inline void ertrs_nco_table(uint32_t* E) {
    for (int32_t k = 0; k < ERTRS_NCO_N; k++) {
        const double c = (double)(1 << ERTRS_E_S) * ertrs_sinpi((double)(k + ERTRS_NCO_N / 4) / (double)(ERTRS_NCO_N / 2));
        const double s = (double)(1 << ERTRS_E_S) * ertrs_sinpi((double)k / (double)(ERTRS_NCO_N / 2));
        const int32_t ci = (int32_t)(c >= 0 ? (int64_t)(c + 0.5) : -(int64_t)(-c + 0.5));
        const int32_t si = (int32_t)(s >= 0 ? (int64_t)(s + 0.5) : -(int64_t)(-s + 0.5));
        E[k] = ((uint32_t)ci & 0xffffu) | ((uint32_t)si << 16);
    }
}

/* phase index of input sample g */
static inline uint32_t ertrs_nco_index(int64_t g, uint32_t W) {
    return ((uint32_t)g * W + (1u << (31 - ERTRS_NCO_BITS))) >> (32 - ERTRS_NCO_BITS);
}

/* s' = s * conj(E[k]) for s = (si, sq) */
static inline void ertrs_mix(int32_t si, int32_t sq, uint32_t e, int32_t* oi, int32_t* oq) {
    const int32_t c = (int32_t)(int16_t)(e & 0xffffu), s = (int32_t)(int16_t)(e >> 16);
    *oi = (si * c + sq * s + (1 << (ERTRS_E_S - 1))) >> ERTRS_E_S;
    *oq = (sq * c - si * s + (1 << (ERTRS_E_S - 1))) >> ERTRS_E_S;
}

/*
 * The wide channel path of a tuned handle (ertgpu_set_channel_gain): the input keeps 15 bits through the mixer and the
 * channel filter, and the decoder's byte is formed only from the last stage's accumulator, with a channel gain 2^k.
 *   Wide component  s_w = isnan(p) ? 0 : clamp(rint(p), -16383, 16383), p = (x * g) * 2^7 with convert.cuh's product
 *                   (fl32(x * g) for components float32 holds exactly, fl64(x * (double)g) otherwise; the * 2^7 is
 *                   exact), so s_w is 64 * (2u - 255) of the narrow path without its half-LSB offset.  cu8 gives
 *                   exactly 64 * (2u - 255).  The input history is carried as s_w pairs.
 *   Mixer           ertrs_mix on s_w.  |s_I C + s_Q S| <= 16383 * max_k(|C| + |S|) = 16383 * 23171 < 2^31, so
 *                   |s'| <= 23170: one staged word of int16 s'_I | s'_Q, as on the narrow path.
 *   Filter          the same tables, taps and interpolation into int32 accumulators.  They cannot overflow while
 *                   (sum_t |c_t| + |delta|) * 23170 < 2^31, i.e. the taps' L1 norm stays below 5.6 * 2^S; the CPU tests
 *                   check sum_t max(|table[p][t]|, |table[p+1][t]|) + 2T over every row pair of every plan of the
 *                   ertrs_plan_tuned and ertrs_plan_decimated sweeps, and sum_t |h_t| of every stage-1 plan (its folded
 *                   pair sums h * (x0 + x1) are bounded by the same |h| (|x0| + |x1|)).
 *   Between stages  a decimating handle's stage 1 writes s_w pairs: ertrs_wide_mid(acc) = clamp((acc + 2^13) >> 14,
 *                   +-16383).  Stage 2 is the tuned resampler on them at W = 0: E[0] = (2^14, 0), so s' = s.
 *   Output byte     u = clamp(((acc + 2^(S+6-k) - 1) >> (S+7-k)) + 128, 0, 255) (ertrs_wide_byte): acc / 2^(S+7) is
 *                   the channel in the decoder's byte units at k = 0, scaled by 2^k and rounded half down, so that a
 *                   constant cu8 input u (s_w = 128 (u - 127.5)) comes out as u at k = 0, and an integer one as itself.
 *   Channel gain    k in [0, ERTRS_GAIN_K_MAX].  At k = 14 the shift S + 7 - k is 7: one s_w unit (2^-7 of a byte at
 *                   k = 0, the input's own quantisation step) spans 2^7 output LSBs, so a larger k only magnifies the
 *                   input's rounding, and the shift keeps an integer rounding bias.
 *   Auto rule       from a histogram of e = floor(log2 |acc|) of the last stage's N output components (bins[e],
 *                   e in [0, 31]; zeros not binned): k is the largest in [0, K_MAX] at which at most floor(N / 65536)
 *                   components would clip, counting as clipping every |acc| * 2^k >= 2^(S+14) (128 output LSBs),
 *                   i.e. e >= S + 14 - k.  k = 0 when no component is non-zero (ertrs_channel_gain).
 */
#define ERTRS_WIDE_MAX 16383     /* |s_w|, and |stage-1 output|                                 */
#define ERTRS_WIDE_BITS 7        /* s_w = rint(x * g * 2^7)                                     */
#define ERTRS_GAIN_K_MAX 14
#define ERTRS_GAIN_BINS 32       /* floor(log2 |acc|) of an int32                                */
#define ERTRS_GAIN_CLIP_SHIFT 16 /* at most N >> 16 components clip                             */

static inline int32_t ertrs_wide_mid(int32_t acc) {
    const int32_t v = (acc + (1 << (ERTRS_S - 1))) >> ERTRS_S;
    return v < -ERTRS_WIDE_MAX ? -ERTRS_WIDE_MAX : v > ERTRS_WIDE_MAX ? ERTRS_WIDE_MAX : v;
}

static inline uint8_t ertrs_wide_byte(int32_t acc, int32_t k) {
    const int32_t sh = ERTRS_S + ERTRS_WIDE_BITS - k;
    const int32_t v = ((acc + (1 << (sh - 1)) - 1) >> sh) + 128;
    return (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v);
}

/* k of the auto rule for bins[ERTRS_GAIN_BINS] of `components` output components */
static inline int32_t ertrs_channel_gain(const int64_t* bins, int64_t components) {
    int64_t nonzero = 0;
    for (int e = 0; e < ERTRS_GAIN_BINS; e++) nonzero += bins[e];
    if (nonzero == 0) return 0;
    const int64_t allow = components >> ERTRS_GAIN_CLIP_SHIFT;
    for (int32_t k = ERTRS_GAIN_K_MAX; k > 0; k--) {
        int64_t over = 0;
        for (int e = ERTRS_S + 14 - k; e < ERTRS_GAIN_BINS; e++) over += bins[e];
        if (over <= allow) return k;
    }
    return 0;
}

/* h(d) * 2^S for the plan's window */
static inline double ertrs_proto(const ertgpu_resampler_info* info, double d) {
    const double nu = info->rate_out < info->rate_in ? (double)info->rate_out / (double)info->rate_in : 1.0;
    const double half = 0.5 * (double)info->T;
    if (d <= -half || d >= half) return 0.0;
    const double beta = 0.1102 * (ERTRS_ATTEN_DB - 8.7);
    const double z = d / half;
    const double w = ertrs_i0(beta * __builtin_sqrt(1.0 - z * z)) / ertrs_i0(beta);
    const double fc = 0.5 * nu; /* cut-off, cycles per input sample */
    const double x = 2.0 * fc * d;
    const double sinc = x == 0.0 ? 1.0 : ertrs_sinpi(x) / (3.14159265358979323846 * x);
    return (double)(1 << info->S) * 2.0 * fc * sinc * w;
}

/* Build the (P+1) x T table.  Returns 0, or -1 if a tap or an interpolation step does not fit
 * (never for plans ertrs_plan makes). */
static inline int ertrs_build_table(const ertgpu_resampler_info* info, int16_t* table) {
    const int32_t T = info->T, P = info->P;
    const int32_t one = 1 << info->S;
    for (int32_t p = 0; p <= P / 2; p++) {
        int16_t* row = table + (int64_t)p * T;
        int64_t sum = 0;
        if (p < P / 2) {
            for (int32_t t = 0; t < T; t++) {
                const double v = ertrs_proto(info, (double)(t - T / 2 + 1) - (double)p / (double)P);
                const double r = v >= 0 ? (double)(int64_t)(v + 0.5) : -(double)(int64_t)(-v + 0.5);
                if (r > 32767.0 || r < -32768.0) return -1;
                row[t] = (int16_t)r;
                sum += row[t];
            }
            const int64_t c = row[T / 2 - 1] + (one - sum);
            if (c > 32767 || c < -32768) return -1;
            row[T / 2 - 1] = (int16_t)c;
        } else { /* the half-sample row mirrors itself: build one half, mirror, split the residual */
            for (int32_t t = 0; t < T / 2; t++) {
                const double v = ertrs_proto(info, (double)(t - T / 2 + 1) - 0.5);
                const double r = v >= 0 ? (double)(int64_t)(v + 0.5) : -(double)(int64_t)(-v + 0.5);
                if (r > 32767.0 || r < -32768.0) return -1;
                row[t] = row[T - 1 - t] = (int16_t)r;
                sum += 2 * (int64_t)row[t];
            }
            const int64_t c = row[T / 2 - 1] + (one - sum) / 2; /* sum is even */
            if (c > 32767 || c < -32768) return -1;
            row[T / 2 - 1] = row[T / 2] = (int16_t)c;
        }
    }
    for (int32_t p = P / 2 + 1; p <= P; p++)
        for (int32_t t = 0; t < T; t++) table[(int64_t)p * T + t] = table[(int64_t)(P - p) * T + (T - 1 - t)];
    /* h0 * 2^F + 2^(F-1) + (h1 - h0) * w must fit int32 */
    for (int32_t p = 0; p < P; p++)
        for (int32_t t = 0; t < T; t++) {
            const int32_t d = (int32_t)table[(int64_t)(p + 1) * T + t] - (int32_t)table[(int64_t)p * T + t];
            if (d >= (1 << (30 - info->F)) || d <= -(1 << (30 - info->F))) return -1;
        }
    return 0;
}

#endif
