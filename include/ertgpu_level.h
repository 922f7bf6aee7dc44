/*
 * ertgpu_level.h -- the automatic gain of a converted input (ertgpu_measure_input), as one header shared by
 * libertgpu.so and the CPU test that restates it.  Not part of the reference API: rtlamr puts its tuner in automatic
 * gain mode instead (main.go:119-121), so its 8-bit ADC always sees a sensible level.
 *
 * The gain multiplies each component x (the value convert.cuh's fmt_x defines: the stored value, byte permuted for
 * a big-endian format, less 2^15 or 2^31 for an unsigned one) before it is rounded and clamped to the decoder's byte,
 * u = clamp(rint(x * G), -128, 127) + 128.  The measurement is a histogram of e = floor(log2 |x|), taken from the
 * bits (never from a logarithm), clamped to [-128, 127]: bins[e + 128], with +-inf in the top bin and zeros
 * (including -0) and NaNs counted on their own.
 *
 * The rule: with N components measured and the allowance A = floor(N / 65536), G = 2^k for the largest integer k in
 * [ERTLV_K_MIN, ERTLV_K_MAX] for which at most A components have |x| * 2^k >= 128, i.e. sum of bins[e + 128] over
 * e >= 7 - k (the infinities included) <= A: at most one component in 65 536 clips.  k = ERTLV_K_MIN when even that
 * clips more; the format's default gain when no component is non-zero and non-NaN.  A power of two keeps the
 * conversion exactly what it is with an explicit gain, needs only the exponents, and its 6 dB steps are small against
 * the byte's 48 dB.
 */
#ifndef ERTGPU_LEVEL_H
#define ERTGPU_LEVEL_H

#include <stdint.h>

#define ERTLV_WINDOW (1 << 22) /* input samples a receiver measures at the start of each stream */
#define ERTLV_BINS 256         /* bins[e + 128], e in [-128, 127]                               */
#define ERTLV_CLIP_SHIFT 16    /* A = N >> 16: at most one component in 65 536 clips           */
#define ERTLV_K_MIN (-120)
#define ERTLV_K_MAX 120

/* k of the rule for the histogram bins[ERTLV_BINS] of `components` components, `zeros` and `nans` of them zero and
 * NaN; default_k (log2 of the format's default gain) when no component is non-zero and non-NaN. */
static inline int32_t ertlv_exponent(const int64_t *bins, int64_t components, int64_t zeros, int64_t nans,
                                     int32_t default_k) {
    if (components - zeros - nans <= 0) return default_k;
    const int64_t allow = components >> ERTLV_CLIP_SHIFT;
    /* over = components with e >= t = 7 - k; k falls from ERTLV_K_MAX, so t rises and over falls */
    int64_t over = 0;
    for (int e = 7 - ERTLV_K_MAX; e <= 127; e++) over += bins[e + 128];
    for (int32_t k = ERTLV_K_MAX; k > ERTLV_K_MIN; k--) {
        if (over <= allow) return k;
        over -= bins[7 - k + 128];
    }
    return ERTLV_K_MIN;
}

#endif
