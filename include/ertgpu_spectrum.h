/*
 * ertgpu_spectrum.h -- the power spectrum of a decode's input (ertgpu_enable_spectrum, ertgpu_fetch_spectrum): what
 * is measured, how rows are formed, and the helpers the CLI uses to print them.  One header shared by libertgpu.so's
 * spectrum_kernel<F>, the host mirror, the CLI and the CPU test harness.  Not part of the reference API.
 *
 * Input value.  Every IQ sample of the call's input, as the caller passed it, becomes the wide component pair s_w of
 * include/ertgpu_resample.h: s_w = clamp(rint(x * g * 2^7), +-16383), NaN -> 0, with g the handle's input gain
 * (ertgpu_set_input_format or ertgpu_set_input_scale); cu8 gives s_w = 64 * (2u - 255).  v = (s_I + i s_Q) / 16320,
 * so a full-scale cu8 complex tone has |v| = 1.  The spectrum measures the capture: it does not depend on the handle's
 * rate, tuning, decimation or channel gain.
 *
 * Frames.  N = 2^n, ERTSPEC_LOG2_MIN <= n <= ERTSPEC_LOG2_MAX.  Frame f is input samples [f N, (f+1) N) of the stream,
 * counted from its start (allocate or ertgpu_reset), without overlap.  A frame is measured once all N of its samples
 * have arrived, however the stream is cut into calls.
 *
 * Window.  The periodic Hann window w[j] = 0.5 - 0.5 cos(2 pi j / N), computed in double and rounded to float
 * (ertspec_window).
 *
 * Power.  P_f[k] = |sum_j w[j] v[j] e^(-2 pi i j k' / N)|^2 / (sum_j w[j])^2, sum_j w[j] = N / 2.  Bins are in ascending
 * frequency order: bin k holds k' = (k - N/2) mod N, centred at Centre + (k - N/2) R_in / N (ertspec_bin_hz).  Centre
 * is the capture frequency of a tuned handle, otherwise the decoder's CenterFreq.  A full-scale tone at a bin centre
 * reads 0 dB in its bin: the scale of ertsig_summary's Level.
 *
 * Rows.  Row r is frames [r F, (r+1) F); N F >= ERTSPEC_ROW_MIN_SAMPLES, so that rows are a small fraction of the input.
 * A row (ertgpu_spectrum_row) carries mean[k] = (sum_f P_f[k]) / F, the integrated power, and peak[k] = max_f P_f[k],
 * which shows a 10 ms burst in a 1 s row.  Both are float32.  The sum is taken in an order fixed by frame index
 * alone, so that rows are bitwise the same however the stream is cut into calls (DESIGN.md section 3.14).
 *
 * dB.  10 log10(P), clamped below at ERTSPEC_DB_FLOOR (ertspec_db).
 *
 * CSV.  ertspec_csv_line prints one row in rtl_power's column layout:
 *   date, time, Hz low, Hz high, Hz step, samples, dB, dB, ...
 * with Hz low = Centre - R_in / 2 and Hz high = Centre + R_in / 2 (integer division), Hz step = R_in / N to two
 * decimals, samples = frames N, and N dB values to two decimals.  date and time are UTC.
 */
#ifndef ERTGPU_SPECTRUM_H
#define ERTGPU_SPECTRUM_H

#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include "ertgpu.h"

#define ERTSPEC_LOG2_MIN 6
#define ERTSPEC_LOG2_MAX 14
#define ERTSPEC_ROW_MIN_SAMPLES (1 << 18) /* N F at least                        */
#define ERTSPEC_FULL_SCALE 16320.0         /* |s_w| of a full-scale cu8 component  */
#define ERTSPEC_DB_FLOOR (-200.0)
#define ERTSPEC_PI 3.14159265358979323846

/* The periodic Hann window of N = 2^log2_n points, rounded to float. */
static inline void ertspec_window(int32_t log2_n, float* w) {
    const int32_t N = 1 << log2_n;
    for (int32_t j = 0; j < N; j++) w[j] = (float)(0.5 - 0.5 * cos(2.0 * ERTSPEC_PI * (double)j / (double)N));
}

/* The factor |X|^2 is multiplied by: 1 / (16320 sum_j w[j])^2, sum_j w[j] = N / 2, rounded to float. */
static inline float ertspec_power_scale(int32_t log2_n) {
    const double s = ERTSPEC_FULL_SCALE * (double)(1 << log2_n) / 2.0;
    return (float)(1.0 / (s * s));
}

/* Power in dB, clamped below at ERTSPEC_DB_FLOOR. */
static inline double ertspec_db(double p) {
    if (!(p > 0)) return ERTSPEC_DB_FLOOR;
    const double d = 10.0 * log10(p);
    return d > ERTSPEC_DB_FLOOR ? d : ERTSPEC_DB_FLOOR;
}

/* log2 of the smallest power of two N with rate_hz / N <= bin_hz, clamped to [ERTSPEC_LOG2_MIN, ERTSPEC_LOG2_MAX]. */
static inline int32_t ertspec_log2_for_bin(int64_t rate_hz, double bin_hz) {
    int32_t n = ERTSPEC_LOG2_MIN;
    while (n < ERTSPEC_LOG2_MAX && (double)rate_hz / (double)(1 << n) > bin_hz) n++;
    return n;
}

/* Frames per row for rows of duration_ns at rate_hz: max(ceil(2^18 / N), round(duration * rate_hz / N)). */
static inline int64_t ertspec_frames_per_row(int32_t log2_n, int64_t duration_ns, int64_t rate_hz) {
    const int64_t N = (int64_t)1 << log2_n;
    const int64_t least = (ERTSPEC_ROW_MIN_SAMPLES + N - 1) / N;
    const int64_t f = llround((double)duration_ns * 1e-9 * (double)rate_hz / (double)N);
    return f > least ? f : least;
}

/* Centre frequency of bin k (0 <= k < N) in Hz. */
static inline double ertspec_bin_hz(int64_t centre_hz, int64_t rate_hz, int32_t log2_n, int32_t k) {
    const int32_t N = 1 << log2_n;
    return (double)centre_hz + (double)(k - N / 2) * (double)rate_hz / (double)N;
}

/* UTC calendar date of a day count since 1970-01-01 (proleptic Gregorian). */
static inline void ertspec_civil(int64_t days, int64_t* y, int32_t* m, int32_t* d) {
    days += 719468;
    const int64_t era = (days >= 0 ? days : days - 146096) / 146097;
    const int64_t doe = days - era * 146097;
    const int64_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
    const int64_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
    const int64_t mp = (5 * doy + 2) / 153;
    *d = (int32_t)(doy - (153 * mp + 2) / 5 + 1);
    *m = (int32_t)(mp < 10 ? mp + 3 : mp - 9);
    *y = yoe + era * 400 + (*m <= 2);
}

/* One row as a CSV line (with its newline) into out[0 .. cap): unix_s the time of its first sample in whole seconds,
 * samples = frames N, p its N powers.  Returns the length the whole line needs, as snprintf does. */
static inline int ertspec_csv_line(char* out, size_t cap, int64_t unix_s, int64_t centre_hz, int64_t rate_hz,
                                   int32_t log2_n, int64_t samples, const float* p) {
    const int32_t N = 1 << log2_n;
    const int64_t days = unix_s >= 0 ? unix_s / 86400 : -((-unix_s + 86399) / 86400);
    const int64_t sod = unix_s - days * 86400;
    int64_t y;
    int32_t mo, d;
    ertspec_civil(days, &y, &mo, &d);
    size_t len = 0;
#define ERTSPEC_PUT(...)                                                                  \
    do {                                                                                  \
        const int k_ = snprintf(out ? out + (len < cap ? len : cap) : NULL,               \
                                len < cap ? cap - len : 0, __VA_ARGS__);                  \
        if (k_ < 0) return -1;                                                            \
        len += (size_t)k_;                                                                \
    } while (0)
    ERTSPEC_PUT("%04lld-%02d-%02d, %02d:%02d:%02d, %lld, %lld, %.2f, %lld", (long long)y, mo, d, (int)(sod / 3600),
                (int)(sod / 60 % 60), (int)(sod % 60), (long long)(centre_hz - rate_hz / 2),
                (long long)(centre_hz + rate_hz / 2), (double)rate_hz / (double)N, (long long)samples);
    for (int32_t k = 0; k < N; k++) ERTSPEC_PUT(", %.2f", ertspec_db((double)p[k]));
    ERTSPEC_PUT("\n");
#undef ERTSPEC_PUT
    return (int)len;
}

#endif
