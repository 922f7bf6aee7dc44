/* spectrum_ref.c -- include/ertgpu_spectrum.h's helpers for ctypes (tests/spectrum_ref.py). */
#include "ertgpu_spectrum.h"

void specref_window(int32_t log2_n, float* w) { ertspec_window(log2_n, w); }
float specref_power_scale(int32_t log2_n) { return ertspec_power_scale(log2_n); }
double specref_db(double p) { return ertspec_db(p); }
int32_t specref_log2_for_bin(int64_t rate_hz, double bin_hz) { return ertspec_log2_for_bin(rate_hz, bin_hz); }
int64_t specref_frames_per_row(int32_t log2_n, int64_t duration_ns, int64_t rate_hz) {
    return ertspec_frames_per_row(log2_n, duration_ns, rate_hz);
}
double specref_bin_hz(int64_t centre_hz, int64_t rate_hz, int32_t log2_n, int32_t k) {
    return ertspec_bin_hz(centre_hz, rate_hz, log2_n, k);
}
int specref_csv_line(char* out, size_t cap, int64_t unix_s, int64_t centre_hz, int64_t rate_hz, int32_t log2_n,
                     int64_t samples, const float* p) {
    return ertspec_csv_line(out, cap, unix_s, centre_hz, rate_hz, log2_n, samples, p);
}
