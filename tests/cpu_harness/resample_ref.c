/*
 * CPU restatement of the input-rate resampler (include/ertgpu_resample.h), independent of the CUDA kernel:
 * every output's position, phase and sub-phase come from direct 128-bit divisions (the kernel steps them
 * incrementally), and the input is one flat buffer (the kernel stages tiles).  Only the table builder is
 * shared.  Test infrastructure: tests/resample_ref.py compiles it with gcc.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "ertgpu_resample.h"

typedef struct {
    ertgpu_resampler_info info;
    int16_t table[(ERTRS_P + 1) * ERTRS_MAX_T];
    int64_t in_total;   /* input samples fed so far            */
    int64_t out_next;   /* first output not yet produced       */
    int64_t hist_first; /* first input sample kept in hist     */
    int64_t hist_n;
    uint8_t hist[2 * ERTRS_MAX_T];
} rsref_state;

size_t rsref_state_size(void) { return sizeof(rsref_state); }

int rsref_init(rsref_state* st, int64_t rate_in, int64_t rate_out) {
    memset(st, 0, sizeof(*st));
    if (ertrs_plan(rate_in, rate_out, &st->info) != 0) return -1;
    return ertrs_build_table(&st->info, st->table);
}

const int16_t* rsref_table(const rsref_state* st) { return st->table; }
const ertgpu_resampler_info* rsref_info(const rsref_state* st) { return &st->info; }

static int64_t kpos(const ertgpu_resampler_info* r, int64_t n) { return (int64_t)((__int128)n * r->M / r->L); }

/* One output from the flat input x[] holding input samples [x_first, x_first + x_n). */
static void one_output(const rsref_state* st, int64_t n, const uint8_t* x, int64_t x_first, uint8_t* o) {
    const ertgpu_resampler_info* r = &st->info;
    const int32_t T = r->T, P = r->P;
    const int64_t k = kpos(r, n);
    const int64_t phi = (int64_t)((__int128)n * r->M - (__int128)k * r->L);
    const int64_t q = (int64_t)(((__int128)phi * ((int64_t)P << r->F)) / r->L);
    const int32_t p = (int32_t)(q >> r->F), w = (int32_t)(q & ((1 << r->F) - 1));
    int32_t c[ERTRS_MAX_T];
    int32_t sum = 0;
    for (int32_t t = 0; t < T; t++) {
        const int32_t h0 = st->table[p * T + t], h1 = st->table[(p + 1) * T + t];
        int32_t step = (h1 - h0) * w + (1 << (r->F - 1));
        step = step >= 0 ? step / (1 << r->F) : -((-step + (1 << r->F) - 1) / (1 << r->F)); /* floor */
        c[t] = h0 + step;
        sum += c[t];
    }
    c[T / 2 - 1 + (p >= P / 2)] += (1 << r->S) - sum;
    for (int comp = 0; comp < 2; comp++) {
        int32_t acc = 0;
        for (int32_t t = 0; t < T; t++) {
            const int64_t j = k - T / 2 + 1 + t;
            const int32_t s = j < 0 ? 0 : 2 * (int32_t)x[2 * (j - x_first) + comp] - 255;
            acc += c[t] * s;
        }
        int64_t v = (int64_t)acc + (1 << (r->S + 8));
        v = v >= 0 ? v / (1 << (r->S + 1)) : -((-v + (1 << (r->S + 1)) - 1) / (1 << (r->S + 1))); /* floor */
        o[comp] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
    }
}

/* Feed n input samples (2n bytes); writes every output whose window is now complete (2 bytes each) to out,
 * at most cap outputs.  Returns the number written, or -1 if cap is too small (nothing changes then). */
int64_t rsref_feed(rsref_state* st, const uint8_t* in, int64_t n, uint8_t* out, int64_t cap) {
    const ertgpu_resampler_info* r = &st->info;
    const int64_t half = r->T / 2;
    const int64_t in_new = st->in_total + n;
    int64_t ne = 0;
    if (in_new - half > 0) ne = (int64_t)(((__int128)(in_new - half) * r->L + r->M - 1) / r->M);
    if (ne - st->out_next > cap) return -1;
    uint8_t* x = (uint8_t*)malloc((size_t)(st->hist_n + n) * 2 + 2);
    if (!x) return -1;
    memcpy(x, st->hist, (size_t)st->hist_n * 2);
    if (n) memcpy(x + st->hist_n * 2, in, (size_t)n * 2);
    const int64_t written = ne - st->out_next;
    for (int64_t i = 0; i < written; i++) one_output(st, st->out_next + i, x, st->hist_first, out + 2 * i);
    int64_t first = kpos(r, ne) - half + 1;
    if (first < 0) first = 0;
    if (first > in_new) first = in_new;
    memmove(st->hist, x + 2 * (first - st->hist_first), (size_t)(in_new - first) * 2);
    st->hist_first = first;
    st->hist_n = in_new - first;
    st->in_total = in_new;
    st->out_next = ne;
    free(x);
    return written;
}
