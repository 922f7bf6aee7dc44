/*
 * CPU restatement of the tuned input resampler (ertrs_plan_tuned in include/ertgpu_resample.h), independent of the
 * CUDA kernel: each input sample is mixed once, with its phase index taken straight from its absolute index, and
 * kept as an int32 pair in one flat buffer; every output's position, phase and sub-phase come from direct 128-bit
 * divisions.  The table builders, the NCO step and the mix are the header's.  tests/resample_ref.c stays the
 * untuned reference.  Test infrastructure: tests/tune_ref.py compiles it with gcc.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "ertgpu_resample.h"

typedef struct {
    ertgpu_resampler_info info;
    int16_t table[(ERTRS_P + 1) * ERTRS_MAX_T];
    uint32_t E[ERTRS_NCO_N];
    uint32_t W;
    int64_t in_total;   /* input samples fed so far                  */
    int64_t out_next;   /* first output not yet produced             */
    int64_t hist_first; /* first input sample kept in hist           */
    int64_t hist_n;
    int32_t hist[2 * ERTRS_MAX_T]; /* mixed samples s'_I, s'_Q        */
} tuneref_state;

size_t tuneref_state_size(void) { return sizeof(tuneref_state); }

int tuneref_init(tuneref_state* st, int64_t rate_in, int64_t rate_out, int64_t offset_hz) {
    memset(st, 0, sizeof(*st));
    if (ertrs_plan_tuned(rate_in, rate_out, offset_hz, &st->info) != 0) return -1;
    ertrs_nco_table(st->E);
    st->W = ertrs_nco_step(offset_hz, rate_in);
    return ertrs_build_table(&st->info, st->table);
}

const int16_t* tuneref_table(const tuneref_state* st) { return st->table; }
const ertgpu_resampler_info* tuneref_info(const tuneref_state* st) { return &st->info; }
uint32_t tuneref_nco_step(int64_t offset_hz, int64_t rate_in) { return ertrs_nco_step(offset_hz, rate_in); }
void tuneref_nco_table(uint32_t* E) { ertrs_nco_table(E); }
int tuneref_plan(int64_t rate_in, int64_t rate_out, int64_t offset_hz, ertgpu_resampler_info* info) {
    return ertrs_plan_tuned(rate_in, rate_out, offset_hz, info);
}

static int64_t kpos(const ertgpu_resampler_info* r, int64_t n) { return (int64_t)((__int128)n * r->M / r->L); }

static int64_t floor_div(int64_t v, int64_t d) { return v >= 0 ? v / d : -((-v + d - 1) / d); }

/* One output from the mixed samples x[] holding input samples [x_first, x_first + x_n). */
static void one_output(const tuneref_state* st, int64_t n, const int32_t* x, int64_t x_first, uint8_t* o) {
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
        c[t] = h0 + (int32_t)floor_div((int64_t)(h1 - h0) * w + (1 << (r->F - 1)), (int64_t)1 << r->F);
        sum += c[t];
    }
    c[T / 2 - 1 + (p >= P / 2)] += (1 << r->S) - sum;
    for (int comp = 0; comp < 2; comp++) {
        int64_t acc = 0;
        for (int32_t t = 0; t < T; t++) {
            const int64_t j = k - T / 2 + 1 + t;
            acc += (int64_t)c[t] * (j < 0 ? 0 : x[2 * (j - x_first) + comp]);
        }
        const int64_t v = floor_div(acc + (1 << (r->S + 8)), (int64_t)1 << (r->S + 1));
        o[comp] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
    }
}

/* Feed n uint8 IQ input samples (2n bytes); writes every output whose window is now complete (2 bytes each) to
 * out, at most cap outputs.  Returns the number written, or -1 if cap is too small (nothing changes then). */
int64_t tuneref_feed(tuneref_state* st, const uint8_t* in, int64_t n, uint8_t* out, int64_t cap) {
    const ertgpu_resampler_info* r = &st->info;
    const int64_t half = r->T / 2;
    const int64_t in_new = st->in_total + n;
    int64_t ne = 0;
    if (in_new - half > 0) ne = (int64_t)(((__int128)(in_new - half) * r->L + r->M - 1) / r->M);
    if (ne - st->out_next > cap) return -1;
    int32_t* x = (int32_t*)malloc((size_t)(st->hist_n + n) * 2 * sizeof(int32_t) + 8);
    if (!x) return -1;
    memcpy(x, st->hist, (size_t)st->hist_n * 2 * sizeof(int32_t));
    for (int64_t i = 0; i < n; i++) {
        const int64_t g = st->in_total + i;
        const uint32_t e = st->E[ertrs_nco_index(g, st->W)];
        ertrs_mix(2 * (int32_t)in[2 * i] - 255, 2 * (int32_t)in[2 * i + 1] - 255, e, &x[2 * (st->hist_n + i)],
                  &x[2 * (st->hist_n + i) + 1]);
    }
    const int64_t written = ne - st->out_next;
    for (int64_t i = 0; i < written; i++) one_output(st, st->out_next + i, x, st->hist_first, out + 2 * i);
    int64_t first = kpos(r, ne) - half + 1;
    if (first < 0) first = 0;
    if (first > in_new) first = in_new;
    memmove(st->hist, x + 2 * (first - st->hist_first), (size_t)(in_new - first) * 2 * sizeof(int32_t));
    st->hist_first = first;
    st->hist_n = in_new - first;
    st->in_total = in_new;
    st->out_next = ne;
    free(x);
    return written;
}
