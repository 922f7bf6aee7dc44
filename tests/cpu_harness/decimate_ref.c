/*
 * CPU restatement of the first stage of a decimating tuned input (ertrs_plan_decimated in include/ertgpu_resample.h),
 * independent of the CUDA kernel: each input sample is mixed once, with its phase index taken straight from its
 * absolute index, and kept as an int32 pair in one flat buffer; every output applies all T1 taps one by one (the kernel
 * folds the symmetric pairs and stages tiles).  The plan, the taps, the NCO step and the mix are the header's.  The
 * second stage is the untuned resampler, restated by resample_ref.c.  Test infrastructure: tests/decimate_ref.py
 * compiles it with gcc.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "ertgpu_resample.h"

#define DCREF_MAX_T1 512

typedef struct {
    ertgpu_decimator_info dec;
    ertgpu_resampler_info info; /* the second stage's plan */
    int16_t taps[DCREF_MAX_T1];
    uint32_t E[ERTRS_NCO_N];
    uint32_t W;
    int64_t in_total;   /* input samples fed so far                  */
    int64_t out_next;   /* first output not yet produced             */
    int64_t hist_first; /* first input sample kept in hist           */
    int64_t hist_n;
    int32_t hist[2 * DCREF_MAX_T1]; /* mixed samples s'_I, s'_Q      */
} dcref_state;

size_t dcref_state_size(void) { return sizeof(dcref_state); }

int dcref_plan(int64_t rate_in, int64_t rate_out, int64_t offset_hz, ertgpu_decimator_info* dec, ertgpu_resampler_info* info) {
    return ertrs_plan_decimated(rate_in, rate_out, offset_hz, dec, info);
}

/* 0, or -1 when the plan is rejected, has D = 1 or its taps do not fit */
int dcref_init(dcref_state* st, int64_t rate_in, int64_t rate_out, int64_t offset_hz) {
    memset(st, 0, sizeof(*st));
    if (ertrs_plan_decimated(rate_in, rate_out, offset_hz, &st->dec, &st->info) != 0) return -1;
    if (st->dec.D < 2 || st->dec.T1 > DCREF_MAX_T1) return -1;
    ertrs_nco_table(st->E);
    st->W = ertrs_nco_step(offset_hz, rate_in);
    return ertrs_build_decimator(&st->dec, st->taps);
}

const ertgpu_decimator_info* dcref_dec(const dcref_state* st) { return &st->dec; }
const ertgpu_resampler_info* dcref_info(const dcref_state* st) { return &st->info; }
const int16_t* dcref_taps(const dcref_state* st) { return st->taps; }

static int64_t floor_div(int64_t v, int64_t d) { return v >= 0 ? v / d : -((-v + d - 1) / d); }

/* Feed n uint8 IQ input samples (2n bytes); writes every stage-1 output whose window is now complete (2 bytes each)
 * to out, at most cap outputs.  Returns the number written, or -1 if cap is too small (nothing changes then). */
int64_t dcref_feed(dcref_state* st, const uint8_t* in, int64_t n, uint8_t* out, int64_t cap) {
    const int64_t D = st->dec.D, T1 = st->dec.T1, half = T1 / 2;
    const int64_t in_new = st->in_total + n;
    const int64_t ne = in_new - half > 0 ? (in_new - half + D - 1) / D : 0;
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
    for (int64_t i = 0; i < written; i++) {
        const int64_t k = (st->out_next + i) * D;
        for (int comp = 0; comp < 2; comp++) {
            int64_t acc = 0;
            for (int64_t t = 0; t < T1; t++) {
                const int64_t j = k - half + 1 + t;
                acc += (int64_t)st->taps[t] * (j < 0 ? 0 : x[2 * (j - st->hist_first) + comp]);
            }
            const int64_t v = floor_div(acc + (1 << (st->dec.S + 8)), (int64_t)1 << (st->dec.S + 1));
            out[2 * i + comp] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
        }
    }
    int64_t first = ne * D - half + 1;
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
