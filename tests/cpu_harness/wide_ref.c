/*
 * CPU restatement of the wide channel path of a tuned handle (include/ertgpu_resample.h, ertgpu_set_channel_gain),
 * independent of the CUDA kernels and written in the manner of tune_ref.c and decimate_ref.c: each input sample is mixed
 * once, with its phase index taken straight from its absolute index, and kept as an int32 pair in one flat buffer; every
 * output applies all of its taps one by one, with its position, phase and sub-phase from direct 128-bit divisions, into
 * a 64-bit accumulator.  The plan, tables, taps, NCO and the wide formulas are the header's.  The input is the wide
 * components s_w (tests/wide_ref.py converts every format to them).  Test infrastructure: tests/wide_ref.py compiles it
 * with gcc.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "ertgpu_resample.h"

#define WR_MAX_T1 512

typedef struct { /* one tuned stage: the one stage of D = 1, or the second stage at W = 0 */
    ertgpu_resampler_info info;
    int16_t table[(ERTRS_P + 1) * ERTRS_MAX_T];
    uint32_t W;
    int64_t in_total, out_next, hist_first, hist_n;
    int32_t hist[2 * (ERTRS_MAX_T + 64)];
} wr_tuned;

typedef struct { /* the first stage of D >= 2 */
    ertgpu_decimator_info dec;
    int16_t taps[WR_MAX_T1];
    uint32_t W;
    int64_t in_total, out_next, hist_first, hist_n;
    int32_t hist[2 * (WR_MAX_T1 + ERTRS_MAX_D + 16)];
} wr_dec;

typedef struct {
    int32_t k;
    uint32_t E[ERTRS_NCO_N];
    wr_dec s1;
    wr_tuned s2;
    int64_t max_acc; /* largest |acc| of any stage so far (int32 is what the kernels hold) */
} wideref_state;

size_t wideref_state_size(void) { return sizeof(wideref_state); }

/* 0, or -1 when the plan is rejected or a table or the taps do not fit */
int wideref_init(wideref_state* st, int64_t rate_in, int64_t rate_out, int64_t offset_hz, int32_t k) {
    memset(st, 0, sizeof(*st));
    st->k = k;
    if (ertrs_plan_decimated(rate_in, rate_out, offset_hz, &st->s1.dec, &st->s2.info) != 0) return -1;
    ertrs_nco_table(st->E);
    if (st->s1.dec.D > 1) {
        if (st->s1.dec.T1 > WR_MAX_T1 || ertrs_build_decimator(&st->s1.dec, st->s1.taps) != 0) return -1;
        st->s1.W = ertrs_nco_step(offset_hz, rate_in);
        st->s2.W = 0;
    } else {
        st->s2.W = ertrs_nco_step(offset_hz, rate_in);
    }
    return ertrs_build_table(&st->s2.info, st->s2.table);
}

const ertgpu_resampler_info* wideref_info(const wideref_state* st) { return &st->s2.info; }
const ertgpu_decimator_info* wideref_dec(const wideref_state* st) { return &st->s1.dec; }
const int16_t* wideref_table(const wideref_state* st) { return st->s2.table; }
const int16_t* wideref_taps(const wideref_state* st) { return st->s1.taps; }
int64_t wideref_max_acc(const wideref_state* st) { return st->max_acc; }
void wideref_set_gain(wideref_state* st, int32_t k) { st->k = k; }

static int64_t floor_div(int64_t v, int64_t d) { return v >= 0 ? v / d : -((-v + d - 1) / d); }
static int64_t kpos(const ertgpu_resampler_info* r, int64_t n) { return (int64_t)((__int128)n * r->M / r->L); }
static void note(wideref_state* st, int64_t acc) {
    const int64_t a = acc < 0 ? -acc : acc;
    if (a > st->max_acc) st->max_acc = a;
}

/* the input samples [hist, new) of a stage, mixed at step W, as one flat int32 pair buffer (freed by the caller) */
static int32_t* mixed(const uint32_t* E, uint32_t W, const int32_t* hist, int64_t hist_n, int64_t in_total, const int32_t* s,
                      int64_t n) {
    int32_t* x = (int32_t*)malloc((size_t)(hist_n + n) * 2 * sizeof(int32_t) + 8);
    if (!x) return NULL;
    memcpy(x, hist, (size_t)hist_n * 2 * sizeof(int32_t));
    for (int64_t i = 0; i < n; i++)
        ertrs_mix(s[2 * i], s[2 * i + 1], E[ertrs_nco_index(in_total + i, W)], &x[2 * (hist_n + i)], &x[2 * (hist_n + i) + 1]);
    return x;
}

/* The tuned stage over n new s pairs: the accumulators of every output whose window is now complete into acc (pairs).
 * Returns their number, or -1. */
static int64_t tuned_feed(wideref_state* w, wr_tuned* st, const int32_t* s, int64_t n, int32_t* acc) {
    const ertgpu_resampler_info* r = &st->info;
    const int32_t T = r->T, P = r->P;
    const int64_t in_new = st->in_total + n;
    const int64_t ne = in_new - T / 2 > 0 ? (int64_t)(((__int128)(in_new - T / 2) * r->L + r->M - 1) / r->M) : 0;
    int32_t* x = mixed(w->E, st->W, st->hist, st->hist_n, st->in_total, s, n);
    if (!x) return -1;
    const int64_t cnt = ne - st->out_next;
    for (int64_t i = 0; i < cnt; i++) {
        const int64_t nn = st->out_next + i, k = kpos(r, nn);
        const int64_t phi = (int64_t)((__int128)nn * r->M - (__int128)k * r->L);
        const int64_t q = (int64_t)(((__int128)phi * ((int64_t)P << r->F)) / r->L);
        const int32_t p = (int32_t)(q >> r->F), wt = (int32_t)(q & ((1 << r->F) - 1));
        int32_t c[ERTRS_MAX_T];
        int32_t sum = 0;
        for (int32_t t = 0; t < T; t++) {
            const int32_t h0 = st->table[p * T + t], h1 = st->table[(p + 1) * T + t];
            c[t] = h0 + (int32_t)floor_div((int64_t)(h1 - h0) * wt + (1 << (r->F - 1)), (int64_t)1 << r->F);
            sum += c[t];
        }
        c[T / 2 - 1 + (p >= P / 2)] += (1 << r->S) - sum;
        for (int comp = 0; comp < 2; comp++) {
            int64_t a = 0;
            for (int32_t t = 0; t < T; t++) {
                const int64_t j = k - T / 2 + 1 + t;
                a += (int64_t)c[t] * (j < 0 ? 0 : x[2 * (j - st->hist_first) + comp]);
            }
            note(w, a);
            acc[2 * i + comp] = (int32_t)a;
        }
    }
    int64_t first = kpos(r, ne) - T / 2 + 1;
    if (first < 0) first = 0;
    if (first > in_new) first = in_new;
    memmove(st->hist, x + 2 * (first - st->hist_first), (size_t)(in_new - first) * 2 * sizeof(int32_t));
    st->hist_first = first;
    st->hist_n = in_new - first;
    st->in_total = in_new;
    st->out_next = ne;
    free(x);
    return cnt;
}

/* The first stage over n new s_w pairs: its outputs ertrs_wide_mid(acc) into mid (pairs).  Returns their number. */
static int64_t dec_feed(wideref_state* w, wr_dec* st, const int32_t* s, int64_t n, int32_t* mid) {
    const int64_t D = st->dec.D, T1 = st->dec.T1, half = T1 / 2;
    const int64_t in_new = st->in_total + n;
    const int64_t ne = in_new - half > 0 ? (in_new - half + D - 1) / D : 0;
    int32_t* x = mixed(w->E, st->W, st->hist, st->hist_n, st->in_total, s, n);
    if (!x) return -1;
    const int64_t cnt = ne - st->out_next;
    for (int64_t i = 0; i < cnt; i++) {
        const int64_t k = (st->out_next + i) * D;
        for (int comp = 0; comp < 2; comp++) {
            int64_t a = 0;
            for (int64_t t = 0; t < T1; t++) {
                const int64_t j = k - half + 1 + t;
                a += (int64_t)st->taps[t] * (j < 0 ? 0 : x[2 * (j - st->hist_first) + comp]);
            }
            note(w, a);
            mid[2 * i + comp] = ertrs_wide_mid((int32_t)a);
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
    return cnt;
}

/* Feed n input samples as s_w pairs (int32, |s_w| <= 16383).  Every output whose window is now complete goes to out
 * (2 bytes each, ertrs_wide_byte at the current k) when out != NULL, and its two accumulators to acc when acc != NULL;
 * at most cap outputs.  Returns the number of outputs, or -1 if cap is too small (nothing changes then). */
int64_t wideref_feed(wideref_state* st, const int32_t* s, int64_t n, uint8_t* out, int32_t* acc, int64_t cap) {
    const ertgpu_resampler_info* r = &st->s2.info;
    const int64_t D = st->s1.dec.D;
    int64_t n2 = n;
    if (D > 1) {
        const int64_t in_new = st->s1.in_total + n, half = st->s1.dec.T1 / 2;
        n2 = (in_new - half > 0 ? (in_new - half + D - 1) / D : 0) - st->s1.out_next;
    }
    const int64_t in_new2 = st->s2.in_total + n2;
    const int64_t ne = in_new2 - r->T / 2 > 0 ? (int64_t)(((__int128)(in_new2 - r->T / 2) * r->L + r->M - 1) / r->M) : 0;
    if (ne - st->s2.out_next > cap) return -1;
    int32_t* a = (int32_t*)malloc((size_t)(ne - st->s2.out_next + 1) * 2 * sizeof(int32_t));
    int64_t got;
    if (D > 1) {
        int32_t* mid = (int32_t*)malloc((size_t)(n2 + 1) * 2 * sizeof(int32_t));
        dec_feed(st, &st->s1, s, n, mid);
        got = tuned_feed(st, &st->s2, mid, n2, a);
        free(mid);
    } else {
        got = tuned_feed(st, &st->s2, s, n, a);
    }
    for (int64_t i = 0; i < 2 * got; i++) {
        if (out) out[i] = ertrs_wide_byte(a[i], st->k);
        if (acc) acc[i] = a[i];
    }
    free(a);
    return got;
}

/* the header's rule, for the tests */
int32_t wideref_channel_gain(const int64_t* bins, int64_t components) { return ertrs_channel_gain(bins, components); }
