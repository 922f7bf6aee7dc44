/*
 * ertgpu_signal.h -- per-packet signal reports (ertgpu_enable_signal, ertgpu_fetch_signal): where a candidate's
 * samples are, which of them are measured, and how the host turns the exact integer record into Hz and dB.  One
 * header shared by libertgpu.so's packet_signal_kernel, the host mirror and the CPU test harness.  Not part of the
 * reference API: rtlamr reports what a meter sent, never how it was received.
 *
 * Notation: a handle's merged geometry CL, SL = 2 CL, BS, PKL (PacketLength), BUF = PKL + BS; a candidate of block b
 * (counted from the stream's first block) at Idx idx.
 *
 * Where the packet is.  After the Decode of block b, Signal[j] is decoder sample b*BS + j - SL (decode.go:165-169)
 * and Quantized[PKL + i] is the matched filter at Signal[i] (decode.go:229-245), so Quantized[q] is the symbol that
 * starts at sample (b+1)*BS - BUF + q - SL.  Slice takes bit k of the packet from Quantized[idx + k*SL]
 * (decode.go:369): symbol k starts at a0 + k*SL with a0 = (b+1)*BS - BUF + idx - SL.
 *
 * Which symbols.  The protocol is the first registered one filed under the candidate's preamble whose check_mask bit
 * is set, or the first one filed under it when no bit is.  Its span is its PacketSymbols (PreambleSymbols for an
 * ERTGPU_CHECK_R900 protocol, whose payload is not Manchester coded), and symbols 1 .. span-1 are measured.  Symbol 0
 * is skipped: it can begin up to SL samples before the PKL samples of history a handle keeps in front of a call, every
 * later one lies inside history and call, so a record does not depend on how the stream is cut into calls.
 *
 * High and low chips.  Bit k of the candidate's bytes (MSB first; a trailing partial byte holds its PK%8 bits in the
 * low bits) is 1 when the symbol's first chip is the high one (decode.go:243, f >= 0).  Only a chip's inner samples
 * [c0 + g, c0 + CL - g), g = CL >> 2, count: chip edges and the channel filter's ringing stay out.
 *
 * Sample value.  s = 2u - 255 per component of the decoder's byte u: always odd, so |s|^2 >= 2 and no power is 0.
 * Samples before the stream's first sample are not counted.
 *
 * The record (ertgpu_signal in ertgpu.h), exact integers summed in any order:
 *   n_on, e_on = sum(sI^2 + sQ^2) over high-chip inner samples; n_off, e_off over low-chip inner samples;
 *   r = sum s[n] conj(s[n-1]) over adjacent pairs inside one high-chip inner span (r_re, r_im), and n_pairs.
 * An idm packet at CL 96 keeps every sum below 2^40.
 *
 * The summary (ertsig_summary), with P_on = e_on / n_on and P_off = e_off / n_off:
 *   Level  = 10 log10(P_on / 65025)   dB of the decoder's bytes; a full-scale complex tone is 0 dB
 *   Noise  = 10 log10(P_off / 65025)
 *   SNR    = 10 log10((P_on - P_off) / P_off), clamped below at -99.99
 *   Offset = atan2(r_im, r_re) * R_out / (2 pi), R_out = DataRate * ChipLength: unambiguous within +-R_out/2, which
 *            holds the channel filter's +-0.4 R_out passband
 *   Freq   = Channel + Offset rounded to Hz; Channel is the tuned channel's centre, or the decoder's CenterFreq.
 * A record with n_on = 0 or n_off = 0 (only a packet that starts before the stream) has no summary.
 */
#ifndef ERTGPU_SIGNAL_H
#define ERTGPU_SIGNAL_H

#include <math.h>
#include <stdint.h>

#include "ertgpu.h"

#ifdef __CUDACC__
#define ERTSIG_HD __host__ __device__ __forceinline__
#else
#define ERTSIG_HD static inline
#endif

#define ERTSIG_FULL_SCALE 65025.0 /* |s|^2 of one full-scale component: 255^2 */
#define ERTSIG_SNR_MIN (-99.99)
#define ERTSIG_PI 3.14159265358979323846 /* M_PI is not in strict C */

/* What packet_signal_kernel needs of a handle: its merged geometry and, per registered protocol, the preamble it is
 * filed under and the symbols of its span. */
typedef struct {
    int32_t CL, SL, BS, BUF, PK;
    int32_t nproto;
    int32_t preamble_id[ERTGPU_MAX_PROTOCOLS];
    int32_t span[ERTGPU_MAX_PROTOCOLS];
} ertsig_geometry;

/* Decoder sample at which symbol 0 of the candidate (block b, idx) starts; b counted from the first sample of the
 * samples the caller indexes. */
ERTSIG_HD int64_t ertsig_first_sample(const ertsig_geometry* g, int64_t b, int32_t idx) {
    return (b + 1) * g->BS - g->BUF + idx - g->SL;
}

/* The protocol whose span is measured, -1 when none is filed under the preamble. */
ERTSIG_HD int32_t ertsig_protocol(const ertsig_geometry* g, int32_t preamble_id, uint32_t check_mask) {
    int32_t first = -1;
    for (int32_t i = 0; i < g->nproto; i++) {
        if (g->preamble_id[i] != preamble_id) continue;
        if ((check_mask >> i) & 1u) return i;
        if (first < 0) first = i;
    }
    return first;
}

/* Bit k of a candidate's bytes. */
ERTSIG_HD int ertsig_bit(const uint8_t* bytes, int32_t k, int32_t PK) {
    const int32_t byte = k >> 3;
    const int shift = ((PK & 7) && byte == (PK >> 3)) ? (PK & 7) - 1 - (k & 7) : 7 - (k & 7);
    return (bytes[byte] >> shift) & 1;
}

/* One record in Hz and dB. */
typedef struct {
    double level_db, noise_db, snr_db;
    double offset_hz;
    int64_t freq_hz;
} ertsig_summary_t;

/* 1 and *s for a record with a summary, 0 otherwise.  channel_hz: the channel the handle decodes; rate_out: R_out. */
static inline int ertsig_summary(const ertgpu_signal* r, int64_t channel_hz, int64_t rate_out, ertsig_summary_t* s) {
    if (r->n_on <= 0 || r->n_off <= 0) return 0;
    const double p_on = (double)r->e_on / (double)r->n_on, p_off = (double)r->e_off / (double)r->n_off;
    const double x = (p_on - p_off) / p_off;
    s->level_db = 10.0 * log10(p_on / ERTSIG_FULL_SCALE);
    s->noise_db = 10.0 * log10(p_off / ERTSIG_FULL_SCALE);
    s->snr_db = x > 0 ? fmax(10.0 * log10(x), ERTSIG_SNR_MIN) : ERTSIG_SNR_MIN;
    s->offset_hz = atan2((double)r->r_im, (double)r->r_re) * (double)rate_out / (2.0 * ERTSIG_PI);
    s->freq_hz = (int64_t)llround((double)channel_hz + s->offset_hz);
    return 1;
}

#endif
