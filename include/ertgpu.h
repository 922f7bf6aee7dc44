/*
 * ertgpu.h -- C ABI of libertgpu.so: a Hopper (sm_90a) implementation of the
 * rtlamr `protocol.Decoder` hot path (uint8 IQ -> magnitude -> Manchester
 * matched filter -> quantize -> pack -> preamble search -> slice -> CRC screen).
 *
 * This is the drop-in boundary.  A thin cgo shim (go/protocol/decode_cuda.go,
 * shown in INTEGRATION.md) keeps the reference's Go names and calls these
 * entry points instead of running decode.go's loops.  Every entry point cites
 * the reference interface it replaces (paths relative to the rtlamr checkout).
 *
 * Conventions
 *  - plain C types only; no C++/torch types cross the boundary; nothing throws.
 *  - every function returns 0 (ERTGPU_OK) or a negative ERTGPU_E* code;
 *    ertgpu_last_error(h) gives the message.  The Go shim turns errors into
 *    panics where the reference panics (short input: decode.go:222).
 *  - one handle == one protocol.Decoder == one sample stream.  Calls on a handle
 *    must be serialised by the caller (the reference's Decode is not re-entrant
 *    either: it is called from one goroutine, main.go:235).  Different handles
 *    are independent; any OS thread may call (the library sets the device per
 *    call and keeps no thread-local state).
 *  - the library never keeps a caller pointer after a call returns (cgo rule).
 *  - there is NO CPU fallback: without a usable CUDA device every call fails
 *    with ERTGPU_ECUDA.
 */
#ifndef ERTGPU_H
#define ERTGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ERTGPU_ABI_VERSION 2

/* error codes */
#define ERTGPU_OK 0
#define ERTGPU_EINVAL (-1)    /* bad argument / call order                       */
#define ERTGPU_ECUDA (-2)     /* CUDA runtime error, no device, wrong arch       */
#define ERTGPU_ENOMEM (-3)    /* host or device allocation failed                */
#define ERTGPU_ECAPACITY (-4) /* output array (or max_candidates) too small:    *
                               * *n_out holds the need, see ertgpu_decode       */
#define ERTGPU_ESIZE (-5)     /* nbytes not a multiple of BlockSize2 / too large */

#define ERTGPU_MAX_PROTOCOLS 8
#define ERTGPU_MAX_PREAMBLE 32
#define ERTGPU_MAX_CHANNELS 64 /* most handles of one ertgpu_decode_channels call */
#define ERTGPU_MAX_PACKET_BYTES 92 /* (PacketSymbols+7)>>3 for idm/netidm */
#define ERTGPU_R900_DIGITS 42      /* r900.PayloadSymbols, r900/r900.go:30 */

/* integrity screens the GPU can run per candidate (the parsers re-check on the
 * host exactly as the reference does; the mask only lets the shim skip the
 * candidates every parser would reject) */
#define ERTGPU_CHECK_NONE 0
#define ERTGPU_CHECK_CRC16 1 /* Checksum(init, Bytes[from:to]) == residue: scm/scm.go:76, scmplus/scmplus.go:77 */
#define ERTGPU_CHECK_IDM 2   /* packet CRC Bytes[4:92] and serial CRC Bytes[9:13]+Bytes[88:90]: idm/idm.go:77-87, netidm/netidm.go:88-98;
                              * crc_from/crc_to are ignored, crc_init/crc_poly/crc_residue apply to both CRCs */
#define ERTGPU_CHECK_R900 3  /* base-6 digit pairs <= 31 and RS syndrome == 0: r900/r900.go:199-221 */

/* One registered parser's PacketConfig (protocol/decode.go:27-42) as the parser's
 * NewParser literal fills it (scm/scm.go:42-50 ...), plus the integrity screen. */
typedef struct {
    char name[16];                          /* PacketConfig.Protocol          */
    char preamble[ERTGPU_MAX_PREAMBLE + 1]; /* PacketConfig.Preamble, '0'/'1' */
    int32_t data_rate;                      /* PacketConfig.DataRate          */
    int32_t chip_length;                    /* PacketConfig.ChipLength (the -symbollength flag, main.go:77) */
    int32_t preamble_symbols;               /* PacketConfig.PreambleSymbols   */
    int32_t packet_symbols;                 /* PacketConfig.PacketSymbols     */
    uint32_t center_freq;                   /* PacketConfig.CenterFreq        */
    int32_t check_kind;                     /* ERTGPU_CHECK_* (any other value: EINVAL) */
    uint16_t crc_init, crc_poly, crc_residue; /* crc.NewCRC arguments, crc/crc.go:16-24 */
    uint16_t reserved;
    int32_t crc_from, crc_to;               /* byte range for ERTGPU_CHECK_CRC16 (ignored otherwise) */
} ertgpu_protocol;

/* Decoder.Cfg after Allocate (protocol/decode.go:131-141) */
typedef struct {
    int32_t data_rate;
    int32_t block_size, block_size2;
    int32_t chip_length, symbol_length;
    int32_t sample_rate;
    int32_t preamble_symbols, packet_symbols;
    int32_t preamble_length, packet_length;
    int32_t buffer_length;
    uint32_t center_freq;
    int32_t n_protocols;
    int32_t n_preambles;   /* distinct preambles, decode.go:121-124 */
    int32_t packet_bytes;  /* (packet_symbols+7)>>3, decode.go:154 */
} ertgpu_decoder_config;

/* One protocol.Data (protocol/parse.go:55-59) as produced by Search+Slice
 * (decode.go:255-375), tagged with the Decode call ("block") it belongs to. */
typedef struct {
    int64_t block;        /* index of the reference Decode call since stream start */
    int32_t idx;          /* Data.Idx in [0, BlockSize)                            */
    int32_t preamble_id;  /* distinct preamble, in registration order              */
    uint32_t check_mask;  /* bit i: i-th registered protocol passed its screen     */
    uint32_t flags;       /* ERTGPU_CAND_*                                         */
    uint8_t bytes[ERTGPU_MAX_PACKET_BYTES]; /* Data.Bytes (merged PacketSymbols, MSB first; a trailing partial byte holds its PK%8 bits in the low bits, like decode.go:363-366 on a zeroed pkt) */
    uint8_t r900_digits[ERTGPU_R900_DIGITS]; /* r900 quantized[] at the 42 payload positions, r900/r900.go:187-193 */
    uint8_t pad[2];
} ertgpu_candidate;

#define ERTGPU_CAND_HAS_R900 1u /* r900_digits[] is filled */

/* How one candidate was received (ertgpu_fetch_signal): exact integer sums over its own samples, as
 * include/ertgpu_signal.h defines them; ertsig_summary there turns them into Level, Noise, SNR and Freq. */
typedef struct {
    int64_t n_on, e_on;   /* high-chip inner samples, and the sum of their sI^2 + sQ^2 (s = 2u - 255) */
    int64_t n_off, e_off; /* the same over low-chip inner samples                                     */
    int64_t r_re, r_im;   /* sum of s[n] conj(s[n-1]) over adjacent pairs inside one high-chip span    */
    int64_t n_pairs;      /* pairs in r                                                                */
    int32_t protocol;     /* registered protocol whose span was measured                              */
    int32_t symbols;      /* symbols measured (1 .. span-1 of that protocol)                           */
} ertgpu_signal;

/* One row of a handle's input spectrum (ertgpu_fetch_spectrum; include/ertgpu_spectrum.h defines it). */
typedef struct {
    int64_t first_sample; /* input sample of the stream at which its first frame starts */
    int64_t frames;       /* frames in it: frames_per_row, or fewer for the open row     */
} ertgpu_spectrum_row;

/* decode flags */
#define ERTGPU_DECODE_ONLY_VALID 1u /* return only candidates with check_mask != 0 */

/* parity taps (state of the most recent decode call) */
#define ERTGPU_TAP_SIGNAL 0    /* float32[BS+SL]   Decoder.Signal  after block b (decode.go:144,169)  */
#define ERTGPU_TAP_CSUM 1      /* float32[BS+SL+1] Decoder.csum    after block b (decode.go:147,232-236) */
#define ERTGPU_TAP_QUANTIZED 2 /* uint8[BUF]       Decoder.Quantized after block b (decode.go:145,166,243) */
#define ERTGPU_TAP_PACKED 3    /* uint8[(BS+PL+7)>>3] Decoder.packed after block b (decode.go:159,259-265) */
#define ERTGPU_TAP_R900_QUANTIZED 4 /* uint8[BUF]  r900 Parser.quantized after block b (r900/r900.go:82-150) */
#define ERTGPU_TAP_RESAMPLED 5 /* uint8[BlockSize2] the uint8 IQ bytes of block b as the decoder read them (handles that resample or convert their input) */

/* input sample formats (ertgpu_set_input_format) */
#define ERTGPU_FORMAT_CU8 0  /* interleaved uint8 I,Q (rtl_sdr, rtl_tcp): 2 bytes per sample, decoded as they are */
#define ERTGPU_FORMAT_CS8 1  /* interleaved int8 I,Q (hackrf_transfer): 2 bytes per sample        */
#define ERTGPU_FORMAT_CS16 2 /* interleaved little-endian int16 I,Q: 4 bytes per sample              */
#define ERTGPU_FORMAT_CF32 3 /* interleaved little-endian float32 I,Q: 8 bytes per sample            */
/* The other complex SigMF datatypes, named by their SigMF names; x is the component the scale multiplies. */
#define ERTGPU_FORMAT_CS16BE 16 /* ci16_be: big-endian int16, 4 bytes per sample, x = v          */
#define ERTGPU_FORMAT_CF32BE 17 /* cf32_be: big-endian float32, 8 bytes per sample, x = v        */
#define ERTGPU_FORMAT_CU16 18   /* cu16_le: little-endian uint16, 4 bytes, x = v - 2^15          */
#define ERTGPU_FORMAT_CU16BE 19 /* cu16_be: big-endian uint16, 4 bytes, x = v - 2^15             */
#define ERTGPU_FORMAT_CS32 20   /* ci32_le: little-endian int32, 8 bytes, x = v                  */
#define ERTGPU_FORMAT_CS32BE 21 /* ci32_be: big-endian int32, 8 bytes, x = v                     */
#define ERTGPU_FORMAT_CU32 22   /* cu32_le: little-endian uint32, 8 bytes, x = v - 2^31          */
#define ERTGPU_FORMAT_CU32BE 23 /* cu32_be: big-endian uint32, 8 bytes, x = v - 2^31             */
#define ERTGPU_FORMAT_CF64 24   /* cf64_le: little-endian float64, 16 bytes, x = v               */
#define ERTGPU_FORMAT_CF64BE 25 /* cf64_be: big-endian float64, 16 bytes, x = v                  */

typedef struct ertgpu_handle ertgpu_handle;

/* The input-rate resampler of a handle (ertgpu_set_input_rate; include/ertgpu_resample.h has the
 * arithmetic).  Output rate R_out = DataRate * ChipLength; R_out / R_in = L / M reduced. */
typedef struct {
    int64_t rate_in, rate_out;
    int64_t L, M;
    int32_t T;  /* taps per output sample                      */
    int32_t P;  /* table sub-phases per input sample            */
    int32_t S;  /* DC gain of every coefficient set is 2^S      */
    int32_t F;  /* bits of the sub-phase interpolation weight   */
} ertgpu_resampler_info;

/* The first stage of a decimating tuned handle (ertgpu_allow_input_decimation; include/ertgpu_resample.h has the
 * arithmetic): mix, lowpass and keep every D-th sample, R_in -> R_mid = R_in / D.  D = 1 means no first stage. */
typedef struct {
    int64_t rate_in, rate_out; /* the capture's rate and the decoder's rate R_out             */
    int32_t D;                 /* decimation of the first stage                              */
    int32_t T1;                /* its taps (0 when D = 1)                                    */
    int32_t S;                 /* the taps sum to 2^S                                        */
    int32_t reserved;
} ertgpu_decimator_info;

/* The tuning of a handle (ertgpu_set_input_tuning; include/ertgpu_resample.h has the arithmetic). */
typedef struct {
    int64_t capture_center_hz; /* the frequency at the centre of the capture                    */
    int64_t center_hz;         /* the channel decoded (the decoder's CenterFreq when given as 0) */
    int64_t offset_hz;         /* center_hz - capture_center_hz                                  */
    uint32_t nco_step;         /* W = round(offset * 2^32 / R_in) mod 2^32                        */
    int32_t nco_bits;          /* bits of the mixer's phase index (2^nco_bits table entries)     */
} ertgpu_tuning_info;

/* ---- lifecycle -------------------------------------------------------- */

/* protocol.NewDecoder (decode.go:65-71).  No CUDA work yet. */
int ertgpu_create(ertgpu_handle **out);

/* Decoder.RegisterProtocol (decode.go:100-128): merge the parser's config
 * (max of DataRate/ChipLength/PreambleSymbols/PacketSymbols, last CenterFreq)
 * and file it under its preamble.  Must precede ertgpu_allocate. */
int ertgpu_register_protocol(ertgpu_handle *h, const ertgpu_protocol *p);

/* Convenience: fill *p with the stock PacketConfig + screen of a parser by its
 * -msgtype name ("scm","scm+","idm","netidm","r900","r900bcd";
 * protocol/parse.go:42-51 NewParser).  Returns ERTGPU_EINVAL for unknown names
 * (the reference returns an error there, parse.go:49). */
int ertgpu_stock_protocol(const char *msgtype, int32_t chip_length, ertgpu_protocol *p);

/* Decoder.Allocate (decode.go:131-160): derive SymbolLength, BlockSize, ...,
 * select the CUDA device, allocate device buffers for up to
 * max_blocks_per_call blocks per decode call and max_candidates candidates.
 * max_blocks_per_call <= 0 or max_candidates <= 0 pick defaults (2^18
 * candidates).
 *
 * max_candidates bounds the preamble matches ("hits") of one pipeline step: a
 * decode call runs in steps of up to max_blocks_per_call decoder blocks, and
 * every start position of a step whose bits match a registered preamble takes
 * one slot, whatever the decode flags are (ERTGPU_DECODE_ONLY_VALID drops
 * candidates after their screens, so it does not lower the need).  A call
 * with a step of more hits returns ERTGPU_ECAPACITY with "internal" in
 * ertgpu_last_error (see ertgpu_decode).
 *
 * Before any device call it returns ERTGPU_EINVAL, with a message naming the
 * rule, for a merged configuration (PS, PK, CL, SL, PL, PKL, BS, BUF of
 * decode.go:131-141; n = bits of a registered preamble) in which the reference
 * reads something it did not compute for the candidate at hand:
 *   R1  8*ceil((BS+PL)/8) <= BUF: Search packs that many Quantized bits
 *       (decode.go:259-265);
 *   R2  for every preamble, n - 1 <= PK and (n-1)*(SL>>3) + BS/8 <=
 *       ceil((BS+PL)/8): the exact pass and the byte pre-filter stay inside
 *       Quantized and packed (decode.go:268-325);
 *   R3  with an ERTGPU_CHECK_R900 protocol, PK >= PS + 83: every payload digit
 *       lies below BUF - 4*CL, the positions the r900 filter writes
 *       (r900.go:117,187-193).  This also rejects PK = PS+81 and PS+82, where
 *       the reference reads digits it never wrote (zeros) instead of panicking;
 *       decoding them would need a zero-digit branch in two r900 kernels;
 *   R4  when PK % 8 != 0, no ERTGPU_CHECK_CRC16 range [crc_from, crc_to)
 *       holds byte PK>>3: in the reference that byte still carries the
 *       previous candidate's high bits (decode.go:363-366), so its CRC
 *       verdict depends on the order the preambles are searched in.
 * Every stock -msgtype set passes these rules at any chip length. */
int ertgpu_allocate(ertgpu_handle *h, int32_t device, int64_t max_blocks_per_call,
                    int64_t max_candidates);

/* Decoder.Cfg (decode.go:46), valid after ertgpu_allocate. */
int ertgpu_get_config(const ertgpu_handle *h, ertgpu_decoder_config *cfg);

/* Forget the stream history (Signal tail, Quantized history, block counter, and the
 * resampler's input history and partial block): the next decode behaves like the first
 * Decode of a fresh Decoder. */
int ertgpu_reset(ertgpu_handle *h);

/* Declare the sample rate of the IQ the handle will be fed (Hz), between the last
 * ertgpu_register_protocol and ertgpu_allocate.  The decoder keeps its own rate
 * R_out = DataRate * ChipLength (and its geometry, blocks, Idx and taps); when hz != R_out the
 * input is converted to R_out by an exact integer resampler on the GPU, and Block / Idx refer to
 * the resampled stream.  hz == R_out (or never calling this) changes nothing.  R_out / hz must
 * lie in [1/4, 4] ([1/10, 4] on a handle tuned by ertgpu_set_input_tuning, [1/256, 4] on one that also called
 * ertgpu_allow_input_decimation), otherwise ERTGPU_EINVAL.  With resampling, ertgpu_decode and
 * ertgpu_decode_device_async take any whole number of IQ samples (nbytes even, else
 * ERTGPU_ESIZE): the handle carries the input history, the outputs still waiting for look-ahead
 * and the partial output block across calls and decodes every whole block it has.
 * ertgpu_decode_sharded rejects such handles (ERTGPU_EINVAL).  A call that completes no whole block
 * runs only resample_kernel; ertgpu_last_kernels then keeps the list of the last call that ran the
 * decoder (demod first, resample_kernel last). */
int ertgpu_set_input_rate(ertgpu_handle *h, int64_t hz);

/* Decode the channel at center_hz of a capture recorded centred at capture_center_hz (both Hz;
 * center_hz == 0 selects the decoder's CenterFreq, what rtlamr tunes to by default).  Call it after
 * the last ertgpu_register_protocol and before ertgpu_set_input_rate and ertgpu_allocate; otherwise,
 * or for capture_center_hz <= 0 or center_hz < 0, ERTGPU_EINVAL (and ertgpu_register_protocol after
 * it is ERTGPU_EINVAL too).  The resampler then multiplies each input sample by
 * e^(-j 2 pi (center_hz - capture_center_hz) g / R_in) before its lowpass, which is the channel filter,
 * all in integers (include/ertgpu_resample.h).  A tuned handle takes R_out / R_in in [1/10, 4], and
 * the channel must lie inside the capture: |offset| + 0.4 * min(R_in, R_out) <= 0.5 * R_in, checked by
 * ertgpu_set_input_rate, or by ertgpu_allocate when the input is at the decoder's own rate.  An offset
 * of 0 decodes exactly like an untuned handle.  ertgpu_reset restarts the mixer's phase;
 * ERTGPU_TAP_RESAMPLED returns the mixed and filtered bytes; ertgpu_decode_sharded rejects tuned
 * handles.  Several channels of one capture are several handles, fed the same bytes in one pass by
 * ertgpu_decode_channels. */
int ertgpu_set_input_tuning(ertgpu_handle *h, int64_t capture_center_hz, int64_t center_hz);

/* Let a tuned handle take captures at up to 256 times the decoder's rate R_out.  Call it after
 * ertgpu_set_input_tuning and before ertgpu_set_input_rate and ertgpu_allocate; otherwise, and on an untuned handle,
 * ERTGPU_EINVAL.  Up to 10:1 nothing changes: the handle runs the tuned resampler alone, with the same plan, bytes and
 * kernels.  Above 10:1, up to 256:1, the input goes through two stages on the GPU (include/ertgpu_resample.h):
 * decimate_kernel mixes the channel to 0 Hz, lowpasses and keeps every D-th sample, D = ceil(R_in / (4 R_out)), and the
 * untuned uint8 resample_kernel takes R_mid = R_in / D to R_out.  The channel must lie inside the capture,
 * |offset| + 0.4 R_out <= 0.5 R_in.  ertgpu_last_kernels names both kernels (demod first, decimate_kernel<F> and
 * resample_kernel<cu8> last), ERTGPU_TAP_RESAMPLED returns the bytes at R_out, ertgpu_get_resampler describes the
 * second stage and ertgpu_reset restarts both and the mixer's phase. */
int ertgpu_allow_input_decimation(ertgpu_handle *h);

/* The first stage of a handle that allows decimation, once its rate is known (after ertgpu_set_input_rate, or after
 * ertgpu_allocate at the decoder's own rate): *info, and the T1 int16 taps when taps != NULL and cap (entries) is
 * large enough; *n_out = T1.  D = 1 and T1 = 0 when the handle does not decimate.  ERTGPU_EINVAL otherwise. */
int ertgpu_get_decimator(const ertgpu_handle *h, ertgpu_decimator_info *info, int16_t *taps, size_t cap,
                         size_t *n_out);

/* The tuning of a handle; ERTGPU_EINVAL when ertgpu_set_input_tuning was not called. */
int ertgpu_get_tuning(const ertgpu_handle *h, ertgpu_tuning_info *info);

/* Declare the sample format of the IQ the handle will be fed (ERTGPU_FORMAT_*), before
 * ertgpu_allocate (its order relative to ertgpu_set_input_rate is free).  Each component x is
 * converted on the GPU to the byte the decoder reads,
 *     u = (isnan(p) ? 0 : clamp(rint(p), -128, 127)) + 128,   p = fl32(x * scale)
 * (one float32 multiply, both roundings to nearest even).  The 32-bit integer and float64 formats,
 * whose x is not exact in float32, take p = fl64(x * (double)scale) instead and clamp and round it
 * in double.  scale == 0 selects the format's default: 1 for cs8, 2^-8 for the 16-bit formats,
 * 2^7 for the float formats, 2^-24 for the 32-bit integer formats, which map full scale to full scale.
 * ERTGPU_FORMAT_CU8 (or never calling this) changes nothing; it takes no scale.  ERTGPU_EINVAL
 * for an unknown format, a negative or non-finite scale, cu8 with a scale other than 0, or a
 * call after ertgpu_allocate.  With s bytes per IQ sample, a handle that resamples takes any
 * nbytes that is a multiple of s (device input s-byte aligned); one at the decoder's own rate
 * takes a multiple of BlockSize * s (device input 16-byte aligned); otherwise ERTGPU_ESIZE /
 * ERTGPU_EINVAL as for uint8 input.  ertgpu_decode_sharded rejects converting handles. */
int ertgpu_set_input_format(ertgpu_handle *h, int32_t format, float scale);

/* The format and the scale in effect (the default filled in). */
int ertgpu_get_input_format(const ertgpu_handle *h, int32_t *format, float *scale);

/* The level of a converted input (include/ertgpu_level.h has the rule): a histogram of e = floor(log2 |x|) over the
 * components x of the samples measured, and the gain the rule picks from it. */
typedef struct {
    int64_t components, zeros, nans; /* components measured (2 per IQ sample); of them zero (+-0) and NaN         */
    int64_t bins[256];   /* bins[e + 128]: components with 2^e <= |x| < 2^(e+1), e clamped to [-128, 127]; +-inf in bins[255] */
    int32_t exponent;    /* k of the rule (log2 of the format's default gain when no component is non-zero and non-NaN) */
    float scale;         /* 2^k, or the format's default                                                                 */
} ertgpu_input_level;

/* Measure nbytes of samples in HOST memory (pinned or pageable) in the handle's input format: *out gets their
 * histogram and the gain ertgpu_level.h's rule picks.  Any whole number of IQ samples is accepted (otherwise
 * ERTGPU_ESIZE); they are copied through the handle's staging buffers and counted on the GPU on the handle's device
 * and stream.  Nothing of the decode stream changes: a decode after a measure returns exactly what it returns
 * without it.  Nothing is applied either: ertgpu_set_input_scale does that.  ERTGPU_EINVAL before ertgpu_allocate
 * and for ERTGPU_FORMAT_CU8. */
int ertgpu_measure_input(ertgpu_handle *h, const void *samples, size_t nbytes, ertgpu_input_level *out);

/* Change the gain of an allocated, converting handle (scale as for ertgpu_set_input_format, 0: the format's default),
 * at a stream start only: after ertgpu_allocate or ertgpu_reset and before the next decode call.  The gain stays for
 * the stream and survives ertgpu_reset.  ERTGPU_EINVAL otherwise, for ERTGPU_FORMAT_CU8, and for a negative or
 * non-finite scale. */
int ertgpu_set_input_scale(ertgpu_handle *h, float scale);

/* The wide channel path of a tuned handle (include/ertgpu_resample.h has the arithmetic).  Called before
 * ertgpu_allocate, it makes the handle keep its input at 15 bits (s_w = rint(x * scale * 2^7)) through the mixer and
 * the channel filter, and form the decoder's byte only from the last stage's accumulator, scaled by the channel gain
 * 2^k, k in [0, 14].  The gain is then chosen after channel selection, so a weak channel next to a strong one is not
 * cut to the few bits the strong one leaves it.  Every rate and offset the tuned handle takes is accepted, and a wide
 * handle at the decoder's own rate and offset 0 still filters (L = M = 1, T = 22).  After ertgpu_allocate it changes k
 * only at a stream start (after allocate or ertgpu_reset, before the next decode call); k survives ertgpu_reset.
 * ertgpu_last_kernels names the wide instances (resample_kernel<F,tuned,wide>, or decimate_kernel<F,wide> and
 * resample_kernel<mid16,tuned,wide>), ERTGPU_TAP_RESAMPLED returns the wide path's bytes.  ERTGPU_EINVAL on an
 * untuned handle, on a handle allocated without the wide path, for k outside [0, 14], and after a decode call.
 * Handles that never call it decode exactly as before. */
int ertgpu_set_channel_gain(ertgpu_handle *h, int32_t k);

/* The channel gain k of a wide handle; ERTGPU_EINVAL when it is not one. */
int ertgpu_get_channel_gain(const ertgpu_handle *h, int32_t *k);

/* The level of a wide handle's channel: floor(log2 |acc|) of the last stage's output accumulators, and the k the
 * rule of include/ertgpu_resample.h (ertrs_channel_gain) picks from it. */
typedef struct {
    int64_t components;  /* output components measured (2 per output sample)                   */
    int64_t zeros;       /* of them with acc = 0                                                 */
    int64_t bins[32];    /* bins[e]: components with 2^e <= |acc| < 2^(e+1)                     */
    int32_t k;           /* the channel gain the rule picks                                      */
    int32_t reserved;
} ertgpu_channel_level;

/* Run the handle's wide input stage over nbytes of samples in HOST memory (pinned or pageable, any whole number of IQ
 * samples, copied through the handle's staging buffers) as the start of a stream, and histogram the last stage's
 * accumulators instead of forming bytes.  Nothing of the decode stream changes: its position, history, taps and the
 * last call's counts are those before the call.  Nothing is applied either: ertgpu_set_channel_gain does that.
 * ERTGPU_EINVAL before ertgpu_allocate and on a handle without the wide path; ERTGPU_ESIZE for a partial sample. */
int ertgpu_measure_channel(ertgpu_handle *h, const void *samples, size_t nbytes, ertgpu_channel_level *out);

/* The resampler of a handle with an input rate: *info, and the (P+1)*T int16 prototype table
 * when table != NULL and cap (entries) is large enough; *n_out = number of table entries.
 * ERTGPU_EINVAL when the handle does not resample. */
int ertgpu_get_resampler(const ertgpu_handle *h, ertgpu_resampler_info *info, int16_t *table,
                         size_t cap, size_t *n_out);

void ertgpu_destroy(ertgpu_handle *h);

const char *ertgpu_last_error(const ertgpu_handle *h);
int ertgpu_abi_version(void);

/* ---- decode ----------------------------------------------------------- */

/* N consecutive Decoder.Decode(input) calls (decode.go:163-197, called from
 * main.go:235) in one go: iq holds nbytes = N*BlockSize2 interleaved uint8 IQ
 * bytes in HOST memory.  Semantically identical to N sequential reference
 * Decodes: history (Signal tail, Quantized) is carried inside the handle
 * between calls.  Candidates (all preambles) are written in ascending
 * (block, preamble_id, idx) order.  Synchronous; copies are pipelined with
 * the kernels internally.  If more than cap candidates exist the call returns
 * ERTGPU_ECAPACITY with *n_out = the number needed and the stream state
 * already advanced (call ertgpu_fetch with a larger array to get them).
 *
 * ERTGPU_ECAPACITY has a second meaning: a step of the call found more hits
 * than the handle's max_candidates (ertgpu_allocate), and ertgpu_last_error
 * says "internal".  Then *n_out = the most hits of any step of the call: the
 * smallest max_candidates at which the same call succeeds.  The call's
 * candidates (and signal reports) are lost: ertgpu_fetch and
 * ertgpu_fetch_signal return the same code and *n_out until the next decode
 * call or ertgpu_reset.  The stream still advances exactly as it would have
 * without the overflow, so the next call decodes as on a handle that never
 * overflowed; and ertgpu_last_counts counts every hit of the call. */
int ertgpu_decode(ertgpu_handle *h, const uint8_t *iq, size_t nbytes, uint32_t flags,
                  ertgpu_candidate *out, size_t cap, size_t *n_out);

/* Same, with the IQ bytes already in DEVICE memory of the handle's device.
 * `stream` is a cudaStream_t (NULL = the handle's own stream).  Enqueues all
 * kernels on that stream and returns without synchronising; the results are
 * read with ertgpu_fetch.  d_iq must stay valid until then. */
int ertgpu_decode_device_async(ertgpu_handle *h, const void *d_iq, size_t nbytes, uint32_t flags,
                               void *stream);

/* Several channels of ONE capture in one pass: handles[0..n) are tuned to different channels of the same capture, and
 * each decodes the nbytes of iq (HOST memory, pinned or pageable, staged as ertgpu_decode stages it) exactly as
 * ertgpu_decode would on that handle alone: the same candidates, taps, block counts and stream state.  The input crosses
 * the host link once per chunk, into handles[0]'s staging buffers, and every channel reads that device copy.  Above
 * 10:1 (a first stage with D > 1) one decimate_channels_kernel converts each input sample once and runs the first stage
 * of every channel; then each handle runs its own second stage and pipeline.  Up to 10:1 each handle's tuned resampler
 * reads the shared copy.  Synchronous; read each handle's candidates with ertgpu_fetch(handles[c], ...).  Call splits
 * are free: n calls on a group equal one call over the same bytes.  The rules, each broken one ERTGPU_EINVAL with the
 * rule named in ertgpu_last_error(handles[0]):
 *   1 <= n <= ERTGPU_MAX_CHANNELS, and no handle appears twice;
 *   every handle is allocated, on one device, with the same protocols, equal field for field even where a screen
 *   ignores the field (and so the same chip length);
 *   every handle is tuned (ertgpu_set_input_tuning), with the same capture centre, input rate, format and scale;
 *   every handle is at the same stream position (fresh, or reset together, and fed together since);
 *   every handle takes the wide channel path (ertgpu_set_channel_gain), each with its own k, or none does.  Wide
 *   handles run their first stage each on its own.
 * Otherwise every rule of ertgpu_decode holds for each handle. */
int ertgpu_decode_channels(ertgpu_handle *const *handles, int32_t n, const uint8_t *iq, size_t nbytes, uint32_t flags);

/* The same with the input in DEVICE memory of the handles' device, enqueued on `stream` (a cudaStream_t, NULL = the
 * handles[0]'s own stream) without synchronising, as ertgpu_decode_device_async does for one handle.  d_iq must stay
 * valid until every handle's candidates are fetched. */
int ertgpu_decode_channels_device_async(ertgpu_handle *const *handles, int32_t n, const void *d_iq, size_t nbytes,
                                        uint32_t flags, void *stream);

/* Wait for the decode enqueued last and copy its candidates out (sorted as
 * above).  May be repeated (e.g. after ERTGPU_ECAPACITY): an array too small
 * loses nothing.  ERTGPU_ECAPACITY as ertgpu_decode returns it, in both
 * meanings (*n_out = the candidates, or the hits of the largest step). */
int ertgpu_fetch(ertgpu_handle *h, ertgpu_candidate *out, size_t cap, size_t *n_out);

/* Per-packet signal reports.  ertgpu_enable_signal, called before ertgpu_allocate (after it: ERTGPU_EINVAL), makes
 * every decode of the handle also measure each candidate it returns on its own samples, on the GPU behind the slice
 * stage (packet_signal_kernel, counted in ertgpu_last_launches and named last in ertgpu_last_kernels).  The candidates
 * themselves are exactly those of a handle without reports.  ertgpu_fetch_signal returns one ertgpu_signal per
 * candidate the last ertgpu_decode or ertgpu_fetch returned, in the same order, with ertgpu_fetch's capacity rules
 * (ERTGPU_ECAPACITY with *n_out = the number needed); it works after ertgpu_decode, ertgpu_decode_device_async +
 * ertgpu_fetch and, per handle, ertgpu_decode_channels[_device_async].  ERTGPU_EINVAL on a handle without reports.
 * ertgpu_decode_sharded rejects handles with reports. */
int ertgpu_enable_signal(ertgpu_handle *h);
int ertgpu_fetch_signal(ertgpu_handle *h, ertgpu_signal *out, size_t cap, size_t *n_out);

/* The power spectrum of the input (include/ertgpu_spectrum.h).  ertgpu_enable_spectrum, called before ertgpu_allocate
 * (after it: ERTGPU_EINVAL), makes every decode of the handle also measure its input samples, as the caller passed them,
 * in frames of N = 2^log2_n samples (ERTSPEC_LOG2_MIN <= log2_n <= ERTSPEC_LOG2_MAX), frames_per_row F frames to a row,
 * N F >= ERTSPEC_ROW_MIN_SAMPLES (else ERTGPU_EINVAL).  Any handle takes it, whatever its format, rate and tuning.  The
 * kernel (spectrum_kernel<F>) runs on the handle's stream behind each step of the decode, is counted in
 * ertgpu_last_launches and named last in ertgpu_last_kernels; candidates and signal reports are those of a handle
 * without a spectrum.  Rows do not depend on how the stream is cut into calls.
 * Rows wait on the device until they are fetched.  allocate sizes that buffer for the rows of one call of up to
 * max_blocks_per_call blocks of the decoder, times the input rate over the decoder's rate (rounded up) input samples,
 * plus two; a decode call whose rows would not fit beside the rows not yet fetched returns ERTGPU_ECAPACITY before it
 * enqueues anything (fetch, then repeat the call).
 * ertgpu_fetch_spectrum waits for the handle's work and returns the rows completed since the last fetch, in order:
 * rows[i], and mean[i * N .. (i+1) * N) and peak[i * N ..] by ascending bin.  With partial = 1 it also returns the open
 * row, when it has at least one frame, last and without consuming it.  *n_out = the rows returned, or, with
 * ERTGPU_ECAPACITY, the rows needed (nothing is consumed).  ERTGPU_EINVAL on a handle without a spectrum.  ertgpu_reset
 * restarts frames, rows and the carried samples.  ertgpu_decode_channels[_device_async] takes at most one handle with a
 * spectrum, which measures the group's input once; ertgpu_decode_sharded rejects handles with a spectrum. */
int ertgpu_enable_spectrum(ertgpu_handle *h, int32_t log2_n, int64_t frames_per_row);
int ertgpu_fetch_spectrum(ertgpu_handle *h, int32_t partial, ertgpu_spectrum_row *rows, float *mean, float *peak,
                          size_t cap, size_t *n_out);

/* Number of candidates of the last decode, and how many passed a screen.
 * n_candidates counts every hit of the call (with flags 0, one candidate
 * each), also after an overflow of max_candidates; n_valid then counts only
 * the hits the handle held, and may fall short. */
int ertgpu_last_counts(ertgpu_handle *h, int64_t *n_candidates, int64_t *n_valid);

/* Kernels launched by the last decode call (for bench.py's gpu_launches). */
int64_t ertgpu_last_launches(const ertgpu_handle *h);

/* Per-stage device timing of the decode pipeline (CUDA events recorded on the
 * launching stream around each stage; for bench.py's roofline).  After a decode
 * with timing enabled, ms4[] = {demod (magnitude+filter+quantize+pack),
 * search, slice+screens (+r900 replay), history carry} of the last pipeline. */
int ertgpu_set_stage_timing(ertgpu_handle *h, int32_t enable);
int ertgpu_last_stage_ms(ertgpu_handle *h, float *ms4);
/* Mean of the same four stage times over every pipeline since timing was enabled. */
int ertgpu_stage_ms_mean(ertgpu_handle *h, float *ms4, int64_t *n_pipelines);

/* Parity tap: reference buffer `which` as it would be after the Decode of
 * block `block` (absolute index; must lie inside the last decode call).
 * Writes up to cap bytes to dst (host), *n_out = bytes of the full tap. */
int ertgpu_tap(ertgpu_handle *h, int32_t which, int64_t block, void *dst, size_t cap,
               size_t *n_out);

/* Test hook: variant 0 forces the generic (any chip length) demod kernel,
 * -1 restores the automatic choice of a chip-length-specialised kernel. */
int ertgpu_set_demod_variant(ertgpu_handle *h, int32_t variant);

/* Pinned host memory for callers that can use it (cudaHostAlloc/cudaFreeHost).  ertgpu_decode
 * accepts any host memory: pinned input is copied to the device directly; ordinary (pageable)
 * input -- a Go slice, the block buffer of main.go:166 -- is staged through pinned buffers the
 * handle owns (the copy into them runs on a few host threads and overlaps the H2D transfer of
 * the previous chunk), so the caller never has to know. */
int ertgpu_host_alloc(void **out, size_t nbytes);
int ertgpu_host_free(void *p);

/* Restrict the CALLING thread to the CPUs next to `device` (the PCI device's local_cpulist in
 * sysfs), so that the pinned buffers it allocates afterwards and the staging copies it runs are
 * NUMA-local to the GPU.  Optional; *ncpus = CPUs in the new mask, *numa_node = the device's
 * node (-1 unknown).  Returns ERTGPU_EINVAL when the topology cannot be read (nothing changed). */
int ertgpu_bind_host_thread(int32_t device, int32_t *ncpus, int32_t *numa_node);

/* Names of the kernel instantiations the last decode launched (for bench.py's roofline label). */
const char *ertgpu_last_kernels(const ertgpu_handle *h);

/* ---- one stream over several GPUs (SURVEY.md section 8e; main.go:207-235 is where the
 * reference would hang such a driver) ------------------------------------------------- */

/* Shard r of a stream of total_blocks reference blocks cut into nshards contiguous block-aligned
 * shards: the shard REPORTS the candidates of blocks [first_block, last_block) and must be FED
 * from first_fed_block (halo: ceil(PacketLength/BlockSize) blocks of Quantized history,
 * decode.go:166, plus one block of Signal lead-in, decode.go:165). */
typedef struct {
    int64_t first_block, last_block, first_fed_block;
} ertgpu_shard;
int ertgpu_plan_shards(int64_t total_blocks, int32_t nshards, int32_t block_size, int32_t packet_length,
                       ertgpu_shard *out /* [nshards] */);

/* N consecutive Decoder.Decode calls on a FRESH stream, spread over nhandles handles (normally
 * one per GPU; several on one GPU also work): handle r decodes shard r (halo + owned blocks) of
 * the host buffer on its own device from its own host thread, candidates of halo blocks are
 * dropped, block numbers are made global and the lists are concatenated in (block, preamble,
 * idx) order -- the same list one handle returns for the whole buffer after ertgpu_reset.
 * All handles must be allocated with the same protocols; each is reset first.  There is no
 * collective: shards are independent (every candidate is decided inside one shard + halo).
 * The call empties every handle's ertgpu_last_error first; a shard's failure leaves its
 * message on its handle.  When shards overflow their handle's max_candidates (shard and halo
 * are one ertgpu_decode), it returns ERTGPU_ECAPACITY with *n_out = the largest need of those
 * shards; when only the output array is too small, *n_out = the candidates. */
int ertgpu_decode_sharded(ertgpu_handle *const *handles, int32_t nhandles, const uint8_t *iq, size_t nbytes,
                          uint32_t flags, ertgpu_candidate *out, size_t cap, size_t *n_out);

/* ---- synthetic input (bench/test tooling, not part of the reference API) -- */

/* One injected packet: chips are OOK "high"/"low" flags, MSB first. */
typedef struct {
    int64_t start_sample;  /* first sample of chip 0 in the global stream */
    int32_t n_chips;       /* <= 1536                                      */
    int32_t chip_length;   /* samples per chip                             */
    int16_t amp_i, amp_q;  /* carrier added to I,Q on high chips           */
    uint8_t chips[192];
    int32_t pad;
} ertgpu_synth_packet;

/* Fill d_out (device) with nsamples IQ samples of the synthetic stream
 * starting at global sample index first_sample: counter-based noise keyed by
 * (seed, sample index) plus the given packets (host array, sorted by
 * start_sample, non-overlapping).  Bit-identical to synth_reference_fill() in
 * include/ertgpu_synth.h on the host. */
int ertgpu_synth_fill(int32_t device, void *d_out, int64_t first_sample, int64_t nsamples,
                      uint64_t seed, const ertgpu_synth_packet *packets, int64_t npackets,
                      void *stream);

#ifdef __cplusplus
}
#endif
#endif
