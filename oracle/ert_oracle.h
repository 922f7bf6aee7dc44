/*
 * ert_oracle.h -- CPU restatement of rtlamr's protocol.Decoder hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product:
 * only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load this library, and only as the checker or as
 * the timed CPU baseline.  The product path (rtlamr_b200/, libertgpu.so) never
 * links, imports or calls it.
 *
 * Parity pinning: the reference's own tests pin only CRC algebra
 * (crc/crc_test.go:22-41).  This oracle is pinned against (a) those CRC
 * identities and the standard "123456789" check values, (b) the LUT/geometry
 * known answers of SURVEY.md section 8c/8d, and (c) the 14 self-verifying
 * (CRC-valid) SCM messages recovered from the reference's assets/sample.bin
 * fixture (tests/golden/).  The Go toolchain is absent from this image, so the
 * reference itself could not be run: decoder-level parity is "unpinned by the
 * reference's own tests" beyond those items -- see DESIGN.md.
 *
 * Every function cites the reference file:line it restates (paths relative to
 * the reference checkout).
 */
#ifndef ERT_ORACLE_H
#define ERT_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* protocol ids (registration names: protocol/parse.go:28, each parser's init()) */
enum {
    ERT_SCM = 0,     /* scm/scm.go:33     */
    ERT_SCMPLUS = 1, /* scmplus/scmplus.go:32 */
    ERT_IDM = 2,     /* idm/idm.go:30     */
    ERT_NETIDM = 3,  /* netidm/netidm.go:30 */
    ERT_R900 = 4,    /* r900/r900.go:34   */
    ERT_R900BCD = 5, /* r900bcd/r900bcd.go:27 */
    ERT_NPROTO = 6
};

/* search modes */
enum {
    ERT_SEARCH_GO = 0,   /* literal decode.go:255-328 (byte pre-filter with SL>>3) */
    ERT_SEARCH_EXACT = 1 /* exact stride-SL test of every idx in [0,BlockSize)      */
};

/* mirrors protocol.PacketConfig (decode.go:27-42) */
typedef struct {
    int32_t data_rate;
    int32_t block_size, block_size2;
    int32_t chip_length, symbol_length;
    int32_t sample_rate;
    int32_t preamble_symbols, packet_symbols;
    int32_t preamble_length, packet_length;
    int32_t buffer_length;
    uint32_t center_freq;
} ert_oracle_cfg;

#define ERT_ORACLE_MAX_PKT 96

/* one protocol.Data (parse.go:55-59) produced by Slice (decode.go:353-375) */
typedef struct {
    int64_t block;       /* 0-based index of the Decode call            */
    int32_t idx;         /* Data.Idx                                    */
    int32_t preamble_id; /* distinct preamble, in registration order    */
    int32_t nbytes;      /* (PacketSymbols+7)>>3 of the merged config   */
    uint8_t bytes[ERT_ORACLE_MAX_PKT];
} ert_oracle_cand;

/* one protocol.Message as emitted by a parser's Parse */
typedef struct {
    int64_t block;
    int32_t idx;
    int32_t proto;        /* ERT_* */
    uint32_t meter_id;    /* Message.MeterID()   */
    uint32_t meter_type;  /* Message.MeterType() */
    uint32_t consumption; /* SCM/SCM+ Consumption, IDM LastConsumptionCount,
                             NetIDM LastConsumptionNet, R900 Consumption */
    int32_t nchecksum;    /* 2 (CRC) or 5 (r900 RS symbols) */
    uint8_t checksum[8];  /* Message.Checksum() */
    int32_t nbytes;       /* parser's own prefix length (r900: 21 symbols) */
    uint8_t bytes[ERT_ORACLE_MAX_PKT];
} ert_oracle_msg;

typedef struct ert_oracle ert_oracle;

#define ERT_ORACLE_MAX_PROTOS 8 /* protocols one decoder registers (ERTGPU_MAX_PROTOCOLS) */
#define ERT_PARSER_NONE (-1)    /* candidates only: no parser runs on them */

/* One parser's PacketConfig (decode.go:27-42) and the parser that runs on its
 * candidates: a stock ERT_* parser (ERT_R900 / ERT_R900BCD: the r900 DSP parser,
 * r900.go:160-245) or ERT_PARSER_NONE. */
typedef struct {
    char preamble[33]; /* '0'/'1', 1..32 bits */
    int32_t data_rate, chip_length;
    int32_t preamble_symbols, packet_symbols;
    uint32_t center_freq;
    int32_t parser;
} ert_oracle_proto;

/* NewDecoder + RegisterProtocol for every entry of p[] (in that order, merged
 * per protocol as decode.go:100-128 does, ChipLength included) + Allocate
 * (decode.go:131-160).  Returns NULL on bad input. */
ert_oracle *ert_oracle_new_protocols(const ert_oracle_proto *p, int32_t n, int32_t search_mode);

/* The same for the stock parsers protos[] (ERT_* ids), all at one chip length. */
ert_oracle *ert_oracle_new(const int32_t *protos, int32_t nprotos, int32_t chip_length,
                           int32_t search_mode);
void ert_oracle_free(ert_oracle *o);

const ert_oracle_cfg *ert_oracle_config(const ert_oracle *o);
int32_t ert_oracle_npreambles(const ert_oracle *o);

/* One Decoder.Decode(input) call (decode.go:163-197) on block_size2 bytes,
 * followed by every registered parser's Parse.  Candidates and messages of
 * this block are appended to the caller's arrays (up to the caps); the
 * return value is 0, or -1 if a cap was hit (counts are still exact), or
 * ERT_ORACLE_PANIC when the reference would index a slice past its length
 * here (Search's packing, byte pre-filter or exact pass, Slice, the r900 digit
 * reads): nothing is read out of bounds, the block's results are incomplete
 * and every later call returns ERT_ORACLE_PANIC too (the reference has died). */
#define ERT_ORACLE_PANIC (-2)
int32_t ert_oracle_decode(ert_oracle *o, const uint8_t *input, ert_oracle_cand *cands,
                          int32_t cand_cap, int32_t *ncands, ert_oracle_msg *msgs,
                          int32_t msg_cap, int32_t *nmsgs);

/* Convenience: feed nblocks consecutive blocks. Totals returned in ncands/nmsgs. */
int32_t ert_oracle_decode_stream(ert_oracle *o, const uint8_t *input, int64_t nblocks,
                                 ert_oracle_cand *cands, int32_t cand_cap, int32_t *ncands,
                                 ert_oracle_msg *msgs, int32_t msg_cap, int32_t *nmsgs);

/* DSP only (shift + magnitude + Filter, no Search/Parse): used by the timed CPU
 * baseline to separate DSP cost, and by parity taps. */
void ert_oracle_dsp_only(ert_oracle *o, const uint8_t *input);

/* parity taps: state after the most recent Decode */
const float *ert_oracle_signal(const ert_oracle *o, int32_t *n);      /* Decoder.Signal    */
const float *ert_oracle_csum(const ert_oracle *o, int32_t *n);        /* Decoder.csum      */
const uint8_t *ert_oracle_quantized(const ert_oracle *o, int32_t *n); /* Decoder.Quantized */
const uint8_t *ert_oracle_packed(const ert_oracle *o, int32_t *n);    /* Decoder.packed    */
const uint8_t *ert_oracle_r900_quantized(const ert_oracle *o, int32_t *n); /* r900 Parser.quantized */
const float *ert_oracle_maglut(void);                                 /* NewMagLUT, 256 entries */

/* crc/crc.go */
void ert_crc_table(uint16_t poly, uint16_t table[256]);                       /* crc.go:34-47 */
uint16_t ert_crc_checksum(uint16_t init, const uint8_t *data, size_t n,
                          const uint16_t table[256]);                         /* crc.go:49-55 */

/* r900/gf/gf.go: GF(32), poly 37, generator 2; Syndrome(message,5,29) */
void ert_gf32_syndrome(const uint8_t *message, int32_t n, int32_t nparity, int32_t offset,
                       uint8_t *syndrome);

/* ert_oracle_bench.c: the timed CPU baseline.  `nthreads` independent decoders (one per thread,
 * like the reference's single DSP goroutine, main.go:207-235) over contiguous block-aligned
 * shards of one stream of `nblocks` blocks, each decoded `repeats` times in BlockSize2-byte
 * Decode calls.  Returns wall seconds (common start to last finish), < 0 on failure. */
double ert_oracle_bench_threads(const int32_t *protos, int32_t nprotos, int32_t chip_length,
                                int32_t search_mode, const uint8_t *iq, int64_t nblocks,
                                int32_t nthreads, int32_t repeats, int32_t pin,
                                int64_t *ncands, int64_t *nmsgs);
int32_t ert_oracle_host_cpus(void);

#ifdef __cplusplus
}
#endif
#endif
