/*
 * ert_oracle.c -- CPU restatement of rtlamr's protocol.Decoder hot path.
 *
 * TEST INFRASTRUCTURE ONLY (see ert_oracle.h).  Plain C, strict IEEE float32
 * in the reference's operation order; build with -O2 -ffp-contract=off and
 * without -ffast-math (oracle/Makefile).  Go on amd64 evaluates the same
 * expressions as scalar SSE float32 with no fused multiply-add, so `float`
 * arithmetic here is bit-identical to the reference's.
 *
 * Citations are reference file:line.
 */
#include "ert_oracle.h"

#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------ */
/* protocol descriptors: the PacketConfig literal of each NewParser    */
/* ------------------------------------------------------------------ */
typedef struct {
    const char *name;
    const char *preamble;
    int32_t preamble_symbols, packet_symbols;
    int32_t data_rate;
    uint32_t center_freq;
} proto_desc;

static const proto_desc PROTO[ERT_NPROTO] = {
    /* scm/scm.go:42-50 */
    {"scm", "111110010101001100000", 21, 96, 32768, 912600155u},
    /* scmplus/scmplus.go:49-57 */
    {"scm+", "0001011010100011", 16, 128, 32768, 912600155u},
    /* idm/idm.go:48-56 */
    {"idm", "01010101010101010001011010100011", 32, 736, 32768, 912600155u},
    /* netidm/netidm.go:60-68 */
    {"netidm", "01010101010101010001011010100011", 32, 736, 32768, 912600155u},
    /* r900/r900.go:57-65 */
    {"r900", "00000000000000001110010101100100", 32, 116, 32768, 912380000u},
    /* r900bcd/r900bcd.go:35-37 wraps r900.NewParser */
    {"r900bcd", "00000000000000001110010101100100", 32, 116, 32768, 912380000u},
};

#define MAX_PREAMBLE_BITS 32

typedef struct {
    uint8_t bits[MAX_PREAMBLE_BITS]; /* numeric 0/1, decode.go:113-118 */
    int32_t nbits;
    int32_t parsers[ERT_ORACLE_MAX_PROTOS]; /* registration indices sharing this preamble, decode.go:124 */
    int32_t nparsers;
} preamble_entry;

/* r900 parser private state (r900/r900.go:42-55,161-166) */
typedef struct {
    int32_t active;
    float *signal;      /* BufferLength   */
    float *csum;        /* BufferLength+1 */
    uint8_t *quantized; /* BufferLength   */
    uint8_t rs_buf[31];
} r900_state;

struct ert_oracle {
    ert_oracle_cfg cfg;
    int32_t search_mode;
    int64_t block; /* number of Decode calls so far */
    int panicked;  /* the reference indexed past a slice: it has died */

    float lut[256];

    float *signal;      /* BlockSize+SymbolLength, decode.go:144 */
    float *csum;        /* len(signal)+1,         decode.go:147 */
    uint8_t *quantized; /* BufferLength,          decode.go:145 */
    uint8_t *packed;    /* (BS+PL+7)>>3,          decode.go:159 */
    int32_t npacked;
    uint8_t pkt[ERT_ORACLE_MAX_PKT]; /* d.pkt, reused and never cleared: decode.go:154,363-366 */
    int32_t npkt;
    int32_t *idx_a, *idx_b; /* sIdxA/sIdxB, decode.go:156-157 (sized 8x for the expand step) */

    preamble_entry pre[ERT_ORACLE_MAX_PROTOS];
    int32_t npre;

    int32_t parser[ERT_ORACLE_MAX_PROTOS];   /* ERT_* or ERT_PARSER_NONE, by registration index */
    r900_state r900[ERT_ORACLE_MAX_PROTOS]; /* by registration index: each registered r900 parser owns its buffers */

    uint16_t bch[256];   /* crc.NewTable(0x6F63) */
    uint16_t ccitt[256]; /* crc.NewTable(0x1021) */
    uint8_t gf_exp[62], gf_log[32];
};

/* ------------------------------------------------------------------ */
/* crc/crc.go                                                          */
/* ------------------------------------------------------------------ */
/* crc.go:34-47 NewTable */
void ert_crc_table(uint16_t poly, uint16_t table[256]) {
    for (int t = 0; t < 256; t++) {
        uint16_t crc = (uint16_t)(t << 8);
        for (int b = 0; b < 8; b++) {
            if (crc & 0x8000)
                crc = (uint16_t)((crc << 1) ^ poly);
            else
                crc = (uint16_t)(crc << 1);
        }
        table[t] = crc;
    }
}

/* crc.go:49-55 Checksum */
uint16_t ert_crc_checksum(uint16_t init, const uint8_t *data, size_t n, const uint16_t table[256]) {
    uint16_t crc = init;
    for (size_t i = 0; i < n; i++)
        crc = (uint16_t)((crc << 8) ^ table[(crc >> 8) ^ data[i]]);
    return crc;
}

/* ------------------------------------------------------------------ */
/* r900/gf/gf.go: NewField(32, 37, 2)                                  */
/* ------------------------------------------------------------------ */
/* gf.go:88-101 mul */
static int gf_slow_mul(int x, int y, int order, int poly) {
    int z = 0;
    while (x > 0) {
        if (x & 1) z ^= y;
        x >>= 1;
        y <<= 1;
        if (y & order) y ^= poly;
    }
    return z;
}

/* gf.go:20-57 NewField: exp has 2*(order-1) entries, log[0] = order-1 */
static void gf32_tables(uint8_t exp[62], uint8_t log[32]) {
    int x = 1;
    for (int i = 0; i < 31; i++) {
        exp[i] = (uint8_t)x;
        exp[i + 31] = (uint8_t)x;
        log[x] = (uint8_t)i;
        x = gf_slow_mul(x, 2, 32, 37);
    }
    log[0] = 31;
}

/* gf.go:143-148 Mul, gf.go:118-123 Exp */
static uint8_t gf32_mul(const uint8_t exp[62], const uint8_t log[32], uint8_t x, uint8_t y) {
    if (x == 0 || y == 0) return 0;
    return exp[(int)log[x] + (int)log[y]];
}

/* gf.go:152-172 Syndrome */
static void gf32_syndrome_tbl(const uint8_t exp[62], const uint8_t log[32], const uint8_t *message,
                              int32_t n, int32_t nparity, int32_t offset, uint8_t *syndrome) {
    for (int idx = 0; idx < nparity; idx++) {
        uint8_t syn = message[0];
        uint8_t root = exp[(offset + idx) % 31];
        for (int j = 1; j < n; j++) syn = (uint8_t)(gf32_mul(exp, log, syn, root) ^ message[j]);
        syndrome[idx] = syn;
    }
}

void ert_gf32_syndrome(const uint8_t *message, int32_t n, int32_t nparity, int32_t offset,
                       uint8_t *syndrome) {
    uint8_t exp[62], log[32];
    gf32_tables(exp, log);
    gf32_syndrome_tbl(exp, log, message, n, nparity, offset, syndrome);
}

/* ------------------------------------------------------------------ */
/* decode.go:209-216 NewMagLUT                                         */
/* ------------------------------------------------------------------ */
static void make_maglut(float lut[256]) {
    for (int i = 0; i < 256; i++) {
        /* untyped constants take the float32 type of the expression */
        float v = (127.5f - (float)i) / 127.5f;
        v = v * v;
        lut[i] = v;
    }
}

const float *ert_oracle_maglut(void) {
    static float lut[256];
    make_maglut(lut);
    return lut;
}

/* decode.go:377-379 NextPowerOf2 = 1 << ceil(log2(v)) */
static int32_t next_pow2(int32_t v) {
    int32_t p = 1;
    while (p < v) p <<= 1;
    return p;
}

static int32_t imax(int32_t a, int32_t b) { return a > b ? a : b; }

/* bits of a preamble string in a 33-byte field (MAX_PREAMBLE_BITS + 1 when unterminated) */
static int32_t preamble_len(const char *s) {
    int32_t n = 0;
    while (n <= MAX_PREAMBLE_BITS && s[n]) n++;
    return n;
}

/* ------------------------------------------------------------------ */
/* construction: NewDecoder, RegisterProtocol, Allocate                */
/* ------------------------------------------------------------------ */
ert_oracle *ert_oracle_new(const int32_t *protos, int32_t nprotos, int32_t chip_length,
                           int32_t search_mode) {
    if (!protos || nprotos <= 0 || nprotos > ERT_ORACLE_MAX_PROTOS || chip_length <= 0) return NULL;
    ert_oracle_proto p[ERT_ORACLE_MAX_PROTOS];
    memset(p, 0, sizeof(p));
    for (int i = 0; i < nprotos; i++) {
        const int32_t id = protos[i];
        if (id < 0 || id >= ERT_NPROTO) return NULL;
        const proto_desc *d = &PROTO[id];
        strcpy(p[i].preamble, d->preamble);
        p[i].data_rate = d->data_rate;
        p[i].chip_length = chip_length;
        p[i].preamble_symbols = d->preamble_symbols;
        p[i].packet_symbols = d->packet_symbols;
        p[i].center_freq = d->center_freq;
        p[i].parser = id;
    }
    return ert_oracle_new_protocols(p, nprotos, search_mode);
}

ert_oracle *ert_oracle_new_protocols(const ert_oracle_proto *protos, int32_t nprotos, int32_t search_mode) {
    if (!protos || nprotos <= 0 || nprotos > ERT_ORACLE_MAX_PROTOS) return NULL;
    for (int i = 0; i < nprotos; i++) {
        const ert_oracle_proto *p = &protos[i];
        const int32_t n = preamble_len(p->preamble);
        if (n == 0 || n > MAX_PREAMBLE_BITS || p->chip_length <= 0 || p->preamble_symbols <= 0 ||
            p->packet_symbols <= 0 || (p->packet_symbols + 7) / 8 > ERT_ORACLE_MAX_PKT ||
            p->parser < ERT_PARSER_NONE || p->parser >= ERT_NPROTO)
            return NULL;
        for (int32_t k = 0; k < n; k++)
            if (p->preamble[k] != '0' && p->preamble[k] != '1') return NULL;
    }
    ert_oracle *o = (ert_oracle *)calloc(1, sizeof(*o));
    if (!o) return NULL;
    o->search_mode = search_mode;

    /* decode.go:100-128 RegisterProtocol, in the caller's order */
    for (int i = 0; i < nprotos; i++) {
        const ert_oracle_proto *p = &protos[i];
        o->cfg.center_freq = p->center_freq;                                         /* :105 */
        o->cfg.data_rate = imax(o->cfg.data_rate, p->data_rate);                     /* :106 */
        o->cfg.chip_length = imax(o->cfg.chip_length, p->chip_length);               /* :107 */
        o->cfg.preamble_symbols = imax(o->cfg.preamble_symbols, p->preamble_symbols); /* :108 */
        o->cfg.packet_symbols = imax(o->cfg.packet_symbols, p->packet_symbols);      /* :109 */

        preamble_entry e;
        memset(&e, 0, sizeof(e));
        e.nbits = preamble_len(p->preamble);
        for (int k = 0; k < e.nbits; k++) e.bits[k] = (uint8_t)(p->preamble[k] == '1'); /* :113-118 */
        int found = -1;
        for (int j = 0; j < o->npre; j++)
            if (o->pre[j].nbits == e.nbits && memcmp(o->pre[j].bits, e.bits, (size_t)e.nbits) == 0)
                found = j;
        if (found < 0) {
            found = o->npre++;
            o->pre[found] = e;
        }
        o->pre[found].parsers[o->pre[found].nparsers++] = i; /* :124 */
        o->parser[i] = p->parser;
        if (p->parser == ERT_R900 || p->parser == ERT_R900BCD) o->r900[i].active = 1;
    }

    /* decode.go:131-141 Allocate */
    ert_oracle_cfg *c = &o->cfg;
    c->symbol_length = c->chip_length << 1;
    c->sample_rate = c->data_rate * c->chip_length;
    c->preamble_length = c->preamble_symbols * c->symbol_length;
    c->packet_length = c->packet_symbols * c->symbol_length;
    c->block_size = next_pow2(c->preamble_length);
    c->block_size2 = c->block_size << 1;
    c->buffer_length = c->packet_length + c->block_size;

    /* decode.go:144-159 buffers (zero-initialised like Go's make) */
    o->signal = (float *)calloc((size_t)(c->block_size + c->symbol_length), sizeof(float));
    o->csum = (float *)calloc((size_t)(c->block_size + c->symbol_length + 1), sizeof(float));
    o->quantized = (uint8_t *)calloc((size_t)c->buffer_length, 1);
    o->npacked = (c->block_size + c->preamble_length + 7) >> 3;
    o->packed = (uint8_t *)calloc((size_t)o->npacked, 1);
    o->npkt = (c->packet_symbols + 7) >> 3;
    o->idx_a = (int32_t *)calloc((size_t)c->block_size + 8, sizeof(int32_t));
    o->idx_b = (int32_t *)calloc((size_t)c->block_size + 8, sizeof(int32_t));
    make_maglut(o->lut);

    /* r900.go:161-166 once.Do: buffers sized from the merged decoder config */
    for (int k = 0; k < ERT_ORACLE_MAX_PROTOS; k++) {
        if (!o->r900[k].active) continue;
        o->r900[k].signal = (float *)calloc((size_t)c->buffer_length, sizeof(float));
        o->r900[k].csum = (float *)calloc((size_t)c->buffer_length + 1, sizeof(float));
        o->r900[k].quantized = (uint8_t *)calloc((size_t)c->buffer_length, 1);
    }

    ert_crc_table(0x6F63, o->bch);
    ert_crc_table(0x1021, o->ccitt);
    gf32_tables(o->gf_exp, o->gf_log);
    return o;
}

void ert_oracle_free(ert_oracle *o) {
    if (!o) return;
    free(o->signal);
    free(o->csum);
    free(o->quantized);
    free(o->packed);
    free(o->idx_a);
    free(o->idx_b);
    for (int k = 0; k < ERT_ORACLE_MAX_PROTOS; k++) {
        free(o->r900[k].signal);
        free(o->r900[k].csum);
        free(o->r900[k].quantized);
    }
    free(o);
}

const ert_oracle_cfg *ert_oracle_config(const ert_oracle *o) { return &o->cfg; }
int32_t ert_oracle_npreambles(const ert_oracle *o) { return o->npre; }

/* ------------------------------------------------------------------ */
/* DSP: decode.go:165-172                                              */
/* ------------------------------------------------------------------ */
void ert_oracle_dsp_only(ert_oracle *o, const uint8_t *input) {
    const ert_oracle_cfg *c = &o->cfg;
    const int32_t bs = c->block_size, sl = c->symbol_length, cl = c->chip_length;
    const int32_t nsig = bs + sl;

    /* :165-166 slide history */
    memmove(o->signal, o->signal + bs, (size_t)(nsig - bs) * sizeof(float));
    memmove(o->quantized, o->quantized + bs, (size_t)(c->buffer_length - bs));

    /* :169 MagLUT.Execute (:219-225) into Signal[SL:] */
    float *out = o->signal + sl;
    for (int32_t j = 0; j < bs; j++) out[j] = o->lut[input[2 * j]] + o->lut[input[2 * j + 1]];

    /* :172 Filter (:229-245): sequential float32 running sum restarted at 0 */
    float sum = 0.0f;
    for (int32_t k = 0; k < nsig; k++) {
        sum += o->signal[k];
        o->csum[k + 1] = sum;
    }
    uint8_t *q = o->quantized + c->packet_length;
    for (int32_t i = 0; i < bs; i++) {
        float l = o->csum[i + cl];
        float f = (l - o->csum[i]) - (o->csum[i + sl] - l);
        uint32_t bits;
        memcpy(&bits, &f, sizeof(bits));
        q[i] = (uint8_t)(1u - (bits >> 31)); /* :243 */
    }
}

/* ------------------------------------------------------------------ */
/* Search: decode.go:255-348                                           */
/* ------------------------------------------------------------------ */
/* Every index below is checked against the length Go's slice has; past it the reference panics and the search
 * returns ERT_ORACLE_PANIC without reading. */
static int32_t pack_quantized(ert_oracle *o) {
    /* :259-265: d.Quantized[bIdx<<3 : (bIdx+1)<<3] */
    if ((int64_t)o->npacked * 8 > o->cfg.buffer_length) return ERT_ORACLE_PANIC;
    for (int32_t b = 0; b < o->npacked; b++) {
        uint8_t v = 0;
        for (int k = 0; k < 8; k++) v = (uint8_t)((v << 1) | o->quantized[(b << 3) + k]);
        o->packed[b] = v;
    }
    return 0;
}

/* returns number of indices left in o->idx_a, or ERT_ORACLE_PANIC */
static int32_t search_go(ert_oracle *o, const preamble_entry *p) {
    const ert_oracle_cfg *c = &o->cfg;
    const int32_t sym_len_byte = c->symbol_length >> 3; /* :256 */
    int32_t *a = o->idx_a, *b = o->idx_b, na = 0, nb = 0;

    if (pack_quantized(o)) return ERT_ORACLE_PANIC;

    for (int32_t k = 0; k < p->nbits; k++) {
        uint8_t mask = (uint8_t)((p->bits[k] ^ 1) * 0xFF); /* :270 */
        int32_t offset = k * sym_len_byte;
        if (k == 0) {
            na = 0;
            for (int32_t qi = 0; qi < (c->block_size >> 3); qi++) /* :277 */
                if (o->packed[qi] != mask) a[na++] = qi;
        } else {
            nb = 0; /* searchPassByte :330-338 over d.packed[offset:] (:287) */
            if (offset > o->npacked) return ERT_ORACLE_PANIC;
            for (int32_t j = 0; j < na; j++) {
                if (offset + a[j] >= o->npacked) return ERT_ORACLE_PANIC;
                if (o->packed[offset + a[j]] != mask) b[nb++] = a[j];
            }
            int32_t *t = a; a = b; b = t; na = nb;
            if (na == 0) return 0; /* :290-292 */
        }
    }

    /* :298-307 expand byte indices to 8 sample indices.  na <= BS/8 so 8*na <= BS. */
    nb = 0;
    for (int32_t j = 0; j < na; j++)
        for (int32_t k = 0; k < 8; k++) b[nb++] = (a[j] << 3) + k;
    { int32_t *t = a; a = b; b = t; na = nb; }

    /* :313-325 exact pass, searchPass :340-348 */
    for (int32_t k = 0; k < p->nbits; k++) {
        /* d.Quantized[offset : offset+BlockSize] (:315) */
        if ((int64_t)k * c->symbol_length + c->block_size > c->buffer_length) return ERT_ORACLE_PANIC;
        const uint8_t *sig = o->quantized + k * c->symbol_length;
        nb = 0;
        for (int32_t j = 0; j < na; j++)
            if (sig[a[j]] == p->bits[k]) b[nb++] = a[j];
        int32_t *t = a; a = b; b = t; na = nb;
        if (na == 0) return 0;
    }
    if (a != o->idx_a) memcpy(o->idx_a, a, (size_t)na * sizeof(int32_t));
    return na;
}

static int32_t search_exact(ert_oracle *o, const preamble_entry *p) {
    const ert_oracle_cfg *c = &o->cfg;
    int32_t n = 0;
    if (pack_quantized(o)) return ERT_ORACLE_PANIC; /* keeps the `packed` tap identical in both modes */
    for (int32_t i = 0; i < c->block_size; i++) {
        int ok = 1;
        for (int32_t k = 0; k < p->nbits && ok; k++) {
            if ((int64_t)i + (int64_t)k * c->symbol_length >= c->buffer_length) return ERT_ORACLE_PANIC;
            ok = o->quantized[i + k * c->symbol_length] == p->bits[k];
        }
        if (ok) o->idx_a[n++] = i;
    }
    return n;
}

/* ------------------------------------------------------------------ */
/* helpers on a Data's bit string                                      */
/* ------------------------------------------------------------------ */
static uint32_t bits_uint(const uint8_t *bytes, int32_t from, int32_t to) {
    /* strconv.ParseUint(data.Bits[from:to], 2, ..) over the "%08b" rendering, parse.go:64-66 */
    uint32_t v = 0;
    for (int32_t i = from; i < to; i++) v = (v << 1) | ((bytes[i >> 3] >> (7 - (i & 7))) & 1u);
    return v;
}

static uint32_t be32(const uint8_t *p) {
    return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
}
static uint16_t be16(const uint8_t *p) { return (uint16_t)(((uint16_t)p[0] << 8) | p[1]); }

typedef struct {
    uint8_t (*keys)[ERT_ORACLE_MAX_PKT + 16];
    int32_t n, cap, klen;
} seen_set;

static int seen_test_and_set(seen_set *s, const uint8_t *key) {
    for (int32_t i = 0; i < s->n; i++)
        if (memcmp(s->keys[i], key, (size_t)s->klen) == 0) return 1;
    if (s->n == s->cap) {
        s->cap = s->cap ? s->cap * 2 : 64;
        s->keys = realloc(s->keys, (size_t)s->cap * sizeof(*s->keys));
    }
    memcpy(s->keys[s->n++], key, (size_t)s->klen);
    return 0;
}

typedef struct {
    ert_oracle_msg *msgs;
    int32_t cap;
    int32_t n;
    int overflow;
} msg_sink;

static void emit(msg_sink *sink, const ert_oracle_msg *m) {
    if (sink->msgs && sink->n < sink->cap)
        sink->msgs[sink->n] = *m;
    else
        sink->overflow = 1;
    sink->n++;
}

/* ------------------------------------------------------------------ */
/* CRC-checked parsers                                                  */
/* ------------------------------------------------------------------ */
/* scm/scm.go:61-90 Parse + :103-119 NewSCM */
static void parse_scm(ert_oracle *o, const ert_oracle_cand *pk, int32_t npk, msg_sink *sink) {
    seen_set seen = {0};
    seen.klen = 12;
    for (int32_t i = 0; i < npk; i++) {
        uint8_t b[12];
        memcpy(b, pk[i].bytes, 12); /* :66-67 copy into the parser's 12-byte buffer */
        if (seen_test_and_set(&seen, b)) continue; /* :69-73 */
        if (ert_crc_checksum(0, b + 2, 10, o->bch) != 0) continue; /* :76 */
        ert_oracle_msg m;
        memset(&m, 0, sizeof(m));
        m.block = pk[i].block;
        m.idx = pk[i].idx;
        m.proto = ERT_SCM;
        m.meter_id = (bits_uint(b, 21, 23) << 24) | bits_uint(b, 56, 80); /* :104 */
        m.meter_type = bits_uint(b, 26, 30);                               /* :105 */
        m.consumption = bits_uint(b, 32, 56);                              /* :108 */
        uint16_t ck = (uint16_t)bits_uint(b, 80, 96);                      /* :109 */
        m.nchecksum = 2;
        m.checksum[0] = (uint8_t)(ck >> 8);
        m.checksum[1] = (uint8_t)ck;
        m.nbytes = 12;
        memcpy(m.bytes, b, 12);
        if (m.meter_id == 0) continue; /* :83-85 */
        emit(sink, &m);
    }
    free(seen.keys);
}

/* scmplus/scmplus.go:60-90 Parse + :105-109 NewSCM (big-endian struct read) */
static void parse_scmplus(ert_oracle *o, const ert_oracle_cand *pk, int32_t npk, msg_sink *sink) {
    seen_set seen = {0};
    seen.klen = 16;
    for (int32_t i = 0; i < npk; i++) {
        uint8_t b[16];
        memcpy(b, pk[i].bytes, 16);
        if (seen_test_and_set(&seen, b)) continue;
        if (ert_crc_checksum(0xFFFF, b + 2, 14, o->ccitt) != 0x1D0F) continue; /* :77 */
        ert_oracle_msg m;
        memset(&m, 0, sizeof(m));
        m.block = pk[i].block;
        m.idx = pk[i].idx;
        m.proto = ERT_SCMPLUS;
        uint8_t protocol_id = b[2];
        m.meter_type = b[3];          /* EndpointType */
        m.meter_id = be32(b + 4);     /* EndpointID   */
        m.consumption = be32(b + 8);  /* Consumption  */
        m.nchecksum = 2;
        m.checksum[0] = b[14];
        m.checksum[1] = b[15];
        m.nbytes = 16;
        memcpy(m.bytes, b, 16);
        if (m.meter_id == 0 || protocol_id != 0x1E) continue; /* :84-86 */
        emit(sink, &m);
    }
    free(seen.keys);
}

/* idm/idm.go:59-98 and netidm/netidm.go:71-109: identical checks, different field map */
static void parse_idm_like(ert_oracle *o, int32_t proto, const ert_oracle_cand *pk, int32_t npk,
                           msg_sink *sink) {
    seen_set seen = {0};
    seen.klen = 92;
    for (int32_t i = 0; i < npk; i++) {
        uint8_t b[92];
        memcpy(b, pk[i].bytes, 92);
        if (seen_test_and_set(&seen, b)) continue;
        if (ert_crc_checksum(0xFFFF, b + 4, 88, o->ccitt) != 0x1D0F) continue; /* idm.go:77 */
        uint8_t buf[6];
        memcpy(buf, b + 9, 4);      /* idm.go:82-84 */
        memcpy(buf + 4, b + 88, 2);
        if (ert_crc_checksum(0xFFFF, buf, 6, o->ccitt) != 0x1D0F) continue; /* idm.go:85 */
        ert_oracle_msg m;
        memset(&m, 0, sizeof(m));
        m.block = pk[i].block;
        m.idx = pk[i].idx;
        m.proto = proto;
        m.meter_type = b[8] & 0x0F;  /* idm.go:124, netidm.go:136 */
        m.meter_id = be32(b + 9);    /* idm.go:125, netidm.go:137 */
        if (proto == ERT_IDM)
            m.consumption = be32(b + 29); /* LastConsumptionCount idm.go:132 */
        else
            m.consumption = be32(b + 34); /* LastConsumptionNet netidm.go:143 */
        m.nchecksum = 2;
        m.checksum[0] = b[90];
        m.checksum[1] = b[91];
        (void)be16;
        m.nbytes = 92;
        memcpy(m.bytes, b, 92);
        if (m.meter_id == 0) continue; /* idm.go:90-92 */
        emit(sink, &m);
    }
    free(seen.keys);
}

/* ------------------------------------------------------------------ */
/* r900: r900/r900.go:82-150 filter, :160-245 Parse                    */
/* ------------------------------------------------------------------ */
static float absf(float x) { return x < 0 ? -x : x; } /* r900.go:152-157 */

static void r900_filter(ert_oracle *o, r900_state *r) {
    const ert_oracle_cfg *c = &o->cfg;
    float sum = 0.0f;
    for (int32_t k = 0; k < c->buffer_length; k++) { /* :96-100 */
        sum += r->signal[k];
        r->csum[k + 1] = sum;
    }
    const int32_t cl = c->chip_length, cl2 = cl * 2, cl3 = cl * 3, cl4 = cl * 4;
    const int32_t limit = c->buffer_length - cl4; /* :117 */
    for (int32_t i = 0; i < limit; i++) {
        float c0 = r->csum[i];
        float c1 = r->csum[i + cl] + r->csum[i + cl];
        float c2 = r->csum[i + cl2] + r->csum[i + cl2];
        float c3 = r->csum[i + cl3] + r->csum[i + cl3];
        float c4 = r->csum[i + cl4];
        float a0 = (c2 - c4) - c0;                 /* :126 */
        float a1 = (((c1 - c2) + c3) - c4) - c0;   /* :127 */
        float a2 = ((c1 - c3) + c4) - c0;          /* :128 */
        float max_abs = absf(a0);
        uint8_t arg = 0;
        float win = a0;
        if (absf(a1) > max_abs) { max_abs = absf(a1); arg = 1; win = a1; }
        if (absf(a2) > max_abs) { max_abs = absf(a2); arg = 2; win = a2; }
        if (win > 0) arg = (uint8_t)(arg + 3); /* :145-148 */
        r->quantized[i] = arg;
    }
}

static int32_t parse_r900(ert_oracle *o, int32_t proto, r900_state *r, const ert_oracle_cand *pk,
                          int32_t npk, msg_sink *sink) {
    const ert_oracle_cfg *c = &o->cfg;
    /* :168-170 slide own history, append the decoder's new magnitudes */
    memmove(r->signal, r->signal + c->block_size, (size_t)(c->buffer_length - c->block_size) * sizeof(float));
    memcpy(r->signal + c->packet_length, o->signal + c->symbol_length, (size_t)c->block_size * sizeof(float));
    r900_filter(o, r); /* :172 -- runs every block, candidates or not */

    seen_set seen = {0};
    seen.klen = 21; /* `bits` is a function of the 21 symbols */
    for (int32_t i = 0; i < npk; i++) {
        if (pk[i].idx > c->block_size) break; /* :183-185 */
        int32_t payload = pk[i].idx + c->preamble_length - c->symbol_length; /* :187 */
        uint8_t symbols[21 + 16];
        memset(symbols, 0, sizeof(symbols));
        int bad = 0;
        /* p.quantized[payloadIdx + 41*4*ChipLength] is the last digit :189-192 reads */
        if ((int64_t)payload + 41ll * 4 * c->chip_length >= c->buffer_length) {
            free(seen.keys);
            return ERT_ORACLE_PANIC;
        }
        for (int32_t k = 0; k < 21; k++) { /* :188-207: two base-6 digits per symbol */
            int32_t d0 = r->quantized[payload + (2 * k) * 4 * c->chip_length];
            int32_t d1 = r->quantized[payload + (2 * k + 1) * 4 * c->chip_length];
            int32_t sym = d0 * 6 + d1;
            if (sym > 31) { bad = 1; break; }
            symbols[k] = (uint8_t)sym;
        }
        if (bad) continue;
        if (seen_test_and_set(&seen, symbols)) continue; /* :209-213 */
        memcpy(r->rs_buf, symbols, 16);            /* :215 */
        memcpy(r->rs_buf + 26, symbols + 16, 5);   /* :216 */
        uint8_t syn[5];
        gf32_syndrome_tbl(o->gf_exp, o->gf_log, r->rs_buf, 31, 5, 29, syn); /* :217 */
        if (syn[0] | syn[1] | syn[2] | syn[3] | syn[4]) continue;          /* :219-221 */

        /* :199-207 bits = concatenation of "%05b" per symbol -> 105 bits */
        uint8_t bitbuf[16];
        memset(bitbuf, 0, sizeof(bitbuf));
        for (int32_t k = 0; k < 21; k++)
            for (int32_t j = 0; j < 5; j++) {
                int32_t pos = k * 5 + j;
                if ((symbols[k] >> (4 - j)) & 1) bitbuf[pos >> 3] |= (uint8_t)(0x80 >> (pos & 7));
            }
        ert_oracle_msg m;
        memset(&m, 0, sizeof(m));
        m.block = pk[i].block;
        m.idx = pk[i].idx;
        m.proto = proto;
        m.meter_id = bits_uint(bitbuf, 0, 32);      /* :223 */
        m.meter_type = bits_uint(bitbuf, 32, 40);   /* Unkn1, :224, MeterType() :277-279 */
        m.consumption = bits_uint(bitbuf, 48, 72);  /* :227 */
        if (proto == ERT_R900BCD) {
            /* r900bcd.go:63-65: hex digits re-read as decimal; ParseUint error -> 0 */
            uint32_t v = m.consumption, out = 0, mul = 1;
            int ok = 1;
            if (v == 0) out = 0;
            while (v) {
                uint32_t d = v & 0xF;
                if (d > 9) { ok = 0; break; }
                out += d * mul;
                mul *= 10;
                v >>= 4;
            }
            m.consumption = ok ? out : 0;
        }
        m.nchecksum = 5;
        memcpy(m.checksum, symbols + 16, 5); /* :242 */
        m.nbytes = 21;
        memcpy(m.bytes, symbols, 21);
        emit(sink, &m);
    }
    free(seen.keys);
    return 0;
}

/* ------------------------------------------------------------------ */
/* Decode: decode.go:163-197                                           */
/* ------------------------------------------------------------------ */
int32_t ert_oracle_decode(ert_oracle *o, const uint8_t *input, ert_oracle_cand *cands,
                          int32_t cand_cap, int32_t *ncands, ert_oracle_msg *msgs,
                          int32_t msg_cap, int32_t *nmsgs) {
    const ert_oracle_cfg *c = &o->cfg;
    int overflow = 0;
    int32_t nc = ncands ? *ncands : 0;
    msg_sink sink = {msgs, msg_cap, nmsgs ? *nmsgs : 0, 0};

    if (o->panicked) return ERT_ORACLE_PANIC;
    ert_oracle_dsp_only(o, input);

    ert_oracle_cand *local = NULL;
    int32_t local_cap = 0;

    for (int32_t pi = 0; pi < o->npre; pi++) { /* :177 (Go map order is random; ours is fixed) */
        const preamble_entry *p = &o->pre[pi];
        int32_t n = (o->search_mode == ERT_SEARCH_GO) ? search_go(o, p) : search_exact(o, p);
        if (n < 0) {
            o->panicked = 1;
            break;
        }

        if (n > local_cap) {
            local_cap = n;
            local = (ert_oracle_cand *)realloc(local, (size_t)local_cap * sizeof(*local));
        }
        /* Slice :353-375 */
        int32_t npk = 0;
        for (int32_t j = 0; j < n; j++) {
            int32_t qi = o->idx_a[j];
            if (qi > c->block_size) continue; /* :358 */
            if (qi + (int64_t)(c->packet_symbols - 1) * c->symbol_length >= c->buffer_length) {
                o->panicked = 1;
                break;
            }
            for (int32_t s = 0; s < c->packet_symbols; s++) { /* :363-366, pkt never cleared */
                o->pkt[s >> 3] = (uint8_t)(o->pkt[s >> 3] << 1);
                o->pkt[s >> 3] |= o->quantized[qi + s * c->symbol_length];
            }
            ert_oracle_cand *d = &local[npk++];
            memset(d, 0, sizeof(*d));
            d->block = o->block;
            d->idx = qi;
            d->preamble_id = pi;
            d->nbytes = o->npkt;
            memcpy(d->bytes, o->pkt, (size_t)o->npkt);
        }
        if (o->panicked) break;
        for (int32_t j = 0; j < npk; j++) {
            if (cands && nc < cand_cap)
                cands[nc] = local[j];
            else
                overflow = 1;
            nc++;
        }
        for (int32_t k = 0; k < p->nparsers && !o->panicked; k++) { /* :185-187 */
            const int32_t i = p->parsers[k];
            switch (o->parser[i]) {
            case ERT_SCM: parse_scm(o, local, npk, &sink); break;
            case ERT_SCMPLUS: parse_scmplus(o, local, npk, &sink); break;
            case ERT_IDM: parse_idm_like(o, ERT_IDM, local, npk, &sink); break;
            case ERT_NETIDM: parse_idm_like(o, ERT_NETIDM, local, npk, &sink); break;
            case ERT_R900:
            case ERT_R900BCD:
                if (parse_r900(o, o->parser[i], &o->r900[i], local, npk, &sink)) o->panicked = 1;
                break;
            }
        }
        if (o->panicked) break;
    }
    free(local);
    o->block++;
    if (ncands) *ncands = nc;
    if (nmsgs) *nmsgs = sink.n;
    if (o->panicked) return ERT_ORACLE_PANIC;
    return (overflow || sink.overflow) ? -1 : 0;
}

int32_t ert_oracle_decode_stream(ert_oracle *o, const uint8_t *input, int64_t nblocks,
                                 ert_oracle_cand *cands, int32_t cand_cap, int32_t *ncands,
                                 ert_oracle_msg *msgs, int32_t msg_cap, int32_t *nmsgs) {
    int32_t rc = 0;
    for (int64_t b = 0; b < nblocks; b++) {
        const int32_t r = ert_oracle_decode(o, input + (size_t)b * (size_t)o->cfg.block_size2, cands, cand_cap,
                                            ncands, msgs, msg_cap, nmsgs);
        if (r == ERT_ORACLE_PANIC) return r;
        if (r != 0) rc = -1;
    }
    return rc;
}

/* ------------------------------------------------------------------ */
/* taps                                                                */
/* ------------------------------------------------------------------ */
const float *ert_oracle_signal(const ert_oracle *o, int32_t *n) {
    if (n) *n = o->cfg.block_size + o->cfg.symbol_length;
    return o->signal;
}
const float *ert_oracle_csum(const ert_oracle *o, int32_t *n) {
    if (n) *n = o->cfg.block_size + o->cfg.symbol_length + 1;
    return o->csum;
}
const uint8_t *ert_oracle_quantized(const ert_oracle *o, int32_t *n) {
    if (n) *n = o->cfg.buffer_length;
    return o->quantized;
}
const uint8_t *ert_oracle_packed(const ert_oracle *o, int32_t *n) {
    if (n) *n = o->npacked;
    return o->packed;
}
const uint8_t *ert_oracle_r900_quantized(const ert_oracle *o, int32_t *n) {
    if (n) *n = o->cfg.buffer_length;
    for (int k = 0; k < ERT_ORACLE_MAX_PROTOS; k++)
        if (o->r900[k].active) return o->r900[k].quantized; /* every r900 parser filters the same signal */
    return NULL;
}
