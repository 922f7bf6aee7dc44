// search.cuh -- preamble Search, Slice and the per-candidate integrity screens on the packed
// bit-plane produced by the demod kernels.
//
// Replaces Decoder.Search (protocol/decode.go:255-328), Decoder.Slice (decode.go:353-375) and
// the CRC calls each parser makes on every candidate (scm/scm.go:76, scmplus/scmplus.go:77,
// idm/idm.go:77-87, netidm/netidm.go:88-98; crc/crc.go:49-55), plus the DSP half of
// r900.Parser.Parse for the candidates it inspects (r900/r900.go:160-207).
//
// Search semantics: the reference's byte pre-filter (decode.go:268-294) is only a CPU
// shortcut; for every legal chip length (SL % 8 == 0) its net result is "every idx in
// [0, BlockSize) whose bits at idx + k*SL equal the preamble" (SURVEY.md section 2.1 step 5).
// The kernel computes exactly that set, 32 start positions at a time: the hit mask of a word
// of starts is the AND over the preamble bits k of (plane window at +k*SL) XNOR P[k].
#pragma once

#include <cstring>
#include <type_traits>

#include "demod_fast.cuh"
#include "demod_generic.cuh"
#include "ert_common.cuh"

namespace ert {

constexpr int kSearchMaxPre = 4;  // preambles the sliding-window kernel takes in one pass

__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}

// A word of starts with surviving bits m (MSB = first start of the word): reserve its RawHits (one reservation
// per word: same-address atomics serialise in L2) and file the word itself for Slice.  counters = the pipeline's
// counter block (kCntHits, kCntWords).
__device__ __forceinline__ void emit_hit_word(uint32_t m, long long gw, int p, RawHit* __restrict__ hits,
                                              HitWord* __restrict__ words, unsigned long long hit_cap,
                                              unsigned long long* __restrict__ counters) {
    unsigned long long slot = atomicAdd(&counters[kCntHits], (unsigned long long)__popc(m));
    const unsigned long long wslot = atomicAdd(&counters[kCntWords], 1ull);
    if (wslot < hit_cap) {
        HitWord w;
        w.gw = (unsigned long long)gw;
        w.slot = slot;
        w.mask = m;
        w.preamble_id = p;
        words[wslot] = w;
    }
    while (m) {
        const int lead = __clz(m);  // MSB = first start of the word
        m &= ~(0x80000000u >> lead);
        if (slot < hit_cap) {
            RawHit h;
            h.s = (unsigned long long)((gw << 5) + lead);
            h.preamble_id = p;
            h.pad = 0;
            hits[slot] = h;
        }
        slot++;
    }
}

// ---- sliding-window Search (every stock geometry: SL % 16 == 0, first start word aligned) ----
//
// Two preamble bits are SL/16 = q whole words apart, so for the chain of start words j, j+q, j+2q, ...
// the window of bit k+2 at step i is the window of bit k at step i+1.  A thread walks kSlideSeg steps
// of one chain with the windows of the even bits (E) and of the odd bits (O: q/2 words further on, half
// a word in when SL % 32 == 16) in registers: a step costs 2-3 LDS for the two NEW windows plus one LOP3
// per probed bit, instead of one or two LDS per bit.  The first 16 bits are probed this way (2^-16 of the
// starts survive on noise); the rare word with a live start finishes its bits from shared memory in
// slide_finish, one copy of cold code outside the unrolled loop.
//
// Thread c = c_hi * q + c_lo owns residue c_lo, segment c_hi: start word c_lo + q * (33 * c_hi + i).
// 33 steps per segment (= 1 mod 32) make the 32 lanes of a warp read 32 consecutive banks at every
// step, whatever q is; 33 = 3 x 11 lets the registers be a ring of 11 with compile-time indices.
constexpr int kSlideSeg = 33;    // steps per thread per tile
constexpr int kSlideRing = 11;   // register ring per parity (unroll factor)
constexpr int kSlideProbe = 16;  // preamble bits probed from the rings
constexpr int kSlideWin = kSlideProbe / 2;  // windows kept per parity
constexpr int kSlideThreads = 256;  // q * nseg of them work: 252 for SL = 144 (smaller CTAs leave more lanes idle)
constexpr uint32_t kSlideRuntimePat = 0xFFFFFFFFu;
constexpr int kSlideMaxLoad = 8448 + 200;  // words per stage: the largest tile (q = 4, 8) + the largest halo (q = 12)

struct SlideParams {
    uint32_t inv[kSearchMaxPre][ERTGPU_MAX_PREAMBLE];  // 0 where P[k]=1, ~0 where P[k]=0
    int32_t nbits[kSearchMaxPre];
    int32_t q;           // SL / 16: words between the windows of bits k and k+2
    int32_t odd_off;     // SL >> 5: word offset of the odd bits' window
    int32_t half;        // 16 when SL % 32 == 16, else 0: bit shift of the odd bits' window
    int32_t nseg;        // segments per residue; q * nseg threads work
    int32_t tile_words;  // q * kSlideSeg * nseg, a multiple of 4
    int32_t load_words;  // tile + halo, a multiple of 4
    int32_t w0;          // plane word of start 0 (p0 >> 5)
    long long nwords;    // words of starts
};

// A word of starts that survived the probe: test bits kSlideProbe .. nbits-1 from shared memory and emit.
// wa = shared address of the word's bit-0 window, gw = call-relative word of starts.
__device__ __noinline__ void slide_finish(const SlideParams* sp, int p, uint32_t wa, uint32_t m, long long gw,
                                          RawHit* __restrict__ hits, HitWord* __restrict__ words, unsigned long long hit_cap,
                                          unsigned long long* __restrict__ hit_count) {
    const int nb = sp->nbits[p];
    for (int k = kSlideProbe; k < nb && m; k++) {
        uint32_t a = wa + 4u * (uint32_t)((k >> 1) * sp->q);
        uint32_t x;
        if (k & 1) {
            a += 4u * (uint32_t)sp->odd_off;
            x = __funnelshift_l(lds_u32(a + 4), lds_u32(a), sp->half);
        } else {
            x = lds_u32(a);
        }
        m &= x ^ sp->inv[p][k];
    }
    if (m == 0 || gw >= sp->nwords) return;
    emit_hit_word(m, gw, p, hits, words, hit_cap, hit_count);
}

// PATp: the first 16 bits of preamble p as a compile-time constant (bit 15 = preamble bit 0) for launches of the
// stock protocol sets (one preamble; scm,scm+,idm; scm,scm+,idm,r900 = "-msgtype=all"): the compiler then folds
// two or three window words into each LOP3 (the probe is bound by the half-rate integer pipe);
// kSlideRuntimePat = any preamble, bits taken from the launch constants.
template <int NPRE, bool HALF, uint32_t PAT0 = kSlideRuntimePat, uint32_t PAT1 = kSlideRuntimePat,
          uint32_t PAT2 = kSlideRuntimePat, uint32_t PAT3 = kSlideRuntimePat>
__global__ void __launch_bounds__(kSlideThreads)
search_slide_kernel(const uint32_t* __restrict__ plane, const __grid_constant__ SlideParams sp,
                    RawHit* __restrict__ hits, HitWord* __restrict__ words, unsigned long long hit_cap,
                    unsigned long long* __restrict__ hit_count) {
    extern __shared__ __align__(128) uint32_t slide_smem[];  // [2][load_words] then two mbarriers
    const uint32_t buf0 = smem_u32(slide_smem);
    const uint32_t stage_bytes = (uint32_t)sp.load_words * 4u;
    const uint32_t bar0 = buf0 + 2u * stage_bytes;
    const long long ntiles = (sp.nwords + sp.tile_words - 1) / sp.tile_words;
    if (threadIdx.x == 0) {
        mbar_init(bar0, 1);
        mbar_init(bar0 + 8, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    pdl_launch_dependents();
    pdl_wait();   // the plane is complete (the demod kernel in front of this one has finished)
    __syncthreads();
    auto issue = [&](long long tile, int st) {
        mbar_arrive_expect_tx(bar0 + 8 * st, stage_bytes);
        bulk_g2s(buf0 + st * stage_bytes, plane + tile * sp.tile_words, stage_bytes, bar0 + 8 * st);
    };
    if (threadIdx.x == 0 && blockIdx.x < ntiles) issue(blockIdx.x, 0);

    const int q = sp.q;
    const bool active = (int)threadIdx.x < q * sp.nseg;
    const int c_lo = (int)threadIdx.x % q, c_hi = (int)threadIdx.x / q;
    const int j0 = c_lo + q * kSlideSeg * c_hi;  // first start word of this thread inside a tile
    const uint32_t step = 4u * (uint32_t)q;
    const uint32_t odd = 4u * (uint32_t)sp.odd_off;

    uint32_t phases = 0;
    int it = 0;
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x, it++) {
        const int st = it & 1;
        const long long next = tile + gridDim.x;
        if (threadIdx.x == 0 && next < ntiles) issue(next, st ^ 1);  // that stage was released by the barrier below
        mbar_wait(bar0 + 8 * st, (phases >> st) & 1u);
        phases ^= 1u << st;
        const long long t0 = tile * sp.tile_words;
        if (active) {
            // window n of this segment: E[n] = word j0 + w0 + q*n, O[n] = the same + odd_off (+ 16 bits)
            const uint32_t a0 = buf0 + st * stage_bytes + 4u * (uint32_t)(j0 + sp.w0);
            uint32_t a = a0;
            auto load_o = [&](uint32_t addr) -> uint32_t {
                if (HALF) return __byte_perm(lds_u32(addr + odd + 4), lds_u32(addr + odd), 0x5432);
                return lds_u32(addr + odd);
            };
            uint32_t E[kSlideRing], O[kSlideRing];  // rings with compile-time indices
#pragma unroll
            for (int n = 0; n < kSlideWin; n++) {  // one window ahead: a step never waits for its own loads
                E[n] = lds_u32(a);
                O[n] = load_o(a);
                a += step;
            }
#pragma unroll 1
            for (int rep = 0; rep < kSlideSeg / kSlideRing; rep++) {
#pragma unroll
                for (int i = 0; i < kSlideRing; i++) {
                    E[(i + kSlideWin) % kSlideRing] = lds_u32(a);  // the newest window of step i+1
                    O[(i + kSlideWin) % kSlideRing] = load_o(a);
                    a += step;
#pragma unroll
                    for (int p = 0; p < NPRE; p++) {
                        uint32_t me = 0xFFFFFFFFu, mo = 0xFFFFFFFFu;  // two chains: half the dependent latency
#pragma unroll
                        for (int k = 0; k < kSlideProbe; k += 2) {
                            const uint32_t e = E[(i + k / 2) % kSlideRing], o = O[(i + k / 2) % kSlideRing];
                            // p comes from a fully unrolled loop: the pattern and the branch below are compile-time
                            const uint32_t pat = (p == 0) ? PAT0 : (p == 1) ? PAT1 : (p == 2) ? PAT2 : PAT3;
                            if (pat != kSlideRuntimePat) {
                                me &= ((pat >> (15 - k)) & 1u) ? e : ~e;
                                mo &= ((pat >> (14 - k)) & 1u) ? o : ~o;
                            } else {
                                me &= e ^ sp.inv[p][k];
                                mo &= o ^ sp.inv[p][k + 1];
                            }
                        }
                        const uint32_t m = me & mo;
                        if (m != 0) {
                            const int s = rep * kSlideRing + i;
                            slide_finish(&sp, p, a0 + (uint32_t)s * step, m, t0 + j0 + (long long)q * s, hits, words, hit_cap,
                                         hit_count);
                        }
                    }
                }
            }
        }
        __syncthreads();  // everyone is done with this stage: it may be refilled next iteration
    }
}

// the first 16 bits of preamble p as search_slide_kernel's PAT
inline uint32_t slide_pattern(const DevCfg& c, int p) {
    uint32_t v = 0;
    for (int k = 0; k < 16; k++) v = (v << 1) | (c.pre_bits[p][k] ? 1u : 0u);
    return v;
}

// host: launch constants of the sliding-window kernel; false when the geometry does not fit it
inline bool make_slide_params(const DevCfg& c, long long p0, long long nwords, SlideParams* sp) {
    if (c.npre > kSearchMaxPre || p0 < 0 || (p0 & 31) != 0 || p0 >= 128) return false;
    if (c.SL % 16 != 0 || c.SL < 64 || c.SL > 192) return false;
    memset(sp, 0, sizeof(*sp));
    for (int p = 0; p < c.npre; p++) {
        if (c.pre_nbits[p] < 16 || c.pre_nbits[p] > 32) return false;
        sp->nbits[p] = c.pre_nbits[p];
        for (int k = 0; k < ERTGPU_MAX_PREAMBLE; k++)
            sp->inv[p][k] = (k < c.pre_nbits[p]) ? (c.pre_bits[p][k] ? 0u : 0xFFFFFFFFu) : 0u;
    }
    sp->q = c.SL / 16;
    sp->odd_off = c.SL >> 5;
    sp->half = c.SL % 32;
    sp->nseg = (kSlideThreads / sp->q) & ~3;  // a multiple of 4 keeps the tile a multiple of 16 bytes
    sp->tile_words = sp->q * kSlideSeg * sp->nseg;
    sp->w0 = (int32_t)(p0 >> 5);
    // the last start word of a tile reaches bit 31's window: 15 strides + the odd offset + 2 words
    const int halo = sp->q * 15 + sp->odd_off + 2 + sp->w0;  // also covers the one-ahead window loads (8 strides)
    sp->load_words = (sp->tile_words + halo + 3) & ~3;
    if (sp->load_words > kSlideMaxLoad) return false;
    sp->nwords = nwords;
    return true;
}

// ---- Search for every other geometry: SL % 16 != 0 (e.g. chip length 78), SL outside [64, 192], more than
// kSearchMaxPre preambles, preambles shorter than 16 bits, halos beyond kSlideMaxLoad.  One thread per word of
// starts, every preamble bit read from global memory: exact for any geometry.
__device__ __forceinline__ uint32_t plane_window2(const uint32_t* __restrict__ plane, long long pos) {
    const long long w = pos >> 5;
    return __funnelshift_l(plane[w + 1], plane[w], (int)(pos & 31));
}

__global__ void __launch_bounds__(256)
search_generic_kernel(const uint32_t* __restrict__ plane, long long p0, long long nwords, DevCfg cfg,
                      RawHit* __restrict__ hits, HitWord* __restrict__ words, unsigned long long hit_cap,
                      unsigned long long* __restrict__ hit_count) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    pdl_launch_dependents();
    pdl_wait();
    for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < nwords; w += stride) {
        const long long base = p0 + (w << 5);
        for (int p = 0; p < cfg.npre; p++) {
            uint32_t m = 0xFFFFFFFFu;
            const int nb = cfg.pre_nbits[p];
            for (int k = 0; k < nb && m; k++) {
                const uint32_t x = plane_window2(plane, base + (long long)k * cfg.SL);
                m &= cfg.pre_bits[p][k] ? x : ~x;
            }
            if (m) emit_hit_word(m, w, p, hits, words, hit_cap, hit_count);
        }
    }
}

// GF(32) log/exp for the r900 syndrome screen (r900/gf/gf.go:20-57 with order 32, poly 37, generator 2)
struct Gf32 {
    uint8_t exp[62];
    uint8_t log[32];
};

constexpr int kExtractWarps = 8;
constexpr int kExtractRowWords = 25;  // packet words per candidate row in shared memory: odd pitch, conflict free

// 32 x 32 bit transpose across a warp, MSB-first on both sides: in = lane r's word, bit 31-k = element (r, k);
// out = lane c's word, bit 31-r = element (r, c).  Five exchange steps of off-diagonal blocks (16 .. 1).
__device__ __forceinline__ uint32_t warp_transpose32(uint32_t x, int lane) {
#pragma unroll
    for (int j = 16; j >= 1; j >>= 1) {
        const uint32_t keep = (j == 16) ? 0xFFFF0000u : (j == 8) ? 0xFF00FF00u : (j == 4) ? 0xF0F0F0F0u
                              : (j == 2) ? 0xCCCCCCCCu : 0xAAAAAAAAu;
        const uint32_t partner = __shfl_xor_sync(0xFFFFFFFFu, x, j);
        x = (lane & j) ? ((x & ~keep) | ((partner & ~keep) << j)) : ((x & keep) | ((partner & keep) >> j));
    }
    return x;
}

// Carry the last `hist_words` words of a call's plane to the front of the other plane, and the last
// `hist_samples` IQ samples into the other history buffer (ping-pong: no overlap hazards).  Grid-stride work
// done by the threads of the Slice kernel (the plane and the IQ bytes are read-only by then).
struct CarryArgs {
    const uint32_t* plane_src;
    uint32_t* plane_dst;
    long long src_offset_words;
    int hist_words;
    const uint8_t* iq;
    const uint8_t* hist_src;
    uint8_t* hist_dst;
    int hist_samples;
    long long nsamples;
};
__device__ __forceinline__ void carry_part(const CarryArgs& c, int i0, int stride) {
    for (int i = i0; i < c.hist_words; i += stride) c.plane_dst[i] = c.plane_src[c.src_offset_words + i];
    // hist_dst[k] (k in [0,hist_samples)) = sample (nsamples - hist_samples + k) relative to the call
    for (int k = i0; k < c.hist_samples; k += stride) {
        const long long j = c.nsamples - c.hist_samples + k;
        uint16_t v;
        if (j >= 0) v = reinterpret_cast<const uint16_t*>(c.iq)[j];
        else v = reinterpret_cast<const uint16_t*>(c.hist_src)[c.hist_samples + j];
        reinterpret_cast<uint16_t*>(c.hist_dst)[k] = v;
    }
}

// Slice (decode.go:353-375) + the parsers' integrity screens, one WARP per word of starts that holds a hit.
//  * gather: bit p of the packet that starts at s is plane bit base + s + p*SL, so the 32 starts of the word
//    share their loads: lane r reads the 32-bit window of symbol 32*ch + r (one funnel shift of two words) and a
//    warp transpose hands lane c the 32 symbols of start c.  Adjacent sample phases of one transmission (~70
//    starts in a row pass the preamble test) cost one pass instead of 70.
//  * screens: lane c runs the checks of every parser filed under the preamble on ITS packet (byte-serial table
//    CRC, crc/crc.go:49-55, tables and packet rows in shared memory); the r900 syndrome check stays warp-parallel
//    per candidate (few candidates, 31 symbols each).
//  * records: one slot reservation per word; every lane writes its own 160-byte record with 16-byte stores.
// KMAX: chunks of 32 symbols gathered (4 covers PacketSymbols <= 128: scm, scm+, r900).
template <int KMAX>
__global__ void __launch_bounds__(kExtractWarps * 32)
extract_words_kernel(const uint32_t* __restrict__ plane, long long p0, const __grid_constant__ DevCfg cfg,
                     const HitWord* __restrict__ words, unsigned long long word_cap,
                     const uint16_t* __restrict__ crc_tables, const __grid_constant__ Gf32 gf,
                     const uint8_t* __restrict__ r900_digits, long long first_block, uint32_t flags,
                     ertgpu_candidate* __restrict__ out, unsigned long long out_cap,
                     unsigned long long* __restrict__ counters, const __grid_constant__ CarryArgs carry) {
    __shared__ uint16_t tab_s[ERTGPU_MAX_PROTOCOLS][256];
    __shared__ uint32_t rows_s[kExtractWarps][32 * kExtractRowWords];
    __shared__ uint32_t rs_s[21][32];   // r900: packed syndromes (5 x 5 bits) of symbol value v at message position pi
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    pdl_wait();   // Search (and with it everything in front of it) has finished
    carry_part(carry, blockIdx.x * blockDim.x + threadIdx.x, gridDim.x * blockDim.x);
    unsigned long long n = counters[kCntWords];
    if (n > word_cap) n = word_cap;
    if ((unsigned long long)blockIdx.x * kExtractWarps >= n) return;
    for (int i = threadIdx.x; i < cfg.nproto * 256; i += blockDim.x) tab_s[i >> 8][i & 255] = crc_tables[i];
    if (r900_digits != nullptr) {
        for (int i = threadIdx.x; i < 21 * 32; i += blockDim.x) {
            const int pi = i >> 5, v = i & 31;
            const int q = pi < 16 ? pi : pi + 10;   // position in the 31-symbol word (r900.go:215-216)
            uint32_t e5 = 0;
            if (v != 0) {
                const int lg = gf.log[v];
#pragma unroll
                for (int s2 = 0; s2 < 5; s2++) e5 |= (uint32_t)gf.exp[(lg + ((29 + s2) * (30 - q)) % 31) % 31] << (5 * s2);
            }
            rs_s[pi][v] = e5;
        }
    }
    __syncthreads();
    uint32_t* const row = &rows_s[warp][lane * kExtractRowWords];
    const uint8_t* const rowb = reinterpret_cast<const uint8_t*>(row);
    const int nchunks = (cfg.PK + 31) >> 5;
    const int shift = bs_shift(cfg);
    for (unsigned long long w = (unsigned long long)blockIdx.x * kExtractWarps + warp; w < n;
         w += (unsigned long long)gridDim.x * kExtractWarps) {
        const HitWord hw = words[w];
        const long long base = p0 + (long long)(hw.gw << 5);
        // ---- gather + transpose: row[ch] = symbols 32*ch .. 32*ch+31 of start `lane`, in packet byte order
#pragma unroll
        for (int ch = 0; ch < KMAX; ch++) {
            uint32_t win = 0;
            const int sym = ch * 32 + lane;
            if (ch < nchunks && sym < cfg.PK) {
                const long long pos = base + (long long)sym * cfg.SL;
                const uint32_t* pw = plane + (pos >> 5);
                win = __funnelshift_l(pw[1], pw[0], (int)(pos & 31));
            }
            if (ch < nchunks) row[ch] = __byte_perm(warp_transpose32(win, lane), 0u, 0x0123);
            else row[ch] = 0u;
        }
        for (int ch = KMAX; ch < ERTGPU_MAX_PACKET_BYTES / 4; ch++) row[ch] = 0u;
        if (cfg.PK & 7) {
            // a trailing partial byte holds its PK%8 bits in the LOW bits, like d.pkt after PK%8 shifts of a zeroed
            // buffer (decode.go:363-366)
            uint8_t* rb = reinterpret_cast<uint8_t*>(row);
            rb[cfg.PK >> 3] = (uint8_t)(rb[cfg.PK >> 3] >> (8 - (cfg.PK & 7)));
        }
        __syncwarp();
        const bool active = (hw.mask >> (31 - lane)) & 1u;
        const int rank = __popc(hw.mask >> (31 - lane)) - 1;   // set bits above this lane's = index among the word's hits
        // Hit slots and word slots come from two counters: a word below word_cap (= the hit capacity) may still hold
        // hits whose slots are past it, with no digits computed (the call overflowed and delivers nothing).
        const bool has_dig = r900_digits != nullptr && cfg.pre_has_r900[hw.preamble_id] &&
                             hw.slot + (unsigned long long)rank < word_cap;
        // ---- screens
        uint32_t mask = 0;
        for (int i = 0; i < cfg.nproto; i++) {
            const DevProto& pr = cfg.proto[i];
            if (pr.preamble_id != hw.preamble_id) continue;
            bool ok = false;
            if (pr.check_kind == ERTGPU_CHECK_NONE) {
                ok = true;
            } else if (pr.check_kind == ERTGPU_CHECK_CRC16 || pr.check_kind == ERTGPU_CHECK_IDM) {
                const uint16_t* tb = tab_s[pr.table];
                uint32_t crc = pr.crc_init;
                if (active) {
                    for (int q = pr.crc_from; q < pr.crc_to; q++) crc = ((crc << 8) & 0xFFFFu) ^ tb[(crc >> 8) ^ rowb[q]];
                    ok = crc == pr.crc_residue;
                    if (ok && pr.check_kind == ERTGPU_CHECK_IDM) {   // Bytes[9:13] + Bytes[88:90], idm.go:82-87
                        crc = pr.crc_init;
#pragma unroll
                        for (int q = 0; q < 6; q++) crc = ((crc << 8) & 0xFFFFu) ^ tb[(crc >> 8) ^ rowb[q < 4 ? 9 + q : 84 + q]];
                        ok = crc == pr.crc_residue;
                    }
                }
            } else if (pr.check_kind == ERTGPU_CHECK_R900 && has_dig) {
                // r900.go:199-221, one candidate per lane: 21 message symbols (two base-6 digits each) must be <= 31 and the
                // five syndromes of the 31-symbol RS word (16 data symbols, 10 zeros, 5 parity symbols) must vanish.  The
                // Horner evaluation of gf.go:163-169 at root a^(29+s) is linear over GF(32): S_s = XOR_q msg[q] * root_s^(30-q),
                // so the five syndromes of symbol value v at position q are one packed table entry and a check is 21 lookups.
                if (active) {
                    const uint16_t* d16 = reinterpret_cast<const uint16_t*>(r900_digits + (hw.slot + (unsigned long long)rank) * ERTGPU_R900_DIGITS);
                    uint32_t synd = 0;
                    bool bad = false;
#pragma unroll
                    for (int pi = 0; pi < 21; pi++) {
                        const uint32_t dd = d16[pi];                       // digits 2*pi (low byte) and 2*pi+1
                        const uint32_t sym = (dd & 0xFFu) * 6u + (dd >> 8);
                        bad = bad || sym > 31u;
                        synd ^= rs_s[pi][sym & 31u];
                    }
                    ok = !bad && synd == 0;
                }
            }
            if (ok) mask |= 1u << i;
        }
        // ---- records
        const bool emit = active && (mask != 0 || !(flags & ERTGPU_DECODE_ONLY_VALID));
        const uint32_t emit_b = __ballot_sync(0xFFFFFFFFu, emit);
        const uint32_t valid_b = __ballot_sync(0xFFFFFFFFu, active && mask != 0);
        unsigned long long slot0 = 0;
        if (lane == 0) {
            if (valid_b) atomicAdd(&counters[kCntValid], (unsigned long long)__popc(valid_b));
            if (emit_b) slot0 = atomicAdd(&counters[kCntOut], (unsigned long long)__popc(emit_b));
        }
        slot0 = __shfl_sync(0xFFFFFFFFu, slot0, 0);
        const unsigned long long slot = slot0 + (unsigned long long)__popc(emit_b & ((1u << lane) - 1u));
        if (emit && slot < out_cap) {
            const unsigned long long s = (hw.gw << 5) + (unsigned long long)lane;
            const long long block = first_block + (long long)(s >> shift);
            uint32_t dg[11];   // 42 digits + 2 pad bytes
#pragma unroll
            for (int k = 0; k < 11; k++) dg[k] = 0;
            if (has_dig) {
                const uint16_t* d16 = reinterpret_cast<const uint16_t*>(r900_digits + (hw.slot + (unsigned long long)rank) * ERTGPU_R900_DIGITS);
#pragma unroll
                for (int k = 0; k < 21; k++) dg[k >> 1] |= (uint32_t)d16[k] << (16 * (k & 1));
            }
            uint4* dst = reinterpret_cast<uint4*>(out + slot);
            dst[0] = make_uint4((uint32_t)block, (uint32_t)((unsigned long long)block >> 32),
                                (uint32_t)(s & (unsigned long long)(cfg.BS - 1)), (uint32_t)hw.preamble_id);
            dst[1] = make_uint4(mask, has_dig ? ERTGPU_CAND_HAS_R900 : 0u, row[0], row[1]);
#pragma unroll
            for (int k = 0; k < 5; k++) dst[2 + k] = make_uint4(row[2 + 4 * k], row[3 + 4 * k], row[4 + 4 * k], row[5 + 4 * k]);
            dst[7] = make_uint4(row[22], dg[0], dg[1], dg[2]);
            dst[8] = make_uint4(dg[3], dg[4], dg[5], dg[6]);
            dst[9] = make_uint4(dg[7], dg[8], dg[9], dg[10]);
        }
        __syncwarp();   // the rows are rewritten by the next word
    }
}

// ---- r900 DSP half, once per detecting block ------------------------------------------------
//
// The r900 parser restarts its float32 running sum at the start of ITS buffer in every block
// (r900/r900.go:96-100), i.e. at sample (b+1)*BS - BUF of the block b that detects a candidate, and
// reads 42 digits at payload + k*4*CL, payload = Idx + PL - SL (r900.go:187-193).  All candidates of
// one block therefore share one chain, and only its first r900_span = BS + PL - SL + 168*CL + 1 running
// sums can ever be read.  Three small kernels: (1) give every block that has an r900 hit a scratch
// slot, (2) r900_chain2_kernel rebuilds the chain of every slot, (3) one thread per (hit, digit)
// evaluates the three 4-chip correlators.  Blocks beyond the scratch capacity, and every block of a
// geometry whose chain starts are not multiples of 8 samples, fall back to r900_replay_kernel.

// Scratch row of a slot: csum[i] sits at row[i] with row = base + slot * pitch + 3, so that csum[1], csum[5], ... are 16-byte
// aligned (the chain kernel stores four running sums per instruction; csum[0] = 0 is never produced by an add).
__host__ __device__ __forceinline__ size_t r900_pitch(int span) { return (size_t)((span + 255) / 256) * 256 + 8; }   // whole hand-off units + the 3-float offset: the chain kernel stores whole vectors
__device__ __forceinline__ float* r900_row(float* scratch, long long slot, int span) { return scratch + (size_t)slot * r900_pitch(span) + 3; }
__device__ __forceinline__ const float* r900_row(const float* scratch, long long slot, int span) { return scratch + (size_t)slot * r900_pitch(span) + 3; }

__global__ void r900_mark_kernel(DevCfg cfg, const RawHit* __restrict__ hits, unsigned long long hit_cap,
                                 const unsigned long long* __restrict__ hit_count, int* __restrict__ block_slot,
                                 int* __restrict__ slot_block, int slot_cap, unsigned int* __restrict__ slot_count) {
    unsigned long long n = *hit_count;
    if (n > hit_cap) n = hit_cap;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    for (unsigned long long c = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; c < n; c += stride) {
        const RawHit h = hits[c];
        if (!cfg.pre_has_r900[h.preamble_id]) continue;
        const long long b = (long long)(h.s >> bs_shift(cfg));
        if (block_slot[b] != -1) continue;
        if (atomicCAS(&block_slot[b], -1, -3) == -1) {  // -3: being assigned
            const unsigned int slot = atomicAdd(slot_count, 1u);
            if ((int)slot < slot_cap) {
                slot_block[slot] = (int)b;
                block_slot[b] = (int)slot;
            } else {
                block_slot[b] = -2;  // no scratch left: per-candidate replay
            }
        }
    }
}

// ---- the chain, software-pipelined over producer and consumer warps ----------------------------
//
// A chain is span-1 (about 24 700) DEPENDENT float32 adds: its latency, not its work, is what the r900 path
// pays (all chains of a call run concurrently).  One warp cannot both feed and run the serial section without
// the feeding instructions sitting inside the dependent chain's issue stream (~10 cycles per add).  Here a
// CTA is two warps and kChainsPerCta chains:
//  * the PRODUCER warp fetches IQ bytes kChainAhead units ahead, looks the magnitudes up and hands units of
//    kChainUnit samples per chain through a shared-memory ring; afterwards it streams the finished running sums
//    of a unit to the chains' scratch rows;
//  * the CONSUMER warp runs one chain on each of its lanes 0, 8, 16, 24 (SIMT: one FADD instruction advances all
//    of them, so four chains cost the issue slots and registers of one) and does nothing but LDS.128 -> 32 dependent
//    FADD -> STS.128 per 32 samples; the next 32 magnitudes are loaded before the adds, and the next unit's
//    barrier is PROBED (mbarrier.test_wait) at the start of the current unit, so neither the shared-memory latency
//    nor the barrier's sits in the dependent chain.
// mbarrier pairs (full / empty) per ring slot carry the hand-offs, one pair of operations per kChainUnit samples.
// Same additions in the same order as r900.go:96-100.  Four chains per CTA keep every chain of a 4 GiB call
// resident at once (the kernel's time is ONE chain's latency as long as that holds).
constexpr int kChainsPerCta = 16;        // chains per consumer warp (its even lanes)
constexpr int kChainProducers = 8;       // producer warps per CTA, kChainsPerCta / kChainProducers chains each (a lone warp issues at ~0.4 IPC: the
                                         // conversion work wants two warps per scheduler)
constexpr int kChainUnit = 128;          // samples per hand-off: kChainUnit / 64 16-byte loads (8 IQ samples each) per producer lane
constexpr int kChainRing = 3;            // units in flight between producers and consumer (static shared memory: 48 KB)
constexpr int kChainAhead = 4;           // units of raw IQ in flight in a producer's registers (a warp has 6 scoreboards: more loads in flight share them, and a wait on a shared scoreboard waits for its NEWEST load)
constexpr int kChainPitch = kChainUnit + 4;  // floats per chain row of a ring slot: consecutive consumer lanes hit different bank groups
constexpr int kChainsPerWarp = kChainsPerCta / kChainProducers;   // chains of one producer warp
constexpr int kChainLanes = 32 / kChainsPerWarp;                    // its lanes per chain, 8 samples (16 bytes) each per load
constexpr int kChainLoads = kChainUnit / (8 * kChainLanes);         // 16-byte loads per producer lane and unit
static_assert(kChainsPerCta % kChainProducers == 0 && 32 % kChainsPerWarp == 0 && kChainUnit % (8 * kChainLanes) == 0, "producer geometry");

// 8 consecutive IQ samples (16 bytes) of the call-relative sample range [j0, j0 + 8), j0 a multiple of 8: from the call's
// bytes, from the history of the previous call (j0 < 0), or nothing (before the start of the stream).  The chain starts
// (b + 1) * BS - BUF and the hand-off unit are multiples of 8 samples, so a group never straddles the call boundary.
__device__ __forceinline__ const uint8_t* raw8_addr(const uint8_t* __restrict__ iq, const uint8_t* __restrict__ hist, int hist_samples,
                                                    long long j0, bool wanted) {
    // ALWAYS a valid address: groups that must not be read (before the history, past the chain) read the call's first bytes
    // instead; the caller zeroes their magnitudes.
    const bool in_hist = j0 < 0;
    const bool ok = wanted && (!in_hist || -j0 <= (long long)hist_samples);
    const uint8_t* p = in_hist ? hist + 2 * ((long long)hist_samples + j0) : iq + 2 * j0;
    return ok ? p : iq;
}
// Ampere-style asynchronous copies (LDGSTS): 16 bytes global -> shared per lane, completion in ORDER per commit group.
// Register loads cannot give this kernel its prefetch depth: a warp has six scoreboards, the loads of the ring share
// them, and waiting for the oldest load of a shared scoreboard waits for the newest one too (seen as long_scoreboard on the
// first use of every unit, whatever the depth).  wait_group<N> waits until at most N groups are pending.
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// Spinning wait on a phase with the NON-blocking probe: mbarrier.try_wait may suspend the warp for a system-dependent time
// when the phase is not complete yet -- fine for a TMA refill that takes a microsecond, ruinous for hand-offs between two
// warps that happen every few hundred cycles.
__device__ __forceinline__ void mbar_spin(uint32_t bar, uint32_t parity) {
    while (!mbar_test(bar, parity)) {}
}
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// lut[v] of decode.go:209-216 without the table: x = fl((127.5 - v) / 127.5) is exactly fma(n, rhi, fl(n * rlo)) with
// n = 127.5 - v for all 256 byte values (checked exhaustively with exact arithmetic, tests/test_oracle.py), then fl(x * x).
// `mag` = 0x4700vv00 as a float = 32768 + v.
__device__ __forceinline__ float lut_of_magic(float mag) {
    const float kRhi = __uint_as_float(1006665857u), kRlo = __uint_as_float(2952724223u);
    const float n = __fsub_rn(32895.5f, mag);
    const float x = __fmaf_rn(n, kRhi, __fmul_rn(n, kRlo));
    return __fmul_rn(x, x);
}

// Why this shape.  A chain is ~24 700 DEPENDENT float32 adds, and the kernel's time is one chain's time as long as every
// chain of the call is resident.  What the chain pays on top is every shared- or global-memory instruction that sits in
// the in-order instruction stream of the warp that runs the adds -- little of it hides behind the add latency.  So the
// consumer warp does the minimum: one LDS.128 and one STG.128 per four adds, sixteen chains side by side (one SIMT
// instruction advances all of them; the whole-vector stores go straight to the padded scratch rows, no second ring), and
// everything else lives in the producer warps: asynchronous 16-byte copies (in-order completion, any depth), magnitudes
// COMPUTED instead of looked up (the table lookups of 16 chains would take the shared-memory bandwidth the hand-offs
// need), mbarrier rings between the two sides.
__global__ void __launch_bounds__((kChainProducers + 1) * 32)
r900_chain2_kernel(const uint8_t* __restrict__ iq, const uint8_t* __restrict__ hist, int hist_samples, int hist_valid,
                   DevCfg cfg, const int* __restrict__ slot_block, int slot_cap,
                   const unsigned int* __restrict__ slot_count, int span, float* __restrict__ scratch) {
    __shared__ __align__(16) float m_s[kChainRing][kChainsPerCta][kChainPitch];
    __shared__ __align__(16) uint4 raw_s[kChainProducers][kChainAhead][kChainLoads][32];   // a producer lane's own prefetch ring
    __shared__ __align__(8) unsigned long long bars[2 * kChainRing];  // [0, R): full, [R, 2R): empty
    const uint32_t full0 = smem_u32(&bars[0]), empty0 = smem_u32(&bars[kChainRing]);
    if (threadIdx.x == 0) {
        for (int r = 0; r < kChainRing; r++) {
            mbar_init(full0 + 8 * r, kChainProducers);   // lane 0 of every producer warp
            mbar_init(empty0 + 8 * r, 1);                // lane 0 of the consumer warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned int nslots = *slot_count;
    if (nslots > (unsigned)slot_cap) nslots = (unsigned)slot_cap;
    const int nunits = (span - 1 + kChainUnit - 1) / kChainUnit;   // magnitudes 0 .. span-2 give csum[1 .. span-1]
    uint32_t ph = 0;  // producer: parity to wait for on empty[r]; consumer: on full[r]  (bit r)
    auto arrive = [](uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); };
    for (unsigned int slot0 = blockIdx.x * kChainsPerCta; slot0 < nslots; slot0 += gridDim.x * kChainsPerCta) {
        if (warp < kChainProducers) {
            // ---- producer: lane = (chain kChainsPerWarp * warp + lane / kChainLanes, 8 samples per load at 8 * (lane % kChainLanes))
            const int ch = warp * kChainsPerWarp + lane / kChainLanes, off = (lane % kChainLanes) * 8;
            const unsigned int slot = slot0 + ch;
            const bool valid = slot < nslots;
            const long long first = ((long long)(valid ? slot_block[slot] : 0) + 1) * cfg.BS - cfg.BUF;   // sample of the parser's signal[0]
            const uint32_t ring0 = smem_u32(&raw_s[warp][0][0][lane]);
            auto fetch = [&](int u) {   // unit u's bytes of this lane into ring slot u % Ahead; one commit group per unit
#pragma unroll
                for (int l = 0; l < kChainLoads; l++) {
                    const int i = u * kChainUnit + l * (8 * kChainLanes) + off;
                    cp_async16(ring0 + (uint32_t)((u % kChainAhead) * kChainLoads + l) * 32u * 16u,
                               raw8_addr(iq, hist, hist_samples, first + i, valid && u < nunits && i < span - 1));
                }
                cp_async_commit();
            };
            for (int a = 0; a < kChainAhead; a++) fetch(a);
            for (int u = 0; u < nunits; u++) {
                const int r = u % kChainRing;
                cp_async_wait<kChainAhead - 1>();   // unit u's bytes have landed (groups complete in order)
                float m[kChainLoads][8];
#pragma unroll
                for (int l = 0; l < kChainLoads; l++) {
                    const uint4 rv = raw_s[warp][u % kChainAhead][l][lane];
                    const uint32_t w[4] = {rv.x, rv.y, rv.z, rv.w};
                    // magnitudes of the 8 samples (decode.go:219-225), bytes as "magic" floats 32768 + v
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        const float i0 = lut_of_magic(__uint_as_float(__byte_perm(w[k], 0x47000000u, 0x7604)));
                        const float q0 = lut_of_magic(__uint_as_float(__byte_perm(w[k], 0x47000000u, 0x7614)));
                        const float i1 = lut_of_magic(__uint_as_float(__byte_perm(w[k], 0x47000000u, 0x7624)));
                        const float q1 = lut_of_magic(__uint_as_float(__byte_perm(w[k], 0x47000000u, 0x7634)));
                        m[l][2 * k] = __fadd_rn(i0, q0);
                        m[l][2 * k + 1] = __fadd_rn(i1, q1);
                    }
                    // samples before the start of the stream or past the last running sum the parser reads contribute 0.0
                    // (checked per sample only in the rare group at an edge)
                    const int i0s = u * kChainUnit + l * (8 * kChainLanes) + off;
                    const long long j0 = first + i0s;
                    const bool whole = valid && i0s + 8 <= span - 1 && (j0 >= 0 || -j0 <= (long long)hist_valid);
                    if (!whole) {
#pragma unroll
                        for (int k = 0; k < 8; k++) {
                            const long long j = j0 + k;
                            const bool ok = valid && i0s + k < span - 1 && (j >= 0 || -j <= (long long)hist_valid);
                            if (!ok) m[l][k] = 0.0f;
                        }
                    }
                }
                fetch(u + kChainAhead);   // refills the slot just read (its bytes are in registers: data dependence above)
                if (u >= kChainRing) {   // the consumer has read this ring slot's previous unit
                    mbar_spin(empty0 + 8 * r, (ph >> r) & 1u);
                    ph ^= 1u << r;
                }
#pragma unroll
                for (int l = 0; l < kChainLoads; l++) {
                    float4* d4 = reinterpret_cast<float4*>(&m_s[r][ch][l * (8 * kChainLanes) + off]);
                    d4[0] = make_float4(m[l][0], m[l][1], m[l][2], m[l][3]);
                    d4[1] = make_float4(m[l][4], m[l][5], m[l][6], m[l][7]);
                }
                __syncwarp();
                if (lane == 0) arrive(full0 + 8 * r);
            }
            cp_async_wait<0>();
            // drain: the consumer's last hand-backs (keeps the barrier phases in step for the next group of chains)
            for (int u = (nunits > kChainRing ? nunits - kChainRing : 0); u < nunits; u++) {
                const int r = u % kChainRing;
                mbar_spin(empty0 + 8 * r, (ph >> r) & 1u);
                ph ^= 1u << r;
            }
        } else {
            // ---- consumer: sixteen serial sections side by side (even lanes), and nothing else: LDS.128 of the next 32
            // magnitudes into the other register set, 32 dependent adds, STG.128 of the sums (r900.go:96-100 order)
            const int ch = lane >> 1;
            const bool active = (lane & 1) == 0 && slot0 + ch < nslots;
            float* out = r900_row(scratch, slot0 + (active ? ch : 0), span);   // out[i] = csum[i]
            if (active) out[0] = 0.0f;
            float acc = 0.0f;
            float4 va[8], vb[8];
            mbar_spin(full0, ph & 1u);
            ph ^= 1u;
            {
                const float4* mv = reinterpret_cast<const float4*>(&m_s[0][ch][0]);
#pragma unroll
                for (int k = 0; k < 8; k++) va[k] = mv[k];
            }
            static_assert((kChainUnit / 32) % 2 == 0, "the register sets swap roles once per group of 32");
            for (int u = 0; u < nunits; u++) {
                const int r = u % kChainRing, rn = (u + 1) % kChainRing;
                const bool have_next = u + 1 < nunits;
                // probe the next unit's barrier now: the answer is needed a few hundred cycles from here
                bool ready = have_next ? mbar_test(full0 + 8 * rn, (ph >> rn) & 1u) : false;
                float4* o4 = reinterpret_cast<float4*>(out + u * kChainUnit + 1);   // csum[i0 + 1 ..]: 16-byte aligned
                auto group = [&](int g, float4 (&cur)[8], float4 (&nxt)[8]) {
                    if (g + 1 < kChainUnit / 32) {
                        const float4* mv = reinterpret_cast<const float4*>(&m_s[r][ch][(g + 1) * 32]);
#pragma unroll
                        for (int k = 0; k < 8; k++) nxt[k] = mv[k];
                    } else {
                        // this unit's magnitudes are all in registers: hand the slot back, then take the next unit's
                        __syncwarp();
                        if (lane == 0) arrive(empty0 + 8 * r);
                        if (have_next) {
                            if (!ready) mbar_spin(full0 + 8 * rn, (ph >> rn) & 1u);
                            ph ^= 1u << rn;
                            const float4* mv = reinterpret_cast<const float4*>(&m_s[rn][ch][0]);
#pragma unroll
                            for (int k = 0; k < 8; k++) nxt[k] = mv[k];
                        }
                    }
#pragma unroll
                    for (int k = 0; k < 8; k++) {          // strictly left to right, r900.go:97-99
                        acc = __fadd_rn(acc, cur[k].x); cur[k].x = acc;
                        acc = __fadd_rn(acc, cur[k].y); cur[k].y = acc;
                        acc = __fadd_rn(acc, cur[k].z); cur[k].z = acc;
                        acc = __fadd_rn(acc, cur[k].w); cur[k].w = acc;
                    }
                    // whole vectors always: the rows are padded to whole units (sums past span - 1 are never read)
                    if (active) {
#pragma unroll
                        for (int k = 0; k < 8; k++) o4[g * 8 + k] = cur[k];
                    }
                };
#pragma unroll
                for (int g = 0; g < kChainUnit / 32; g += 2) {
                    group(g, va, vb);
                    group(g + 1, vb, va);
                }
            }
        }
    }
}

__global__ void r900_digits_kernel(DevCfg cfg, const RawHit* __restrict__ hits, unsigned long long hit_cap,
                                   const unsigned long long* __restrict__ hit_count, const int* __restrict__ block_slot,
                                   int span, const float* __restrict__ scratch, uint8_t* __restrict__ digits) {
    unsigned long long n = *hit_count;
    if (n > hit_cap) n = hit_cap;
    const unsigned long long total = n * ERTGPU_R900_DIGITS;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    for (unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
        // lanes run across HITS (neighbouring hits are neighbouring sample phases of one packet: their five running
        // sums are neighbouring floats of the scratch row), digit positions across the outer index
        const unsigned long long c = t % n;
        const int k = (int)(t / n);
        const RawHit h = hits[c];
        if (!cfg.pre_has_r900[h.preamble_id]) continue;
        const long long b = (long long)(h.s >> bs_shift(cfg));
        const int slot = block_slot[b];
        if (slot < 0) continue;  // handled by the replay kernel
        const int idx = (int)(h.s & (unsigned long long)(cfg.BS - 1));
        const float* cs = r900_row(scratch, slot, span) + (idx + cfg.PL - cfg.SL + 4 * k * cfg.CL);
        digits[c * ERTGPU_R900_DIGITS + k] = r900_digit(cs[0], cs[cfg.CL], cs[2 * cfg.CL], cs[3 * cfg.CL], cs[4 * cfg.CL]);
    }
}

// r900 payload digits for each raw hit of an r900 preamble: exact replay of the parser's own
// running sum (r900/r900.go:96-100), which restarts at sample (b+1)*BS - BUF of the block b
// that detects the candidate, up to the last payload correlator window.  One thread per hit;
// only the 169 running-sum values at payload + t*CL (t = 0..168) are kept.
__global__ void r900_replay_kernel(const uint8_t* __restrict__ iq, const uint8_t* __restrict__ hist,
                                   int hist_samples, int hist_valid, const float* __restrict__ lut_g,
                                   DevCfg cfg, const RawHit* __restrict__ hits, unsigned long long hit_cap,
                                   const unsigned long long* __restrict__ hit_count,
                                   const int* __restrict__ block_slot, uint8_t* __restrict__ digits,
                                   const unsigned int* __restrict__ slot_count = nullptr, int slot_cap = 0) {
    if (slot_count && *slot_count <= (unsigned)slot_cap) return;   // every detecting block found a scratch slot
    __shared__ float lut[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = lut_g[i];
    __syncthreads();
    unsigned long long n = *hit_count;
    if (n > hit_cap) n = hit_cap;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    for (unsigned long long c = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; c < n; c += stride) {
        const RawHit h = hits[c];
        if (!cfg.pre_has_r900[h.preamble_id]) continue;
        const long long b = (long long)(h.s >> bs_shift(cfg));
        if (block_slot && block_slot[b] >= 0) continue;      // served by the per-block chain
        const int idx = (int)(h.s & (unsigned long long)(cfg.BS - 1));
        const long long first = (b + 1) * cfg.BS - cfg.BUF;  // sample of r900 signal[0]
        const int payload = idx + cfg.PL - cfg.SL;           // r900.go:187
        const int last = payload + 4 * ERTGPU_R900_DIGITS * cfg.CL;  // csum index of the final tap
        float taps[4 * ERTGPU_R900_DIGITS + 1];
        float s = 0.0f;
        int next = payload, ti = 0;
        if (next == 0) { taps[ti++] = 0.0f; next += cfg.CL; }
        for (int t = 0; t < last; t++) {
            s = __fadd_rn(s, mag_at(iq, hist, hist_samples, hist_valid, first + t, lut));
            if (t + 1 == next) { taps[ti++] = s; next += cfg.CL; }
        }
        uint8_t* d = digits + c * ERTGPU_R900_DIGITS;
        for (int k = 0; k < ERTGPU_R900_DIGITS; k++)
            d[k] = r900_digit(taps[4 * k], taps[4 * k + 1], taps[4 * k + 2], taps[4 * k + 3], taps[4 * k + 4]);
    }
}

}  // namespace ert
