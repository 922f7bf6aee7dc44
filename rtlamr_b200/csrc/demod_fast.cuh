// demod_fast.cuh -- the hot kernel: magnitude + Manchester matched filter + quantize + pack with
// the chip length as a compile-time constant.
//
// Replaces, fused into one pass over the IQ bytes: MagLUT.Execute (protocol/decode.go:219-225),
// Filter (decode.go:229-245) and the bit packing of Search (decode.go:259-265).
//
// Design (see DESIGN.md "demod_fast"):
//  * One thread per reference block ("chain"); a warp owns 32 consecutive blocks.  The float32
//    running sum of Filter is sequential within a block and restarts at every block
//    (decode.go:232-236), so this is the only parallelism that keeps the sign bits exact.
//  * Per sample: running sum c += m; chip sum A = c - c[CL steps ago]; filter f = A[CL steps ago] - A.
//    Both histories are rings held in REGISTERS.  The rings have L > CL slots (L = the unrolled
//    body length): a new value is born into the slot that died L - CL steps earlier, so no value
//    ever has to be moved -- every ring slot is a fixed register and the steady state is
//    2 PRMT + 2 LDS + 4 FADD + 1 SHF per sample.
//  * Magnitude lut[I] + lut[Q]: the 256-entry table is replicated per lane in shared memory as
//    [value][lane] with a 256-byte row pitch, so a lookup address is ONE byte-permute
//    (PRMT: {lane*4, value, base>>16}) and the 32 lanes always hit 32 different banks.  Column 32
//    of every row holds 0.0f: samples that must not contribute (the alignment pad in front of the
//    lead-in, and the lead-in of the first block of a stream, whose Signal buffer starts as zeros,
//    decode.go:144) are looked up there.
//  * IQ bytes reach the thread that needs them through shared memory: body t of a warp's 32 chains
//    is one [32 rows][2*L bytes] box of the IQ matrix (row = reference block), a single TMA tile
//    load (cp.async.bulk.tensor.2d) issued by one lane into a 2-stage ring with an mbarrier per
//    stage.  L/8 is odd, so rows have an odd 16-byte pitch and the per-lane LDS.128 reads are bank
//    conflict free.  HBM is read in whole sectors, each byte once.
//  * Sign bits are shifted into words with one funnel shift per sample and appended to the
//    per-block bit-plane row.
//
// Stream of one chain, in steps: [pad = 2L - SL zero-magnitude steps][SL lead-in samples = tail of the
// previous block][BS samples of the block]; bodies 0 and 1 are pad + lead-in, f[0] is produced by the
// last step of body 1, bodies >= 2 produce L bits each.
#pragma once

#include <cuda.h>

#include <algorithm>
#include <type_traits>

#include "ert_common.cuh"

namespace ert {

constexpr int kLutBytes = 65536;  // 256 rows x 256 B (lanes 0..31 + zero column at byte 128)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(bar), "r"(parity)
        : "memory");
}
// non-blocking probe of a phase (acquire on success, like the waiting form)
__device__ __forceinline__ bool mbar_test(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
// 2D tiled TMA load: box (x = byte column, y = block row) -> dense smem tile
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int x, int y, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
        "l"(map), "r"(x), "r"(y), "r"(bar)
        : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
// LUT read: not volatile, the table is constant after the prologue barrier
__device__ __forceinline__ float lds_f32(uint32_t addr) {
    float v;
    asm("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
    return v;
}

// body length for a chip length: the smallest L >= CL + 1 with L % 8 == 0 and L / 8 odd
constexpr int fast_body_len(int CL) {
    int L = ((CL + 1 + 7) / 8) * 8;
    if (((L / 8) & 1) == 0) L += 8;
    return L;
}

// The fast kernel reads two bodies of L samples from one block (a shorter block: PreambleSymbols = 1 at chip length 32,
// 56 or 64) ...
constexpr bool fast_block_fits(int L, int BS) { return 2 * L <= BS; }
// ... and a lead-in of 2L samples from the history of PacketLength samples, with bulk copies from 2*PacketLength - 4L
// bytes into the history, which must be 16-byte aligned (a shorter packet: PacketSymbols = 1; PacketLength % 8 != 0: an
// odd PacketSymbols at chip length 78).  Geometries that do not fit take demod_generic_kernel.
constexpr bool fast_history_fits(int L, int PacketLength) { return PacketLength >= 2 * L && PacketLength % 8 == 0; }

template <int CL>
struct FastGeom {
    static constexpr int L = fast_body_len(CL);
    static constexpr int kPad = 2 * L - 2 * CL;        // zero-magnitude steps in front of the lead-in
    static constexpr int kRowBytes = 2 * L;            // one body's IQ bytes per chain
    static constexpr int kRowUnits = kRowBytes / 16;   // odd: conflict-free LDS.128
    static constexpr int kStageBytes = 32 * kRowBytes;
    static constexpr int kStages = 2;                   // bodies in flight per warp (3 measured no faster than 2: the refill is not what the warps wait for)
    static constexpr int kWarpBytes = kStages * kStageBytes;
    static constexpr int kFullWords = L / 32;           // whole output words per body
    static constexpr int kTailBits = L % 32;
    static_assert(L % 8 == 0 && (kRowUnits & 1) == 1 && L >= CL && kPad >= 0 && kPad < L, "bad body length");
    static_assert(CL % 2 == 0, "the two samples of a word take neighbouring ring slots: needs an even chip length");
};

// smem map (byte offsets inside the dynamic segment, computed at run time):
//   [bars: 2 x 8 B per warp][pad][staging of the first warps ...][LUT at the next 64 KiB boundary]
//   [staging of the remaining warps ...]
template <int CL, int WARPS>
__global__ void __launch_bounds__(WARPS * 32, 1)
demod_fast_kernel(const __grid_constant__ CUtensorMap iq_map, const uint8_t* __restrict__ iq,
                  const uint8_t* __restrict__ hist, int hist_samples, int hist_valid,
                  const float* __restrict__ lut_g, uint32_t* __restrict__ plane_out, long long nblocks, int BS,
                  unsigned long long* __restrict__ tile_counter, long long dyn_tiles) {
    using G = FastGeom<CL>;
    constexpr int L = G::L;
    extern __shared__ __align__(128) uint8_t fast_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t sbase = smem_u32(fast_smem);
    const uint32_t lut_base = (sbase + 1024 + 0xFFFFu) & ~0xFFFFu;  // 64 KiB aligned, after the barriers
    // staging areas: as many warps as fit below the LUT, the rest above it
    const uint32_t below0 = sbase + 1024;
    const int nbelow = (int)((lut_base - below0) / G::kWarpBytes);
    const uint32_t stage0 = (warp < nbelow) ? below0 + warp * G::kWarpBytes
                                            : lut_base + kLutBytes + (warp - nbelow) * G::kWarpBytes;
    const uint32_t bar0 = sbase + warp * 32;  // kStages (<= 4) mbarriers per warp
    {   // the staging areas must fit the dynamic segment (they do for every instantiated geometry)
        uint32_t dyn;
        asm("mov.u32 %0, %%dynamic_smem_size;" : "=r"(dyn));
        const int nabove = (WARPS > nbelow) ? WARPS - nbelow : 0;
        if (lut_base + kLutBytes + (uint32_t)nabove * G::kWarpBytes > sbase + dyn) __trap();
    }

    pdl_launch_dependents();   // Search's CTAs may move in as this kernel's CTAs leave (they wait for the whole grid)
    // ---- prologue: LUT [v][lane] + zero column, barriers ----
    for (int v = warp; v < 256; v += WARPS) {   // row v: the value in the 32 lane columns, 0.0 in column 32
        const float x = lut_g[v];
        asm volatile("st.shared.f32 [%0], %1;" ::"r"(lut_base + v * 256 + lane * 4), "f"(x) : "memory");
        if (lane == 0) asm volatile("st.shared.f32 [%0], %1;" ::"r"(lut_base + v * 256 + 128), "f"(0.0f) : "memory");
    }
    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < G::kStages; s++) mbar_init(bar0 + s * 8, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int wpb = BS >> 5;                         // words per block
    const int nbody = (2 * L + BS - 1 + L - 1) / L;  // bodies covering steps 0 .. 2L+BS-2
    const long long ntiles = (nblocks + 31) / 32;
    const uint32_t lo_main = lut_base | (uint32_t)(lane * 4);
    const uint32_t lo_zero = lut_base | 128u;
    const uint32_t row = stage0 + lane * G::kRowBytes;
    const bool have_hist = hist_valid >= 2 * L;      // hist_valid is 0 or >= BlockSize
    uint32_t phases = 0;  // bit s = parity to wait for on stage s
    int st = 0;           // stage of the next body (runs on across work tiles)
    bool ready = false;   // the next body's stage was seen complete
    int npref = 0;        // leading bodies of this work tile that were already issued during the previous one

    // Work tiles are claimed one ahead: the id of the NEXT tile is asked for when a tile starts and is known long
    // before the tile's last bodies, which refill the staging ring with the next tile's first bodies instead of
    // letting it drain -- a warp pays the TMA latency once, not once per tile.
    //
    // The first dyn_tiles tiles go out dynamically (atomic counter).  When the call does not fill the last round of
    // SMs x WARPS tiles, the remaining tiles (at most 4 per SM) are pre-assigned instead: tile dyn_tiles + SM +
    // SMs * w to warp w < 4 of each CTA, i.e. at most ONE per scheduler -- a warp that runs alone on its scheduler
    // finishes a tile in ~0.6 of the shared time, while a dynamic hand-out lets two late tiles land on one scheduler
    // next to an idle one.
    constexpr unsigned long long kNoTile = 0x7FFFFFFFFFFFFFFFull;   // compares above every tile as a signed value too
    bool static_used = false;
    auto resolve = [&](unsigned long long claimed) -> unsigned long long {   // warp-uniform
        if ((long long)claimed < dyn_tiles) return claimed;
        if (!static_used && warp < 4) {
            static_used = true;
            const long long s = dyn_tiles + blockIdx.x + (long long)gridDim.x * warp;
            if (s < ntiles) return (unsigned long long)s;
        }
        return kNoTile;
    };
    unsigned long long tile = 0;
    if (lane == 0) tile = atomicAdd(tile_counter, 1ull);
    tile = resolve(__shfl_sync(0xFFFFFFFFu, tile, 0));
    while ((long long)tile < ntiles) {
        unsigned long long next_raw = 0, next_tile = kNoTile;
        int npref_next = 0;
        if (lane == 0) next_raw = atomicAdd(tile_counter, 1ull);  // consumed after the lead-in bodies

        long long b = (long long)tile * 32 + lane;
        const bool live = b < nblocks;
        if (!live) b = nblocks - 1;  // the lane-copy path needs a valid source; results are discarded
        const bool first = (b == 0);
        // lead-in of the stream's very first block: magnitude 0.0 (zero column)
        const uint32_t lo_lead = (first && !have_hist) ? lo_zero : lo_main;

        // Body t of the 32 chains of this work tile = one [32 rows][2L bytes] box of the IQ matrix:
        // bodies 0,1 come from the tail of the previous row (block), bodies >= 2 from the row itself.
        // Rows past the end of the call and columns past the end of a row are zero-filled by the TMA
        // unit (the steps that read them produce no output).  The first work tile of a call is the
        // exception: block 0 takes its lead-in from the history buffer, so that tile uses one 1D bulk
        // copy per lane instead (its own instantiation of the tile code: the hot loop carries neither
        // that path nor the lead-in special cases).
        float cr[L], ar[L];  // rings of the running sums and the chip sums
#pragma unroll
        for (int j = 0; j < L; j++) { cr[j] = 0.0f; ar[j] = 0.0f; }
        uint32_t acc = 0;   // pending output bits (low nacc bits), still as SIGN bits (inverted at store)
        int nacc = 0;       // warp-uniform
        uint32_t ow0 = 0, ow1 = 0, ow2 = 0;  // the last words of the current 16-byte output group
        uint4 pend = make_uint4(0, 0, 0, 0); // the group that fills the first half of the current 32-byte sector
        // Each lane writes its own row, so every store of the warp touches 32 lines.  The 16-byte groups go out a
        // whole 32-byte sector at a time (two stores back to back): with lone 16-byte stores (half sectors) the 1 GiB
        // scm demod took 9 % longer on H100.  The rows may start in the middle of a sector (r900's plane history is
        // 16 mod 32 bytes), so which groups share a sector is read from the plane's base address (ph = 4: group 0
        // is a second half).  A row of BS/32 words is a whole number of sectors for every block size >= 256; with a
        // row of 4 mod 8 words the odd rows would pair across sectors, slower but storing the same words.  A group
        // is stored iff its last word is < wlimit.
        int wi = 0;
        const int wlimit = live ? wpb : 0;   // words this lane may store
        uint4* const out4 = reinterpret_cast<uint4*>(plane_out + b * wpb);
        auto ph = [&]() { return (int)((uint32_t)reinterpret_cast<uintptr_t>(plane_out) >> 2) & 4; };   // warp-uniform
        auto put = [&](uint32_t o) {
            if ((wi & 3) == 3) {
                const uint4 q = make_uint4(~ow0, ~ow1, ~ow2, ~o);
                if ((wi ^ ph()) & 4) {   // second half: the sector is complete
                    // (unsigned): no first half in front of group 0
                    if ((unsigned)(wi - 4) < (unsigned)wlimit) out4[(wi >> 2) - 1] = pend;
                    if (wi < wlimit) out4[wi >> 2] = q;
                } else {
                    pend = q;
                }
            }
            ow0 = ow1; ow1 = ow2; ow2 = o;
            wi++;
        };

        auto run_tile = [&](auto lc_tag) {
            constexpr bool kLaneCopies = decltype(lc_tag)::value;
            // one [32 rows][2L bytes] box: body tb of work tile tl
            auto issue_box = [&](unsigned long long tl, int tb, int stage) {
                if (lane == 0) {
                    const uint32_t bar = bar0 + stage * 8;
                    mbar_arrive_expect_tx(bar, 32u * G::kRowBytes);
                    const int x = (tb < 2) ? 2 * BS - 2 * G::kRowBytes + tb * G::kRowBytes : (tb - 2) * G::kRowBytes;
                    const int y = (int)(tl * 32) - (tb < 2 ? 1 : 0);
                    tma_load_2d(stage0 + stage * G::kStageBytes, &iq_map, x, y, bar);
                }
            };
            auto issue = [&](int t, int stage) {
                if (t >= nbody) {   // past the end of this tile: the next tile's first bodies (never the call's first tile)
                    if ((long long)next_tile < ntiles) {
                        issue_box(next_tile, t - nbody, stage);
                        npref_next++;
                    }
                    return;
                }
                const uint32_t bar = bar0 + stage * 8;
                if constexpr (!kLaneCopies) {
                    issue_box(tile, t, stage);
                } else {
                    // stream byte offset of body t relative to the block start: (t - 2) * 2L
                    const long long off = (long long)(t - 2) * G::kRowBytes;
                    long long n = 2ll * BS - off;  // bytes left in the block
                    if (n > G::kRowBytes) n = G::kRowBytes;
                    const uint8_t* src;
                    if (t < 2 && first) src = have_hist ? hist + 2ll * hist_samples + off : iq;  // off < 0: tail of the history
                    else src = iq + b * 2ll * BS + off;
                    if (lane == 0) mbar_arrive_expect_tx(bar, 32u * (uint32_t)n);
                    __syncwarp();
                    bulk_g2s(row + stage * G::kStageBytes, src, (uint32_t)n, bar);
                }
            };
            // PHASE 0: body 0 = alignment pad (zero column) + start of the lead-in; PHASE 1: body 1 = rest of the
            // lead-in, its last step is f[0]; PHASE 2: the block itself, L output bits per body.
            auto body = [&](auto phase_tag, int t) {
                constexpr int PHASE = decltype(phase_tag)::value;
                // the phase was probed in the middle of the previous body: the wait loop (and the latency of
                // its first probe) is only paid when the refill really is late
                if (!ready) mbar_wait(bar0 + st * 8, (phases >> st) & 1u);
                phases ^= 1u << st;
                const uint32_t lo_b = (PHASE == 2) ? lo_main : lo_lead;
                const uint32_t lo_a = (PHASE == 0) ? lo_zero : lo_b;  // the first kPad steps of body 0
                const uint32_t src = row + st * G::kStageBytes;
                uint32_t w = 0;
                float c = cr[L - 1];  // the running sum = the last slot of the ring

#pragma unroll
                for (int g = 0; g < L / 8; g++) {
                    const uint4 v = lds128(src + g * 16);
                    const uint32_t xs[4] = {v.x, v.y, v.z, v.w};
                    if (g == L / 16) {
                        const int nst = (st + 1 == G::kStages) ? 0 : st + 1;
                        ready = mbar_test(bar0 + nst * 8, (phases >> nst) & 1u);
                    }
#pragma unroll
                    for (int q = 0; q < 4; q++) {
                        // two samples (I0 Q0 I1 Q1) per 32-bit word.  CL, L and kPad are even, so the two samples of
                        // a word never straddle the end of the ring.
                        const int j = g * 8 + q * 2;
                        const int jo = (j + L - CL) % L;  // the slots written CL steps ago
                        const uint32_t lo = (j < G::kPad) ? lo_a : lo_b;
                        // {byte0: lane*4 (or the zero column), byte1: I or Q, bytes 2-3: LUT base >> 16}
                        const float li0 = lds_f32(__byte_perm(xs[q], lo, 0x7604));
                        const float li1 = lds_f32(__byte_perm(xs[q], lo, 0x7624));
                        const float lq0 = lds_f32(__byte_perm(xs[q], lo, 0x7614));
                        const float lq1 = lds_f32(__byte_perm(xs[q], lo, 0x7634));
                        const float m0 = __fadd_rn(li0, lq0), m1 = __fadd_rn(li1, lq1);   // decode.go:222
                        const float c0 = __fadd_rn(c, m0);                            // csum[k+1], decode.go:234
                        c = __fadd_rn(c0, m1);
                        const float a0 = __fsub_rn(c0, cr[jo]), a1 = __fsub_rn(c, cr[jo + 1]);   // csum[k+1] - csum[k+1-CL]
                        const float f0 = __fsub_rn(ar[jo], a0), f1 = __fsub_rn(ar[jo + 1], a1);  // decode.go:242
                        ar[j] = a0;
                        ar[j + 1] = a1;
                        cr[j] = c0;  // slots j, j+1 died L-CL steps ago
                        cr[j + 1] = c;
                        w = __funnelshift_l(__float_as_uint(f0), w, 1);           // sign bits in
                        w = __funnelshift_l(__float_as_uint(f1), w, 1);
                        if (((j + 1) & 31) == 31 && PHASE == 2) {
                            // 32 more bits complete: emit one word (acc keeps the nacc pending bits)
                            put(__funnelshift_r(w, acc, nacc));
                            acc = w;
                        }
                    }
                }
                // every lane has read its row of this stage into registers: refill it with body t+kStages
                __syncwarp();
                issue(t + G::kStages, st);
                st = (st + 1 == G::kStages) ? 0 : st + 1;

                if constexpr (G::kTailBits != 0 && PHASE == 2) {
                    // append the body's last L%32 bits
                    const uint32_t y = w & ((1u << G::kTailBits) - 1u);
                    const uint32_t hi = acc >> (32 - G::kTailBits);
                    const uint32_t lw = (acc << G::kTailBits) | y;
                    const int n2 = nacc + G::kTailBits;
                    if (n2 >= 32) put(__funnelshift_r(lw, hi, n2 & 31));
                    nacc = n2 & 31;
                    acc = lw;
                }
                if constexpr (PHASE == 1) {  // body 1 contributes only its last step = f[0]
                    acc = w & 1u;
                    nacc = 1;
                }
            };
#pragma unroll
            for (int s = 0; s < G::kStages; s++)
                if (s >= npref) issue(s, (st + s) % G::kStages);
            body(std::integral_constant<int, 0>{}, 0);
            body(std::integral_constant<int, 1>{}, 1);
            next_tile = resolve(__shfl_sync(0xFFFFFFFFu, next_raw, 0));
#pragma unroll 1
            for (int t = 2; t < nbody; t++) body(std::integral_constant<int, 2>{}, t);
        };
        if (tile == 0) run_tile(std::true_type{});
        else run_tile(std::false_type{});
        {   // the last whole group, if it is a first half still waiting for the rest of its sector
            const int g = (wi >> 2) - 1;
            if (g >= 0 && !(((4 * g) ^ ph()) & 4) && 4 * g + 3 < wlimit) out4[g] = pend;
        }
        __syncwarp();
        npref = npref_next;
        tile = next_tile;
    }
}

// ---- host side -------------------------------------------------------------------------

template <int CL>
constexpr int fast_warps() {
    // registers: 2*L ring values + ~40 working registers; the register file is handed out in
    // units that make 8/12/16 warps per SM the useful steps (255/168/128 registers per thread)
    return (2 * fast_body_len(CL) + 40 <= 128) ? 16 : ((2 * fast_body_len(CL) + 40 <= 168) ? 12 : 8);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// The driver's entry point, looked up once per process (null when the driver has none).
inline EncodeTiledFn encode_tiled_fn() {
    static const EncodeTiledFn fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        const bool ok = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
                        q == cudaDriverEntryPointSuccess;
        return ok ? (EncodeTiledFn)p : nullptr;
    }();
    return fn;
}

// Shared-space address of the dynamic segment of a kernel without static shared memory (the first KiB
// of the window is reserved by the system).  Asked from the device once per handle (ertgpu_allocate): the demod
// kernel's map depends on where the 64 KiB-aligned LUT lands, and the launch requests exactly the bytes the map needs
// so that CTAs of the Search/extract kernels of another call can share the SM.
__global__ void smem_base_probe_kernel(uint32_t* out) {
    extern __shared__ __align__(128) uint8_t probe_smem[];
    *out = smem_u32(probe_smem);
}

// Dynamic shared memory the kernel's map needs for W warps when the segment starts at shared address sbase:
// [barriers 1 KiB][staging of the warps that fit][LUT at the next 64 KiB boundary][staging of the other warps]
template <class G>
inline int fast_smem_bytes(int W, uint32_t sbase) {
    const uint32_t lut_base = (sbase + 1024 + 0xFFFFu) & ~0xFFFFu;
    const int nbelow = (int)((lut_base - (sbase + 1024)) / G::kWarpBytes);
    const int nabove = W > nbelow ? W - nbelow : 0;
    return (int)(lut_base + kLutBytes + (uint32_t)nabove * G::kWarpBytes - sbase);
}

// Tiles handed out dynamically; the rest (a last round that fills at most one warp per scheduler) is pre-assigned
// inside the kernel.
inline long long fast_dynamic_tiles(long long ntiles, long long grid, int W) {
    const long long cap = grid * W;
    if (W < 4 || cap <= 0) return ntiles;
    const long long full = ntiles / cap, rest = ntiles - full * cap;
    if (full < 1 || rest == 0 || rest > 4 * grid) return ntiles;
    return full * cap;
}
// Rounds of SMs x W tiles a call takes, in units of an 8-warp round.  Model: a 7-warp round costs 0.94 of an 8-warp
// one, and a last round with at most one tile per scheduler 0.62 of one.
inline double fast_round_cost(long long ntiles, long long sms, int W) {
    const long long cap = sms * W, full = ntiles / cap, rest = ntiles - full * cap;
    const double unit = W == 8 ? 1.0 : 0.94;
    double last = 0.0;
    if (rest > 0) last = (full >= 1 && rest <= 4 * sms) ? 0.62 : unit;
    return full * unit + last;
}

// A handle's demod_fast instances, chosen once (fast_demod): <CL, fast_warps<CL>()> and, when that has 8 warps, <CL, 7>,
// each with the dynamic shared memory its launches request; and the tensor map of the handle's last call.
struct FastDemod {
    using Kernel = void (*)(CUtensorMap, const uint8_t*, const uint8_t*, int, int, const float*, uint32_t*, long long, int,
                            unsigned long long*, long long);
    Kernel kern[2] = {nullptr, nullptr};  // [1]: the 7-warp instance, if any
    int warps[2] = {0, 0};
    int smem[2] = {0, 0};
    int row_bytes = 0;                    // the map's box width, FastGeom<CL>::kRowBytes
    // Calls that stream through the same staging buffer reuse the map.  Invariant: the key and the handle's constants are
    // all the map contains -- a buffer freed and re-allocated at the same address with the same number of blocks gives a
    // byte-identical descriptor (addresses and extents, no handle to the allocation), so a stale hit cannot exist.
    const void* map_iq = nullptr;
    long long map_nblocks = 0;
    CUtensorMap map;
};

template <int CL>
FastDemod fast_demod_of(uint32_t sbase) {
    using G = FastGeom<CL>;
    constexpr int W = fast_warps<CL>();
    FastDemod f;
    f.kern[0] = demod_fast_kernel<CL, W>;
    f.warps[0] = W;
    f.smem[0] = fast_smem_bytes<G>(W, sbase);
    if constexpr (W == 8) {
        f.kern[1] = demod_fast_kernel<CL, 7>;
        f.warps[1] = 7;
        f.smem[1] = fast_smem_bytes<G>(7, sbase);
    }
    f.row_bytes = G::kRowBytes;
    return f;
}

// The instances of a chip length when the dynamic segment starts at shared address sbase.  Chip lengths with a
// specialised kernel: every value the reference CLI accepts (flags.go:127-132 allows 8,32,40,...,96) except 8, plus 78,
// the rate the reference's sample.bin fixture was captured at (nothing in the kernel needs CL to be a multiple of 8: only
// L is).  Anything else has no instance and uses the generic kernel.
inline FastDemod fast_demod(int CL, uint32_t sbase) {
    switch (CL) {
        case 32: return fast_demod_of<32>(sbase);
        case 40: return fast_demod_of<40>(sbase);
        case 48: return fast_demod_of<48>(sbase);
        case 56: return fast_demod_of<56>(sbase);
        case 64: return fast_demod_of<64>(sbase);
        case 72: return fast_demod_of<72>(sbase);
        case 78: return fast_demod_of<78>(sbase);
        case 80: return fast_demod_of<80>(sbase);
        case 88: return fast_demod_of<88>(sbase);
        case 96: return fast_demod_of<96>(sbase);
        default: return FastDemod{};
    }
}

// The instance of a chip length and block size (fast_block_fits), whatever the packet: the chip length, or 0.
inline int demod_fast_variant(int CL, int BS) {
    return fast_demod(CL, 0).kern[0] && fast_block_fits(fast_body_len(CL), BS) ? CL : 0;
}
// The instance a decoder runs: the same, if its packet length also gives the lead-in history (fast_history_fits).
inline int demod_fast_variant(int CL, int BS, int PacketLength) {
    const int v = demod_fast_variant(CL, BS);
    return v != 0 && fast_history_fits(fast_body_len(CL), PacketLength) ? v : 0;
}

// Launch one of f's instances over a call of nblocks blocks on a device of sms SMs; *w_out: its warps.  Work tiles are
// handed out in rounds of (SMs x resident warps).  With two warps per scheduler the SM's rate still grows almost
// linearly with the warp count, so when 7 warps need no more rounds than 8 the fuller last round of 7 wins
// (fast_round_cost); long calls keep 8.
inline cudaError_t launch_demod_fast(FastDemod& f, int sms, const uint8_t* iq, const uint8_t* hist, int hist_samples,
                                     int hist_valid, const float* lut, uint32_t* plane_out, long long nblocks, int BS,
                                     unsigned long long* tile_counter, cudaStream_t st, int* w_out) {
    const long long ntiles = (nblocks + 31) / 32;
    const int k = f.kern[1] && fast_round_cost(ntiles, sms, 7) < fast_round_cost(ntiles, sms, 8) ? 1 : 0;
    const int W = f.warps[k];
    *w_out = W;
    if (f.map_iq != iq || f.map_nblocks != nblocks) {
        // the IQ bytes of the call as a 2D uint8 tensor: [nblocks rows][BlockSize2 bytes]
        const EncodeTiledFn enc = encode_tiled_fn();
        if (!enc) return cudaErrorNotSupported;
        const cuuint64_t gdim[2] = {(cuuint64_t)(2 * BS), (cuuint64_t)nblocks};
        const cuuint64_t gstride[1] = {(cuuint64_t)(2 * BS)};
        const cuuint32_t box[2] = {(cuuint32_t)f.row_bytes, 32u};
        const cuuint32_t estr[2] = {1u, 1u};
        // L2 promotion: the L2 fetches 256 B from DRAM around a box row
        const CUresult r = enc(&f.map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<uint8_t*>(iq), gdim, gstride, box, estr,
                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return cudaErrorInvalidValue;
        f.map_iq = iq;
        f.map_nblocks = nblocks;
    }
    const long long grid = std::max(1ll, std::min<long long>((ntiles + W - 1) / W, sms));
    const long long dyn = fast_dynamic_tiles(ntiles, grid, W);
    f.kern[k]<<<(unsigned)grid, W * 32, f.smem[k], st>>>(f.map, iq, hist, hist_samples, hist_valid, lut, plane_out, nblocks,
                                                          BS, tile_counter, dyn);
    return cudaGetLastError();
}

}  // namespace ert
