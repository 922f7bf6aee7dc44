// ertgpu.cu -- C ABI of libertgpu.so (see include/ertgpu.h) and the host-side pipeline that
// drives the sm_90a kernels.  One handle mirrors one reference protocol.Decoder
// (protocol/decode.go:45-63).
//
// Device data layout (all per handle):
//   iq      : the call's interleaved uint8 I,Q bytes (caller's device buffer or a staging chunk; the input stage's
//             output buffer when the handle has an input rate or format, input_stage.cuh)
//   hist[2] : last PKL samples of the previous call (ping-pong) -- replaces the Signal tail
//             (decode.go:165) and the r900 parser's private signal history (r900.go:169)
//   plane[2]: packed quantizer output, 1 bit per sample, MSB first (bit g is bit 31-(g&31) of word g>>5, like
//             the reference's packed bytes, decode.go:259-265), laid out as
//             [hist_words of history | BS/32 words per block of the call] (ping-pong) --
//             replaces Decoder.Quantized (1 byte per bit) and Decoder.packed
//   hits    : (start, preamble) pairs found by the Search kernel (search_slide_kernel or search_generic_kernel)
//   out     : ertgpu_candidate records produced by extract_kernel
//   sig     : ertgpu_signal records of the same slots (packet_signal_kernel; handles with signal reports only)
//   spec    : the input's spectrum rows, and what spectrum_kernel carries between calls (spectrum.cuh; handles with a
//             spectrum only)
#include <ctype.h>
#include <sched.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#include "../../include/ertgpu_level.h"
#include "copy_pool.hpp"
#include "demod_fast.cuh"
#include "demod_generic.cuh"
#include "ert_common.cuh"
#include "input_stage.cuh"
#include "search.cuh"
#include "signal.cuh"
#include "spectrum.cuh"
#include "synth.cuh"

using namespace ert;

// The kernels of a handle's pipeline and their launch constants, chosen from its configuration at allocate (the demod
// again by ertgpu_set_demod_variant).  A pipeline only picks demod_fast's warp count and sizes its grids.
struct PipelineKernels {
    uint32_t smem_base = 0;      // shared address of a kernel's dynamic segment on the handle's device (demod_fast's map)
    int demod_variant = 0;       // 0 generic, else specialised chip length
    FastDemod fast;              // demod_variant != 0
    int generic_threads = 0;     // demod_variant == 0: demod_generic_kernel's CTA size and shared memory (more than
    size_t generic_smem = 0;     // 227 KiB: the decode call fails)
    // Search: the sliding-window instance (none: search_generic_kernel), its constants but nwords, smem and most CTAs
    decltype(&search_slide_kernel<1, false>) slide = nullptr;
    SlideParams sl{};
    int slide_smem = 0;
    long long slide_cap = 0;
    std::string search_label;    // ";search_slide_kernel<...>" or ";search_generic_kernel"
    decltype(&extract_words_kernel<4>) extract = nullptr;
    std::string extract_label;
    bool r900_chain = false;     // PKL % 8 == 0: r900 chains start on 8-sample (16-byte) boundaries (else replay only)
};

// The decode stream position: all that a stream start resets.
struct DecodePos {
    int cur_plane = 0, cur_hist = 0;  // the ping-pong plane and history the next pipeline reads
    int hist_valid = 0;
    int64_t block_counter = 0;  // number of reference Decode calls consumed so far
    bool fresh = true;          // next pipeline must see zeroed history
    bool started = false;       // a decode call was accepted (ertgpu_set_input_scale)
};

// What is enqueued and not yet read back.
struct InFlight {
    cudaStream_t stream = nullptr;    // work is enqueued on it and not yet synchronised (null: none)
    bool counts = false;              // ... and it copies counters back (a resample_kernel launch alone does not)
    unsigned long long uncopied = 0;  // candidates of a synchronised pipeline still only on the device
};

// What the last enqueued pipeline read (ertgpu_tap).
struct LastPipeline {
    const uint8_t* iq = nullptr;
    const uint8_t* hist = nullptr;
    int hist_valid = 0;
    const uint32_t* plane = nullptr;  // null: no pipeline yet
    int64_t first_block = 0, nblocks = 0;
};

// The results of the current decode call.
struct CallResults {
    std::vector<ertgpu_candidate> cands;
    std::vector<ertgpu_signal> sigs;  // cands' records, in the same order (signal reports only)
    bool overflow = false;            // a pipeline found more hits than the handle holds ...
    unsigned long long need = 0;      // ... the most it found
    int64_t hits = 0, valid = 0;      // ertgpu_last_counts
    // Empty, with the vectors' capacity kept: a call does not grow them again.
    void clear() {
        cands.clear();
        sigs.clear();
        *this = {std::move(cands), std::move(sigs)};
    }
};

// Stage timing: a pool of event sets so that nothing has to be read back between steps; the elapsed times of finished
// pipelines are folded into the sums when the pool is full or when somebody asks.
struct StageTiming {
    static constexpr int kSets = 64;
    bool on = false;     // ertgpu_set_stage_timing
    bool valid = false;  // the last pipeline recorded sets[last]
    Event sets[kSets][5];
    int last = 0;        // the set of the last enqueued pipeline
    int next = 0;        // set the next pipeline will use
    int unread = 0;      // finished or pending sets not yet folded (the last `unread` sets)
    double sum[4] = {};  // accumulated since ertgpu_set_stage_timing(1)
    int64_t n = 0;

    // Fold the sets of finished pipelines into the sums (only called with no pipeline pending).
    void fold() {
        for (int i = unread; i > 0; i--) {
            const Event* set = sets[(next - i + 2 * kSets) % kSets];
            float ms[4];
            bool ok = true;
            for (int k = 0; k < 4; k++) ok = ok && cudaEventElapsedTime(&ms[k], set[k], set[k + 1]) == cudaSuccess;
            if (ok) {
                for (int k = 0; k < 4; k++) sum[k] += ms[k];
                n++;
            }
        }
        unread = 0;
    }
};

struct ertgpu_handle {
    std::string err;
    std::vector<ertgpu_protocol> protos;
    ertgpu_decoder_config cfg{};
    bool allocated = false;
    int device = 0;

    DevCfg dcfg{};
    Gf32 gf{};

    // The handle's CUDA resources but the input stage's, the spectrum's and the timing events: free_device clears them.
    // The streams come last, so they are destroyed after the rest.
    struct Device {
        DeviceArray<float> lut;
        DeviceArray<uint16_t> crc;
        DeviceArray<uint32_t> plane[2];
        DeviceArray<uint8_t> hist[2];
        DeviceArray<uint8_t> stage[2];
        size_t stage_bytes = 0;
        PinnedArray<uint8_t> h_stage[2];  // pinned staging of pageable input (allocated on first use)
        size_t h_stage_bytes = 0;
        DeviceArray<RawHit> hits;
        DeviceArray<HitWord> words;       // words of starts that hold a hit (what Slice works from)
        DeviceArray<uint8_t> digits;
        DeviceArray<int> block_slot;      // r900: scratch slot of each block of the call (-1 none)
        DeviceArray<int> slot_block;
        DeviceArray<unsigned int> slot_count;
        DeviceArray<float> r900_scratch;  // [slot][r900_span] running sums
        DeviceArray<ertgpu_candidate> out;
        DeviceArray<ertgpu_signal> sig;
        DeviceArray<unsigned long long> counters;  // kCntHits, kCntOut, kCntValid, kCntTile (demod work tiles), kCntWords
        PinnedArray<unsigned long long> h_counters;  // pinned mirror
        DeviceArray<float> tap;                    // scratch for taps
        Event ev_h2d[2], ev_done[2];
        Stream stream, copy_stream;
    } dev;

    std::unique_ptr<CopyPool> copy_pool;   // host threads of the pageable-input staging
    std::string kernels;                        // instantiations launched by the last pipeline
    int r900_slots = 0, r900_span = 0;
    unsigned long long cand_cap = 0;
    bool signal = false;              // ertgpu_enable_signal: a record per candidate in dev.sig
    ertsig_geometry sig_geo{};

    int64_t max_blocks = 0;
    DecodePos pos;
    bool has_r900 = false;
    int sm_count = 132;
    PipelineKernels pipe;

    InFlight fly;
    LastPipeline last;
    CallResults res;
    int64_t launches = 0;
    StageTiming timing;

    InputStage in{err};  // input format, rate and tuning, and the kernel in front of the pipeline
    Spectrum spec;       // ertgpu_enable_spectrum
};

namespace {

template <class... A>
int fail(ertgpu_handle* h, int code, const char* fmt, A... args) { return h ? ert::fail(h->err, code, fmt, args...) : code; }

int64_t decoder_rate(const ertgpu_handle* h) { return (int64_t)h->cfg.data_rate * h->cfg.chip_length; }

// decode.go:377-379
int32_t next_pow2(int32_t v) {
    int32_t p = 1;
    while (p < v) p <<= 1;
    return p;
}

// decode.go:209-216 -- computed on the host with IEEE float32 division and multiplication
void make_maglut(float* lut) {
    for (int i = 0; i < 256; i++) {
        volatile float x = (127.5f - (float)i) / 127.5f;
        volatile float y = x * x;
        lut[i] = y;
    }
}

// crc.go:34-47
void make_crc_table(uint16_t poly, uint16_t* t) {
    for (int i = 0; i < 256; i++) {
        uint16_t crc = (uint16_t)(i << 8);
        for (int b = 0; b < 8; b++) crc = (crc & 0x8000) ? (uint16_t)((crc << 1) ^ poly) : (uint16_t)(crc << 1);
        t[i] = crc;
    }
}

// gf.go:20-57 for NewField(32, 37, 2)
void make_gf32(Gf32* g) {
    int x = 1;
    for (int i = 0; i < 31; i++) {
        g->exp[i] = g->exp[i + 31] = (uint8_t)x;
        g->log[x] = (uint8_t)i;
        x <<= 1;
        if (x & 32) x ^= 37;
    }
    g->log[0] = 31;
}

// The merged configurations the reference decodes: every index it takes for a candidate lies inside what it computed
// for that candidate (include/ertgpu.h, ertgpu_allocate).  Anything else is ERTGPU_EINVAL, naming the rule.
int check_decodable(ertgpu_handle* h) {
    const ertgpu_decoder_config& c = h->cfg;
    const int64_t BS = c.block_size, PL = c.preamble_length, SL = c.symbol_length, CL = c.chip_length;
    const int64_t PS = c.preamble_symbols, PK = c.packet_symbols, BUF = c.buffer_length;
    const int64_t npacked = (BS + PL + 7) >> 3;  // len(d.packed), decode.go:159
    // R1: Search packs d.packed from Quantized[8*i : 8*i+8] (decode.go:259-265)
    if (8 * npacked > BUF)
        return fail(h, ERTGPU_EINVAL, "R1: Search packs %lld Quantized bits of %lld (PreambleSymbols %lld, PacketSymbols %lld)",
                    (long long)(8 * npacked), (long long)BUF, (long long)PS, (long long)PK);
    bool r900 = false;
    for (const ertgpu_protocol& p : h->protos) {
        const int64_t n = (int64_t)strnlen(p.preamble, sizeof(p.preamble));
        // R2: the exact pass reads Quantized[(n-1)*SL : (n-1)*SL + BS] (decode.go:313-318), the byte pre-filter
        // d.packed[(n-1)*(SL>>3) + BS/8 - 1] (decode.go:268-287)
        if (n - 1 > PK || (n - 1) * (SL >> 3) + BS / 8 > npacked)
            return fail(h, ERTGPU_EINVAL, "R2: the Search of the %lld-bit preamble %s reads past Quantized (PacketSymbols %lld)",
                        (long long)n, p.preamble, (long long)PK);
        r900 = r900 || p.check_kind == ERTGPU_CHECK_R900;
        // R4: the partial last byte holds the previous candidate's bits in the reference (decode.go:363-366)
        if (p.check_kind == ERTGPU_CHECK_CRC16 && (PK & 7) && p.crc_from <= (PK >> 3) && (PK >> 3) < p.crc_to)
            return fail(h, ERTGPU_EINVAL, "R4: CRC range [%d, %d) of %.16s holds the partial last byte %lld (PacketSymbols %lld)",
                        p.crc_from, p.crc_to, p.name, (long long)(PK >> 3), (long long)PK);
    }
    // R3: the last r900 payload digit (r900.go:187-193) lies below BufferLength - 4*ChipLength, the last position the
    // r900 filter writes (r900.go:117): PacketSymbols >= PreambleSymbols + 83
    if (r900 && BS - 1 + PL - SL + 4 * (ERTGPU_R900_DIGITS - 1) * CL >= BUF - 4 * CL)
        return fail(h, ERTGPU_EINVAL, "R3: r900 payload digits need PacketSymbols >= PreambleSymbols + 83 (%lld < %lld)",
                    (long long)PK, (long long)(PS + 83));
    return ERTGPU_OK;
}

void free_device(ertgpu_handle* h) {
    if (!h->allocated) return;
    cudaSetDevice(h->device);
    h->in.dev = {};
    h->spec.dev = {};
    h->timing = {};
    h->dev = {};
    h->fly = {};
    h->last = {};
    h->allocated = false;
}

// Launch `kern` as a programmatic dependent of the kernel in front of it on the stream (its CTAs may become resident
// while that kernel drains; the kernel itself calls pdl_wait() before it reads anything).  pdl == false: ordinary launch.
template <class K, class... Args>
cudaError_t launch_dep(bool pdl, K kern, dim3 grid, dim3 block, size_t smem, cudaStream_t st, const Args&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, args...);
}

// h's demod instance for a variant (0: demod_generic_kernel), and the shared-memory limit of every instance it launches.
int choose_demod(ertgpu_handle* h, int variant) {
    PipelineKernels& k = h->pipe;
    k.demod_variant = variant;
    if (variant != 0) {
        k.fast = fast_demod(variant, k.smem_base);
        for (int i = 0; i < 2 && k.fast.kern[i]; i++)
            if (const int rc = allow_dynamic_smem(h->err, (const void*)k.fast.kern[i], k.fast.smem[i], "demod_fast_kernel")) return rc;
        return ERTGPU_OK;
    }
    const int CL = h->dcfg.CL;
    int nthr = 128;
    while (nthr > 32 && (256 + 2 * (size_t)CL * nthr) * sizeof(float) > 200 * 1024) nthr >>= 1;
    k.generic_threads = nthr;
    k.generic_smem = (256 + 2 * (size_t)CL * nthr) * sizeof(float);
    if (k.generic_smem > 227 * 1024) return ERTGPU_OK;  // the decode call reports it
    return allow_dynamic_smem(h->err, (const void*)demod_generic_kernel, k.generic_smem, "demod_generic_kernel");
}

// search_slide_kernel<NPRE, HALF, PAT...> and its label; PAT...: the preambles' first 16 bits as compile-time constants
// (none: read from sl), spelt as in the source ("0xF953u, 0x16A3u").
template <int NPRE, uint32_t... PAT>
void slide_instance(PipelineKernels& k, bool half) {
    k.slide = half ? search_slide_kernel<NPRE, true, PAT...> : search_slide_kernel<NPRE, false, PAT...>;
    k.search_label = ";search_slide_kernel<" + std::to_string(NPRE) + (half ? ",true" : ",false");
    const uint32_t pat[] = {PAT..., kSlideRuntimePat};
    for (int i = 0; pat[i] != kSlideRuntimePat; i++) {
        char s[16];
        snprintf(s, sizeof(s), "%s0x%04Xu", i ? ", " : ",", pat[i]);
        k.search_label += s;
    }
    k.search_label += ">";
}

// h's Search: the sliding-window kernel where the geometry fits it, search_generic_kernel for every other geometry.
int choose_search(ertgpu_handle* h) {
    const DevCfg& c = h->dcfg;
    PipelineKernels& k = h->pipe;
    if (!make_slide_params(c, (long long)c.hist_words * 32 - c.PKL, 0, &k.sl)) {
        k.search_label = ";search_generic_kernel";
        return ERTGPU_OK;
    }
    const bool half = (c.SL % 32) == 16;
    if (c.npre == 1) {
        // single preamble: the stock protocols' first 16 bits are compile-time constants
        // (scm 0xF953, scm+ 0x16A3, idm/netidm 0x5555, r900 0x0000), anything else runs the generic probe
        switch (slide_pattern(c, 0)) {
            case 0xF953u: slide_instance<1, 0xF953u>(k, half); break;
            case 0x16A3u: slide_instance<1, 0x16A3u>(k, half); break;
            case 0x5555u: slide_instance<1, 0x5555u>(k, half); break;
            case 0x0000u: slide_instance<1, 0x0000u>(k, half); break;
            default: slide_instance<1>(k, half); break;
        }
    } else if (c.npre == 2) {
        slide_instance<2>(k, half);
    } else if (c.npre == 3) {
        // scm, scm+, idm (or netidm) registered in that order: BASELINE.json configs[2]
        if (slide_pattern(c, 0) == 0xF953u && slide_pattern(c, 1) == 0x16A3u && slide_pattern(c, 2) == 0x5555u)
            slide_instance<3, 0xF953u, 0x16A3u, 0x5555u>(k, half);
        else
            slide_instance<3>(k, half);
    } else {
        // "-msgtype=all" = scm, scm+, idm, r900 (main.go:67-73)
        if (c.npre == 4 && slide_pattern(c, 0) == 0xF953u && slide_pattern(c, 1) == 0x16A3u &&
            slide_pattern(c, 2) == 0x5555u && slide_pattern(c, 3) == 0x0000u)
            slide_instance<4, 0xF953u, 0x16A3u, 0x5555u, 0x0000u>(k, half);
        else
            slide_instance<4>(k, half);
    }
    k.slide_smem = 2 * k.sl.load_words * 4 + 16;
    k.slide_cap = (long long)h->sm_count * std::min((227 * 1024) / (k.slide_smem + 1024), 2048 / kSlideThreads);
    return allow_dynamic_smem(h->err, (const void*)k.slide, k.slide_smem, "search_slide_kernel");
}

// Enqueue the whole per-call pipeline for the s.nblocks blocks whose IQ bytes are at s.iq, behind the input stage's
// kernel that writes them (its time counts as demod time).
int enqueue_pipeline(ertgpu_handle* h, const InputStep& s, uint32_t flags, cudaStream_t st) {
    const uint8_t* d_iq = s.iq;
    const int64_t nblocks = s.nblocks;
    const DevCfg& c = h->dcfg;
    DecodePos& pos = h->pos;
    uint32_t* plane = h->dev.plane[pos.cur_plane];
    uint32_t* plane_next = h->dev.plane[pos.cur_plane ^ 1];
    const uint8_t* hist = h->dev.hist[pos.cur_hist];
    uint8_t* hist_next = h->dev.hist[pos.cur_hist ^ 1];
    const long long nwords = nblocks * c.words_per_block;
    const long long p0 = (long long)c.hist_words * 32 - c.PKL;
    h->launches = 0;

    CUDA_TRY(h, cudaMemsetAsync(h->dev.counters, 0, kCntN * sizeof(unsigned long long), st));
    if (pos.fresh) {  // Quantized starts as zeros (decode.go:145); only the history in front of the call is read
        CUDA_TRY(h, cudaMemsetAsync(plane, 0, (size_t)c.hist_words * sizeof(uint32_t), st));
        pos.fresh = false;
    }

    StageTiming& t = h->timing;
    const bool tm = t.on;
    const bool pdl = !tm;   // events recorded between the kernels would sit between primary and dependent
    if (tm) {
        if (t.unread == StageTiming::kSets) t.fold();  // every earlier pipeline has been waited for
        t.last = t.next;
        t.next = (t.next + 1) % StageTiming::kSets;
        t.unread++;
    }
    const Event* ev = t.sets[t.last];
    if (tm) CUDA_TRY(h, cudaEventRecord(ev[0], st));
    if (const int rc = h->in.launch(s, st, &h->launches)) return rc;
    // 1. magnitude + matched filter + quantize + pack
    PipelineKernels& k = h->pipe;
    if (k.demod_variant != 0) {
        int w_used = 0;
        const cudaError_t e = launch_demod_fast(k.fast, h->sm_count, d_iq, hist, c.hist_samples, pos.hist_valid, h->dev.lut,
                                                plane + c.hist_words, nblocks, c.BS, h->dev.counters + kCntTile, st, &w_used);
        if (e != cudaSuccess) return fail(h, ERTGPU_ECUDA, "demod_fast launch failed: %s", cudaGetErrorString(e));
        h->kernels = "demod_fast_kernel<" + std::to_string(k.demod_variant) + "," + std::to_string(w_used) + ">";
    } else {
        h->kernels = "demod_generic_kernel";
        if (k.generic_smem > 227 * 1024) return fail(h, ERTGPU_EINVAL, "chip length %d too large for the generic kernel", c.CL);
        const unsigned grid = (unsigned)((nblocks + k.generic_threads - 1) / k.generic_threads);
        demod_generic_kernel<<<grid, k.generic_threads, k.generic_smem, st>>>(d_iq, hist, c.hist_samples, pos.hist_valid,
                                                                             h->dev.lut, plane + c.hist_words, nblocks, c.BS, c.CL);
        CUDA_TRY(h, cudaGetLastError());
    }
    h->launches++;
    if (tm) CUDA_TRY(h, cudaEventRecord(ev[1], st));

    // 2. preamble search over every start position of the call: the sliding-window kernel where the geometry fits
    //    it, search_generic_kernel for every other geometry
    if (k.slide) {
        SlideParams sl = k.sl;
        sl.nwords = nwords;
        const long long tiles = (nwords + sl.tile_words - 1) / sl.tile_words;
        const unsigned grid = (unsigned)std::max<long long>(1, std::min<long long>(tiles, k.slide_cap));
        CUDA_TRY(h, launch_dep(pdl, k.slide, dim3(grid), dim3(kSlideThreads), (size_t)k.slide_smem, st, (const uint32_t*)plane, sl,
                               h->dev.hits, h->dev.words, h->cand_cap, h->dev.counters));
    } else {
        const int nthr = 256;
        const long long blocks = std::max(1ll, std::min<long long>((nwords + nthr - 1) / nthr, (long long)h->sm_count * 16));
        CUDA_TRY(h, launch_dep(pdl, search_generic_kernel, dim3((unsigned)blocks), dim3(nthr), 0, st, (const uint32_t*)plane, p0, nwords, c,
                               h->dev.hits, h->dev.words, h->cand_cap, h->dev.counters));
    }
    h->kernels += k.search_label;
    CUDA_TRY(h, cudaGetLastError());
    h->launches++;

    if (tm) CUDA_TRY(h, cudaEventRecord(ev[2], st));
    // 3. r900 payload digits for hits of an r900 preamble
    const uint8_t* digits = nullptr;
    if (h->has_r900) {
        CUDA_TRY(h, cudaMemsetAsync(h->dev.block_slot, 0xFF, (size_t)nblocks * sizeof(int), st));
        CUDA_TRY(h, cudaMemsetAsync(h->dev.slot_count, 0, sizeof(unsigned int), st));
        // the chain kernel loads 8 samples (16 bytes) at a time from chain starts (b + 1) * BS - BUF: without that
        // alignment no block gets a scratch slot and every r900 hit takes the exact per-candidate replay
        const int slots = k.r900_chain ? h->r900_slots : 0;
        r900_mark_kernel<<<(unsigned)h->sm_count, 256, 0, st>>>(c, h->dev.hits, h->cand_cap, h->dev.counters, h->dev.block_slot, h->dev.slot_block,
                                              slots, h->dev.slot_count);
        CUDA_TRY(h, cudaGetLastError());
        if (k.r900_chain) {   // producer warps + one consumer warp per 16 chains, hand-offs through shared memory
            r900_chain2_kernel<<<(unsigned)h->sm_count * 2, (kChainProducers + 1) * 32, 0, st>>>(d_iq, hist, c.hist_samples, pos.hist_valid, c, h->dev.slot_block,
                                                        slots, h->dev.slot_count, h->r900_span, h->dev.r900_scratch);
            CUDA_TRY(h, cudaGetLastError());
            r900_digits_kernel<<<(unsigned)h->sm_count * 16, 256, 0, st>>>(c, h->dev.hits, h->cand_cap, h->dev.counters, h->dev.block_slot, h->r900_span,
                                                        h->dev.r900_scratch, h->dev.digits);
            CUDA_TRY(h, cudaGetLastError());
            h->launches += 2;
            h->kernels += ";r900_chain2_kernel";
        } else {
            h->kernels += ";r900_replay_kernel";
        }
        // blocks that found no scratch slot: exact per-candidate replay
        r900_replay_kernel<<<(unsigned)h->sm_count, 64, 0, st>>>(d_iq, hist, c.hist_samples, pos.hist_valid, h->dev.lut, c, h->dev.hits,
                                               h->cand_cap, h->dev.counters, h->dev.block_slot, h->dev.digits, h->dev.slot_count, slots);
        CUDA_TRY(h, cudaGetLastError());
        h->launches += 2;
        digits = h->dev.digits;
    }

    // 4. slice + integrity screens, one warp per word of starts with a hit; the same kernel carries the history to
    //    the other plane / history buffers (both only read what the earlier kernels wrote)
    {
        CarryArgs ca;
        ca.plane_src = plane; ca.plane_dst = plane_next; ca.src_offset_words = nwords; ca.hist_words = c.hist_words;
        ca.iq = d_iq; ca.hist_src = hist; ca.hist_dst = hist_next; ca.hist_samples = c.hist_samples;
        ca.nsamples = nblocks * c.BS;
        const unsigned grid = (unsigned)h->sm_count * 4;
        const bool dep = pdl && !h->has_r900;   // the r900 kernels between Search and Slice are ordinary launches
        CUDA_TRY(h, launch_dep(dep, k.extract, dim3(grid), dim3(kExtractWarps * 32), 0, st, (const uint32_t*)plane, p0, c,
                               (const HitWord*)h->dev.words, h->cand_cap, (const uint16_t*)h->dev.crc, h->gf, digits, (long long)pos.block_counter,
                               flags, h->dev.out, h->cand_cap, h->dev.counters, ca));
        CUDA_TRY(h, cudaGetLastError());
        h->launches++;
        h->kernels += k.extract_label;
    }
    if (h->in.mode != InputStage::kPass) h->kernels += ";" + h->in.label(s.shared_first);
    // 5. signal reports of the emitted candidates; they read d_iq, so they are enqueued before the caller records the
    //    event that frees its staging buffer; five CTAs per SM fill it at 48 registers, to hide the loads' latency
    if (h->signal) {
        packet_signal_kernel<<<(unsigned)h->sm_count * 5, kSignalWarps * 32, 0, st>>>(
            d_iq, hist, c.hist_samples, pos.hist_valid, h->sig_geo, (long long)pos.block_counter, h->dev.out, h->cand_cap,
            h->dev.counters, h->dev.sig);
        CUDA_TRY(h, cudaGetLastError());
        h->launches++;
        h->kernels += ";packet_signal_kernel";
    }

    if (tm) CUDA_TRY(h, cudaEventRecord(ev[3], st));
    if (tm) CUDA_TRY(h, cudaEventRecord(ev[4], st));
    t.valid = tm;
    CUDA_TRY(h, cudaMemcpyAsync(h->dev.h_counters, h->dev.counters, 3 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));

    h->last = {d_iq, hist, pos.hist_valid, plane, pos.block_counter, nblocks};
    h->fly.stream = st;
    h->fly.counts = true;

    pos.cur_plane ^= 1;
    pos.cur_hist ^= 1;
    pos.hist_valid = (int)std::min<long long>((long long)pos.hist_valid + nblocks * c.BS, c.hist_samples);
    pos.block_counter += nblocks;
    return ERTGPU_OK;
}

bool cand_less(const ertgpu_candidate& a, const ertgpu_candidate& b) {
    if (a.block != b.block) return a.block < b.block;
    if (a.preamble_id != b.preamble_id) return a.preamble_id < b.preamble_id;
    return a.idx < b.idx;
}

// Wait for the pending work and read the counters of its pipeline (candidates stay on the device).  A resample_kernel
// launch alone is waited for too: it read the caller's input and wrote the resampler state the next call reads.
int collect_sync(ertgpu_handle* h) {
    if (!h->fly.stream) return ERTGPU_OK;
    CUDA_TRY(h, cudaStreamSynchronize(h->fly.stream));
    h->fly.stream = nullptr;
    if (!h->fly.counts) return ERTGPU_OK;
    const unsigned long long nh = h->dev.h_counters[0], no = h->dev.h_counters[1], nv = h->dev.h_counters[2];
    CallResults& r = h->res;
    r.hits += (int64_t)nh;
    r.valid += (int64_t)nv;
    if (nh > h->cand_cap) {
        r.overflow = true;
        r.need = std::max(r.need, nh);
    }
    h->fly.uncopied = std::min(no, h->cand_cap);
    return ERTGPU_OK;  // stage times are folded lazily (StageTiming::fold)
}

// ... and append its candidates to h->res.
int collect(ertgpu_handle* h) {
    int rc = collect_sync(h);
    if (rc) return rc;
    if (const unsigned long long n = h->fly.uncopied) {
        std::vector<ertgpu_candidate>& res = h->res.cands;
        const size_t old = res.size();
        res.resize(old + n);
        CUDA_TRY(h, cudaMemcpy(res.data() + old, h->dev.out, n * sizeof(ertgpu_candidate), cudaMemcpyDeviceToHost));
        h->fly.uncopied = 0;
        // Slots are handed out by atomics, so a pipeline's records arrive unordered.  Pipelines of one
        // call cover ascending, disjoint block ranges: sorting each segment as it arrives (while the next
        // chunk's H2D copy is in flight) leaves the whole list in (block, preamble, idx) order.
        if (!h->signal) {
            std::sort(res.begin() + (std::ptrdiff_t)old, res.end(), cand_less);
            return ERTGPU_OK;
        }
        // with reports, the signal records take the candidates' order (the key is unique per candidate)
        std::vector<ertgpu_signal> sig(n);
        CUDA_TRY(h, cudaMemcpy(sig.data(), h->dev.sig, sig.size() * sizeof(ertgpu_signal), cudaMemcpyDeviceToHost));
        std::vector<uint32_t> order(sig.size());
        for (size_t i = 0; i < order.size(); i++) order[i] = (uint32_t)i;
        const ertgpu_candidate* seg = res.data() + old;
        std::sort(order.begin(), order.end(), [seg](uint32_t a, uint32_t b) { return cand_less(seg[a], seg[b]); });
        const std::vector<ertgpu_candidate> cands(seg, seg + order.size());
        for (size_t i = 0; i < order.size(); i++) {
            res[old + i] = cands[order[i]];
            h->res.sigs.push_back(sig[order[i]]);
        }
    }
    return ERTGPU_OK;
}

// The call's records v (candidates, or their signal reports: `what`) into out[0..cap), unless a pipeline found more hits
// than the handle holds.
template <class T>
int deliver(ertgpu_handle* h, const std::vector<T>& v, T* out, size_t cap, size_t* n_out, const char* what) {
    if (h->res.overflow) {
        if (n_out) *n_out = (size_t)h->res.need;
        return fail(h, ERTGPU_ECAPACITY, "internal candidate capacity %llu exceeded (%llu hits): allocate with a larger max_candidates",
                    h->cand_cap, h->res.need);
    }
    if (n_out) *n_out = v.size();  // in order already (collect)
    if (v.size() > cap) return fail(h, ERTGPU_ECAPACITY, "output array holds %zu %s, %zu needed", cap, what, v.size());
    if (!v.empty() && out) memcpy(out, v.data(), v.size() * sizeof(T));
    return ERTGPU_OK;
}

// Device staging buffers of `bytes` each (kept when large enough) and, for pageable input, the pinned staging
// buffers and the copy threads.
int prepare_staging(ertgpu_handle* h, size_t bytes, const void* iq, bool* pageable) {
    if (h->dev.stage_bytes < bytes) {
        h->dev.stage_bytes = 0;
        for (int k = 0; k < 2; k++) CUDA_TRY(h, h->dev.stage[k].alloc(bytes));
        h->dev.stage_bytes = bytes;
    }
    // Pinned (or registered / managed) input goes to the device directly.  Ordinary pageable memory -- a Go slice,
    // main.go:166's block buffer -- would make every cudaMemcpyAsync a synchronous driver-staged copy: it is staged
    // through two pinned buffers of the handle instead, filled by a few host threads while the previous chunk's
    // transfer is in flight.
    {
        cudaPointerAttributes at{};
        if (cudaPointerGetAttributes(&at, iq) == cudaSuccess) *pageable = at.type == cudaMemoryTypeUnregistered;
        else cudaGetLastError();
    }
    if (*pageable && h->dev.h_stage_bytes < h->dev.stage_bytes) {
        h->dev.h_stage_bytes = 0;
        for (int k = 0; k < 2; k++) CUDA_TRY(h, h->dev.h_stage[k].alloc(h->dev.stage_bytes));
        h->dev.h_stage_bytes = h->dev.stage_bytes;
    }
    if (*pageable) {
        int copy_threads = (int)std::min(8u, std::max(1u, std::thread::hardware_concurrency() / 4));  // ~6 GB/s per memcpy stream; 8 fill a PCIe 5 x16 link
        if (const char* e = getenv("ERTGPU_STAGE_THREADS")) copy_threads = std::min(64, std::max(1, atoi(e)));
        if (!h->copy_pool || h->copy_pool->size() != copy_threads) h->copy_pool.reset(new CopyPool(copy_threads - 1));
    }
    return ERTGPU_OK;
}

// Stream `total` host samples of s bytes at src through h's two staging slots, chunk i into slot k = i & 1: it is copied
// to dev.stage[k] on dev.copy_stream (through dev.h_stage[k] when the input is pageable), and its work is enqueued on dev.stream
// behind that copy, so that the copy of chunk i + 1 overlaps chunk i's kernels.  The callbacks:
//   next(left)        the samples of the next chunk when `left` remain; 0 ends the call with ERTGPU_EINVAL, the
//                     message already in place;
//   between()         before the work of every chunk but the first (collect the previous one's);
//   enqueue(d_in, n)  enqueue the work on the n samples at d_in on dev.stream.
// Staging buffers of `bytes` each (prepare_staging).
template <class Next, class Between, class Enqueue>
int upload(ertgpu_handle* h, const void* src, int64_t total, size_t s, size_t bytes, Next next, Between between,
           Enqueue enqueue) {
    if (total == 0) return ERTGPU_OK;
    bool pageable = true;
    if (const int rc = prepare_staging(h, bytes, src, &pageable)) return rc;
    const uint8_t* src0 = static_cast<const uint8_t*>(src);
    int64_t done = 0;
    for (int64_t i = 0; done < total; i++) {
        const int k = (int)(i & 1);
        const int64_t c = next(total - done);
        if (c <= 0) return ERTGPU_EINVAL;
        if (i >= 2) CUDA_TRY(h, cudaEventSynchronize(h->dev.ev_done[k]));  // the kernels that read dev.stage[k] (and its H2D) are done
        const uint8_t* p = src0 + (size_t)done * s;
        if (pageable) {
            h->copy_pool->copy(h->dev.h_stage[k], p, (size_t)c * s);
            p = h->dev.h_stage[k];
        }
        CUDA_TRY(h, cudaMemcpyAsync(h->dev.stage[k], p, (size_t)c * s, cudaMemcpyHostToDevice, h->dev.copy_stream));
        CUDA_TRY(h, cudaEventRecord(h->dev.ev_h2d[k], h->dev.copy_stream));
        if (i >= 1)
            if (const int rc = between()) return rc;
        CUDA_TRY(h, cudaStreamWaitEvent(h->dev.stream, h->dev.ev_h2d[k], 0));
        if (const int rc = enqueue(h->dev.stage[k], c)) return rc;
        CUDA_TRY(h, cudaEventRecord(h->dev.ev_done[k], h->dev.stream));
        done += c;
    }
    return ERTGPU_OK;
}

// Only an input stage launch is pending on st: it is waited for like a pipeline, with no counters to read.
void stage_pending(ertgpu_handle* h, cudaStream_t st) {
    h->fly.stream = st;
    h->fly.counts = false;
}

// Enqueue spectrum_kernel over the n input samples at d_in on st, last in the step: it reads the staging buffer too.
int launch_spectrum(ertgpu_handle* h, const uint8_t* d_in, int64_t n, cudaStream_t st) {
    if (const int rc = h->spec.launch(h->err, d_in, n, h->in.scale, st, &h->launches)) return rc;
    const std::string lab = ";" + h->spec.label;
    if (h->kernels.size() < lab.size() || h->kernels.compare(h->kernels.size() - lab.size(), lab.size(), lab) != 0)
        h->kernels += lab;  // a step without a pipeline keeps the last pipeline's list, which names it already
    if (!h->fly.stream) stage_pending(h, st);
    return ERTGPU_OK;
}

// Enqueue the work for the next n input samples, at d_in on the device, on st: the input stage's step, the pipeline
// over the whole blocks it completes and, with a spectrum, spectrum_kernel over the n samples.
int run_step(ertgpu_handle* h, const InputStep& s, uint32_t flags, cudaStream_t st, const uint8_t* d_in, int64_t n) {
    int rc;
    if (s.nblocks > 0) {
        rc = enqueue_pipeline(h, s, flags, st);
    } else {  // no pipeline: the stage's launch alone is pending, with no counters to read
        h->launches = 0;
        rc = h->in.launch(s, st, &h->launches);
        if (rc == ERTGPU_OK && h->launches) {
            stage_pending(h, st);
            if (h->kernels.empty()) h->kernels = h->in.label(s.shared_first);  // otherwise the last pipeline's list stays
        }
    }
    if (rc) return rc;
    h->in.commit(s);
    return h->spec.on ? launch_spectrum(h, d_in, n, st) : ERTGPU_OK;
}

int enqueue_step(ertgpu_handle* h, const uint8_t* d_in, int64_t n, uint32_t flags, cudaStream_t st) {
    return run_step(h, h->in.plan(d_in, n), flags, st, d_in, n);
}

// The same for the channels hs[0..n) of one capture (check_channels holds) over the same input.  Decimating channels
// share one decimate_channels_kernel launch, counted in hs[0]'s launches; the rest is each handle's own step.
int enqueue_channels(ertgpu_handle* const* hs, int n, const uint8_t* d_in, int64_t cnt, uint32_t flags, cudaStream_t st) {
    if (n == 1 || hs[0]->in.mode != InputStage::kDecimate || hs[0]->in.wide) {  // wide: per handle (DESIGN §3.12)
        for (int k = 0; k < n; k++)
            if (const int rc = enqueue_step(hs[k], d_in, cnt, flags, st)) return rc;
        return ERTGPU_OK;
    }
    InputStep steps[ERTGPU_MAX_CHANNELS];
    for (int k = 0; k < n; k++) steps[k] = hs[k]->in.plan(d_in, cnt);
    int64_t shared = 0;
    if (const int rc = hs[0]->in.launch_channels(steps, n, st, &shared)) return fail(hs[0], rc, "%s", hs[0]->err.c_str());
    for (int k = 0; k < n; k++)
        if (const int rc = run_step(hs[k], steps[k], flags, st, d_in, cnt)) return rc;
    ertgpu_handle* h = hs[0];
    h->launches += shared;
    if (shared && !h->fly.stream) stage_pending(h, st);  // the shared launch wrote every channel's history
    return ERTGPU_OK;
}

void begin_call(ertgpu_handle* h) {
    h->res.clear();
    h->fly.uncopied = 0;
}

// The start of both decode calls.  The input is checked by the input stage's rules before anything is collected, so
// that a rejected call leaves the stream as it was.  Then the previous call's work is collected and this call's results
// start empty.
int check_decode(ertgpu_handle* h, const void* iq, size_t nbytes, bool device) {
    if (const int rc = h ? h->in.check_samples(nbytes) : ERTGPU_OK) return rc;
    if (!h || !h->allocated) return ERTGPU_EINVAL;
    if (!iq && nbytes) return fail(h, ERTGPU_EINVAL, "null input");
    if (const int rc = h->in.check_call(iq, nbytes, device)) return rc;
    if (h->spec.on) {
        const Spectrum& sp = h->spec;
        const int64_t waiting = sp.rows_done() - sp.pos.rows_fetched, more = sp.rows_after((int64_t)(nbytes / h->in.sample_bytes));
        if (waiting + more > sp.row_cap)
            return fail(h, ERTGPU_ECAPACITY, "spectrum: %lld rows not fetched and %lld more from this call, the handle holds %lld: "
                        "ertgpu_fetch_spectrum first, or make the call shorter", (long long)waiting, (long long)more, (long long)sp.row_cap);
    }
    return ERTGPU_OK;
}

int begin_decode(ertgpu_handle* h, const void* iq, size_t nbytes, bool device) {
    if (const int rc = check_decode(h, iq, nbytes, device)) return rc;
    CUDA_TRY(h, cudaSetDevice(h->device));
    h->pos.started = true;
    if (h->fly.stream) {
        int rc = collect(h);
        if (rc) return rc;
    }
    begin_call(h);
    return ERTGPU_OK;
}

bool same_protocol(const ertgpu_protocol& a, const ertgpu_protocol& b) {
    return strncmp(a.name, b.name, sizeof(a.name)) == 0 && strncmp(a.preamble, b.preamble, sizeof(a.preamble)) == 0 &&
           a.data_rate == b.data_rate && a.chip_length == b.chip_length && a.preamble_symbols == b.preamble_symbols &&
           a.packet_symbols == b.packet_symbols && a.center_freq == b.center_freq && a.check_kind == b.check_kind &&
           a.crc_init == b.crc_init && a.crc_poly == b.crc_poly && a.crc_residue == b.crc_residue &&
           a.crc_from == b.crc_from && a.crc_to == b.crc_to;
}

// The rules of ertgpu_decode_channels and then each handle's own call rules (ertgpu.h), before anything changes.  The
// message of a broken rule goes to hs[0].
int check_channels(ertgpu_handle* const* hs, int32_t n, const void* iq, size_t nbytes, bool device) {
    if (!hs || n < 1) return ERTGPU_EINVAL;
    ertgpu_handle* h0 = hs[0];
    if (n > ERTGPU_MAX_CHANNELS) return fail(h0, ERTGPU_EINVAL, "%d channels: one call takes 1 ... %d", n, ERTGPU_MAX_CHANNELS);
    for (int k = 0; k < n; k++) {
        if (!hs[k] || !hs[k]->allocated) return fail(h0, ERTGPU_EINVAL, "channel %d: the handle is not allocated", k);
        for (int j = 0; j < k; j++)
            if (hs[j] == hs[k]) return fail(h0, ERTGPU_EINVAL, "channel %d is the handle of channel %d again", k, j);
    }
    for (int k = 0; k < n; k++) {
        const ertgpu_handle* h = hs[k];
        if (!h->in.tuned) return fail(h0, ERTGPU_EINVAL, "channel %d is not tuned (ertgpu_set_input_tuning)", k);
        if (h->device != h0->device)
            return fail(h0, ERTGPU_EINVAL, "channel %d is on device %d, channel 0 on device %d", k, h->device, h0->device);
        bool same = h->protos.size() == h0->protos.size();
        for (size_t i = 0; same && i < h->protos.size(); i++) same = same_protocol(h->protos[i], h0->protos[i]);
        if (!same) return fail(h0, ERTGPU_EINVAL, "channel %d decodes other protocols or another chip length than channel 0", k);
        if (h->in.fmt != h0->in.fmt || h->in.scale != h0->in.scale)
            return fail(h0, ERTGPU_EINVAL, "channel %d has another input format or scale than channel 0", k);
        // (the same rate gives every decimating handle the same first stage: D and T1 do not depend on the channel)
        if (h->in.rate_in != h0->in.rate_in || h->in.capture_hz != h0->in.capture_hz)
            return fail(h0, ERTGPU_EINVAL, "channel %d has another input rate or capture centre than channel 0", k);
        if (h->in.wide != h0->in.wide)
            return fail(h0, ERTGPU_EINVAL, "channel %d %s the wide channel path and channel 0 %s: every channel of a group takes it or none does",
                        k, h->in.wide ? "takes" : "does not take", h0->in.wide ? "does" : "does not");
        if (h->in.received() != h0->in.received())
            return fail(h0, ERTGPU_EINVAL, "channel %d is at input sample %lld of its stream, channel 0 at %lld: reset the channels together",
                        k, (long long)h->in.received(), (long long)h0->in.received());
    }
    for (int k = 0; k < n; k++)
        for (int j = 0; j < k; j++)
            if (hs[k]->spec.on && hs[j]->spec.on)
                return fail(h0, ERTGPU_EINVAL, "channels %d and %d both have a spectrum: a group measures its input once, on one handle", j, k);
    for (int k = 0; k < n; k++)
        if (const int rc = check_decode(hs[k], iq, nbytes, device)) {
            if (k) fail(h0, rc, "channel %d: %s", k, hs[k]->err.c_str());
            return rc;
        }
    return ERTGPU_OK;
}

}  // namespace

// ertgpu_decode_sharded's rule for signal reports and spectra, with its message on h.  Shared with sharded.cpp inside
// the library only: hidden, so libertgpu.so exports nothing beyond include/ertgpu.h.
__attribute__((visibility("hidden"))) int sharded_reject_signal(ertgpu_handle* h) {
    if (h->spec.on) return fail(h, ERTGPU_EINVAL, "decode_sharded: the handle has a spectrum (ertgpu_enable_spectrum), which sharded decodes do not measure");
    return h->signal ? fail(h, ERTGPU_EINVAL, "decode_sharded: the handle has signal reports (ertgpu_enable_signal), which sharded decodes do not keep")
                     : ERTGPU_OK;
}

extern "C" {

int ertgpu_abi_version(void) { return ERTGPU_ABI_VERSION; }

const char* ertgpu_last_error(const ertgpu_handle* h) { return h ? h->err.c_str() : "null handle"; }

int ertgpu_create(ertgpu_handle** out) {
    if (!out) return ERTGPU_EINVAL;
    ertgpu_handle* h = new (std::nothrow) ertgpu_handle();
    if (!h) return ERTGPU_ENOMEM;
    *out = h;
    return ERTGPU_OK;
}

void ertgpu_destroy(ertgpu_handle* h) {
    if (!h) return;
    free_device(h);
    delete h;
}

int ertgpu_stock_protocol(const char* msgtype, int32_t chip_length, ertgpu_protocol* p) {
    if (!msgtype || !p) return ERTGPU_EINVAL;
    memset(p, 0, sizeof(*p));
    p->data_rate = 32768;
    p->chip_length = chip_length;
    p->center_freq = 912600155u;
    snprintf(p->name, sizeof(p->name), "%s", msgtype);
    if (!strcmp(msgtype, "scm")) {  // scm/scm.go:40-50
        snprintf(p->preamble, sizeof(p->preamble), "%s", "111110010101001100000");
        p->preamble_symbols = 21;
        p->packet_symbols = 96;
        p->check_kind = ERTGPU_CHECK_CRC16;
        p->crc_init = 0; p->crc_poly = 0x6F63; p->crc_residue = 0;
        p->crc_from = 2; p->crc_to = 12;
    } else if (!strcmp(msgtype, "scm+")) {  // scmplus/scmplus.go:47-57
        snprintf(p->preamble, sizeof(p->preamble), "%s", "0001011010100011");
        p->preamble_symbols = 16;
        p->packet_symbols = 128;
        p->check_kind = ERTGPU_CHECK_CRC16;
        p->crc_init = 0xFFFF; p->crc_poly = 0x1021; p->crc_residue = 0x1D0F;
        p->crc_from = 2; p->crc_to = 16;
    } else if (!strcmp(msgtype, "idm") || !strcmp(msgtype, "netidm")) {  // idm/idm.go:46-56, netidm/netidm.go:58-68
        snprintf(p->preamble, sizeof(p->preamble), "%s", "01010101010101010001011010100011");
        p->preamble_symbols = 32;
        p->packet_symbols = 92 * 8;
        p->check_kind = ERTGPU_CHECK_IDM;
        p->crc_init = 0xFFFF; p->crc_poly = 0x1021; p->crc_residue = 0x1D0F;
        p->crc_from = 4; p->crc_to = 92;
    } else if (!strcmp(msgtype, "r900") || !strcmp(msgtype, "r900bcd")) {  // r900/r900.go:54-65
        snprintf(p->preamble, sizeof(p->preamble), "%s", "00000000000000001110010101100100");
        p->preamble_symbols = 32;
        p->packet_symbols = 116;
        p->center_freq = 912380000u;
        p->check_kind = ERTGPU_CHECK_R900;
    } else {
        return ERTGPU_EINVAL;  // parse.go:49 "invalid message type"
    }
    return ERTGPU_OK;
}

int ertgpu_register_protocol(ertgpu_handle* h, const ertgpu_protocol* p) {
    if (!h || !p) return ERTGPU_EINVAL;
    if (h->allocated) return fail(h, ERTGPU_EINVAL, "register_protocol after allocate");
    if (h->in.rate_in) return fail(h, ERTGPU_EINVAL, "register_protocol after set_input_rate");
    if (h->in.tuned) return fail(h, ERTGPU_EINVAL, "register_protocol after set_input_tuning");
    if (h->protos.size() >= ERTGPU_MAX_PROTOCOLS) return fail(h, ERTGPU_EINVAL, "too many protocols");
    const size_t n = strnlen(p->preamble, sizeof(p->preamble));
    if (n == 0 || n > ERTGPU_MAX_PREAMBLE) return fail(h, ERTGPU_EINVAL, "bad preamble length %zu", n);
    for (size_t i = 0; i < n; i++)
        if (p->preamble[i] != '0' && p->preamble[i] != '1') return fail(h, ERTGPU_EINVAL, "preamble must be '0'/'1'");
    if (p->chip_length <= 0 || p->preamble_symbols <= 0 || p->packet_symbols <= 0)
        return fail(h, ERTGPU_EINVAL, "non-positive geometry");
    if ((p->packet_symbols + 7) / 8 > ERTGPU_MAX_PACKET_BYTES) return fail(h, ERTGPU_EINVAL, "packet too long");
    if (p->check_kind == ERTGPU_CHECK_CRC16 &&
        (p->crc_from < 0 || p->crc_to > (p->packet_symbols + 7) / 8 || p->crc_from >= p->crc_to))
        return fail(h, ERTGPU_EINVAL, "bad crc range");
    if (p->check_kind == ERTGPU_CHECK_IDM && p->packet_symbols < 92 * 8) return fail(h, ERTGPU_EINVAL, "idm screen needs 92 bytes");
    h->protos.push_back(*p);
    // decode.go:105-109
    ertgpu_decoder_config& c = h->cfg;
    c.center_freq = p->center_freq;
    c.data_rate = std::max(c.data_rate, p->data_rate);
    c.chip_length = std::max(c.chip_length, p->chip_length);
    c.preamble_symbols = std::max(c.preamble_symbols, p->preamble_symbols);
    c.packet_symbols = std::max(c.packet_symbols, p->packet_symbols);
    c.n_protocols = (int32_t)h->protos.size();
    return ERTGPU_OK;
}

static int allocate_impl(ertgpu_handle* h, int32_t device, int64_t max_blocks_per_call, int64_t max_candidates);

int ertgpu_allocate(ertgpu_handle* h, int32_t device, int64_t max_blocks_per_call, int64_t max_candidates) {
    if (!h) return ERTGPU_EINVAL;
    if (h->allocated) return fail(h, ERTGPU_EINVAL, "already allocated");
    const int rc = allocate_impl(h, device, max_blocks_per_call, max_candidates);
    if (rc != ERTGPU_OK) {
        // a half-built handle must not pass the `allocated` checks of decode/tap/reset: release whatever was
        // created (the message of the failure is kept) and leave the handle ready for another ertgpu_allocate
        const std::string msg = h->err;
        free_device(h);
        h->cfg.n_preambles = 0;
        h->err = msg;
    }
    return rc;
}

static int allocate_impl(ertgpu_handle* h, int32_t device, int64_t max_blocks_per_call, int64_t max_candidates) {
    if (h->protos.empty()) return fail(h, ERTGPU_EINVAL, "no protocol registered");
    if (const int rc = h->in.plan_native(decoder_rate(h))) return rc;

    // decode.go:131-141
    ertgpu_decoder_config& c = h->cfg;
    c.symbol_length = c.chip_length << 1;
    c.sample_rate = c.data_rate * c.chip_length;
    c.preamble_length = c.preamble_symbols * c.symbol_length;
    c.packet_length = c.packet_symbols * c.symbol_length;
    c.block_size = next_pow2(c.preamble_length);
    c.block_size2 = c.block_size << 1;
    c.buffer_length = c.packet_length + c.block_size;
    c.packet_bytes = (c.packet_symbols + 7) >> 3;
    if (c.block_size < 32) return fail(h, ERTGPU_EINVAL, "block size %d below 32", c.block_size);
    if (const int rc = check_decodable(h)) return rc;

    DevCfg& d = h->dcfg;
    memset(&d, 0, sizeof(d));
    d.CL = c.chip_length; d.SL = c.symbol_length; d.BS = c.block_size;
    d.PS = c.preamble_symbols; d.PK = c.packet_symbols;
    d.PL = c.preamble_length; d.PKL = c.packet_length; d.BUF = c.buffer_length;
    d.words_per_block = d.BS / 32;
    d.hist_words = ((d.PKL + 31) / 32 + 3) & ~3;  // multiple of 4: the call's first word is 16-byte aligned
    d.hist_samples = d.PKL;
    d.packet_bytes = c.packet_bytes;
    d.nproto = (int32_t)h->protos.size();
    std::vector<uint16_t> tables;
    h->has_r900 = false;
    for (int i = 0; i < d.nproto; i++) {
        const ertgpu_protocol& p = h->protos[i];
        const int nb = (int)strnlen(p.preamble, sizeof(p.preamble));
        int found = -1;
        for (int j = 0; j < d.npre; j++) {
            if (d.pre_nbits[j] != nb) continue;
            bool same = true;
            for (int k = 0; k < nb; k++) same = same && d.pre_bits[j][k] == (uint8_t)(p.preamble[k] == '1');
            if (same) found = j;
        }
        if (found < 0) {  // decode.go:121-124
            found = d.npre++;
            d.pre_nbits[found] = nb;
            for (int k = 0; k < nb; k++) d.pre_bits[found][k] = (uint8_t)(p.preamble[k] == '1');
        }
        DevProto& dp = d.proto[i];
        dp.preamble_id = found;
        dp.check_kind = p.check_kind;
        dp.packet_bytes = (p.packet_symbols + 7) >> 3;
        dp.crc_from = p.crc_from; dp.crc_to = p.crc_to;
        dp.crc_init = p.crc_init; dp.crc_residue = p.crc_residue;
        dp.table = i;
        tables.resize((size_t)(i + 1) * 256);
        make_crc_table(p.crc_poly, tables.data() + (size_t)i * 256);
        if (p.check_kind == ERTGPU_CHECK_IDM) dp.crc_from = 4;   // the IDM screen's first CRC starts at byte 4 whatever crc_from says (idm.go:77-87)
        if (p.check_kind == ERTGPU_CHECK_R900) {
            d.pre_has_r900[found] = 1;
            h->has_r900 = true;
        }
    }
    c.n_preambles = d.npre;

    int ndev = 0;
    CUDA_TRY(h, cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev) return fail(h, ERTGPU_ECUDA, "device %d not available (%d devices)", device, ndev);
    h->device = device;
    CUDA_TRY(h, cudaSetDevice(device));
    cudaDeviceProp prop;
    CUDA_TRY(h, cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) return fail(h, ERTGPU_ECUDA, "libertgpu is built for sm_90a only; device %d is sm_%d%d", device, prop.major, prop.minor);

    if (max_blocks_per_call <= 0) max_blocks_per_call = std::max<int64_t>(1, (64ll << 20) / c.block_size2);
    if (max_candidates <= 0) max_candidates = 1 << 18;
    h->max_blocks = max_blocks_per_call;
    h->cand_cap = (unsigned long long)max_candidates;
    h->allocated = true;  // from here free_device() cleans up on failure

    CUDA_TRY(h, h->dev.stream.create(cudaStreamNonBlocking));
    CUDA_TRY(h, h->dev.copy_stream.create(cudaStreamNonBlocking));
    for (int k = 0; k < 2; k++) {
        CUDA_TRY(h, h->dev.ev_h2d[k].create(cudaEventDisableTiming));
        CUDA_TRY(h, h->dev.ev_done[k].create(cudaEventDisableTiming));
    }
    for (auto& set : h->timing.sets) for (Event& e : set) CUDA_TRY(h, e.create(cudaEventDefault));
    std::vector<float> lut(256);
    make_maglut(lut.data());
    make_gf32(&h->gf);
    CUDA_TRY(h, h->dev.lut.upload(lut));
    CUDA_TRY(h, h->dev.crc.upload(tables));

    // Slack behind the largest call's words, for the Search kernels' reads past the call's last word:
    //  * search_slide_kernel's last tile starts at a word below nwords and loads load_words <= kSlideMaxLoad words;
    //  * search_generic_kernel (and extract_words_kernel) read the word under plane bit p0 + 32*w + k*SL and the next
    //    one, w < nwords; with p0 + PKL = 32*hist_words the bits they use lie inside the call's words while k <= PK
    //    (the next word may be the first one behind them).  Rule R2 (check_decodable) keeps every preamble at most
    //    PK + 1 bits long, so no Search result depends on bits past the call's words.
    const size_t plane_words = (size_t)d.hist_words + (size_t)max_blocks_per_call * d.words_per_block + kSlideMaxLoad + 8;
    for (int k = 0; k < 2; k++) {
        CUDA_TRY(h, h->dev.plane[k].alloc(plane_words));
        CUDA_TRY(h, cudaMemset(h->dev.plane[k], 0, plane_words * sizeof(uint32_t)));
        CUDA_TRY(h, h->dev.hist[k].alloc((size_t)d.hist_samples * 2 + 16));
        CUDA_TRY(h, cudaMemset(h->dev.hist[k], 0, (size_t)d.hist_samples * 2 + 16));
    }
    CUDA_TRY(h, h->dev.hits.alloc(h->cand_cap));
    CUDA_TRY(h, h->dev.words.alloc(h->cand_cap));
    CUDA_TRY(h, h->dev.out.alloc(h->cand_cap));
    if (h->signal) {
        CUDA_TRY(h, h->dev.sig.alloc(h->cand_cap));
        ertsig_geometry& g = h->sig_geo;
        g = {};
        g.CL = d.CL; g.SL = d.SL; g.BS = d.BS; g.BUF = d.BUF; g.PK = d.PK;
        g.nproto = d.nproto;
        for (int i = 0; i < d.nproto; i++) {
            const ertgpu_protocol& p = h->protos[i];
            g.preamble_id[i] = d.proto[i].preamble_id;
            g.span[i] = p.check_kind == ERTGPU_CHECK_R900 ? p.preamble_symbols : p.packet_symbols;
        }
    }
    if (h->has_r900) {
        CUDA_TRY(h, h->dev.digits.alloc(h->cand_cap * ERTGPU_R900_DIGITS));
        h->r900_span = d.BS + d.PL - d.SL + 4 * ERTGPU_R900_DIGITS * d.CL + 1;
        if (h->r900_span > d.BUF + 1) h->r900_span = d.BUF + 1;
        // scratch slots: one per block that holds an r900 hit.  Sized for one packet per 16 blocks
        // (at least 64 slots), at most 1 GiB; blocks beyond that use the per-candidate replay.
        {
            const int64_t per_slot = (int64_t)h->r900_span * 4;
            int64_t want = std::max<int64_t>(64, max_blocks_per_call / 16);
            want = std::min<int64_t>(want, (1ll << 30) / per_slot);
            h->r900_slots = (int)std::max<int64_t>(1, std::min<int64_t>(want, max_blocks_per_call));
        }
        if (const char* e = getenv("ERTGPU_R900_SLOTS")) h->r900_slots = std::max(1, atoi(e));  // test hook: force the replay fallback
        CUDA_TRY(h, h->dev.block_slot.alloc((size_t)max_blocks_per_call));
        CUDA_TRY(h, h->dev.slot_block.alloc((size_t)h->r900_slots));
        CUDA_TRY(h, h->dev.slot_count.alloc(1));
        CUDA_TRY(h, h->dev.r900_scratch.alloc((size_t)h->r900_slots * r900_pitch(h->r900_span) + 16));
    }
    CUDA_TRY(h, h->dev.counters.alloc(kCntN));
    CUDA_TRY(h, h->dev.h_counters.alloc(kCntN));
    CUDA_TRY(h, h->dev.tap.alloc((size_t)std::max(d.BS + d.SL, d.BUF) * 2 + 16));

    cudaDeviceGetAttribute(&h->sm_count, cudaDevAttrMultiProcessorCount, h->device);
    if (h->sm_count < 1) h->sm_count = 132;

    h->pipe = {};
    // where the dynamic shared memory of a kernel starts on this device, through the tap scratch
    smem_base_probe_kernel<<<1, 1, 1024, h->dev.stream>>>(reinterpret_cast<uint32_t*>(h->dev.tap.get()));
    CUDA_TRY(h, cudaGetLastError());
    CUDA_TRY(h, cudaMemcpyAsync(&h->pipe.smem_base, h->dev.tap, sizeof(uint32_t), cudaMemcpyDeviceToHost, h->dev.stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->dev.stream));
    if (const int rc = choose_demod(h, demod_fast_variant(d.CL, d.BS, d.PKL))) return rc;
    if (const int rc = choose_search(h)) return rc;
    constexpr int kFullK = (ERTGPU_MAX_PACKET_BYTES * 8 + 31) / 32;
    const bool short_packets = d.PK <= 128;
    h->pipe.extract = short_packets ? extract_words_kernel<4> : extract_words_kernel<kFullK>;
    h->pipe.extract_label = ";extract_words_kernel<" + std::to_string(short_packets ? 4 : kFullK) + ">";
    // BS is a power of two >= 32 and the call's bytes are 16-byte aligned: chain starts (b + 1) * BS - BUF are
    // multiples of 8 samples when PKL is (BUF = PKL + BS, the history holds PKL samples)
    h->pipe.r900_chain = d.PKL % 8 == 0;

    if (const int rc = h->in.allocate(c.block_size, max_blocks_per_call, h->sm_count)) return rc;
    if (h->spec.on) {  // rows of the largest call: a staging chunk, or a device call of the input stage's largest step
        const int64_t r_out = decoder_rate(h), r_in = h->in.rate_in ? h->in.rate_in : r_out;
        const int64_t in_max = std::max({h->in.chunk(), h->in.max_call_input(),
                                         max_blocks_per_call * c.block_size * ((r_in + r_out - 1) / r_out)});
        if (const int rc = h->spec.allocate(h->err, h->in.fmt, h->in.sample_bytes, ertfmt_name(h->in.fmt), in_max, h->sm_count))
            return rc;
    }
    h->pos = {};
    return ERTGPU_OK;
}

int ertgpu_get_config(const ertgpu_handle* h, ertgpu_decoder_config* cfg) {
    if (!h || !cfg) return ERTGPU_EINVAL;
    if (!h->allocated) return ERTGPU_EINVAL;
    *cfg = h->cfg;
    return ERTGPU_OK;
}

int ertgpu_reset(ertgpu_handle* h) {
    if (!h || !h->allocated) return ERTGPU_EINVAL;
    CUDA_TRY(h, cudaSetDevice(h->device));
    int rc = collect_sync(h);
    if (rc) return rc;
    h->pos = {};  // the history in front of the next call is zeroed on that call's stream (enqueue_pipeline)
    h->in.reset_stream();
    h->spec.pos = {};
    begin_call(h);
    return ERTGPU_OK;
}

int ertgpu_set_input_rate(ertgpu_handle* h, int64_t hz) {
    if (!h) return ERTGPU_EINVAL;
    if (h->allocated) return fail(h, ERTGPU_EINVAL, "set_input_rate after allocate");
    if (h->protos.empty()) return fail(h, ERTGPU_EINVAL, "set_input_rate before register_protocol");
    return h->in.set_rate(hz, decoder_rate(h));
}

int ertgpu_set_input_tuning(ertgpu_handle* h, int64_t capture_center_hz, int64_t center_hz) {
    if (!h) return ERTGPU_EINVAL;
    if (h->allocated) return fail(h, ERTGPU_EINVAL, "set_input_tuning after allocate");
    if (h->protos.empty()) return fail(h, ERTGPU_EINVAL, "set_input_tuning before register_protocol");
    return h->in.set_tuning(capture_center_hz, center_hz, (int64_t)h->cfg.center_freq, decoder_rate(h));
}

int ertgpu_allow_input_decimation(ertgpu_handle* h) {
    if (!h) return ERTGPU_EINVAL;
    if (h->allocated) return fail(h, ERTGPU_EINVAL, "allow_input_decimation after allocate");
    return h->in.allow_decimation();
}

int ertgpu_get_decimator(const ertgpu_handle* h, ertgpu_decimator_info* info, int16_t* taps, size_t cap, size_t* n_out) {
    return h ? h->in.decimator(info, taps, cap, n_out) : ERTGPU_EINVAL;
}

int ertgpu_get_tuning(const ertgpu_handle* h, ertgpu_tuning_info* info) {
    return h ? h->in.tuning(info) : ERTGPU_EINVAL;
}

int ertgpu_set_input_format(ertgpu_handle* h, int32_t format, float scale) {
    if (!h) return ERTGPU_EINVAL;
    if (h->allocated) return fail(h, ERTGPU_EINVAL, "set_input_format after allocate");
    return h->in.set_format(format, scale);
}

int ertgpu_get_input_format(const ertgpu_handle* h, int32_t* format, float* scale) {
    if (!h) return ERTGPU_EINVAL;
    if (format) *format = h->in.fmt;
    if (scale) *scale = h->in.scale;
    return ERTGPU_OK;
}

int ertgpu_set_input_scale(ertgpu_handle* h, float scale) {
    if (!h) return ERTGPU_EINVAL;
    if (!h->allocated) return fail(h, ERTGPU_EINVAL, "set_input_scale before allocate: ertgpu_set_input_format takes the scale");
    if (h->pos.started) return fail(h, ERTGPU_EINVAL, "set_input_scale after a decode call: the gain changes only at a stream start");
    return h->in.set_scale(scale);
}

int ertgpu_set_channel_gain(ertgpu_handle* h, int32_t k) {
    if (!h) return ERTGPU_EINVAL;
    if (h->allocated && h->pos.started)
        return fail(h, ERTGPU_EINVAL, "set_channel_gain after a decode call: the gain changes only at a stream start");
    return h->in.set_channel_gain(k, h->allocated);
}

int ertgpu_get_channel_gain(const ertgpu_handle* h, int32_t* k) {
    if (!h || !h->in.wide) return ERTGPU_EINVAL;
    if (k) *k = h->in.gain;
    return ERTGPU_OK;
}

// ertgpu_measure_input's staging, with the input stage's own steps (begin_measure: from a stream start, on the
// measurement's histories) counting into d_clevel.  The steps end on the handle's stream before the position comes back,
// whether the call succeeds or not.
int ertgpu_measure_channel(ertgpu_handle* h, const void* samples, size_t nbytes, ertgpu_channel_level* out) {
    if (!h || !h->allocated) return ERTGPU_EINVAL;
    if (!h->in.wide) return fail(h, ERTGPU_EINVAL, "measure_channel: the handle does not take the wide channel path");
    if (!out || (!samples && nbytes)) return fail(h, ERTGPU_EINVAL, "null argument");
    const size_t s = (size_t)h->in.sample_bytes;
    if (nbytes % s) return fail(h, ERTGPU_ESIZE, "nbytes %zu is not a whole number of %zu-byte IQ samples", nbytes, s);
    CUDA_TRY(h, cudaSetDevice(h->device));
    if (const int rc = collect_sync(h)) return rc;  // the stream's own last step is done with the histories
    CUDA_TRY(h, cudaMemsetAsync(h->in.dev.clevel, 0, ERTRS_GAIN_BINS * sizeof(unsigned long long), h->dev.stream));
    int64_t outputs = 0, launches = 0;
    h->in.begin_measure();
    const int rc = upload(h, samples, (int64_t)(nbytes / s), s, (size_t)h->in.chunk() * s,
                          [&](int64_t left) { return h->in.next_chunk(left); }, [] { return ERTGPU_OK; },
                          [&](const uint8_t* d_in, int64_t c) {
                              InputStep st = h->in.plan(d_in, c);
                              st.rs.level = h->in.dev.clevel;
                              if (const int rc = h->in.launch(st, h->dev.stream, &launches)) return rc;
                              outputs += st.rs.count;
                              h->in.commit(st);
                              return ERTGPU_OK;
                          });
    unsigned long long cnt[ERTRS_GAIN_BINS];
    const cudaError_t e1 = cudaMemcpyAsync(cnt, h->in.dev.clevel, sizeof(cnt), cudaMemcpyDeviceToHost, h->dev.stream);
    const cudaError_t e2 = cudaStreamSynchronize(h->dev.stream);
    h->in.end_measure();
    if (rc) return rc;
    CUDA_TRY(h, e1);
    CUDA_TRY(h, e2);
    memset(out, 0, sizeof(*out));
    out->components = 2 * outputs;
    int64_t nonzero = 0;
    for (int b = 0; b < ERTRS_GAIN_BINS; b++) nonzero += out->bins[b] = (int64_t)cnt[b];
    out->zeros = out->components - nonzero;
    out->k = ertrs_channel_gain(out->bins, out->components);
    return ERTGPU_OK;
}

// The samples go through ertgpu_decode's staging in chunks of a whole staging buffer, each counted by level_kernel on the
// handle's stream.  The counters live in the input stage and are zeroed first; nothing the decode reads or keeps between
// calls is touched.
int ertgpu_measure_input(ertgpu_handle* h, const void* samples, size_t nbytes, ertgpu_input_level* out) {
    if (!h || !h->allocated) return ERTGPU_EINVAL;
    if (h->in.fmt == ERTGPU_FORMAT_CU8) return fail(h, ERTGPU_EINVAL, "cu8 input is not measured: it takes no gain");
    if (!out || (!samples && nbytes)) return fail(h, ERTGPU_EINVAL, "null argument");
    const size_t s = (size_t)h->in.sample_bytes;
    if (nbytes % s) return fail(h, ERTGPU_ESIZE, "nbytes %zu is not a whole number of %zu-byte IQ samples", nbytes, s);
    CUDA_TRY(h, cudaSetDevice(h->device));
    CUDA_TRY(h, cudaMemsetAsync(h->in.dev.level, 0, kLvCounters * sizeof(unsigned long long), h->dev.stream));
    const int64_t total = (int64_t)(nbytes / s);
    if (const int rc = upload(h, samples, total, s, (size_t)h->in.chunk() * s,
                              [&](int64_t left) { return std::min((int64_t)(h->dev.stage_bytes / s), left); },
                              [] { return ERTGPU_OK; },
                              [&](const uint8_t* d_in, int64_t c) { return h->in.launch_level(d_in, c, h->dev.stream); }))
        return rc;
    unsigned long long cnt[kLvCounters];
    CUDA_TRY(h, cudaMemcpyAsync(cnt, h->in.dev.level, sizeof(cnt), cudaMemcpyDeviceToHost, h->dev.stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->dev.stream));
    memset(out, 0, sizeof(*out));
    out->components = 2 * total;
    out->zeros = (int64_t)cnt[kLvZero];
    out->nans = (int64_t)cnt[kLvNan];
    for (int b = 0; b < ERTLV_BINS; b++) out->bins[b] = (int64_t)cnt[b];
    out->exponent = ertlv_exponent(out->bins, out->components, out->zeros, out->nans, ilogbf(ertfmt_default_scale(h->in.fmt)));
    out->scale = ldexpf(1.0f, out->exponent);
    return ERTGPU_OK;
}

int ertgpu_get_resampler(const ertgpu_handle* h, ertgpu_resampler_info* info, int16_t* table, size_t cap,
                         size_t* n_out) {
    return h ? h->in.resampler(info, table, cap, n_out) : ERTGPU_EINVAL;
}

int ertgpu_set_demod_variant(ertgpu_handle* h, int32_t variant) {
    // test hook: 0 forces the generic kernel, -1 restores the automatic choice
    if (!h || !h->allocated || variant > 0) return ERTGPU_EINVAL;
    CUDA_TRY(h, cudaSetDevice(h->device));
    return choose_demod(h, variant < 0 ? demod_fast_variant(h->dcfg.CL, h->dcfg.BS, h->dcfg.PKL) : 0);
}

int ertgpu_decode_device_async(ertgpu_handle* h, const void* d_iq, size_t nbytes, uint32_t flags, void* stream) {
    const int rc = begin_decode(h, d_iq, nbytes, true);
    if (rc || nbytes == 0) return rc;
    return enqueue_step(h, static_cast<const uint8_t*>(d_iq), (int64_t)(nbytes / h->in.sample_bytes), flags,
                        stream ? (cudaStream_t)stream : h->dev.stream);
}

int ertgpu_fetch(ertgpu_handle* h, ertgpu_candidate* out, size_t cap, size_t* n_out) {
    if (!h || !h->allocated) return ERTGPU_EINVAL;
    CUDA_TRY(h, cudaSetDevice(h->device));
    int rc = collect(h);
    if (rc) return rc;
    return deliver(h, h->res.cands, out, cap, n_out, "candidates");
}

int ertgpu_decode(ertgpu_handle* h, const uint8_t* iq, size_t nbytes, uint32_t flags, ertgpu_candidate* out,
                  size_t cap, size_t* n_out) {
    int rc = begin_decode(h, iq, nbytes, false);
    if (rc) return rc;
    const size_t s = (size_t)h->in.sample_bytes;
    const int64_t total = (int64_t)(nbytes / s);
    if (total == 0) return deliver(h, h->res.cands, out, cap, n_out, "candidates");
    int64_t launches = 0;
    rc = upload(h, iq, total, s, (size_t)h->in.chunk() * s, [&](int64_t left) { return h->in.next_chunk(left); },
                [&] { return collect(h); },
                [&](const uint8_t* d_in, int64_t c) {
                    if (const int rc = enqueue_step(h, d_in, c, flags, h->dev.stream)) return rc;
                    launches += h->launches;
                    return ERTGPU_OK;
                });
    if (rc) return rc;
    rc = collect(h);  // also waits for a last step that completed no block (ertgpu_decode is synchronous)
    if (rc) return rc;
    CUDA_TRY(h, cudaStreamSynchronize(h->dev.copy_stream));  // a step that launched nothing still copied from iq
    h->launches = launches;
    return deliver(h, h->res.cands, out, cap, n_out, "candidates");
}

int ertgpu_decode_channels_device_async(ertgpu_handle* const* hs, int32_t n, const void* d_iq, size_t nbytes, uint32_t flags,
                                        void* stream) {
    if (const int rc = check_channels(hs, n, d_iq, nbytes, true)) return rc;
    for (int k = 0; k < n; k++)
        if (const int rc = begin_decode(hs[k], d_iq, nbytes, true)) return rc;
    if (nbytes == 0) return ERTGPU_OK;
    return enqueue_channels(hs, n, static_cast<const uint8_t*>(d_iq), (int64_t)(nbytes / hs[0]->in.sample_bytes), flags,
                            stream ? (cudaStream_t)stream : hs[0]->dev.stream);
}

// ertgpu_decode's loop over hs[0]'s staging buffers and streams, with every channel's step behind each chunk's copy.
int ertgpu_decode_channels(ertgpu_handle* const* hs, int32_t n, const uint8_t* iq, size_t nbytes, uint32_t flags) {
    if (const int rc = check_channels(hs, n, iq, nbytes, false)) return rc;
    for (int k = 0; k < n; k++)
        if (const int rc = begin_decode(hs[k], iq, nbytes, false)) return rc;
    ertgpu_handle* h = hs[0];
    const size_t s = (size_t)h->in.sample_bytes;
    const int64_t total = (int64_t)(nbytes / s);
    if (total == 0) return ERTGPU_OK;
    int64_t chunk = 0;
    for (int k = 0; k < n; k++) chunk = std::max(chunk, hs[k]->in.chunk());
    // At the decoder's own rate the channel at the capture's centre is not resampled (it only converts, if anything) and
    // takes whole blocks: then every step does.
    bool whole_blocks = false;
    for (int j = 0; j < n; j++) whole_blocks |= !hs[j]->in.resamples();
    const int64_t block = h->dcfg.BS;
    int64_t launches[ERTGPU_MAX_CHANNELS] = {};
    auto next = [&](int64_t left) {
        int64_t c = left;
        for (int j = 0; j < n; j++) c = std::min(c, hs[j]->in.next_chunk(left));  // a step every channel takes
        if (whole_blocks) c -= c % block;
        if (c <= 0) fail(h, ERTGPU_EINVAL, "no step of whole blocks fits every channel's buffers");
        return c;
    };
    auto collect_all = [&] {
        for (int j = 0; j < n; j++)
            if (const int rc = collect(hs[j])) return rc;
        return ERTGPU_OK;
    };
    int rc = upload(h, iq, total, s, (size_t)chunk * s, next, collect_all, [&](const uint8_t* d_in, int64_t c) {
        if (const int rc = enqueue_channels(hs, n, d_in, c, flags, h->dev.stream)) return rc;
        for (int j = 0; j < n; j++) launches[j] += hs[j]->launches;
        return ERTGPU_OK;
    });
    if (rc) return rc;
    for (int j = 0; j < n; j++) {
        if ((rc = collect(hs[j]))) return rc;
        hs[j]->launches = launches[j];
    }
    CUDA_TRY(h, cudaStreamSynchronize(h->dev.stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->dev.copy_stream));
    return ERTGPU_OK;
}

int ertgpu_enable_signal(ertgpu_handle* h) {
    if (!h) return ERTGPU_EINVAL;
    if (h->allocated) return fail(h, ERTGPU_EINVAL, "enable_signal after allocate");
    h->signal = true;
    return ERTGPU_OK;
}

int ertgpu_fetch_signal(ertgpu_handle* h, ertgpu_signal* out, size_t cap, size_t* n_out) {
    if (!h || !h->allocated) return ERTGPU_EINVAL;
    if (!h->signal) return fail(h, ERTGPU_EINVAL, "fetch_signal: the handle was allocated without signal reports (ertgpu_enable_signal)");
    CUDA_TRY(h, cudaSetDevice(h->device));
    if (const int rc = collect(h)) return rc;
    return deliver(h, h->res.sigs, out, cap, n_out, "records");
}

int ertgpu_enable_spectrum(ertgpu_handle* h, int32_t log2_n, int64_t frames_per_row) {
    if (!h) return ERTGPU_EINVAL;
    if (h->allocated) return fail(h, ERTGPU_EINVAL, "enable_spectrum after allocate");
    if (log2_n < ERTSPEC_LOG2_MIN || log2_n > ERTSPEC_LOG2_MAX)
        return fail(h, ERTGPU_EINVAL, "spectrum frames of 2^%d samples: log2_n must be within %d ... %d", log2_n, ERTSPEC_LOG2_MIN, ERTSPEC_LOG2_MAX);
    if (frames_per_row < 1 || frames_per_row > (1ll << 40) || (frames_per_row << log2_n) < ERTSPEC_ROW_MIN_SAMPLES)
        return fail(h, ERTGPU_EINVAL, "spectrum rows of %lld frames of 2^%d samples: N * frames_per_row must be at least %d",
                    (long long)frames_per_row, log2_n, ERTSPEC_ROW_MIN_SAMPLES);
    h->spec.on = true;
    h->spec.log2n = log2_n;
    h->spec.F = frames_per_row;
    return ERTGPU_OK;
}

int ertgpu_fetch_spectrum(ertgpu_handle* h, int32_t partial, ertgpu_spectrum_row* rows, float* mean, float* peak, size_t cap,
                          size_t* n_out) {
    if (!h || !h->allocated) return ERTGPU_EINVAL;
    Spectrum& sp = h->spec;
    if (!sp.on) return fail(h, ERTGPU_EINVAL, "fetch_spectrum: the handle was allocated without a spectrum (ertgpu_enable_spectrum)");
    CUDA_TRY(h, cudaSetDevice(h->device));
    if (const int rc = collect_sync(h)) return rc;
    const int64_t first = sp.pos.rows_fetched, done = sp.rows_done();
    const bool open = partial && sp.frames() % sp.F != 0;
    const size_t need = (size_t)(done - first) + (open ? 1 : 0);
    if (n_out) *n_out = need;
    if (need > cap) return fail(h, ERTGPU_ECAPACITY, "output arrays hold %zu rows, %zu needed", cap, need);
    if (need && (!rows || !mean || !peak)) return fail(h, ERTGPU_EINVAL, "null output array");
    const size_t N = (size_t)sp.N;
    for (int64_t r = first; r < done; r++) {
        const size_t i = (size_t)(r - first), slot = (size_t)(r % sp.row_cap);
        CUDA_TRY(h, cudaMemcpy(mean + i * N, sp.dev.mean + slot * N, N * sizeof(float), cudaMemcpyDeviceToHost));
        CUDA_TRY(h, cudaMemcpy(peak + i * N, sp.dev.peak + slot * N, N * sizeof(float), cudaMemcpyDeviceToHost));
        rows[i].first_sample = r * sp.F * sp.N;
        rows[i].frames = sp.F;
    }
    if (open) {
        const size_t i = (size_t)(done - first);
        int64_t frames = 0;
        if (const int rc = sp.open_row(h->err, mean + i * N, peak + i * N, &frames)) return rc;
        rows[i].first_sample = done * sp.F * sp.N;
        rows[i].frames = frames;
    }
    sp.pos.rows_fetched = done;
    return ERTGPU_OK;
}

int ertgpu_last_counts(ertgpu_handle* h, int64_t* n_candidates, int64_t* n_valid) {
    if (!h || !h->allocated) return ERTGPU_EINVAL;
    if (h->fly.stream) {
        CUDA_TRY(h, cudaSetDevice(h->device));
        int rc = collect_sync(h);  // counters only; ertgpu_fetch copies the candidates if wanted
        if (rc) return rc;
    }
    if (n_candidates) *n_candidates = h->res.hits;
    if (n_valid) *n_valid = h->res.valid;
    return ERTGPU_OK;
}

int64_t ertgpu_last_launches(const ertgpu_handle* h) { return h ? h->launches : 0; }

int ertgpu_tap(ertgpu_handle* h, int32_t which, int64_t block, void* dst, size_t cap, size_t* n_out) {
    if (!h || !h->allocated) return ERTGPU_EINVAL;
    CUDA_TRY(h, cudaSetDevice(h->device));
    if (h->fly.stream) {
        int rc = collect(h);
        if (rc) return rc;
    }
    const LastPipeline& l = h->last;
    if (!l.plane) return fail(h, ERTGPU_EINVAL, "no decode call yet");
    const DevCfg& c = h->dcfg;
    const int64_t b = block - l.first_block;
    if (b < 0 || b >= l.nblocks) return fail(h, ERTGPU_EINVAL, "block %lld outside the last (chunk of the) call [%lld,%lld)",
                                             (long long)block, (long long)l.first_block, (long long)(l.first_block + l.nblocks));
    std::vector<uint8_t> bytes;
    if (which == ERTGPU_TAP_SIGNAL || which == ERTGPU_TAP_CSUM) {
        float* sig = h->dev.tap;
        float* cs = h->dev.tap + (c.BS + c.SL);
        tap_signal_csum_kernel<<<1, 32, 0, h->dev.stream>>>(l.iq, l.hist, c.hist_samples, l.hist_valid, h->dev.lut,
                                                        b, c.BS, c.SL, sig, cs);
        CUDA_TRY(h, cudaGetLastError());
        const size_t n = which == ERTGPU_TAP_SIGNAL ? (size_t)(c.BS + c.SL) : (size_t)(c.BS + c.SL + 1);
        bytes.resize(n * sizeof(float));
        CUDA_TRY(h, cudaMemcpyAsync(bytes.data(), which == ERTGPU_TAP_SIGNAL ? sig : cs, bytes.size(), cudaMemcpyDeviceToHost, h->dev.stream));
        CUDA_TRY(h, cudaStreamSynchronize(h->dev.stream));
    } else if (which == ERTGPU_TAP_QUANTIZED || which == ERTGPU_TAP_PACKED) {
        // Quantized after block b = stream bits [(b+1)*BS - BUF, (b+1)*BS)  (decode.go:166,172)
        const long long first_bit = (long long)c.hist_words * 32 + (b + 1) * c.BS - c.BUF;
        const long long w0 = first_bit >> 5, w1 = (first_bit + c.BUF + 31) >> 5;
        std::vector<uint32_t> words((size_t)(w1 - w0));
        CUDA_TRY(h, cudaMemcpy(words.data(), l.plane + w0, words.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
        std::vector<uint8_t> q((size_t)c.BUF);
        for (long long i = 0; i < c.BUF; i++) {
            const long long pos = first_bit + i - (w0 << 5);
            q[(size_t)i] = (uint8_t)((words[(size_t)(pos >> 5)] >> (31 - (pos & 31))) & 1u);
        }
        if (which == ERTGPU_TAP_QUANTIZED) {
            bytes = q;
        } else {  // decode.go:259-265
            bytes.resize((size_t)((c.BS + c.PL + 7) >> 3));
            for (size_t B = 0; B < bytes.size(); B++) {
                uint8_t v = 0;
                for (int k = 0; k < 8; k++) v = (uint8_t)((v << 1) | q[B * 8 + k]);
                bytes[B] = v;
            }
        }
    } else if (which == ERTGPU_TAP_R900_QUANTIZED) {
        float* cs = h->dev.tap;
        uint8_t* qd = reinterpret_cast<uint8_t*>(h->dev.tap + c.BUF + 4);
        tap_r900_csum_kernel<<<1, 32, 0, h->dev.stream>>>(l.iq, l.hist, c.hist_samples, l.hist_valid, h->dev.lut, b,
                                                      c.BS, c.BUF, cs);
        CUDA_TRY(h, cudaGetLastError());
        tap_r900_digits_kernel<<<(c.BUF + 255) / 256, 256, 0, h->dev.stream>>>(cs, c.BUF, c.CL, qd);
        CUDA_TRY(h, cudaGetLastError());
        bytes.resize((size_t)c.BUF);
        CUDA_TRY(h, cudaMemcpyAsync(bytes.data(), qd, bytes.size(), cudaMemcpyDeviceToHost, h->dev.stream));
        CUDA_TRY(h, cudaStreamSynchronize(h->dev.stream));
    } else if (which == ERTGPU_TAP_RESAMPLED) {
        if (h->in.mode == InputStage::kPass) return fail(h, ERTGPU_EINVAL, "the handle neither resamples nor converts its input");
        bytes.resize((size_t)c.BS * 2);
        CUDA_TRY(h, cudaMemcpyAsync(bytes.data(), l.iq + (size_t)b * c.BS * 2, bytes.size(), cudaMemcpyDeviceToHost, h->dev.stream));
        CUDA_TRY(h, cudaStreamSynchronize(h->dev.stream));
    } else {
        return fail(h, ERTGPU_EINVAL, "unknown tap %d", which);
    }
    if (n_out) *n_out = bytes.size();
    if (dst) memcpy(dst, bytes.data(), std::min(cap, bytes.size()));
    return ERTGPU_OK;
}

int ertgpu_set_stage_timing(ertgpu_handle* h, int32_t enable) {
    if (!h || !h->allocated) return ERTGPU_EINVAL;
    CUDA_TRY(h, cudaSetDevice(h->device));
    const int rc = collect_sync(h);
    if (rc) return rc;
    StageTiming& t = h->timing;
    t.on = enable != 0;
    if (enable) {
        for (int k = 0; k < 4; k++) t.sum[k] = 0;
        t.n = 0;
        t.unread = 0;
    }
    return ERTGPU_OK;
}

int ertgpu_last_stage_ms(ertgpu_handle* h, float* ms4) {
    if (!h || !h->allocated || !ms4) return ERTGPU_EINVAL;
    CUDA_TRY(h, cudaSetDevice(h->device));
    const int rc = collect_sync(h);
    if (rc) return rc;
    const StageTiming& t = h->timing;
    if (!t.valid) return fail(h, ERTGPU_EINVAL, "stage timing was not enabled for the last decode");
    for (int k = 0; k < 4; k++) CUDA_TRY(h, cudaEventElapsedTime(&ms4[k], t.sets[t.last][k], t.sets[t.last][k + 1]));
    return ERTGPU_OK;
}

int ertgpu_stage_ms_mean(ertgpu_handle* h, float* ms4, int64_t* n_pipelines) {
    if (!h || !h->allocated || !ms4) return ERTGPU_EINVAL;
    CUDA_TRY(h, cudaSetDevice(h->device));
    const int rc = collect_sync(h);
    if (rc) return rc;
    StageTiming& t = h->timing;
    t.fold();
    for (int k = 0; k < 4; k++) ms4[k] = t.n ? (float)(t.sum[k] / (double)t.n) : 0.0f;
    if (n_pipelines) *n_pipelines = t.n;
    return ERTGPU_OK;
}

// "0-31,64-95" -> cpu_set_t; returns the number of CPUs
static int parse_cpulist(const char* str, cpu_set_t* set) {
    CPU_ZERO(set);
    int n = 0;
    const char* p = str;
    while (*p) {
        char* end = nullptr;
        long a = strtol(p, &end, 10);
        if (end == p) break;
        long b = a;
        p = end;
        if (*p == '-') {
            b = strtol(p + 1, &end, 10);
            if (end == p + 1) break;
            p = end;
        }
        for (long c = a; c <= b && c < CPU_SETSIZE; c++)
            if (c >= 0 && !CPU_ISSET((int)c, set)) { CPU_SET((int)c, set); n++; }
        while (*p == ',' || *p == ' ' || *p == '\n') p++;
    }
    return n;
}

int ertgpu_bind_host_thread(int32_t device, int32_t* ncpus, int32_t* numa_node) {
    if (ncpus) *ncpus = 0;
    if (numa_node) *numa_node = -1;
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) {
        cudaGetLastError();
        return ERTGPU_ECUDA;
    }
    for (char* c = bus; *c; c++) *c = (char)tolower((unsigned char)*c);
    char path[128], buf[4096] = {0};
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
    if (FILE* f = fopen(path, "r")) {
        int node = -1;
        if (fscanf(f, "%d", &node) == 1 && numa_node) *numa_node = node;
        fclose(f);
    }
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/local_cpulist", bus);
    FILE* f = fopen(path, "r");
    if (!f) return ERTGPU_EINVAL;
    const size_t got = fread(buf, 1, sizeof(buf) - 1, f);
    fclose(f);
    buf[got] = 0;
    cpu_set_t want, allowed, both;
    if (parse_cpulist(buf, &want) <= 0) return ERTGPU_EINVAL;
    if (sched_getaffinity(0, sizeof(allowed), &allowed) != 0) return ERTGPU_EINVAL;
    CPU_AND(&both, &want, &allowed);
    const int n = CPU_COUNT(&both);
    if (n <= 0) return ERTGPU_EINVAL;          // the GPU's CPUs are outside this process's cpuset: leave it alone
    if (sched_setaffinity(0, sizeof(both), &both) != 0) return ERTGPU_EINVAL;
    if (ncpus) *ncpus = n;
    return ERTGPU_OK;
}

const char* ertgpu_last_kernels(const ertgpu_handle* h) { return h ? h->kernels.c_str() : ""; }

int ertgpu_host_alloc(void** out, size_t nbytes) {
    if (!out) return ERTGPU_EINVAL;
    cudaError_t e = cudaHostAlloc(out, nbytes, cudaHostAllocDefault);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return e == cudaErrorMemoryAllocation ? ERTGPU_ENOMEM : ERTGPU_ECUDA;
    }
    return ERTGPU_OK;
}

int ertgpu_host_free(void* p) {
    if (!p) return ERTGPU_OK;
    return cudaFreeHost(p) == cudaSuccess ? ERTGPU_OK : ERTGPU_ECUDA;
}

int ertgpu_synth_fill(int32_t device, void* d_out, int64_t first_sample, int64_t nsamples, uint64_t seed,
                      const ertgpu_synth_packet* packets, int64_t npackets, void* stream) {
    if (!d_out || nsamples < 0 || npackets < 0 || (npackets && !packets)) return ERTGPU_EINVAL;
    if (cudaSetDevice(device) != cudaSuccess) return ERTGPU_ECUDA;
    cudaStream_t st = (cudaStream_t)stream;
    ertgpu_synth_packet* d_pk = nullptr;
    // only the packets that can touch [first_sample, first_sample + nsamples) are uploaded
    int64_t lo = 0, hi = npackets;
    while (lo < npackets && packets[lo].start_sample + (int64_t)packets[lo].n_chips * packets[lo].chip_length <= first_sample) lo++;
    while (hi > lo && packets[hi - 1].start_sample >= first_sample + nsamples) hi--;
    const int64_t n = hi - lo;
    if (cudaMalloc(&d_pk, std::max<int64_t>(n, 1) * sizeof(ertgpu_synth_packet)) != cudaSuccess) return ERTGPU_ENOMEM;
    if (n && cudaMemcpyAsync(d_pk, packets + lo, (size_t)n * sizeof(ertgpu_synth_packet), cudaMemcpyHostToDevice, st) != cudaSuccess) {
        cudaFree(d_pk);
        return ERTGPU_ECUDA;
    }
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    long long groups = (nsamples + 7) / 8;
    long long blocks = std::min<long long>((groups + 255) / 256, (long long)sms * 32);
    if (blocks < 1) blocks = 1;
    synth_kernel<<<(unsigned)blocks, 256, 0, st>>>(static_cast<uint8_t*>(d_out), first_sample, nsamples, seed, d_pk, n);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    cudaFree(d_pk);
    return e == cudaSuccess ? ERTGPU_OK : ERTGPU_ECUDA;
}

}  // extern "C"
