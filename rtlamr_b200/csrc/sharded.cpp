// sharded.cpp -- one IQ stream over several handles / GPUs (include/ertgpu.h, "one stream over several GPUs").
//
// The reference decodes on one goroutine (main.go:207-235); its only state between Decode calls is the Signal
// tail (decode.go:165) and the Quantized history (decode.go:166).  A shard that is fed ceil(PKL/BS)+1 blocks
// before its first owned block therefore reproduces every owned block's candidates exactly (SURVEY.md section
// 2.1 "global view", section 8e), and the shards need no exchange step: no collective, only a host-side concat.
// Written against the public C ABI only (each shard is an ordinary ertgpu_decode on its own handle/device from
// its own host thread), so it is the same code path a Go program with one Decoder per GPU would drive.
#include <algorithm>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "../../include/ertgpu.h"

// ertgpu.cu: ERTGPU_EINVAL, with the message on h, when h has signal reports (sharded decodes do not keep them).  Hidden:
// not exported from libertgpu.so.
__attribute__((visibility("hidden"))) int sharded_reject_signal(ertgpu_handle* h);

extern "C" {

int ertgpu_plan_shards(int64_t total_blocks, int32_t nshards, int32_t block_size, int32_t packet_length,
                       ertgpu_shard* out) {
    if (!out || nshards < 1 || total_blocks < 0 || block_size < 1 || packet_length < 0) return ERTGPU_EINVAL;
    // Quantized history of the first owned block (ceil(PKL/BS) blocks) + one block of real Signal lead-in
    const int64_t halo = (packet_length + (int64_t)block_size - 1) / block_size + 1;
    const int64_t base = total_blocks / nshards, rem = total_blocks % nshards;
    int64_t lo = 0;
    for (int32_t r = 0; r < nshards; r++) {
        const int64_t hi = lo + base + (r < rem ? 1 : 0);
        out[r].first_block = lo;
        out[r].last_block = hi;
        out[r].first_fed_block = std::max<int64_t>(0, lo - halo);
        lo = hi;
    }
    return ERTGPU_OK;
}

int ertgpu_decode_sharded(ertgpu_handle* const* handles, int32_t nhandles, const uint8_t* iq, size_t nbytes,
                          uint32_t flags, ertgpu_candidate* out, size_t cap, size_t* n_out) {
    if (n_out) *n_out = 0;
    if (!handles || nhandles < 1 || (!iq && nbytes)) return ERTGPU_EINVAL;
    for (int32_t r = 0; r < nhandles; r++)
        if (!handles[r]) return ERTGPU_EINVAL;
    for (int32_t r = 0; r < nhandles; r++) {  // shards are cut at decoder blocks of uint8 input: no resampling or converting handles
        ertgpu_resampler_info ri;
        if (ertgpu_get_resampler(handles[r], &ri, nullptr, 0, nullptr) == ERTGPU_OK) return ERTGPU_EINVAL;
        if (ertgpu_get_tuning(handles[r], nullptr) == ERTGPU_OK) return ERTGPU_EINVAL;  // tuned, even at the native rate
        int32_t fmt = ERTGPU_FORMAT_CU8;
        if (ertgpu_get_input_format(handles[r], &fmt, nullptr) != ERTGPU_OK || fmt != ERTGPU_FORMAT_CU8) return ERTGPU_EINVAL;
        if (const int rc = sharded_reject_signal(handles[r])) return rc;
    }
    ertgpu_decoder_config c0;
    int rc = ertgpu_get_config(handles[0], &c0);
    if (rc) return rc;
    for (int32_t r = 1; r < nhandles; r++) {
        ertgpu_decoder_config c;
        rc = ertgpu_get_config(handles[r], &c);
        if (rc) return rc;
        if (memcmp(&c, &c0, sizeof(c)) != 0) return ERTGPU_EINVAL;  // every shard must run the same Decoder
    }
    const size_t bs2 = (size_t)c0.block_size2;
    if (nbytes % bs2) return ERTGPU_ESIZE;
    const int64_t total_blocks = (int64_t)(nbytes / bs2);
    std::vector<ertgpu_shard> plan((size_t)nhandles);
    rc = ertgpu_plan_shards(total_blocks, nhandles, c0.block_size, c0.packet_length, plan.data());
    if (rc) return rc;

    struct Part {
        std::vector<ertgpu_candidate> cands;
        int rc = ERTGPU_OK;
    };
    std::vector<Part> parts((size_t)nhandles);
    auto work = [&](int32_t r) {
        Part& p = parts[(size_t)r];
        const ertgpu_shard& s = plan[(size_t)r];
        ertgpu_handle* h = handles[r];
        if ((p.rc = ertgpu_reset(h)) != ERTGPU_OK) return;
        const int64_t fed = s.last_block - s.first_fed_block;
        if (s.last_block == s.first_block) return;  // nothing owned (more handles than blocks)
        const uint8_t* src = iq + (size_t)s.first_fed_block * bs2;
        size_t n = 0;
        p.cands.resize(4096);
        p.rc = ertgpu_decode(h, src, (size_t)fed * bs2, flags, p.cands.data(), p.cands.size(), &n);
        if (p.rc == ERTGPU_ECAPACITY && n > p.cands.size()) {
            p.cands.resize(n);
            p.rc = ertgpu_fetch(h, p.cands.data(), p.cands.size(), &n);
        }
        if (p.rc != ERTGPU_OK) return;
        // drop the halo's candidates, renumber the rest (the handle counted blocks from its first fed block)
        const int64_t halo = s.first_block - s.first_fed_block;
        size_t w = 0;
        for (size_t i = 0; i < n; i++) {
            if (p.cands[i].block < halo) continue;
            p.cands[w] = p.cands[i];
            p.cands[w].block += s.first_fed_block;
            w++;
        }
        p.cands.resize(w);
    };
    std::vector<std::thread> th;
    for (int32_t r = 1; r < nhandles; r++) th.emplace_back(work, r);
    work(0);
    for (auto& t : th) t.join();
    for (int32_t r = 0; r < nhandles; r++)
        if (parts[(size_t)r].rc != ERTGPU_OK) return parts[(size_t)r].rc;  // ertgpu_last_error(handles[r]) has the message
    size_t total = 0;
    for (auto& p : parts) total += p.cands.size();
    if (n_out) *n_out = total;
    if (total > cap) return ERTGPU_ECAPACITY;
    // shards own ascending disjoint block ranges and each list is sorted: concatenation is the global order
    size_t off = 0;
    for (auto& p : parts) {
        if (!p.cands.empty() && out) memcpy(out + off, p.cands.data(), p.cands.size() * sizeof(ertgpu_candidate));
        off += p.cands.size();
    }
    return ERTGPU_OK;
}

}  // extern "C"
