// receiver.cpp -- see receiver.hpp.
#include "receiver.hpp"

#include <algorithm>
#include <cctype>
#include <climits>
#include <iterator>
#include <cerrno>
#include <chrono>
#include <cstdint>
#include <cstring>
#include <sstream>
#include <stdexcept>

#include "../../include/ertgpu_level.h"

namespace receiver {

Digest NewDigest(const protocol::Message& m) { return Digest(m.MsgType(), m.MeterType(), m.MeterID(), m.Checksum()); }

Receiver::Receiver(const std::string& msgtypes, int chipLength, int device, int64_t blocksPerCall,
                   const protocol::Input& input, const std::vector<int64_t>& channels) {
    protocol::RegisterStockParsers();
    if (blocksPerCall <= 0) blocksPerCall = 4096;
    blocks_per_call_ = blocksPerCall;
    for (size_t c = 0; c < std::max<size_t>(1, channels.size()); c++) {
        d_.push_back(std::make_unique<protocol::Decoder>());
        protocol::Decoder& d = *d_.back();
        std::string list = msgtypes == "all" ? "scm,scm+,idm,r900" : msgtypes;  // main.go:67-73
        std::stringstream ss(list);
        std::string name;
        while (std::getline(ss, name, ','))
            if (!name.empty()) d.RegisterProtocol(protocol::NewParser(name, chipLength));  // main.go:77-82
        protocol::Input in = input;
        if (!channels.empty()) in.CenterFreq = channels[c];
        if (c > 0) in.SpectrumLog2 = 0;   // one spectrum of the capture, on channel 0
        d.SetInput(in);
        d.Allocate(device, blocksPerCall, 0);  // main.go:86
    }
    const protocol::Decoder& d0 = *d_[0];
    buf_bytes_ = (size_t)blocksPerCall * (size_t)d0.Cfg.BlockSize * (size_t)d0.BytesPerSample();
    for (int k = 0; k < 2; k++) {
        void* p = nullptr;
        if (ertgpu_host_alloc(&p, buf_bytes_) != ERTGPU_OK) {
            for (int j = 0; j < k; j++) {   // a constructor that throws runs no destructor: give back what it got
                ertgpu_host_free(buf_[j]);
                buf_[j] = nullptr;
            }
            throw std::runtime_error("pinned host allocation failed");
        }
        buf_[k] = static_cast<uint8_t*>(p);
    }
}

Receiver::~Receiver() {
    for (int k = 0; k < 2; k++) ertgpu_host_free(buf_[k]);
}

void Receiver::Filter(std::vector<protocol::MessagePtr>& msgs, bool block_dedup,
                      const std::function<void(const protocol::Message&)>& emit, Stats& st) {
    dedup_.Filter(msgs, block_dedup, emit, st, fc_.empty() ? nullptr : &fc_);
}

void BlockDedup::Filter(std::vector<protocol::MessagePtr>& msgs, bool block_dedup,
                        const std::function<void(const protocol::Message&)>& emit, Stats& st, FilterChain* fc) {
    size_t i = 0;
    while (i < msgs.size()) {
        size_t j = i;
        while (j < msgs.size() && msgs[j]->Block == msgs[i]->Block) j++;
        FilterBlock(msgs.data() + i, j - i, block_dedup, [&](const protocol::Message& m) { emit(m); return true; }, st, fc);
        i = j;
    }
}

bool BlockDedup::FilterBlock(protocol::MessagePtr* msgs, size_t n, bool block_dedup,
                             const std::function<bool(const protocol::Message&)>& emit, Stats& st, FilterChain* fc) {
    return FilterChannels(&msgs, &n, 1, block_dedup, [&](const protocol::Message& m, size_t) { return emit(m); }, st, fc);
}

bool BlockDedup::FilterChannels(protocol::MessagePtr* const* msgs, const size_t* n, size_t nch, bool block_dedup,
                                const std::function<bool(const protocol::Message&, size_t)>& emit, Stats& st, FilterChain* fc) {
    // main.go:221-224,244-260,292: `next` collects the digests of the current block, a message whose digest
    // was seen in the previous block is skipped, and the maps swap after every block -- including blocks
    // without messages, which is why a gap in the block numbers empties `prev`.  `earlier`: the digests the channels
    // before this one recorded for the block.
    size_t c0 = 0;
    while (c0 < nch && !n[c0]) c0++;
    if (c0 == nch) return true;
    const int64_t b = msgs[c0][0]->Block;
    if (b != prev_block_ + 1) prev_.clear();
    std::set<Digest> next, earlier;
    bool go_on = true;
    for (size_t c = c0; c < nch && go_on; c++) {
        if (c > c0) earlier = next;
        for (size_t i = 0; i < n[c] && go_on; i++) {
            const protocol::Message& m = *msgs[c][i];
            if (fc && !fc->Match(m)) {   // main.go:236-239: rejected before the digest is recorded
                st.filtered++;
                continue;
            }
            Digest dg = NewDigest(m);
            next.insert(dg);
            if (block_dedup && (prev_.count(dg) || earlier.count(dg))) {
                st.duplicates++;
                continue;
            }
            st.messages++;
            go_on = emit(m, c);
        }
    }
    prev_.swap(next);
    prev_block_ = b;
    return go_on;
}

bool NextBlock(std::vector<std::vector<protocol::MessagePtr>>& per, std::vector<size_t>& pos,
               std::vector<protocol::MessagePtr*>& at, std::vector<size_t>& n, int64_t* block) {
    int64_t b = INT64_MAX;
    for (size_t c = 0; c < per.size(); c++)
        if (pos[c] < per[c].size()) b = std::min(b, per[c][pos[c]]->Block);
    if (b == INT64_MAX) return false;
    at.resize(per.size());
    n.resize(per.size());
    for (size_t c = 0; c < per.size(); c++) {
        size_t j = pos[c];
        while (j < per[c].size() && per[c][j]->Block == b) j++;
        at[c] = per[c].data() + pos[c];
        n[c] = j - pos[c];
        pos[c] = j;
    }
    *block = b;
    return true;
}

int64_t ParseDuration(const std::string& str) {   // time.ParseDuration
    const auto bad = [&] { return std::invalid_argument("time: invalid duration \"" + str + "\""); };
    std::string s = str;
    bool neg = false;
    if (!s.empty() && (s[0] == '-' || s[0] == '+')) {
        neg = s[0] == '-';
        s = s.substr(1);
    }
    if (s == "0") return 0;
    if (s.empty()) throw bad();
    static const std::pair<const char*, double> units[] = {{"ns", 1}, {"us", 1e3}, {"\xC2\xB5s", 1e3}, {"\xCE\xBCs", 1e3},
                                                           {"ms", 1e6}, {"s", 1e9}, {"m", 60e9}, {"h", 3600e9}};
    double total = 0;
    size_t i = 0;
    while (i < s.size()) {
        const size_t num0 = i;
        while (i < s.size() && isdigit((unsigned char)s[i])) i++;
        const size_t int_digits = i - num0;
        size_t frac_digits = 0;
        if (i < s.size() && s[i] == '.') {
            i++;
            const size_t f0 = i;
            while (i < s.size() && isdigit((unsigned char)s[i])) i++;
            frac_digits = i - f0;
        }
        if (!int_digits && !frac_digits) throw bad();
        const double v = std::stod("0" + s.substr(num0, i - num0));
        const size_t u0 = i;
        while (i < s.size() && s[i] != '.' && !isdigit((unsigned char)s[i])) i++;
        const std::string unit = s.substr(u0, i - u0);
        double scale = 0;
        for (const auto& un : units)
            if (unit == un.first) scale = un.second;
        if (!scale) throw std::invalid_argument(unit.empty() ? "time: missing unit in duration \"" + str + "\""
                                                             : "time: unknown unit \"" + unit + "\" in duration \"" + str + "\"");
        total += v * scale;
    }
    if (total > 9.223372036854775807e18) throw bad();
    return neg ? -(int64_t)total : (int64_t)total;
}

void Receiver::Reset() {
    for (auto& d : d_) d->Reset();
    dedup_.Reset();
    stream_blocks_ = 0;
    history_.clear();
}

// Append block `block`'s sampleBuf to the sample file: blocks [block - sample_blocks_ + 1, block] of the stream,
// clipped at its start.  Blocks from call_first on are in `call`, the earlier ones at the end of history_.
void Receiver::DumpSampleBuf(const uint8_t* call, int64_t call_first, int64_t block) {
    const size_t bs2 = (size_t)d_[0]->Cfg.BlockSize2;
    const int64_t first = std::max<int64_t>(0, block - sample_blocks_ + 1);
    const int64_t hist_first = call_first - (int64_t)(history_.size() / bs2);
    if (first < hist_first) throw std::logic_error("sample history lost a block");
    size_t wrote = 0, want = (size_t)(block + 1 - first) * bs2;
    if (first < call_first) {
        const size_t from = (size_t)(first - hist_first) * bs2;
        wrote += fwrite(history_.data() + from, 1, history_.size() - from, sample_file_);
    }
    const int64_t in_call = std::max(first, call_first);
    wrote += fwrite(call + (size_t)(in_call - call_first) * bs2, 1, (size_t)(block + 1 - in_call) * bs2, sample_file_);
    if (wrote != want) throw std::runtime_error(std::string("writing the sample file: ") + strerror(errno));
    sample_offset_ += (int64_t)wrote;
}

// After a call: keep the stream's last (sample_blocks_ - 1) blocks, the part of a later block's sampleBuf that the
// next call's buffer does not hold.
void Receiver::KeepHistory(const uint8_t* call, size_t nblocks) {
    const size_t bs2 = (size_t)d_[0]->Cfg.BlockSize2;
    const size_t keep = (size_t)(sample_blocks_ - 1) * bs2, n = nblocks * bs2;
    if (n >= keep) {
        history_.assign(call + n - keep, call + n);
        return;
    }
    history_.insert(history_.end(), call, call + n);
    if (history_.size() > keep) history_.erase(history_.begin(), history_.end() - (ptrdiff_t)keep);
}

Stats Receiver::Run(FILE* in, bool block_dedup, const std::function<void(const protocol::Message&, int64_t, int)>& emit,
                    int64_t max_bytes, const std::function<void(const protocol::SpectrumRows&)>& rows) {
    Stats st;
    protocol::Decoder& d0 = *d_[0];
    st.channel_messages.assign(d_.size(), 0);
    const size_t bs2 = (size_t)d0.Cfg.BlockSize2;
    // bytes per input sample, and per Decode unit: the strictest channel's (whole blocks when one is not resampled, the
    // capture's centre at the decoder's own rate)
    const size_t s = (size_t)d0.BytesPerSample();
    size_t q = 0;
    for (auto& d : d_) q = std::max(q, d->InputQuantum());
    if (q != bs2 && sample_file_) throw std::logic_error("-samplefile with converted or resampled input");
    const bool spectrum = d0.SpectrumEnabled() && rows;
    const auto spectrum_rows = [&](bool partial) {
        if (!spectrum) return;
        const protocol::SpectrumRows r = d0.FetchSpectrum(partial);
        if (!r.rows.empty()) rows(r);
    };
    std::vector<protocol::Decoder*> ds;
    for (auto& d : d_) ds.push_back(d.get());
    uint64_t left = max_bytes < 0 ? UINT64_MAX : (uint64_t)max_bytes;
    // main.go:225-230: sampleBuf grows by one block per block until it holds more than BufferLength<<1 bytes
    sample_blocks_ = 2 * (int64_t)d0.Cfg.BufferLength / (int64_t)bs2 + 1;
    FilterChain* fc = fc_.empty() ? nullptr : &fc_;
    const auto t0 = std::chrono::steady_clock::now();
    // Automatic gain: the stream's first min(stream, ERTLV_WINDOW) samples are read and measured before its first Decode,
    // the gain is set, and then those same bytes are decoded, followed by the rest.  Nothing is read twice (stdin works),
    // and the window does not depend on the size of a Decode call.
    std::vector<uint8_t> window;
    size_t window_pos = 0;
    // The channel gain (Input::AutoChannelGain) is measured per channel from the same window, after the input gain.
    if (d0.AutoScale() || d0.AutoChannelGain()) {
        window.resize((size_t)std::min<uint64_t>((uint64_t)ERTLV_WINDOW * s, left));
        size_t have = 0;
        while (have < window.size()) {
            const size_t n = fread(window.data() + have, 1, window.size() - have, in);
            if (n == 0) break;
            have += n;
        }
        window.resize(have);
        if (d0.AutoScale()) {   // every channel would pick the gain of the same samples: measured once, set on each
            level_ = d0.Measure(window.data(), have / s * s);
            for (auto& d : d_) d->SetScale(level_.scale);
            if (level_report_) level_report_(level_);
        }
        if (d0.AutoChannelGain())
            for (size_t c = 0; c < d_.size(); c++) {
                const ertgpu_channel_level lv = d_[c]->MeasureChannel(window.data(), have / s * s);
                d_[c]->SetChannelGain(lv.k);
                if (channel_report_) channel_report_(c, lv);
            }
    }
    const auto read = [&](uint8_t* dst, size_t n) -> size_t {
        if (window_pos < window.size()) {
            const size_t m = std::min(n, window.size() - window_pos);
            memcpy(dst, window.data() + window_pos, m);
            window_pos += m;
            return m;
        }
        return fread(dst, 1, n, in);
    };
    // Channels whose resamplers lag differently complete a block in different calls: a block is reported once every
    // channel has completed it (at the end of the stream, whatever is left), so that the channels of one block meet in
    // one FilterChannels.  One channel reports every block of a call in that call.
    std::vector<std::vector<protocol::MessagePtr>> held(d_.size());
    int64_t call_first = 0, b = 0;
    int k = 0;
    const auto report = [&](int64_t ready) {
        std::vector<std::vector<protocol::MessagePtr>> per(held.size());
        for (size_t c = 0; c < held.size(); c++) {
            auto& h = held[c];
            size_t j = 0;
            while (j < h.size() && h[j]->Block < ready) j++;
            per[c].assign(std::make_move_iterator(h.begin()), std::make_move_iterator(h.begin() + (ptrdiff_t)j));
            h.erase(h.begin(), h.begin() + (ptrdiff_t)j);
        }
        std::vector<size_t> pos(per.size(), 0), cnt;
        std::vector<protocol::MessagePtr*> at;
        while (!st.stopped && NextBlock(per, pos, at, cnt, &b)) {
            const int64_t offset = sample_file_ ? sample_offset_ : 0;
            const int length = sample_file_ ? (int)(std::min(b + 1, sample_blocks_) * (int64_t)bs2) : 0;
            bool found = false;
            dedup_.FilterChannels(at.data(), cnt.data(), per.size(), block_dedup, [&](const protocol::Message& m, size_t c) {
                emit(m, offset, length);
                st.channel_messages[c]++;
                found = true;
                if (!single_) return true;
                if (!single_ids_ || single_ids_->empty()) return false;   // main.go:271-276
                single_ids_->erase(m.MeterID());
                return true;
            }, st, fc);
            if (found && sample_file_) DumpSampleBuf(buf_[k], call_first, b);   // main.go:279-284
            if (found && single_ && (!single_ids_ || single_ids_->empty())) st.stopped = true;   // main.go:285-287
        }
    };
    size_t carry = 0;  // bytes of a partial block (a partial IQ sample when resampling) kept for the next buffer
    bool eof = false;
    for (;;) {
        if (std::chrono::steady_clock::now() >= deadline_) {
            report(INT64_MAX);   // what was read before the deadline is reported in full
            st.stopped = true;
            break;
        }
        size_t have = carry;
        while (have < buf_bytes_ && left) {
            const size_t n = read(buf_[k] + have, (size_t)std::min<uint64_t>(buf_bytes_ - have, left));
            if (n == 0) break;
            have += n;
            left -= n;
        }
        eof = have < buf_bytes_;
        const size_t whole = have / q * q;
        if (whole) {
            std::vector<std::vector<protocol::MessagePtr>> per;
            if (d_.size() == 1) per.push_back(d0.Decode(buf_[k], whole));
            else per = protocol::Decoder::DecodeChannels(ds, buf_[k], whole);
            call_first = stream_blocks_;
            const int64_t nblocks = d0.BlocksDecoded() - stream_blocks_;
            st.blocks += nblocks;
            st.bytes += (int64_t)whole;   // input bytes: s per input sample
            st.samples += (int64_t)(whole / s);
            stream_blocks_ += nblocks;
            spectrum_rows(false);
            int64_t ready = INT64_MAX;
            for (size_t c = 0; c < per.size(); c++) {
                for (auto& m : per[c]) held[c].push_back(std::move(m));
                ready = std::min(ready, d_[c]->BlocksDecoded());
            }
            report(ready);
            if (st.stopped) break;
            if (sample_file_) KeepHistory(buf_[k], (size_t)nblocks);
        }
        carry = have - whole;
        if (carry) memcpy(buf_[k ^ 1], buf_[k] + whole, carry);
        k ^= 1;
        if (eof) break;  // EOF: the trailing partial block is dropped like main.go does
    }
    report(INT64_MAX);   // the blocks a lagging channel never completes, or those read before the deadline
    spectrum_rows(true);
    st.seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    return st;
}

}  // namespace receiver
