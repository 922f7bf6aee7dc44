// receiver.hpp -- SURVEY.md section 8(f1): file/stream ingest in place of rtl_tcp, plus the receive loop's
// cross-block message dedup.  Mirrors the parts of rtlamr's main.go Receiver that sit around
// protocol.Decoder.Decode:
//   * the block reader (main.go:156-205) -- here it reads K*BlockSize2 bytes per iteration from a file or
//     stdin into pinned host buffers (ertgpu_host_alloc) instead of one block from a TCP socket;
//   * the decode loop (main.go:207-294) -- Decode, then the prev/next digest maps that drop a message
//     already reported for the previous block (main.go:244-260,292), the -samplefile dump of the last blocks
//     (main.go:225-230,279-284), -single (main.go:269-287) and -duration (main.go:350-353).
// Whole blocks only: a trailing partial block is never decoded (main.go:166-186).  Input of another sample format
// (cs8, cs16, cf32) is read in whole samples of its own size and converted on the GPU.
#pragma once

#include <chrono>
#include <cstdio>
#include <functional>
#include <memory>
#include <set>
#include <string>
#include <tuple>
#include <vector>

#include "filters.hpp"
#include "protocol.hpp"

namespace receiver {

// protocol.Digest (parse.go:87-101)
using Digest = std::tuple<std::string, uint8_t, uint32_t, std::vector<uint8_t>>;
Digest NewDigest(const protocol::Message& m);

struct Stats {
    int64_t blocks = 0, bytes = 0, samples = 0, messages = 0, duplicates = 0, filtered = 0;   // bytes, samples: input
    std::vector<int64_t> channel_messages;   // messages reported per channel (Receiver::Run)
    double seconds = 0;
    bool stopped = false;  // -single or -duration ended the run: nothing after it is read
};

// Go duration syntax (time.ParseDuration: "500ms", "1h5m10s", "-1.5h", "0") in nanoseconds; throws invalid_argument.
int64_t ParseDuration(const std::string& s);

// The receive loop's prev/next digest maps (main.go:221-224,244-260,292) on their own: a message whose digest was
// reported for the previous block is dropped; a gap in the block numbers empties the memory.  Across the channels of
// one capture (FilterChannels) a message is also dropped when an earlier channel reported its digest for the same
// block, and "the previous block" means any channel's: one channel is exactly the rule above.
class BlockDedup {
public:
    // msgs grouped by ascending Block (what Decode returns); `emit` sees every message that is reported.  `fc` is the
    // receive loop's filter chain (main.go:236-239): a message it rejects is skipped BEFORE its digest is recorded.
    void Filter(std::vector<protocol::MessagePtr>& msgs, bool block_dedup,
                const std::function<void(const protocol::Message&)>& emit, Stats& st, FilterChain* fc = nullptr);
    // The same for the n messages of ONE block.  `emit` returns false to drop the rest of the block (-single's `break`,
    // main.go:275-277); FilterBlock then returns false too.
    bool FilterBlock(protocol::MessagePtr* msgs, size_t n, bool block_dedup,
                     const std::function<bool(const protocol::Message&)>& emit, Stats& st, FilterChain* fc = nullptr);
    // The same for ONE block's messages of nch channels, channel c's n[c] messages at msgs[c], in the order the channels
    // were given; `emit` also sees the channel.
    bool FilterChannels(protocol::MessagePtr* const* msgs, const size_t* n, size_t nch, bool block_dedup,
                        const std::function<bool(const protocol::Message&, size_t)>& emit, Stats& st, FilterChain* fc = nullptr);
    void Reset() {
        prev_.clear();
        prev_block_ = -2;
    }

private:
    std::set<Digest> prev_;
    int64_t prev_block_ = -2;
};

// The next block with a message in any of the channels' Decode results per[c] (each grouped by ascending Block), from
// the cursors pos[c]: its number goes to *block and its messages of channel c to at[c] .. at[c] + n[c], and the cursors
// move past it.  False when every channel is done.
bool NextBlock(std::vector<std::vector<protocol::MessagePtr>>& per, std::vector<size_t>& pos,
               std::vector<protocol::MessagePtr*>& at, std::vector<size_t>& n, int64_t* block);

class Receiver {
public:
    // msgtypes: comma list as for -msgtype ("all" = scm,scm+,idm,r900, main.go:67-73)
    // input: the capture's rate, format and tuning (protocol::Decoder::SetInput); when it is resampled, blocks, dedup
    // and filters work on the resampled stream.
    // channels: the centre frequencies of several channels of one tuned capture (input.CenterFreq is then not read),
    // decoded in one pass with one protocol::Decoder each: Run reads every chunk once and reports ascending blocks,
    // channel by channel in this order, through the cross-channel dedup (BlockDedup::FilterChannels).
    Receiver(const std::string& msgtypes, int chipLength, int device, int64_t blocksPerCall, const protocol::Input& input,
             const std::vector<int64_t>& channels = {});
    ~Receiver();

    protocol::Decoder& decoder(size_t channel = 0) { return *d_[channel]; }
    size_t channels() const { return d_.size(); }
    FilterChain& filters() { return fc_; }   // -filterid / -filtertype / -unique (flags.go:147-170)

    // -samplefile (main.go:225-230,279-284): after every block with at least one reported message, the receive loop's
    // sampleBuf -- the last blocks of the stream, one dropped from the front before a block is appended once it holds
    // more than BufferLength<<1 bytes -- is appended to `f`.  Every message of that block carries Offset = the file's
    // size before the dump and Length = sampleBuf's size.  The file is shared by all streams of a batch.
    void SetSampleFile(FILE* f) { sample_file_ = f; }
    // -single (main.go:269-287).  ids == nullptr (no -filterid): stop after the first reported message.  Otherwise each
    // reported meter ID is erased from `ids` -- the set the chain's MeterIDFilter reads -- and the run stops at the end of
    // the block that empties it.
    void SetSingle(UintMap* ids) {
        single_ = true;
        single_ids_ = ids;
    }
    // -duration: checked before every read, so a call already read is decoded and reported in full.
    void SetDeadline(std::chrono::steady_clock::time_point t) { deadline_ = t; }
    // Input::AutoScale: `report` sees each stream's level and gain once it is measured, before the stream is decoded.
    void SetLevelReport(std::function<void(const ertgpu_input_level&)> report) { level_report_ = std::move(report); }
    // The level measured at the start of the last stream (Input::AutoScale; all zero otherwise).
    const ertgpu_input_level& Level() const { return level_; }
    // Input::AutoChannelGain: `report` sees each channel's level and k once they are measured, before the stream is
    // decoded (after the input gain of Input::AutoScale is set).
    void SetChannelLevelReport(std::function<void(size_t, const ertgpu_channel_level&)> report) {
        channel_report_ = std::move(report);
    }

    // Run over a FILE* until EOF, -single or the deadline.  With Input::AutoScale the stream's gain is set from its first
    // min(stream, ERTLV_WINDOW) samples (include/ertgpu_level.h) before anything is decoded; it stays for the stream.  `emit` is called once per reported message (after the
    // cross-block dedup when block_dedup) with its LogMessage Offset and Length (0 without a sample file).  max_bytes >= 0
    // stops reading after that many bytes (the data chunk of a WAV file).  With a spectrum (Input::SpectrumLog2; with
    // several channels, channel 0's handle measures the capture once) `rows` sees the rows each decode call completed,
    // after the call, and at the end of the stream the open row when it has at least one frame.
    Stats Run(FILE* in, bool block_dedup, const std::function<void(const protocol::Message&, int64_t, int)>& emit,
              int64_t max_bytes = -1, const std::function<void(const protocol::SpectrumRows&)>& rows = {});

    // Start a new, independent stream (the next file of a batch): zeroed Decoder history (decode.go:144-145),
    // block numbers restart at 0, empty dedup set, empty sampleBuf.
    void Reset();

    // The dedup step on one Decode result (messages grouped by ascending Block), exposed for tests.
    void Filter(std::vector<protocol::MessagePtr>& msgs, bool block_dedup,
                const std::function<void(const protocol::Message&)>& emit, Stats& st);

private:
    std::vector<std::unique_ptr<protocol::Decoder>> d_;   // one per channel
    int64_t blocks_per_call_;
    uint8_t* buf_[2] = {nullptr, nullptr};
    size_t buf_bytes_ = 0;
    BlockDedup dedup_;
    FilterChain fc_;

    FILE* sample_file_ = nullptr;
    int64_t sample_offset_ = 0;       // bytes written to sample_file_
    int64_t sample_blocks_ = 0;       // how many blocks sampleBuf holds once full
    int64_t stream_blocks_ = 0;       // blocks decoded since Reset
    std::vector<uint8_t> history_;    // the stream's last (sample_blocks_ - 1) blocks before the current call
    bool single_ = false;
    UintMap* single_ids_ = nullptr;
    std::chrono::steady_clock::time_point deadline_ = std::chrono::steady_clock::time_point::max();
    std::function<void(const ertgpu_input_level&)> level_report_;
    ertgpu_input_level level_{};
    std::function<void(size_t, const ertgpu_channel_level&)> channel_report_;

    void DumpSampleBuf(const uint8_t* call, int64_t call_first, int64_t block);
    void KeepHistory(const uint8_t* call, size_t nblocks);
};

}  // namespace receiver
