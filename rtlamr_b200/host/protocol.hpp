// protocol.hpp -- host side above the C ABI: a C++ mirror of rtlamr's `protocol` package surface
// for the Decoder hot path (reference protocol/decode.go, protocol/parse.go) and of the per-message
// parsers that consume its output (scm/, scmplus/, idm/, netidm/, r900/, r900bcd/).
//
// The reference is Go and no Go toolchain exists in this image, so this mirror stands in for the
// cgo shim (go/protocol/decode_cuda.go, shown in INTEGRATION.md) in the parity tests: same names,
// same argument meaning, same error behaviour.  All DSP runs in libertgpu.so (CUDA); the parsers
// below are the reference's pure byte-level logic (CRC re-check, field extraction) and never
// touch a sample.
//
// Differences forced by the language, not by design:
//   * Parse returns messages through a std::vector instead of a Go channel + WaitGroup
//     (parse.go:72-76); message order inside a block is unspecified in the reference
//     (map iteration + goroutines, decode.go:177-187), here it is registration order.
//   * Decode accepts N*BlockSize2 bytes and is equivalent to N sequential reference Decode calls.
#pragma once

#include <array>
#include <cstdint>
#include <functional>
#include <map>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/ertgpu.h"

namespace crc {  // reference crc/crc.go

using Table = std::array<uint16_t, 256>;
Table NewTable(uint16_t poly);                                                   // crc.go:34-47
uint16_t Checksum(uint16_t init, const uint8_t* data, size_t n, const Table& t); // crc.go:49-55

struct CRC {  // crc.go:7-14
    std::string Name;
    uint16_t Init = 0, Poly = 0, Residue = 0;
    Table tbl{};
    uint16_t Checksum(const uint8_t* data, size_t n) const { return crc::Checksum(Init, data, n, tbl); }  // crc.go:28-30
    std::string String() const;                                                                         // crc.go:24-26
};
CRC NewCRC(const std::string& name, uint16_t init, uint16_t poly, uint16_t residue);  // crc.go:16-22

}  // namespace crc

namespace gf {  // reference r900/gf/gf.go, NewField(32, 37, 2) only

struct Field {
    std::array<uint8_t, 62> exp{};
    std::array<uint8_t, 32> log{};
    Field();                                                                            // gf.go:20-57
    uint8_t Mul(uint8_t x, uint8_t y) const;                                            // gf.go:143-148
    std::vector<uint8_t> Syndrome(const uint8_t* message, int n, int parity, int offset) const;  // gf.go:152-172
};

}  // namespace gf

namespace protocol {

// decode.go:27-42
struct PacketConfig {
    std::string Protocol, Preamble;
    int DataRate = 0;
    int BlockSize = 0, BlockSize2 = 0;
    int ChipLength = 0, SymbolLength = 0;
    int SampleRate = 0;
    int PreambleSymbols = 0, PacketSymbols = 0;
    int PreambleLength = 0, PacketLength = 0;
    int BufferLength = 0;
    uint32_t CenterFreq = 0;
};

// parse.go:55-59 plus what the GPU attaches to each candidate
struct Data {
    int Idx = 0;
    std::string Bits;
    std::vector<uint8_t> Bytes;
    int64_t Block = 0;                 // which reference Decode call produced it
    uint32_t CheckMask = 0;            // GPU integrity screens (ertgpu_candidate.check_mask)
    bool HasR900 = false;
    std::array<uint8_t, ERTGPU_R900_DIGITS> R900Digits{};  // r900 quantized[] at the payload positions
};
Data NewData(const uint8_t* data, size_t n);  // parse.go:61-69

// One exported field of a message struct as encoding/json and encoding/xml see it through reflection.
struct Field {
    enum Kind { UINT, BYTES, UINT16S };  // uintN, []byte, [N]uint16
    const char* Name;                    // Go field name; also the JSON key, since no message carries a json tag Go can parse
    const char* XmlAttr;                 // attribute name of an `xml:"..,attr"` tag; nullptr for an untagged field (child element)
    Kind kind;
    uint64_t Uint = 0;
    std::vector<uint8_t> Bytes;
    std::vector<uint16_t> Uint16s;
};

// How a message was received (include/ertgpu_signal.h), from the record of the candidate it was parsed from: the
// channel the decoder was tuned to (its CenterFreq when untuned) and, when the record has one, its summary.
struct SignalReport {
    int64_t Channel = 0;
    bool Valid = false;   // false: the packet starts before the stream, no summary
    int64_t Freq = 0;
    double Level = 0, Noise = 0, SNR = 0;
};

// parse.go:78-84 (csv.Recorder folded in)
struct Message {
    virtual ~Message() = default;
    virtual std::string MsgType() const = 0;
    virtual uint32_t MeterID() const = 0;
    virtual uint8_t MeterType() const = 0;
    virtual std::vector<uint8_t> Checksum() const = 0;
    virtual std::string String() const = 0;
    virtual std::vector<std::string> Record() const = 0;
    virtual std::vector<Field> Fields() const = 0;  // exported fields in Go declaration order (embedded structs flattened)
    int64_t Block = 0;  // bookkeeping for the parity tests (not in the reference)
    int Idx = 0;
    std::optional<SignalReport> Signal;  // set by a Decoder with signal reports (Decoder::EnableSignal)
};
using MessagePtr = std::unique_ptr<Message>;

class Decoder;

// parse.go:72-76
struct Parser {
    virtual ~Parser() = default;
    virtual void Parse(const std::vector<Data>& pkts, std::vector<MessagePtr>& msgCh) = 0;
    virtual void SetDecoder(Decoder*) {}
    virtual PacketConfig Cfg() const = 0;
    // the GPU-side screen equivalent to this parser's own integrity check (ertgpu_protocol.check_*)
    virtual void Screen(ertgpu_protocol& p) const { p.check_kind = ERTGPU_CHECK_NONE; }
};
using ParserPtr = std::shared_ptr<Parser>;
using NewParserFunc = std::function<ParserPtr(int chipLength)>;  // parse.go:21

void RegisterParser(const std::string& name, NewParserFunc fn);  // parse.go:28-39 (throws like Go panics)
ParserPtr NewParser(const std::string& name, int chipLength);    // parse.go:42-51 (throws invalid_argument)

// The IQ fed to Decode (not part of the reference, which decodes uint8 IQ at DataRate*ChipLength only).  Every field's
// default leaves the input as the reference takes it.
// Bytes per IQ sample of an ERTGPU_FORMAT_*.
inline int FormatBytes(int32_t f) {
    switch (f) {
        case ERTGPU_FORMAT_CU8: case ERTGPU_FORMAT_CS8: return 2;
        case ERTGPU_FORMAT_CS16: case ERTGPU_FORMAT_CS16BE: case ERTGPU_FORMAT_CU16: case ERTGPU_FORMAT_CU16BE: return 4;
        case ERTGPU_FORMAT_CF64: case ERTGPU_FORMAT_CF64BE: return 16;
        default: return 8;
    }
}

struct Input {
    int64_t SampleRate = 0;             // Hz; another rate than DataRate*ChipLength is resampled (ertgpu_set_input_rate)
    int32_t Format = ERTGPU_FORMAT_CU8; // converted on the GPU with gain Scale, 0: the format's default (ertgpu_set_input_format)
    float Scale = 0.0f;
    int64_t CaptureFreq = 0, CenterFreq = 0;  // the capture's centre and the channel, 0: Cfg.CenterFreq (ertgpu_set_input_tuning)
    // The gain of each stream is measured from its first samples (ertgpu_measure_input) and set before its first Decode
    // (ertgpu_set_input_scale); Scale is the gain until then.  Not for cu8.  The Decoder only carries the flag: whoever
    // feeds it (receiver::Receiver::Run, erthost_decode) measures and sets the gain.
    bool AutoScale = false;
    // The wide channel path of a tuned input (ertgpu_set_channel_gain) with gain 2^ChannelGain; -1: not taken.  With
    // AutoChannelGain the path is taken and k of each stream is measured from its first samples (ertgpu_measure_channel,
    // after the automatic input gain) and set before its first Decode; as with AutoScale, whoever feeds the Decoder does it.
    int32_t ChannelGain = -1;
    bool AutoChannelGain = false;
    bool Signal = false;  // per-packet signal reports (Decoder::EnableSignal)
    // The input's spectrum in rows of SpectrumFrames frames of 2^SpectrumLog2 samples (Decoder::EnableSpectrum); 0: none.
    int32_t SpectrumLog2 = 0;
    int64_t SpectrumFrames = 0;
};

// Rows of a Decoder's input spectrum (ertgpu_fetch_spectrum): rows[i] with mean and peak [i * N, (i+1) * N) by bin.
struct SpectrumRows {
    int32_t N = 0;
    std::vector<ertgpu_spectrum_row> rows;
    std::vector<float> mean, peak;
};

// decode.go:45-63.  Signal/Quantized are not materialised on the host: the parity taps of the C ABI
// expose them (ertgpu_tap).
class Decoder {
public:
    PacketConfig Cfg;

    Decoder();   // NewDecoder, decode.go:65-71
    ~Decoder();
    Decoder(const Decoder&) = delete;
    Decoder& operator=(const Decoder&) = delete;

    void RegisterProtocol(ParserPtr p);  // decode.go:100-128
    // The IQ fed to Decode, between the last RegisterProtocol and Allocate: sets the tuning when CaptureFreq > 0 or
    // CenterFreq != 0 (and allows decimation, so a tuned capture may be at up to 256 times the decoder's rate), then the
    // rate when SampleRate > 0, then the format when Format != cu8 or Scale != 0.  A bad value
    // throws std::invalid_argument, and so does Allocate when the channel does not fit a capture at the decoder's rate.
    void SetInput(const Input& in);
    int BytesPerSample() const { return sample_bytes_; }
    bool AutoScale() const { return auto_scale_; }
    // ertgpu_measure_input on len bytes of whole IQ samples: their level and the gain its rule picks.
    ertgpu_input_level Measure(const uint8_t* samples, size_t len);
    // ertgpu_set_input_scale: the gain of the stream that starts now (after Allocate or Reset, before Decode).
    void SetScale(float scale);
    bool AutoChannelGain() const { return auto_channel_gain_; }
    // ertgpu_measure_channel on len bytes of whole IQ samples (a wide channel path): the channel's level and k.
    ertgpu_channel_level MeasureChannel(const uint8_t* samples, size_t len);
    // ertgpu_set_channel_gain after Allocate: k of the stream that starts now (after Allocate or Reset, before Decode).
    void SetChannelGain(int32_t k);
    // ertgpu_enable_signal, before Allocate: every message then carries a SignalReport.
    void EnableSignal();
    bool SignalEnabled() const { return signal_; }
    // The channel and rate the summaries of Dispatch use (set by Allocate; for a Decoder that is never allocated).
    void SetSignalChannel(int64_t channel_hz, int64_t rate_out) {
        signal_channel_ = channel_hz;
        signal_rate_ = rate_out;
    }
    // Decode takes multiples of this many bytes: whole IQ samples when resampling, whole blocks otherwise.
    size_t InputQuantum() const { return (size_t)sample_bytes_ * (resampling_ ? 1 : (size_t)Cfg.BlockSize); }
    void Allocate(int device = 0, int64_t maxBlocksPerCall = 0, int64_t maxCandidates = 0);  // decode.go:131-160
    // decode.go:163-197 for N = len/BlockSize2 consecutive blocks; throws std::length_error when len is not a multiple
    // of InputQuantum() (BlockSize2 for uint8 IQ at the decoder's rate: the reference panics with a slice-bounds error,
    // decode.go:222).  When resampling, the blocks are those of the resampled stream.
    std::vector<MessagePtr> Decode(const uint8_t* input, size_t len);
    // Decode on each of ds[0..n), decoders tuned to different channels of one capture (the same protocols, input and
    // stream position), from ONE pass over input (ertgpu_decode_channels): element c is what ds[c]->Decode returns.  A
    // group the C ABI refuses throws std::invalid_argument.
    static std::vector<std::vector<MessagePtr>> DecodeChannels(const std::vector<Decoder*>& ds, const uint8_t* input, size_t len);
    // Whole blocks decoded since Allocate / Reset (resampled blocks with an input rate).
    int64_t BlocksDecoded() const;
    // The second half of Decode (decode.go:177-187 + parse.go): candidates sorted by (block, preamble, idx) are
    // regrouped into per-block, per-preamble []Data and handed to the parsers filed under that preamble.  Needs
    // RegisterProtocol only (no device), so the parsers can be exercised on candidates from any source.
    // sigs: the candidates' signal records (ertgpu_fetch_signal), or nullptr.  Each message then gets the report of the
    // candidate it was parsed from, found by (block, preamble, idx).
    void Dispatch(const ertgpu_candidate* cands, size_t n, std::vector<MessagePtr>& out, const ertgpu_signal* sigs = nullptr);
    // ertgpu_enable_spectrum, before Allocate.
    void EnableSpectrum(int32_t log2_n, int64_t frames_per_row);
    bool SpectrumEnabled() const { return spectrum_n_ != 0; }
    // ertgpu_fetch_spectrum: the rows completed since the last fetch and, with partial, the open row (not consumed).
    SpectrumRows FetchSpectrum(bool partial = false);
    std::string Log() const;  // decode.go:73-90
    void Reset();
    ertgpu_handle* Handle() const { return h_; }

private:
    ertgpu_handle* h_ = nullptr;
    std::vector<ParserPtr> parsers_;            // registration order
    std::vector<std::string> preambles_;        // distinct, registration order
    std::vector<std::vector<size_t>> by_pre_;   // parser indices per preamble (decode.go:124)
    std::vector<ertgpu_candidate> cands_;
    std::vector<ertgpu_signal> sigs_;
    bool signal_ = false;
    int32_t spectrum_n_ = 0;
    int64_t signal_channel_ = 0, signal_rate_ = 0;
    const ertgpu_signal* FetchSignal(size_t n);   // the last call's records (nullptr without reports)
    bool allocated_ = false;
    bool resampling_ = false;
    ertgpu_resampler_info rs_{};
    int64_t input_samples_ = 0;  // since Allocate / Reset
    int sample_bytes_ = 2;       // bytes per input IQ sample
    bool auto_scale_ = false;
    bool auto_channel_gain_ = false;
};

void RegisterStockParsers();  // the effect of the reference's blank imports (main.go:37-44)

}  // namespace protocol
