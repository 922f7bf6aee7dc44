// host_capi.cpp -- a small C surface over the C++ protocol mirror so that the Python parity tests
// (and a CLI) can drive Decoder/Parser exactly like rtlamr's main.go does (main.go:59-86,235).
#include <algorithm>
#include <cerrno>
#include <cstdio>
#include <cstring>
#include <memory>

#include "../../include/ertgpu_level.h"
#include "protocol.hpp"
#include "receiver.hpp"
#include "sigmf.hpp"
#include "wav.hpp"

extern "C" {

struct erthost_msg {
    int64_t block;
    int32_t idx;
    uint32_t meter_id;
    uint32_t meter_type;
    int32_t nchecksum;
    uint8_t checksum[8];
    char msgtype[12];
    char text[1400];    // Message.String()
    char record[1400];  // Message.Record() joined with ','
    int32_t signal;     // 0: no report (the decoder has none), 1: a report without a summary, 2: with one
    int32_t reserved;
    int64_t channel, freq;
    double level, noise, snr;
};

struct erthost {
    protocol::Decoder d;
    std::string err;
    bool started = false;        // a decode call since erthost_new / erthost_reset
    bool measured = false;       // `level` holds the measurement of this stream's start
    ertgpu_input_level level{};
};

// main.go:59-86: NewDecoder; for each -msgtype NewParser + RegisterProtocol; Allocate.  The input arguments are
// protocol::Input's (all 0: uint8 IQ at the decoder's own rate): IQ sampled at input_rate Hz, in sample format `format`
// (ERTGPU_FORMAT_*) with gain `scale`, recorded centred at capture_freq Hz with the channel at center_freq.  auto_scale:
// the gain of each stream is measured from the first min(len, ERTLV_WINDOW) samples of its first erthost_decode call.
// channel_gain: k of the wide channel path (0 ... 14), -1 none, -2 measured like auto_scale (after it) from the same
// samples (ertgpu_measure_channel).  signal: every message carries its signal report (protocol::Decoder::EnableSignal).
// spectrum_log2 > 0: the input's spectrum in rows of spectrum_frames frames of 2^spectrum_log2 samples
// (protocol::Decoder::EnableSpectrum; erthost_gpu_handle gives the handle ertgpu_fetch_spectrum takes).
erthost* erthost_new(const char* msgtypes_csv, int chip_length, int device, long long max_blocks, long long max_cands,
                     long long input_rate, int format, float scale, long long capture_freq, long long center_freq,
                     int auto_scale, int channel_gain, int signal, int spectrum_log2, long long spectrum_frames,
                     char* errbuf, int errcap) {
    std::unique_ptr<erthost> h;   // released only on success: a throwing NewParser / Allocate must not leak the handle
    try {
        h.reset(new erthost());
        protocol::RegisterProtocols(h->d, msgtypes_csv, chip_length);
        h->d.SetInput({input_rate, format, scale, capture_freq, center_freq, auto_scale != 0, channel_gain < 0 ? -1 : channel_gain,
                       channel_gain == -2, signal != 0, spectrum_log2, spectrum_frames});
        h->d.Allocate(device, max_blocks, max_cands);
        return h.release();
    } catch (const std::exception& e) {
        if (errbuf && errcap > 0) snprintf(errbuf, (size_t)errcap, "%s", e.what());
        return nullptr;
    }
}

// The same without Allocate: no device is touched, only erthost_parse works on such a handle.
erthost* erthost_new_parse_only(const char* msgtypes_csv, int chip_length, char* errbuf, int errcap) {
    std::unique_ptr<erthost> h;
    try {
        h.reset(new erthost());
        protocol::RegisterProtocols(h->d, msgtypes_csv, chip_length);
        return h.release();
    } catch (const std::exception& e) {
        if (errbuf && errcap > 0) snprintf(errbuf, (size_t)errcap, "%s", e.what());
        return nullptr;
    }
}

void erthost_free(erthost* h) { delete h; }

const char* erthost_error(const erthost* h) { return h ? h->err.c_str() : ""; }

int erthost_config(const erthost* h, int32_t* out12) {
    const protocol::PacketConfig& c = h->d.Cfg;
    const int32_t v[12] = {c.DataRate, c.BlockSize, c.BlockSize2, c.ChipLength, c.SymbolLength, c.SampleRate,
                           c.PreambleSymbols, c.PacketSymbols, c.PreambleLength, c.PacketLength, c.BufferLength,
                           (int32_t)c.CenterFreq};
    memcpy(out12, v, sizeof(v));
    return 0;
}

ertgpu_handle* erthost_gpu_handle(erthost* h) { return h->d.Handle(); }

int erthost_reset(erthost* h) {
    try {
        h->d.Reset();
        h->started = h->measured = false;
        return 0;
    } catch (const std::exception& e) {
        h->err = e.what();
        return -1;
    }
}

// rcvr.d.Decode(block) for N blocks (main.go:235); returns the number of messages (all are counted,
// the first `cap` are written), or -1 on error / -2 when len is not a multiple of BlockSize2.
static long long fill_msgs(const std::vector<const protocol::Message*>& msgs, erthost_msg* out, long long cap);
static std::vector<const protocol::Message*> pointers(const std::vector<protocol::MessagePtr>& msgs);

// The parsers alone (decode.go:177-187 + each Parse): candidates sorted by (block, preamble, idx) in, messages out.
long long erthost_parse(erthost* h, const ertgpu_candidate* cands, long long n, erthost_msg* out, long long cap) {
    try {
        std::vector<protocol::MessagePtr> msgs;
        h->d.Dispatch(cands, (size_t)n, msgs);
        return fill_msgs(pointers(msgs), out, cap);
    } catch (const std::exception& e) {
        h->err = e.what();
        return -1;
    }
}

// erthost_parse_filtered without filters over the candidate lists of nch channels of one capture (counts[c] candidates
// of channel c, one list after the other in cands): each list is parsed, and the messages go through the cross-channel
// dedup in the order the receiver prints them (ascending block, then channel).  channel_out[i]: the channel of out[i].
long long erthost_parse_dedup_channels(erthost* h, const ertgpu_candidate* cands, const long long* counts, int nch,
                                       int block_dedup, erthost_msg* out, int* channel_out, long long cap, long long* duplicates) {
    try {
        std::vector<std::vector<protocol::MessagePtr>> per((size_t)nch);
        for (int c = 0; c < nch; c++) {
            h->d.Dispatch(cands, (size_t)counts[c], per[(size_t)c]);
            cands += counts[c];
        }
        receiver::BlockDedup dd;
        receiver::Stats st;
        std::vector<size_t> pos((size_t)nch, 0), cnt;
        std::vector<protocol::MessagePtr*> at;
        std::vector<const protocol::Message*> order;
        std::vector<int> chan;
        int64_t b = 0;
        while (receiver::NextBlock(per, pos, at, cnt, &b))
            dd.FilterChannels(at.data(), cnt.data(), (size_t)nch, block_dedup != 0, [&](const protocol::Message& m, size_t c) {
                order.push_back(&m);
                chan.push_back((int)c);
                return true;
            }, st);
        if (duplicates) *duplicates = st.duplicates;
        for (size_t i = 0; i < chan.size() && (long long)i < cap; i++) channel_out[i] = chan[i];
        return fill_msgs(order, out, cap);
    } catch (const std::exception& e) {
        h->err = e.what();
        return -1;
    }
}

// erthost_parse, then the receive loop of main.go:236-260 on the result with a fresh memory: the filter chain in the order
// flag.Visit builds it (main.go:97-113: filterid, filtertype, unique -- lexicographic, whatever the command line's order),
// then the cross-block digest dedup.  filterid / filtertype: comma lists as for the flags, NULL or "" = flag not given.
// Without filters: the messages rtlamr would print for this candidate list with -blockdedup=`block_dedup`.
long long erthost_parse_filtered(erthost* h, const ertgpu_candidate* cands, long long n, const char* filterid, const char* filtertype,
                                 int unique, int block_dedup, erthost_msg* out, long long cap, long long* duplicates,
                                 long long* filtered) {
    try {
        std::vector<protocol::MessagePtr> msgs;
        h->d.Dispatch(cands, (size_t)n, msgs);
        receiver::FilterChain fc = receiver::NewFilterChain(filterid ? filterid : "", filtertype ? filtertype : "", unique != 0);
        receiver::BlockDedup dd;
        receiver::Stats st;
        std::vector<const protocol::Message*> order;
        dd.Filter(msgs, block_dedup != 0, [&](const protocol::Message& m) { order.push_back(&m); }, st, fc.empty() ? nullptr : &fc);
        if (duplicates) *duplicates = st.duplicates;
        if (filtered) *filtered = st.filtered;
        return fill_msgs(order, out, cap);
    } catch (const std::exception& e) {
        h->err = e.what();
        return -1;
    }
}

// The encoders (flags.go:140-170) on every message of erthost_parse: format 0 = plain (PlainEncoder, flags.go:261-272),
// 1 = csv (csv/csv.go:27-38), 2 = json (encoding/json), 3 = xml (encoding/xml + NewLineEncoder); the LogMessage fields
// (parse.go:103-109) are the caller's.  Returns the number of bytes the lines need (they are written when they fit `cap`),
// or -1.
long long erthost_encode(erthost* h, const ertgpu_candidate* cands, long long n, int format, long long unix_seconds, int nanos,
                         long long offset, int length, int sample_file_is_devnull, char* buf, long long cap) {
    try {
        std::vector<protocol::MessagePtr> msgs;
        h->d.Dispatch(cands, (size_t)n, msgs);
        const receiver::Format f = (receiver::Format)format;
        const bool plain = f != receiver::CSV && f != receiver::JSON && f != receiver::XML;
        std::string all;
        for (auto& m : msgs) {
            receiver::LogMessage lm;
            lm.unix_seconds = unix_seconds;
            lm.nanos = nanos;
            lm.Offset = offset;
            lm.Length = length;
            lm.Message = m.get();
            all += plain ? receiver::PlainLine(lm, sample_file_is_devnull != 0) + "\n" : receiver::Line(f, lm);
        }
        if ((long long)all.size() < cap && buf) memcpy(buf, all.c_str(), all.size() + 1);
        return (long long)all.size();
    } catch (const std::exception& e) {
        h->err = e.what();
        return -1;
    }
}

// erthost_encode with the candidates' signal records sigs[0..n) (ertgpu_fetch_signal), summarised for a decoder on
// channel_hz at rate_out, and format 0 the plain line of ertgpu_decode_file (receiver::BlockLine).
long long erthost_encode_signal(erthost* h, const ertgpu_candidate* cands, const ertgpu_signal* sigs, long long n,
                                long long channel_hz, long long rate_out, int format, long long unix_seconds, int nanos,
                                char* buf, long long cap) {
    try {
        std::vector<protocol::MessagePtr> msgs;
        h->d.SetSignalChannel(channel_hz, rate_out);
        h->d.Dispatch(cands, (size_t)n, msgs, sigs);
        const receiver::Format f = (receiver::Format)format;
        const bool plain = f != receiver::CSV && f != receiver::JSON && f != receiver::XML;
        std::string all;
        for (auto& m : msgs) {
            receiver::LogMessage lm;
            lm.unix_seconds = unix_seconds;
            lm.nanos = nanos;
            lm.Message = m.get();
            all += plain ? receiver::BlockLine(*m) + "\n" : receiver::Line(f, lm);
        }
        if ((long long)all.size() < cap && buf) memcpy(buf, all.c_str(), all.size() + 1);
        return (long long)all.size();
    } catch (const std::exception& e) {
        h->err = e.what();
        return -1;
    }
}

long long erthost_decode(erthost* h, const uint8_t* iq, size_t len, erthost_msg* out, long long cap) {
    try {
        if (!h->started && len % h->d.InputQuantum() == 0)
            receiver::StartStream({&h->d}, iq, len, [h](const ertgpu_input_level& lv) {
                h->level = lv;
                h->measured = true;
            }, {});
        h->started = true;
        return fill_msgs(pointers(h->d.Decode(iq, len)), out, cap);
    } catch (const std::length_error& e) {
        h->err = e.what();
        return -2;
    } catch (const std::exception& e) {
        h->err = e.what();
        return -1;
    }
}

static std::vector<const protocol::Message*> pointers(const std::vector<protocol::MessagePtr>& msgs) {
    std::vector<const protocol::Message*> v;
    for (const auto& m : msgs) v.push_back(m.get());
    return v;
}

static long long fill_msgs(const std::vector<const protocol::Message*>& msgs, erthost_msg* out, long long cap) {
    {
        long long n = 0;
        for (const protocol::Message* m : msgs) {
            if (n < cap) {
                erthost_msg& o = out[n];
                memset(&o, 0, sizeof(o));
                o.block = m->Block;
                o.idx = m->Idx;
                o.meter_id = m->MeterID();
                o.meter_type = m->MeterType();
                auto ck = m->Checksum();
                o.nchecksum = (int32_t)ck.size();
                memcpy(o.checksum, ck.data(), std::min<size_t>(ck.size(), 8));
                snprintf(o.msgtype, sizeof(o.msgtype), "%s", m->MsgType().c_str());
                snprintf(o.text, sizeof(o.text), "%s", m->String().c_str());
                std::string rec;
                for (auto& f : m->Record()) rec += (rec.empty() ? "" : ",") + f;
                snprintf(o.record, sizeof(o.record), "%s", rec.c_str());
                if (m->Signal) {
                    const protocol::SignalReport& r = *m->Signal;
                    o.signal = r.Valid ? 2 : 1;
                    o.channel = r.Channel;
                    o.freq = r.Freq;
                    o.level = r.Level;
                    o.noise = r.Noise;
                    o.snr = r.SNR;
                }
            }
            n++;
        }
        return n;
    }
}

// The header of the WAV file at `path` (wav.hpp), nothing else: *format = ERTGPU_FORMAT_*, *rate in Hz, *data_offset and
// *data_size in bytes (-1: to the end of the file).  Returns 0, or -1 with the message in errbuf.
int erthost_wav_probe(const char* path, int* format, long long* rate, long long* data_offset, long long* data_size,
                      char* errbuf, int errcap) {
    FILE* f = fopen(path, "rb");
    if (!f) {
        if (errbuf && errcap > 0) snprintf(errbuf, (size_t)errcap, "%s: %s", path, strerror(errno));
        return -1;
    }
    try {
        const wav::Header w = wav::ReadHeader(f);
        fclose(f);
        *format = w.format;
        *rate = w.rate;
        *data_offset = w.data_offset;
        *data_size = w.data_size;
        return 0;
    } catch (const std::exception& e) {
        fclose(f);
        if (errbuf && errcap > 0) snprintf(errbuf, (size_t)errcap, "%s", e.what());
        return -1;
    }
}

// The metadata of the SigMF recording at `path` (NAME.sigmf-meta, NAME.sigmf-data or NAME; sigmf.hpp): *format =
// ERTGPU_FORMAT_*, *rate and *frequency in Hz (0: none given), the data file's path and *samples, and per capture segment
// its first sample, header bytes and datetime in ns (dated[k] = 0: none), the first seg_cap of *nseg.  Returns 0, or -1
// with the message in errbuf.
int erthost_sigmf_probe(const char* path, int* format, long long* rate, long long* frequency, char* data_path, int data_cap,
                        long long* samples, long long* starts, long long* header_bytes, long long* datetime_ns, int* dated,
                        int seg_cap, int* nseg, char* errbuf, int errcap) {
    try {
        const sigmf::Recording r = sigmf::Read(path);
        *format = r.format;
        *rate = r.rate;
        *frequency = r.frequency;
        snprintf(data_path, (size_t)data_cap, "%s", r.data_path.c_str());
        *samples = r.samples;
        *nseg = (int)r.segments.size();
        for (int k = 0; k < *nseg && k < seg_cap; k++) {
            starts[k] = r.segments[k].sample_start;
            header_bytes[k] = r.segments[k].header_bytes;
            datetime_ns[k] = r.segments[k].datetime_ns;
            dated[k] = r.segments[k].dated;
        }
        return 0;
    } catch (const std::exception& e) {
        if (errbuf && errcap > 0) snprintf(errbuf, (size_t)errcap, "%s", e.what());
        return -1;
    }
}

// sigmf::BlockTime of decoder block `block` (block_size samples at rate_out Hz) of the recording at `path`, in *ns.
// Returns 0, or -1 with the message in errbuf (also when no segment is dated).
int erthost_sigmf_block_time(const char* path, long long block, long long block_size, long long rate_out, long long* ns,
                             char* errbuf, int errcap) {
    try {
        *ns = sigmf::BlockTime(sigmf::Read(path), block, block_size, rate_out);
        return 0;
    } catch (const std::exception& e) {
        if (errbuf && errcap > 0) snprintf(errbuf, (size_t)errcap, "%s", e.what());
        return -1;
    }
}

// The level measured at the start of the current stream (auto_scale): *exponent = k, *scale = 2^k, *components, and the
// 256 bins when bins != NULL.  Returns 0, or -1 when nothing was measured yet.
int erthost_level(const erthost* h, int* exponent, float* scale, long long* components, long long* bins) {
    if (!h->measured) return -1;
    *exponent = h->level.exponent;
    *scale = h->level.scale;
    *components = h->level.components;
    if (bins) memcpy(bins, h->level.bins, sizeof(h->level.bins));
    return 0;
}

// k of a handle on the wide channel path (channel_gain >= 0, or -2 once its first erthost_decode measured it); -1
// when the handle does not take it.
int erthost_channel_gain(const erthost* h) {
    int32_t k = -1;
    return ertgpu_get_channel_gain(h->d.Handle(), &k) == ERTGPU_OK ? k : -1;
}

int erthost_log(const erthost* h, char* buf, int cap) {
    snprintf(buf, (size_t)cap, "%s", h->d.Log().c_str());
    return 0;
}

}  // extern "C"
