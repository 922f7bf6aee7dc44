// ertgpu_decode_file -- decode an IQ capture (raw uint8 IQ as rtl_sdr and rtlamr -samplefile write it, raw IQ of any
// complex SigMF datatype, a baseband WAV recording or a SigMF recording) or stdin through the C++ mirror of rtlamr's receive loop
// (receiver.hpp) on the GPU and print one line per message in rtlamr's plain format without the time fields
// (protocol/parse.go:119-121 StringNoOffset).
//   ertgpu_decode_file [-msgtype=scm,idm|all] [-symbollength=72] [-blockdedup=true] [-blocks=4096] [-device=0]
//                      [-filterid=1,2] [-filtertype=4,5] [-unique=true] [-format=plain|csv|json|xml]
//                      [-samplefile=PATH] [-single] [-duration=1h5m10s] [-samplerate=HZ] [-signal]
//                      [-sampleformat=cu8|cs8|cs16|cf32|ci16_be|...|cf64_be|wav|sigmf] [-samplescale=G|auto] [-capturefreq=HZ [-centerfreq=HZ[,HZ...]]]
//                      FILE|- [FILE ...]
// -capturefreq names the frequency the capture was recorded centred at; -centerfreq (rtlamr's flag) the channel to
// receive, by default the protocols' CenterFreq (912.6 MHz, or 912.38 MHz for r900 alone).  The channel is mixed to
// 0 Hz exactly inside the GPU resampler, whose lowpass is then the channel filter; a tuned capture may be at up to 256
// times 32768 * -symbollength (above 10 times it is first decimated by D on the GPU, and the decoder log on stderr
// names D and the intermediate rate).  Without -capturefreq nothing is translated; -centerfreq alone is a usage error,
// and so is -samplefile with -capturefreq.
// -samplerate is rtlamr's (rtltcp's) flag name; here it names the capture's sample rate.  The default,
// 32768 * -symbollength, decodes the bytes as they are; any other rate within 1/4 ... 4 times it is resampled
// exactly on the GPU first, and Block / Idx then count resampled samples.
// -sampleformat names the capture's samples: cu8 (the default: uint8, rtl_sdr), cs8 (int8, hackrf_transfer), cs16
// (little-endian int16: airspy_rx, rx_sdr, SoapySDR), cf32 (little-endian float32: GNU Radio, gqrx) or wav (SDR#,
// SDR++, SDRuno, HDSDR: each file's header gives the format and the rate; wav.hpp).  Every complex SigMF datatype name
// (ci8, ci16_le, ci16_be, cu16_le, cu16_be, ci32_le, ci32_be, cu32_le, cu32_be, cf32_le, cf32_be, cf64_le, cf64_be; cu8)
// names raw samples of that type too.  -sampleformat=sigmf reads SigMF recordings (sigmf.hpp): FILE is NAME.sigmf-meta,
// NAME.sigmf-data or NAME, and the metadata gives the format, the rate and the capture frequency (-centerfreq then picks
// the channel as with -capturefreq); -samplerate or -capturefreq that disagree with it are usage errors.  When a capture
// segment carries a core:datetime, the csv, json and xml Time is the moment a live receiver would have finished the
// message's block (sigmf::BlockTime) instead of the wall clock.  Other formats are converted to uint8 on the GPU,
// u = clamp(rint(x * G), -128, 127) + 128; -samplescale=G is that gain (default 1 for cs8, 2^-8 for the 16-bit formats,
// 2^-24 for the 32-bit integers, 2^7 for the floats: full scale to full scale; a 12-bit Airspy wants 0.0625).
// -samplescale=auto picks G = 2^k per stream (each file of a batch, or stdin) from the stream's first 2^22 samples, after
// a WAV header or SigMF core:header_bytes: the largest k in [-120, 120] at which at most one component in 65 536 clips
// (include/ertgpu_level.h).  The gain then stays fixed for the whole stream; it does not follow the level the way a tuner's
// AGC does.  k, G and the number of samples measured go to stderr; stdout is exactly that of -samplescale=G.  A WAV or
// SigMF file is never detected by its content or name.
// -channelgain=G (a power of two, 1 ... 2^14) or auto takes the wide channel path of a tuned input (a capture frequency
// from -capturefreq or the SigMF metadata): the input keeps 15 bits through the mixer and the channel filter, and the
// decoder's byte is formed from the channel's filtered level times G (include/ertgpu_resample.h).  auto picks G per stream
// and channel from the stream's first 2^22 samples, after -samplescale=auto has set the input gain from the same samples,
// and then decodes those bytes; "channel <Hz>: 2^k = G" goes to stderr, and stdout is exactly that of -channelgain=G.  -samplefile takes only untuned uint8 input at
// 32768 * -symbollength (an 8-bit WAV at that rate is uint8).
// -filterid / -filtertype / -unique, -format, -samplefile, -single and -duration are rtlamr's flags of the same names
// (flags.go:37-58,69-70,140-170; the filter chain runs before the cross-block dedup, main.go:236-260).  With -format=csv a
// line is LogMessage.Record() (parse.go:123-129: time, offset, length, then the message's own record) through Go's
// encoding/csv rules; json and xml are the lines of Go's encoding/json and encoding/xml encoders (filters.hpp).  Time is
// written in UTC.  Offset and Length are 0 unless -samplefile names a file.
// -single stops after the first reported message or, with -filterid, once every listed meter has reported.  -duration
// (Go duration syntax, 0 = no limit) is checked before each read of -blocks blocks: the call in progress is decoded and
// reported in full, so the run can last one call longer than asked.  Both end the run with exit status 0.
// -centerfreq=F1,F2,... (with a capture frequency: -capturefreq or the SigMF metadata) decodes several channels of the
// capture in one pass: each chunk is read and sent to the GPU once, every channel is decoded from it exactly as a run
// with that channel alone decodes it, and the messages are printed by ascending block, then channel in the order given.
// The cross-block dedup spans the channels: a message is dropped when its digest was seen for the previous block in any
// channel, or for the same block in an earlier channel, so a packet where two channels overlap is printed once
// (-blockdedup=false prints it from each).  The decoder log's CenterFreq lists every channel and the summary counts each
// channel's messages.  -samplescale=auto measures the stream once and sets that gain on every channel.
// -signal reports how each message was received, measured on the GPU from its packet's own samples (DESIGN.md §3.13,
// include/ertgpu_signal.h): the channel that decoded it (the tuned channel, or the protocols' CenterFreq), the carrier's
// frequency in Hz, and its level, the noise floor between its chips and their ratio in dB of the decoder's bytes (two
// decimals).  plain: {Block:B Idx:I Channel:C Freq:F Level:L Noise:N SNR:S TYPE:{...}}; csv: the five fields after the
// message's own record; json: "Signal":{"Channel":..,"Freq":..,"Level":..,"Noise":..,"SNR":..} after "Message"; xml: a
// <Signal Channel=".." Freq=".." Level=".." Noise=".." SNR=".."> element after <Message>.  A packet that starts before
// the stream has no report: "-" for each field (plain), five empty fields (csv), null (json), no attributes (xml).
// Without -signal every format is exactly as above.
// Several files are a batch of independent streams through ONE decoder (buffers, tables and kernels set up once):
// each starts from zeroed history with block numbers from 0, exactly as if it were decoded alone.  They share the
// sample file, whose offsets keep growing from one file to the next.
#include <cerrno>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <ctime>
#include <iostream>
#include <tuple>
#include <vector>

#include "../../include/ertgpu_resample.h"
#include "receiver.hpp"
#include "sigmf.hpp"
#include "wav.hpp"

int main(int argc, char** argv) {
    const auto start = std::chrono::steady_clock::now();   // main.go:350-353: the time limit covers the whole run
    std::string msgtype = "scm";
    std::vector<std::string> files;
    int chip = 72, device = 0;
    long long blocks = 4096, samplerate = 0;
    bool block_dedup = true, quiet = false, unique = false, single = false, signal = false;
    std::string filterid, filtertype, format = "plain", samplefile, duration, sampleformat = "cu8", samplescale;
    std::string capturefreq, centerfreq, channelgain;
    bool have_scale = false, auto_scale = false;
    for (int i = 1; i < argc; i++) {
        std::string a = argv[i];
        if (a.rfind("-msgtype=", 0) == 0) msgtype = a.substr(9);
        else if (a.rfind("-symbollength=", 0) == 0) chip = atoi(a.c_str() + 14);
        else if (a.rfind("-device=", 0) == 0) device = atoi(a.c_str() + 8);
        else if (a.rfind("-samplerate=", 0) == 0) samplerate = atoll(a.c_str() + 12);
        else if (a.rfind("-sampleformat=", 0) == 0) sampleformat = a.substr(14);
        else if (a.rfind("-capturefreq=", 0) == 0) capturefreq = a.substr(13);
        else if (a.rfind("-centerfreq=", 0) == 0) centerfreq = a.substr(12);
        else if (a.rfind("-channelgain=", 0) == 0) channelgain = a.substr(13);
        else if (a.rfind("-samplescale=", 0) == 0) {
            samplescale = a.substr(13);
            have_scale = true;
        }
        else if (a.rfind("-blocks=", 0) == 0) blocks = atoll(a.c_str() + 8);
        else if (a.rfind("-blockdedup=", 0) == 0) block_dedup = a.substr(12) != "false";
        else if (a.rfind("-filterid=", 0) == 0) filterid = a.substr(10);
        else if (a.rfind("-filtertype=", 0) == 0) filtertype = a.substr(12);
        else if (a.rfind("-unique=", 0) == 0) unique = a.substr(8) == "true";
        else if (a == "-unique") unique = true;
        else if (a.rfind("-format=", 0) == 0) format = a.substr(8);
        else if (a.rfind("-samplefile=", 0) == 0) samplefile = a.substr(12);
        else if (a.rfind("-single=", 0) == 0) single = a.substr(8) == "true";
        else if (a == "-signal" || a == "-signal=true") signal = true;
        else if (a == "-signal=false") signal = false;
        else if (a == "-single") single = true;
        else if (a.rfind("-duration=", 0) == 0) duration = a.substr(10);
        else if (a == "-quiet") quiet = true;
        else files.push_back(a);
    }
    if (files.empty()) {
        fprintf(stderr, "usage: %s [-msgtype=scm,scm+,idm,netidm,r900,r900bcd|all] [-symbollength=N] [-blockdedup=true|false] "
                        "[-blocks=K] [-device=D] [-filterid=ID,..] [-filtertype=T,..] [-unique=true|false] [-format=plain|csv|json|xml] "
                        "[-samplefile=PATH] [-single] [-duration=D] [-samplerate=HZ] [-sampleformat=cu8|cs8|cs16|cf32|ci16_be|...|wav|sigmf] "
                        "[-samplescale=G|auto] [-channelgain=G|auto] [-signal] "
                        "[-capturefreq=HZ [-centerfreq=HZ[,HZ...]]] [-quiet] FILE|- [FILE ...]\n", argv[0]);
        return 2;
    }
    // -capturefreq / -centerfreq: whole Hz, > 0 and >= 0; -centerfreq may be a comma list of channels
    std::vector<std::string> centers;
    for (size_t p = 0; !centerfreq.empty();) {
        const size_t q = centerfreq.find(',', p);
        centers.push_back(centerfreq.substr(p, q == std::string::npos ? std::string::npos : q - p));
        if (q == std::string::npos) break;
        p = q + 1;
    }
    long long capture_hz = 0, center_hz = 0;
    std::vector<long long> list;
    std::vector<std::tuple<const char*, const std::string*, long long*, long long>> freqs = {
        std::make_tuple("-capturefreq", &capturefreq, &capture_hz, 1LL)};
    if (centers.size() == 1) freqs.push_back(std::make_tuple("-centerfreq", &centerfreq, &center_hz, 0LL));
    list.resize(centers.size() > 1 ? centers.size() : 0);
    for (size_t c = 0; c < list.size(); c++) freqs.push_back(std::make_tuple("-centerfreq", &centers[c], &list[c], 1LL));
    for (auto [flag, text, out, min] : freqs) {
        if (text->empty() && text == &capturefreq) continue;
        char* end = nullptr;
        errno = 0;
        *out = strtoll(text->c_str(), &end, 10);
        if (text->empty() || *end || errno || *out < min) {
            fprintf(stderr, "invalid value \"%s\" for flag %s: a frequency in Hz%s\n", text->c_str(), flag, min ? " > 0" : "");
            return 2;
        }
    }
    const std::vector<int64_t> channels(list.begin(), list.end());
    for (size_t c = 0; c < channels.size(); c++)
        for (size_t j = 0; j < c; j++)
            if (channels[c] == channels[j]) {
                fprintf(stderr, "-centerfreq names the channel %lld Hz twice\n", (long long)channels[c]);
                return 2;
            }
    const bool csv = format == "csv", json = format == "json", xml = format == "xml";
    int64_t limit_ns = 0;
    try {
        if (!duration.empty()) limit_ns = receiver::ParseDuration(duration);
    } catch (const std::exception& e) {
        fprintf(stderr, "invalid value \"%s\" for flag -duration: %s\n", duration.c_str(), e.what());
        return 2;
    }
    const bool wav_in = sampleformat == "wav", sigmf_in = sampleformat == "sigmf";
    int32_t fmt = ERTGPU_FORMAT_CU8;
    if (sampleformat == "cs8") fmt = ERTGPU_FORMAT_CS8;
    else if (sampleformat == "cs16") fmt = ERTGPU_FORMAT_CS16;
    else if (sampleformat == "cf32") fmt = ERTGPU_FORMAT_CF32;
    else if (!wav_in && !sigmf_in && (fmt = sigmf::FormatOf(sampleformat)) < 0) {
        fprintf(stderr, "invalid value \"%s\" for flag -sampleformat: cu8, cs8, cs16, cf32, a complex SigMF datatype "
                        "(ci16_be, cf64_le, ...), wav or sigmf\n", sampleformat.c_str());
        return 2;
    }
    float scale = 0.0f;
    if (samplescale == "auto") {
        auto_scale = true;
    } else if (have_scale) {
        char* end = nullptr;
        scale = strtof(samplescale.c_str(), &end);
        if (samplescale.empty() || *end || !std::isfinite(scale) || scale <= 0.0f) {
            fprintf(stderr, "invalid value \"%s\" for flag -samplescale: a finite gain > 0, or auto\n", samplescale.c_str());
            return 2;
        }
    }
    int32_t channel_k = -1;   // -channelgain: k of G = 2^k
    const bool auto_channel = channelgain == "auto";
    if (!channelgain.empty() && !auto_channel) {
        char* end = nullptr;
        const long long g = strtoll(channelgain.c_str(), &end, 10);
        if (*end || g < 1 || g > (1LL << ERTRS_GAIN_K_MAX) || (g & (g - 1))) {
            fprintf(stderr, "invalid value \"%s\" for flag -channelgain: a power of two 1 ... %lld, or auto\n", channelgain.c_str(),
                    1LL << ERTRS_GAIN_K_MAX);
            return 2;
        }
        channel_k = 63 - __builtin_clzll((unsigned long long)g);
    }
    // wav: every file's header, before anything else (stdin's is consumed here, the files' are read again below)
    std::vector<wav::Header> wav_hdr(files.size());
    if (wav_in) {
        for (size_t fi = 0; fi < files.size(); fi++) {
            FILE* in = files[fi] == "-" ? stdin : fopen(files[fi].c_str(), "rb");
            if (!in) {
                perror(files[fi].c_str());
                return 1;
            }
            try {
                wav_hdr[fi] = wav::ReadHeader(in);
            } catch (const std::exception& e) {
                fprintf(stderr, "%s: %s\n", files[fi].c_str(), e.what());
                if (in != stdin) fclose(in);
                return 1;
            }
            if (in != stdin) fclose(in);
            if (wav_hdr[fi].rate != wav_hdr[0].rate || wav_hdr[fi].format != wav_hdr[0].format) {
                fprintf(stderr, "%s: %lld Hz, format %d, but %s: %lld Hz, format %d: the files of a batch share one decoder\n",
                        files[0].c_str(), (long long)wav_hdr[0].rate, wav_hdr[0].format, files[fi].c_str(),
                        (long long)wav_hdr[fi].rate, wav_hdr[fi].format);
                return 2;
            }
        }
        if (samplerate != 0 && samplerate != wav_hdr[0].rate) {
            fprintf(stderr, "-samplerate=%lld disagrees with the WAV header's %lld Hz\n", samplerate, (long long)wav_hdr[0].rate);
            return 2;
        }
        samplerate = wav_hdr[0].rate;
        fmt = wav_hdr[0].format;
    }
    // sigmf: every recording's metadata, before anything else
    std::vector<sigmf::Recording> rec(files.size());
    if (sigmf_in) {
        for (size_t fi = 0; fi < files.size(); fi++) {
            if (files[fi] == "-") {
                fprintf(stderr, "-sampleformat=sigmf reads NAME.sigmf-meta beside NAME.sigmf-data, not stdin\n");
                return 2;
            }
            try {
                rec[fi] = sigmf::Read(files[fi]);
            } catch (const std::exception& e) {
                fprintf(stderr, "%s: %s\n", files[fi].c_str(), e.what());
                return 1;
            }
            if (rec[fi].rate != rec[0].rate || rec[fi].format != rec[0].format || rec[fi].frequency != rec[0].frequency) {
                fprintf(stderr, "%s: %s at %lld Hz, %lld Hz, but %s: %s at %lld Hz, %lld Hz: the files of a batch share one decoder\n",
                        files[0].c_str(), sigmf::FormatName(rec[0].format), (long long)rec[0].rate, (long long)rec[0].frequency,
                        files[fi].c_str(), sigmf::FormatName(rec[fi].format), (long long)rec[fi].rate, (long long)rec[fi].frequency);
                return 2;
            }
        }
        if (samplerate != 0 && samplerate != rec[0].rate) {
            fprintf(stderr, "-samplerate=%lld disagrees with the SigMF core:sample_rate %lld Hz\n", samplerate, (long long)rec[0].rate);
            return 2;
        }
        if (capture_hz != 0 && rec[0].frequency != 0 && capture_hz != rec[0].frequency) {
            fprintf(stderr, "-capturefreq=%lld disagrees with the SigMF core:frequency %lld Hz\n", capture_hz, (long long)rec[0].frequency);
            return 2;
        }
        samplerate = rec[0].rate;
        fmt = rec[0].format;
        if (rec[0].frequency) capture_hz = rec[0].frequency;
    }
    if (!centerfreq.empty() && capture_hz == 0) {
        fprintf(stderr, "-centerfreq needs -capturefreq: the frequency at the centre of the capture\n");
        return 2;
    }
    if (!channels.empty() && !samplefile.empty() && samplefile != "/dev/null") {
        fprintf(stderr, "-samplefile takes one channel, not a -centerfreq list\n");
        return 2;
    }
    for (const int64_t ch : channels) {   // each channel of a list lies inside the capture (ertrs_plan_decimated's rule)
        const int64_t rate = samplerate ? samplerate : 32768LL * chip;
        ertgpu_decimator_info d{};
        ertgpu_resampler_info info{};
        if (ertrs_plan_decimated(rate, 32768LL * chip, ch - capture_hz, &d, &info) != 0) {
            fprintf(stderr, "-centerfreq channel %lld Hz does not fit a %lld Hz capture at %lld Hz: |offset| + 0.4 * %lld Hz "
                            "must be at most half the capture's rate\n", (long long)ch, (long long)rate, capture_hz, 32768LL * chip);
            return 2;
        }
    }
    const bool tuned = capture_hz > 0;
    if (!channelgain.empty() && !tuned) {
        fprintf(stderr, "-channelgain needs -capturefreq (or a SigMF frequency): the channel path of a tuned capture\n");
        return 2;
    }
    if (have_scale && fmt == ERTGPU_FORMAT_CU8) {
        fprintf(stderr, "-samplescale does not apply to uint8 (cu8) input\n");
        return 2;
    }
    // -samplerate names the capture's rate; the default DataRate*ChipLength (32768 * -symbollength) resamples nothing
    const bool resampling = samplerate != 0 && samplerate != 32768LL * chip;
    if (tuned && !samplefile.empty() && samplefile != "/dev/null") {
        fprintf(stderr, "-samplefile does not take tuned (-capturefreq) input\n");
        return 2;
    }
    if ((resampling || fmt != ERTGPU_FORMAT_CU8) && !samplefile.empty() && samplefile != "/dev/null") {
        fprintf(stderr, "-samplefile needs uint8 (cu8) input at 32768 * -symbollength = %lld Hz; this input is %s at %lld Hz\n",
                32768LL * chip, sigmf::FormatName(fmt),
                samplerate ? samplerate : 32768LL * chip);
        return 2;
    }
    FILE* sample = nullptr;   // os.DevNull, the default, is never opened (flags.go:136-141)
    if (!samplefile.empty() && samplefile != "/dev/null") {
        sample = fopen(samplefile.c_str(), "wb");
        if (!sample) {
            perror(samplefile.c_str());
            return 1;
        }
    }
    try {
        receiver::Receiver rcvr(msgtype, chip, device, blocks, {resampling ? samplerate : 0, fmt, scale, capture_hz, center_hz, auto_scale, channel_k, auto_channel, signal},
                                channels);
        std::string log = rcvr.decoder().Log();
        if (!channels.empty()) {   // the channels share everything of the log but CenterFreq, its first line: name them all
            std::string names;
            for (size_t c = 0; c < channels.size(); c++) names += (c ? "," : "") + std::to_string(channels[c]);
            log = "CenterFreq: " + names + log.substr(log.find('\n'));
        }
        fputs(log.c_str(), stderr);
        if (sample) rcvr.SetSampleFile(sample);
        if (limit_ns) rcvr.SetDeadline(start + std::chrono::nanoseconds(limit_ns));
        if (single) rcvr.SetSingle(nullptr);
        // the order flag.Visit gives the chain (main.go:97-113): filterid, filtertype, unique
        if (!filterid.empty()) {
            auto f = std::make_shared<receiver::MeterIDFilter>();
            f->ids.Set(filterid);
            rcvr.filters().Add(f);
            if (single) rcvr.SetSingle(&f->ids);   // main.go:278: -single empties the filter's own set
        }
        if (!filtertype.empty()) {
            auto f = std::make_shared<receiver::MeterTypeFilter>();
            f->types.Set(filtertype);
            rcvr.filters().Add(f);
        }
        if (unique) rcvr.filters().Add(std::make_shared<receiver::UniqueFilter>());
        for (size_t fi = 0; fi < files.size(); fi++) {
            const std::string& file = files[fi];
            FILE* in = sigmf_in ? sigmf::OpenSamples(rec[fi]) : file == "-" ? stdin : fopen(file.c_str(), "rb");
            if (!in) {
                perror(file.c_str());
                return 1;
            }
            if (fi) rcvr.Reset();
            if (auto_scale)
                rcvr.SetLevelReport([&](const ertgpu_input_level& lv) {
                    fprintf(stderr, "%s%s-samplescale=auto: 2^%d = %.9g from %lld samples\n", files.size() > 1 ? file.c_str() : "",
                            files.size() > 1 ? ": " : "", lv.exponent, (double)lv.scale, (long long)(lv.components / 2));
                });
            if (auto_channel)
                rcvr.SetChannelLevelReport([&](size_t c, const ertgpu_channel_level& lv) {
                    ertgpu_tuning_info t{};
                    ertgpu_get_tuning(rcvr.decoder(c).Handle(), &t);
                    fprintf(stderr, "%s%schannel %lld: 2^%d = %lld\n", files.size() > 1 ? file.c_str() : "", files.size() > 1 ? ": " : "",
                            (long long)t.center_hz, lv.k, 1LL << lv.k);
                });
            if (wav_in && in != stdin) wav_hdr[fi] = wav::ReadHeader(in);   // the same header as above: to the samples
            auto st = rcvr.Run(in, block_dedup, [&](const protocol::Message& m, int64_t offset, int length) {
                if (quiet) return;
                if (csv || json || xml) {
                    receiver::LogMessage lm;
                    if (sigmf_in && sigmf::Dated(rec[fi])) {
                        const protocol::PacketConfig& c = rcvr.decoder().Cfg;
                        const int64_t ns = sigmf::BlockTime(rec[fi], m.Block, c.BlockSize, c.SampleRate);
                        lm.unix_seconds = ns / 1000000000 - (ns % 1000000000 < 0);
                        lm.nanos = (int32_t)(ns - lm.unix_seconds * 1000000000);
                    } else {
                        timespec ts{};
                        clock_gettime(CLOCK_REALTIME, &ts);
                        lm.unix_seconds = (int64_t)ts.tv_sec;
                        lm.nanos = (int32_t)ts.tv_nsec;
                    }
                    lm.Offset = offset;
                    lm.Length = length;
                    lm.Message = &m;
                    fputs((csv ? receiver::CsvLine(lm.Record()) : json ? receiver::JsonLine(lm) : receiver::XmlLine(lm)).c_str(), stdout);
                } else {
                    printf("%s\n", receiver::BlockLine(m).c_str());
                }
            }, wav_in ? wav_hdr[fi].data_size : -1);
            if (in != stdin) fclose(in);
            fprintf(stderr, "%s%s%lld messages (%lld duplicates dropped) from %lld blocks, %.1f MB in %.3f s = %.1f Msamples/s\n",
                    files.size() > 1 ? file.c_str() : "", files.size() > 1 ? ": " : "", (long long)st.messages,
                    (long long)st.duplicates, (long long)st.blocks, st.bytes / 1e6, st.seconds,
                    st.samples / 1e6 / (st.seconds > 0 ? st.seconds : 1));
            for (size_t c = 0; c < channels.size(); c++)
                fprintf(stderr, "%s%s%lld Hz: %lld messages\n", files.size() > 1 ? file.c_str() : "", files.size() > 1 ? ": " : "",
                        (long long)channels[c], (long long)st.channel_messages[c]);
            if (st.stopped) break;
        }
    } catch (const std::exception& e) {
        fprintf(stderr, "error: %s\n", e.what());
        if (sample) fclose(sample);
        return 1;
    }
    if (sample && fclose(sample) != 0) {
        perror(samplefile.c_str());
        return 1;
    }
    return 0;
}
