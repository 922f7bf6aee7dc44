// ertgpu_decode_file -- decode an IQ capture (raw uint8 IQ as rtl_sdr and rtlamr -samplefile write it, raw IQ of any
// complex SigMF datatype, a baseband WAV recording or a SigMF recording) or stdin through the C++ mirror of rtlamr's receive loop
// (receiver.hpp) on the GPU and print one line per message in rtlamr's plain format without the time fields
// (protocol/parse.go:119-121 StringNoOffset).
//   ertgpu_decode_file [-msgtype=scm,idm|all] [-symbollength=72] [-blockdedup=true] [-blocks=4096] [-device=0]
//                      [-filterid=1,2] [-filtertype=4,5] [-unique=true] [-format=plain|csv|json|xml]
//                      [-samplefile=PATH] [-single] [-duration=1h5m10s] [-samplerate=HZ] [-signal]
//                      [-spectrum=FILE [-spectrumbin=HZ] [-spectrumint=1s] [-spectrumpeak]]
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
// -spectrum=FILE also measures the power spectrum of the capture on the GPU, from the same uploaded samples as the decode
// (DESIGN.md §3.14, include/ertgpu_spectrum.h), and appends one line per row to FILE in rtl_power's column layout, which
// heat-map (waterfall) scripts read: date, time, Hz low, Hz high, Hz step, samples, dB, dB, ...  Hz low and Hz high are the
// capture's centre (the capture frequency, or the protocols' CenterFreq) -+ half its rate, Hz step the bin width, samples
// the row's input samples, and each dB a bin's mean power over the row (-spectrumpeak: its largest frame power, like
// rtl_power -P) in dB of full scale, 0 dB for a full-scale tone.  -spectrumbin=HZ (default 10000) picks the frame length:
// the smallest power of two N, 64 ... 16384, whose bins are at most HZ wide.  -spectrumint=DURATION (Go syntax, default 1s)
// is a row's length, at least 2^18 samples.  The time is the recording time of the row's first sample (UTC) for a SigMF
// recording with core:datetime, otherwise 1970-01-01 00:00:00 plus the row's offset from the start of its stream, in whole
// seconds: rows shorter than a second may share a time, and the samples column and their order tell them apart.  At the
// end of each stream the open row follows if it holds a frame.  Every file of a batch is its own stream with its own rows.
// stdout is exactly what it is without -spectrum.
// Several files are a batch of independent streams through ONE decoder (buffers, tables and kernels set up once):
// each starts from zeroed history with block numbers from 0, exactly as if it were decoded alone.  They share the
// sample file, whose offsets keep growing from one file to the next.
#include <cerrno>
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <ctime>
#include <functional>
#include <string>
#include <vector>

#include "../../include/ertgpu_format.h"
#include "../../include/ertgpu_resample.h"
#include "../../include/ertgpu_spectrum.h"
#include "receiver.hpp"
#include "sigmf.hpp"
#include "wav.hpp"

namespace {

// An end of the program before the run: main writes the message and a newline to stderr and returns the code, 2 for a
// usage error and 1 for a file that cannot be read.
struct Exit {
    int code;
    std::string message;
};

[[noreturn]] __attribute__((format(printf, 1, 2))) void usage(const char* fmt, ...) {
    va_list ap, ap2;
    va_start(ap, fmt);
    va_copy(ap2, ap);
    std::string msg((size_t)vsnprintf(nullptr, 0, fmt, ap), '\0');
    va_end(ap);
    vsnprintf(&msg[0], msg.size() + 1, fmt, ap2);
    va_end(ap2);
    throw Exit{2, msg};
}

// perror(name)'s line for errno, with status 1.
Exit file_error(const std::string& name) {
    const std::string reason = strerror(errno);
    return Exit{1, (name.empty() ? "" : name + ": ") + reason};
}

// The command line as given: every -flag=value spelling the CLI takes, and anything else as a file name.
struct Options {
    std::vector<std::string> files;
    std::string msgtype = "scm", format = "plain", sampleformat = "cu8";
    int chip = 72, device = 0;
    long long blocks = 4096, samplerate = 0;
    bool block_dedup = true, quiet = false, unique = false, single = false, signal = false, spectrum_peak = false;
    bool have_scale = false;
    std::string filterid, filtertype, samplefile, duration, samplescale, capturefreq, centerfreq, channelgain;
    std::string spectrum_file, spectrum_bin, spectrum_int;
};

Options parse_flags(int argc, char** argv) {
    Options o;
    for (int i = 1; i < argc; i++) {
        std::string a = argv[i];
        if (a.rfind("-msgtype=", 0) == 0) o.msgtype = a.substr(9);
        else if (a.rfind("-symbollength=", 0) == 0) o.chip = atoi(a.c_str() + 14);
        else if (a.rfind("-device=", 0) == 0) o.device = atoi(a.c_str() + 8);
        else if (a.rfind("-samplerate=", 0) == 0) o.samplerate = atoll(a.c_str() + 12);
        else if (a.rfind("-sampleformat=", 0) == 0) o.sampleformat = a.substr(14);
        else if (a.rfind("-capturefreq=", 0) == 0) o.capturefreq = a.substr(13);
        else if (a.rfind("-centerfreq=", 0) == 0) o.centerfreq = a.substr(12);
        else if (a.rfind("-channelgain=", 0) == 0) o.channelgain = a.substr(13);
        else if (a.rfind("-samplescale=", 0) == 0) {
            o.samplescale = a.substr(13);
            o.have_scale = true;
        }
        else if (a.rfind("-blocks=", 0) == 0) o.blocks = atoll(a.c_str() + 8);
        else if (a.rfind("-blockdedup=", 0) == 0) o.block_dedup = a.substr(12) != "false";
        else if (a.rfind("-filterid=", 0) == 0) o.filterid = a.substr(10);
        else if (a.rfind("-filtertype=", 0) == 0) o.filtertype = a.substr(12);
        else if (a.rfind("-unique=", 0) == 0) o.unique = a.substr(8) == "true";
        else if (a == "-unique") o.unique = true;
        else if (a.rfind("-format=", 0) == 0) o.format = a.substr(8);
        else if (a.rfind("-samplefile=", 0) == 0) o.samplefile = a.substr(12);
        else if (a.rfind("-single=", 0) == 0) o.single = a.substr(8) == "true";
        else if (a == "-signal" || a == "-signal=true") o.signal = true;
        else if (a == "-signal=false") o.signal = false;
        else if (a == "-single") o.single = true;
        else if (a.rfind("-duration=", 0) == 0) o.duration = a.substr(10);
        else if (a == "-quiet") o.quiet = true;
        else if (a.rfind("-spectrum=", 0) == 0) o.spectrum_file = a.substr(10);
        else if (a.rfind("-spectrumbin=", 0) == 0) o.spectrum_bin = a.substr(13);
        else if (a.rfind("-spectrumint=", 0) == 0) o.spectrum_int = a.substr(13);
        else if (a == "-spectrumpeak" || a == "-spectrumpeak=true") o.spectrum_peak = true;
        else o.files.push_back(a);
    }
    if (o.files.empty())
        usage("usage: %s [-msgtype=scm,scm+,idm,netidm,r900,r900bcd|all] [-symbollength=N] [-blockdedup=true|false] "
              "[-blocks=K] [-device=D] [-filterid=ID,..] [-filtertype=T,..] [-unique=true|false] [-format=plain|csv|json|xml] "
              "[-samplefile=PATH] [-single] [-duration=D] [-samplerate=HZ] [-sampleformat=cu8|cs8|cs16|cf32|ci16_be|...|wav|sigmf] "
              "[-samplescale=G|auto] [-channelgain=G|auto] [-signal] "
              "[-spectrum=FILE [-spectrumbin=HZ] [-spectrumint=D] [-spectrumpeak]] "
              "[-capturefreq=HZ [-centerfreq=HZ[,HZ...]]] [-quiet] FILE|- [FILE ...]", argv[0]);
    return o;
}

// What the flags and the files' headers say about the capture, checked.
struct Capture {
    int64_t decoder_rate = 0;   // DataRate * ChipLength = 32768 * -symbollength
    int64_t rate = 0;           // the capture's: -samplerate, the WAV header or the SigMF metadata, or decoder_rate
    bool resampling = false;    // rate != decoder_rate
    bool wav_in = false, sigmf_in = false;
    int32_t fmt = ERTGPU_FORMAT_CU8;
    float scale = 0.0f;
    bool auto_scale = false, auto_channel = false;
    int32_t channel_k = -1;    // -channelgain: k of G = 2^k
    long long capture_hz = 0, center_hz = 0;
    std::vector<int64_t> channels;   // -centerfreq=F1,F2,...
    int64_t limit_ns = 0;
    bool writes_samples = false;   // -samplefile names a file: os.DevNull, the default, is never opened (flags.go:136-141)
    receiver::Format out = receiver::PLAIN;
    FILE* spectrum_out = nullptr;
    int32_t spectrum_log2 = 0;
    int64_t spectrum_frames = 0;
    std::vector<wav::Header> wav_hdr;
    std::vector<sigmf::Recording> rec;
};

Capture resolve(const Options& o) {
    Capture c;
    c.decoder_rate = 32768LL * o.chip;
    // -capturefreq / -centerfreq: whole Hz, > 0 and >= 0; -centerfreq may be a comma list of channels
    std::vector<std::string> centers;
    for (size_t p = 0; !o.centerfreq.empty();) {
        const size_t q = o.centerfreq.find(',', p);
        centers.push_back(o.centerfreq.substr(p, q == std::string::npos ? std::string::npos : q - p));
        if (q == std::string::npos) break;
        p = q + 1;
    }
    const auto hz = [](const char* flag, const std::string& text, long long min) {
        char* end = nullptr;
        errno = 0;
        const long long v = strtoll(text.c_str(), &end, 10);
        if (text.empty() || *end || errno || v < min)
            usage("invalid value \"%s\" for flag %s: a frequency in Hz%s", text.c_str(), flag, min ? " > 0" : "");
        return v;
    };
    if (!o.capturefreq.empty()) c.capture_hz = hz("-capturefreq", o.capturefreq, 1);
    if (centers.size() == 1) c.center_hz = hz("-centerfreq", o.centerfreq, 0);
    else
        for (const std::string& t : centers) c.channels.push_back(hz("-centerfreq", t, 1));
    for (size_t i = 0; i < c.channels.size(); i++)
        for (size_t j = 0; j < i; j++)
            if (c.channels[i] == c.channels[j]) usage("-centerfreq names the channel %lld Hz twice", (long long)c.channels[i]);
    c.out = o.format == "csv" ? receiver::CSV : o.format == "json" ? receiver::JSON : o.format == "xml" ? receiver::XML : receiver::PLAIN;
    try {
        if (!o.duration.empty()) c.limit_ns = receiver::ParseDuration(o.duration);
    } catch (const std::exception& e) {
        usage("invalid value \"%s\" for flag -duration: %s", o.duration.c_str(), e.what());
    }
    if (o.spectrum_file.empty() && (!o.spectrum_bin.empty() || !o.spectrum_int.empty() || o.spectrum_peak))
        usage("-spectrumbin, -spectrumint and -spectrumpeak need -spectrum=FILE");
    double spectrum_hz = 10000;
    int64_t spectrum_ns = 1000000000;
    if (!o.spectrum_bin.empty()) {
        char* end = nullptr;
        spectrum_hz = strtod(o.spectrum_bin.c_str(), &end);
        if (*end || !std::isfinite(spectrum_hz) || spectrum_hz <= 0)
            usage("invalid value \"%s\" for flag -spectrumbin: a bin width in Hz > 0", o.spectrum_bin.c_str());
    }
    if (!o.spectrum_int.empty()) {
        try {
            spectrum_ns = receiver::ParseDuration(o.spectrum_int);
        } catch (const std::exception& e) {
            usage("invalid value \"%s\" for flag -spectrumint: %s", o.spectrum_int.c_str(), e.what());
        }
        if (spectrum_ns < 0) usage("invalid value \"%s\" for flag -spectrumint: a duration >= 0", o.spectrum_int.c_str());
    }
    if (!o.spectrum_file.empty() && !(c.spectrum_out = fopen(o.spectrum_file.c_str(), "w")))
        usage("-spectrum=%s: %s", o.spectrum_file.c_str(), strerror(errno));
    c.wav_in = o.sampleformat == "wav";
    c.sigmf_in = o.sampleformat == "sigmf";
    if (!c.wav_in && !c.sigmf_in && (c.fmt = ertfmt_from_name(o.sampleformat.c_str())) < 0)
        usage("invalid value \"%s\" for flag -sampleformat: cu8, cs8, cs16, cf32, a complex SigMF datatype "
              "(ci16_be, cf64_le, ...), wav or sigmf", o.sampleformat.c_str());
    if (o.samplescale == "auto") {
        c.auto_scale = true;
    } else if (o.have_scale) {
        char* end = nullptr;
        c.scale = strtof(o.samplescale.c_str(), &end);
        if (o.samplescale.empty() || *end || !std::isfinite(c.scale) || c.scale <= 0.0f)
            usage("invalid value \"%s\" for flag -samplescale: a finite gain > 0, or auto", o.samplescale.c_str());
    }
    c.auto_channel = o.channelgain == "auto";
    if (!o.channelgain.empty() && !c.auto_channel) {
        char* end = nullptr;
        const long long g = strtoll(o.channelgain.c_str(), &end, 10);
        if (*end || g < 1 || g > (1LL << ERTRS_GAIN_K_MAX) || (g & (g - 1)))
            usage("invalid value \"%s\" for flag -channelgain: a power of two 1 ... %lld, or auto", o.channelgain.c_str(),
                  1LL << ERTRS_GAIN_K_MAX);
        c.channel_k = 63 - __builtin_clzll((unsigned long long)g);
    }
    const std::vector<std::string>& files = o.files;
    long long samplerate = o.samplerate;
    // wav: every file's header, before anything else (stdin's is consumed here, the files' are read again by the run)
    c.wav_hdr.resize(files.size());
    if (c.wav_in) {
        for (size_t fi = 0; fi < files.size(); fi++) {
            FILE* in = files[fi] == "-" ? stdin : fopen(files[fi].c_str(), "rb");
            if (!in) throw file_error(files[fi]);
            try {
                c.wav_hdr[fi] = wav::ReadHeader(in);
            } catch (const std::exception& e) {
                if (in != stdin) fclose(in);
                throw Exit{1, files[fi] + ": " + e.what()};
            }
            if (in != stdin) fclose(in);
            const wav::Header &h0 = c.wav_hdr[0], &h = c.wav_hdr[fi];
            if (h.rate != h0.rate || h.format != h0.format)
                usage("%s: %lld Hz, format %d, but %s: %lld Hz, format %d: the files of a batch share one decoder", files[0].c_str(),
                      (long long)h0.rate, h0.format, files[fi].c_str(), (long long)h.rate, h.format);
        }
        if (samplerate != 0 && samplerate != c.wav_hdr[0].rate)
            usage("-samplerate=%lld disagrees with the WAV header's %lld Hz", samplerate, (long long)c.wav_hdr[0].rate);
        samplerate = c.wav_hdr[0].rate;
        c.fmt = c.wav_hdr[0].format;
    }
    // sigmf: every recording's metadata, before anything else
    c.rec.resize(files.size());
    if (c.sigmf_in) {
        for (size_t fi = 0; fi < files.size(); fi++) {
            if (files[fi] == "-") usage("-sampleformat=sigmf reads NAME.sigmf-meta beside NAME.sigmf-data, not stdin");
            try {
                c.rec[fi] = sigmf::Read(files[fi]);
            } catch (const std::exception& e) {
                throw Exit{1, files[fi] + ": " + e.what()};
            }
            const sigmf::Recording &r0 = c.rec[0], &r = c.rec[fi];
            if (r.rate != r0.rate || r.format != r0.format || r.frequency != r0.frequency)
                usage("%s: %s at %lld Hz, %lld Hz, but %s: %s at %lld Hz, %lld Hz: the files of a batch share one decoder",
                      files[0].c_str(), ertfmt_name(r0.format), (long long)r0.rate, (long long)r0.frequency, files[fi].c_str(),
                      ertfmt_name(r.format), (long long)r.rate, (long long)r.frequency);
        }
        const sigmf::Recording& r0 = c.rec[0];
        if (samplerate != 0 && samplerate != r0.rate)
            usage("-samplerate=%lld disagrees with the SigMF core:sample_rate %lld Hz", samplerate, (long long)r0.rate);
        if (c.capture_hz != 0 && r0.frequency != 0 && c.capture_hz != r0.frequency)
            usage("-capturefreq=%lld disagrees with the SigMF core:frequency %lld Hz", c.capture_hz, (long long)r0.frequency);
        samplerate = r0.rate;
        c.fmt = r0.format;
        if (r0.frequency) c.capture_hz = r0.frequency;
    }
    c.rate = samplerate ? samplerate : c.decoder_rate;
    // -samplerate names the capture's rate; the default DataRate*ChipLength (32768 * -symbollength) resamples nothing
    c.resampling = samplerate != 0 && samplerate != c.decoder_rate;
    c.writes_samples = !o.samplefile.empty() && o.samplefile != "/dev/null";
    if (!o.centerfreq.empty() && c.capture_hz == 0) usage("-centerfreq needs -capturefreq: the frequency at the centre of the capture");
    if (!c.channels.empty() && c.writes_samples) usage("-samplefile takes one channel, not a -centerfreq list");
    for (const int64_t ch : c.channels) {   // each channel of a list lies inside the capture (ertrs_plan_decimated's rule)
        ertgpu_decimator_info d{};
        ertgpu_resampler_info info{};
        if (ertrs_plan_decimated(c.rate, c.decoder_rate, ch - c.capture_hz, &d, &info) != 0)
            usage("-centerfreq channel %lld Hz does not fit a %lld Hz capture at %lld Hz: |offset| + 0.4 * %lld Hz "
                  "must be at most half the capture's rate", (long long)ch, (long long)c.rate, c.capture_hz, (long long)c.decoder_rate);
    }
    const bool tuned = c.capture_hz > 0;
    if (!o.channelgain.empty() && !tuned)
        usage("-channelgain needs -capturefreq (or a SigMF frequency): the channel path of a tuned capture");
    if (o.have_scale && c.fmt == ERTGPU_FORMAT_CU8) usage("-samplescale does not apply to uint8 (cu8) input");
    if (tuned && c.writes_samples) usage("-samplefile does not take tuned (-capturefreq) input");
    if ((c.resampling || c.fmt != ERTGPU_FORMAT_CU8) && c.writes_samples)
        usage("-samplefile needs uint8 (cu8) input at 32768 * -symbollength = %lld Hz; this input is %s at %lld Hz",
              (long long)c.decoder_rate, ertfmt_name(c.fmt), (long long)c.rate);
    if (c.spectrum_out) {
        c.spectrum_log2 = ertspec_log2_for_bin(c.rate, spectrum_hz);
        c.spectrum_frames = ertspec_frames_per_row(c.spectrum_log2, spectrum_ns, c.rate);
    }
    return c;
}

// The batch: every file through one receiver, then the files closed.  Returns the exit status.
int run(const Options& o, Capture& c, std::chrono::steady_clock::time_point start) {
    FILE* sample = nullptr;
    if (c.writes_samples && !(sample = fopen(o.samplefile.c_str(), "wb"))) throw file_error(o.samplefile);
    const std::vector<std::string>& files = o.files;
    try {
        receiver::Receiver rcvr(o.msgtype, o.chip, o.device, o.blocks,
                                {c.resampling ? c.rate : 0, c.fmt, c.scale, c.capture_hz, c.center_hz, c.auto_scale, c.channel_k,
                                 c.auto_channel, o.signal, c.spectrum_log2, c.spectrum_frames},
                                c.channels);
        const protocol::PacketConfig& cfg = rcvr.decoder().Cfg;
        const int64_t spectrum_centre = c.capture_hz ? c.capture_hz : (int64_t)cfg.CenterFreq;
        std::vector<char> line;
        std::string log = rcvr.decoder().Log();
        if (!c.channels.empty()) {   // the channels share everything of the log but CenterFreq, its first line: name them all
            std::string names;
            for (size_t i = 0; i < c.channels.size(); i++) names += (i ? "," : "") + std::to_string(c.channels[i]);
            log = "CenterFreq: " + names + log.substr(log.find('\n'));
        }
        fputs(log.c_str(), stderr);
        if (sample) rcvr.SetSampleFile(sample);
        if (c.limit_ns) rcvr.SetDeadline(start + std::chrono::nanoseconds(c.limit_ns));
        receiver::UintMap* ids = nullptr;
        rcvr.filters() = receiver::NewFilterChain(o.filterid, o.filtertype, o.unique, &ids);
        if (o.single) rcvr.SetSingle(ids);   // main.go:278: -single empties the -filterid filter's own set
        for (size_t fi = 0; fi < files.size(); fi++) {
            const std::string& file = files[fi];
            const std::string prefix = files.size() > 1 ? file + ": " : "";
            const bool dated = c.sigmf_in && sigmf::Dated(c.rec[fi]);
            FILE* in = c.sigmf_in ? sigmf::OpenSamples(c.rec[fi]) : file == "-" ? stdin : fopen(file.c_str(), "rb");
            if (!in) throw file_error(file);
            if (fi) rcvr.Reset();
            if (c.auto_scale)
                rcvr.SetLevelReport([&](const ertgpu_input_level& lv) {
                    fprintf(stderr, "%s-samplescale=auto: 2^%d = %.9g from %lld samples\n", prefix.c_str(), lv.exponent,
                            (double)lv.scale, (long long)(lv.components / 2));
                });
            if (c.auto_channel)
                rcvr.SetChannelLevelReport([&](size_t ch, const ertgpu_channel_level& lv) {
                    ertgpu_tuning_info t{};
                    ertgpu_get_tuning(rcvr.decoder(ch).Handle(), &t);
                    fprintf(stderr, "%schannel %lld: 2^%d = %lld\n", prefix.c_str(), (long long)t.center_hz, lv.k, 1LL << lv.k);
                });
            if (c.wav_in && in != stdin) c.wav_hdr[fi] = wav::ReadHeader(in);   // the same header as before: to the samples
            std::function<void(const protocol::SpectrumRows&)> rows;
            if (c.spectrum_out)
                rows = [&](const protocol::SpectrumRows& r) {
                    for (size_t i = 0; i < r.rows.size(); i++) {
                        const int64_t s0 = r.rows[i].first_sample;
                        int64_t ns = s0 / c.rate * 1000000000 + s0 % c.rate * 1000000000 / c.rate;   // stream time
                        if (dated) ns = sigmf::BlockTime(c.rec[fi], s0 - 1, 1, c.rec[0].rate);
                        const int64_t sec = ns / 1000000000 - (ns % 1000000000 < 0);
                        const float* p = (o.spectrum_peak ? r.peak.data() : r.mean.data()) + i * (size_t)r.N;
                        const int len = ertspec_csv_line(nullptr, 0, sec, spectrum_centre, c.rate, c.spectrum_log2,
                                                         r.rows[i].frames * r.N, p);
                        line.resize((size_t)len + 1);
                        ertspec_csv_line(line.data(), line.size(), sec, spectrum_centre, c.rate, c.spectrum_log2,
                                         r.rows[i].frames * r.N, p);
                        if (fputs(line.data(), c.spectrum_out) < 0) throw std::runtime_error("writing the -spectrum file failed");
                    }
                };
            const auto st = rcvr.Run(in, o.block_dedup, [&](const protocol::Message& m, int64_t offset, int length) {
                if (o.quiet) return;
                if (c.out == receiver::PLAIN) {
                    printf("%s\n", receiver::BlockLine(m).c_str());
                    return;
                }
                receiver::LogMessage lm;
                if (dated) {
                    const int64_t ns = sigmf::BlockTime(c.rec[fi], m.Block, cfg.BlockSize, cfg.SampleRate);
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
                fputs(receiver::Line(c.out, lm).c_str(), stdout);
            }, c.wav_in ? c.wav_hdr[fi].data_size : -1, rows);
            if (in != stdin) fclose(in);
            fprintf(stderr, "%s%lld messages (%lld duplicates dropped) from %lld blocks, %.1f MB in %.3f s = %.1f Msamples/s\n",
                    prefix.c_str(), (long long)st.messages, (long long)st.duplicates, (long long)st.blocks, st.bytes / 1e6,
                    st.seconds, st.samples / 1e6 / (st.seconds > 0 ? st.seconds : 1));
            for (size_t ch = 0; ch < c.channels.size(); ch++)
                fprintf(stderr, "%s%lld Hz: %lld messages\n", prefix.c_str(), (long long)c.channels[ch],
                        (long long)st.channel_messages[ch]);
            if (st.stopped) break;
        }
    } catch (const std::exception& e) {
        fprintf(stderr, "error: %s\n", e.what());
        if (sample) fclose(sample);
        if (c.spectrum_out) fclose(c.spectrum_out);
        return 1;
    }
    if (c.spectrum_out && fclose(c.spectrum_out) != 0) {
        perror(o.spectrum_file.c_str());
        return 1;
    }
    if (sample && fclose(sample) != 0) {
        perror(o.samplefile.c_str());
        return 1;
    }
    return 0;
}

}  // namespace

int main(int argc, char** argv) {
    const auto start = std::chrono::steady_clock::now();   // main.go:350-353: the time limit covers the whole run
    try {
        const Options o = parse_flags(argc, argv);
        Capture c = resolve(o);
        return run(o, c, start);
    } catch (const Exit& e) {
        fprintf(stderr, "%s\n", e.message.c_str());
        return e.code;
    }
}
