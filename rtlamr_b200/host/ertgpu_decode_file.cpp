// ertgpu_decode_file -- decode a raw uint8 IQ capture (rtl_sdr / rtlamr -samplefile format) or stdin
// through the C++ mirror of rtlamr's receive loop (receiver.hpp) on the GPU and print one line per message
// in rtlamr's plain format without the time fields (protocol/parse.go:119-121 StringNoOffset).
//   ertgpu_decode_file [-msgtype=scm,idm|all] [-symbollength=72] [-blockdedup=true] [-blocks=4096] [-device=0]
//                      [-filterid=1,2] [-filtertype=4,5] [-unique=true] [-format=plain|csv|json|xml]
//                      [-samplefile=PATH] [-single] [-duration=1h5m10s] [-samplerate=HZ] FILE|- [FILE ...]
// -samplerate is rtlamr's (rtltcp's) flag name; here it names the capture's sample rate.  The default,
// 32768 * -symbollength, decodes the bytes as they are; any other rate within 1/4 ... 4 times it is resampled
// exactly on the GPU first, and Block / Idx then count resampled samples.  It cannot be combined with -samplefile.
// -filterid / -filtertype / -unique, -format, -samplefile, -single and -duration are rtlamr's flags of the same names
// (flags.go:37-58,69-70,140-170; the filter chain runs before the cross-block dedup, main.go:236-260).  With -format=csv a
// line is LogMessage.Record() (parse.go:123-129: time, offset, length, then the message's own record) through Go's
// encoding/csv rules; json and xml are the lines of Go's encoding/json and encoding/xml encoders (filters.hpp).  Time is
// written in UTC.  Offset and Length are 0 unless -samplefile names a file.
// -single stops after the first reported message or, with -filterid, once every listed meter has reported.  -duration
// (Go duration syntax, 0 = no limit) is checked before each read of -blocks blocks: the call in progress is decoded and
// reported in full, so the run can last one call longer than asked.  Both end the run with exit status 0.
// Several files are a batch of independent streams through ONE decoder (buffers, tables and kernels set up once):
// each starts from zeroed history with block numbers from 0, exactly as if it were decoded alone.  They share the
// sample file, whose offsets keep growing from one file to the next.
#include <chrono>
#include <cstdio>
#include <cstring>
#include <ctime>
#include <iostream>
#include <vector>

#include "receiver.hpp"

int main(int argc, char** argv) {
    const auto start = std::chrono::steady_clock::now();   // main.go:350-353: the time limit covers the whole run
    std::string msgtype = "scm";
    std::vector<std::string> files;
    int chip = 72, device = 0;
    long long blocks = 4096, samplerate = 0;
    bool block_dedup = true, quiet = false, unique = false, single = false;
    std::string filterid, filtertype, format = "plain", samplefile, duration;
    for (int i = 1; i < argc; i++) {
        std::string a = argv[i];
        if (a.rfind("-msgtype=", 0) == 0) msgtype = a.substr(9);
        else if (a.rfind("-symbollength=", 0) == 0) chip = atoi(a.c_str() + 14);
        else if (a.rfind("-device=", 0) == 0) device = atoi(a.c_str() + 8);
        else if (a.rfind("-samplerate=", 0) == 0) samplerate = atoll(a.c_str() + 12);
        else if (a.rfind("-blocks=", 0) == 0) blocks = atoll(a.c_str() + 8);
        else if (a.rfind("-blockdedup=", 0) == 0) block_dedup = a.substr(12) != "false";
        else if (a.rfind("-filterid=", 0) == 0) filterid = a.substr(10);
        else if (a.rfind("-filtertype=", 0) == 0) filtertype = a.substr(12);
        else if (a.rfind("-unique=", 0) == 0) unique = a.substr(8) == "true";
        else if (a == "-unique") unique = true;
        else if (a.rfind("-format=", 0) == 0) format = a.substr(8);
        else if (a.rfind("-samplefile=", 0) == 0) samplefile = a.substr(12);
        else if (a.rfind("-single=", 0) == 0) single = a.substr(8) == "true";
        else if (a == "-single") single = true;
        else if (a.rfind("-duration=", 0) == 0) duration = a.substr(10);
        else if (a == "-quiet") quiet = true;
        else files.push_back(a);
    }
    if (files.empty()) {
        fprintf(stderr, "usage: %s [-msgtype=scm,scm+,idm,netidm,r900,r900bcd|all] [-symbollength=N] [-blockdedup=true|false] "
                        "[-blocks=K] [-device=D] [-filterid=ID,..] [-filtertype=T,..] [-unique=true|false] [-format=plain|csv|json|xml] "
                        "[-samplefile=PATH] [-single] [-duration=D] [-samplerate=HZ] [-quiet] FILE|- [FILE ...]\n", argv[0]);
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
    // -samplerate names the capture's rate; the default DataRate*ChipLength (32768 * -symbollength) resamples nothing
    const bool resampling = samplerate != 0 && samplerate != 32768LL * chip;
    if (resampling && !samplefile.empty() && samplefile != "/dev/null") {
        fprintf(stderr, "-samplefile cannot be combined with -samplerate=%lld (the capture is not at 32768 * -symbollength = %lld Hz)\n",
                samplerate, 32768LL * chip);
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
        receiver::Receiver rcvr(msgtype, chip, device, blocks, resampling ? samplerate : 0);
        fputs(rcvr.decoder().Log().c_str(), stderr);
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
            FILE* in = file == "-" ? stdin : fopen(file.c_str(), "rb");
            if (!in) {
                perror(file.c_str());
                return 1;
            }
            if (fi) rcvr.Reset();
            auto st = rcvr.Run(in, block_dedup, [&](const protocol::Message& m, int64_t offset, int length) {
                if (quiet) return;
                if (csv || json || xml) {
                    receiver::LogMessage lm;
                    timespec ts{};
                    clock_gettime(CLOCK_REALTIME, &ts);
                    lm.unix_seconds = (int64_t)ts.tv_sec;
                    lm.nanos = (int32_t)ts.tv_nsec;
                    lm.Offset = offset;
                    lm.Length = length;
                    lm.Message = &m;
                    fputs((csv ? receiver::CsvLine(lm.Record()) : json ? receiver::JsonLine(lm) : receiver::XmlLine(lm)).c_str(), stdout);
                } else {
                    printf("{Block:%lld Idx:%d %s:%s}\n", (long long)m.Block, m.Idx, m.MsgType().c_str(), m.String().c_str());
                }
            });
            if (in != stdin) fclose(in);
            fprintf(stderr, "%s%s%lld messages (%lld duplicates dropped) from %lld blocks, %.1f MB in %.3f s = %.1f Msamples/s\n",
                    files.size() > 1 ? file.c_str() : "", files.size() > 1 ? ": " : "", (long long)st.messages,
                    (long long)st.duplicates, (long long)st.blocks, st.bytes / 1e6, st.seconds,
                    st.bytes / 2e6 / (st.seconds > 0 ? st.seconds : 1));
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
