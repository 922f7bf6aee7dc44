// filters.hpp -- SURVEY.md section 8(f4): the receive loop's message filters and encoders, mirrored from rtlamr so that
// ertgpu_decode_file prints what `rtlamr -filterid=.. -filtertype=.. -unique=.. -format=plain|csv|json|xml` would.
//   MessageFilter / FilterChain   protocol/parse.go:126-155
//   UintMap (flag syntax)          flags.go:200-224
//   MeterIDFilter, MeterTypeFilter flags.go:226-240
//   UniqueFilter                   flags.go:242-259 (meter id -> last checksum; applied BEFORE the digest of main.go:251-253)
//   LogMessage, PlainEncoder       protocol/parse.go:103-125, flags.go:261-272
//   csv.Encoder                    csv/csv.go:27-38 over Go's encoding/csv writer rules
//   json.Encoder, xml.Encoder      flags.go:147-170 over encoding/json and encoding/xml, driven by protocol::Message::Fields()
// Time is written in UTC (Go writes local time with the same layouts).
// Header-only; nothing here touches a sample or the GPU.
#pragma once

#include <cstdint>
#include <cstdio>
#include <ctime>
#include <map>
#include <memory>
#include <set>
#include <stdexcept>
#include <string>
#include <vector>

#include "protocol.hpp"

namespace receiver {

struct MessageFilter {   // parse.go:153-155
    virtual ~MessageFilter() = default;
    virtual bool Filter(const protocol::Message& msg) = 0;
};

// flags.go:200-224: "1,2,3" -> set; anything that is not an unsigned decimal number is an error (strconv.ParseUint)
struct UintMap : std::set<uint64_t> {
    void Set(const std::string& value) {
        size_t i = 0;
        while (i <= value.size()) {
            size_t j = value.find(',', i);
            if (j == std::string::npos) j = value.size();
            const std::string v = value.substr(i, j - i);
            if (v.empty() || v.find_first_not_of("0123456789") != std::string::npos || v.size() > 20)
                throw std::invalid_argument("strconv.ParseUint: parsing \"" + v + "\": invalid syntax");
            insert(std::stoull(v));
            i = j + 1;
        }
    }
};

struct MeterIDFilter : MessageFilter {   // flags.go:226-232
    UintMap ids;
    bool Filter(const protocol::Message& msg) override { return ids.count(msg.MeterID()) != 0; }
};

struct MeterTypeFilter : MessageFilter {   // flags.go:234-240
    UintMap types;
    bool Filter(const protocol::Message& msg) override { return types.count(msg.MeterType()) != 0; }
};

struct UniqueFilter : MessageFilter {   // flags.go:242-259
    std::map<uint32_t, std::vector<uint8_t>> last;
    bool Filter(const protocol::Message& msg) override {
        const std::vector<uint8_t> checksum = msg.Checksum();
        const uint32_t mid = msg.MeterID();
        auto it = last.find(mid);
        if (it != last.end() && it->second == checksum) return false;
        last[mid] = checksum;
        return true;
    }
};

struct FilterChain {   // parse.go:126-149
    std::vector<std::shared_ptr<MessageFilter>> filters;
    void Add(std::shared_ptr<MessageFilter> f) { filters.push_back(std::move(f)); }
    bool Match(const protocol::Message& msg) {
        for (auto& f : filters)
            if (!f->Filter(msg)) return false;   // later filters are not consulted (a rejected message never reaches -unique)
        return true;
    }
    bool empty() const { return filters.empty(); }
};

// The receive loop's filter chain from -filterid, -filtertype and -unique ("" and false: the flag is not given), in the
// order flag.Visit builds it (main.go:97-113: filterid, filtertype, unique -- lexicographic, whatever the command line's
// order).  *ids, when asked for, is the MeterIDFilter's set, which -single empties (main.go:278), or nullptr without one.
inline FilterChain NewFilterChain(const std::string& filterid, const std::string& filtertype, bool unique,
                                  UintMap** ids = nullptr) {
    FilterChain fc;
    if (ids) *ids = nullptr;
    if (!filterid.empty()) {
        auto f = std::make_shared<MeterIDFilter>();
        f->ids.Set(filterid);
        fc.Add(f);
        if (ids) *ids = &f->ids;
    }
    if (!filtertype.empty()) {
        auto f = std::make_shared<MeterTypeFilter>();
        f->types.Set(filtertype);
        fc.Add(f);
    }
    if (unique) fc.Add(std::make_shared<UniqueFilter>());
    return fc;
}

// parse.go:103-125.  Time is kept as (seconds, nanoseconds) UTC; the reference formats local time with the same layouts.
struct LogMessage {
    int64_t unix_seconds = 0;
    int32_t nanos = 0;
    int64_t Offset = 0;
    int Length = 0;
    const protocol::Message* Message = nullptr;

    std::string time_layout(bool rfc3339nano) const {
        std::tm tm{};
        const time_t t = (time_t)unix_seconds;
        gmtime_r(&t, &tm);
        char buf[64];
        if (!rfc3339nano) {   // TimeFormat = "2006-01-02T15:04:05.000" (parse.go:13)
            snprintf(buf, sizeof(buf), "%04d-%02d-%02dT%02d:%02d:%02d.%03d", tm.tm_year + 1900, tm.tm_mon + 1, tm.tm_mday, tm.tm_hour,
                     tm.tm_min, tm.tm_sec, nanos / 1000000);
            return buf;
        }
        // time.RFC3339Nano: fractional seconds with trailing zeros removed, "Z" for UTC
        snprintf(buf, sizeof(buf), "%04d-%02d-%02dT%02d:%02d:%02d", tm.tm_year + 1900, tm.tm_mon + 1, tm.tm_mday, tm.tm_hour,
                 tm.tm_min, tm.tm_sec);
        std::string s = buf;
        if (nanos) {
            char f[16];
            snprintf(f, sizeof(f), ".%09d", nanos);
            std::string fs = f;
            while (fs.back() == '0') fs.pop_back();
            s += fs;
        }
        return s + "Z";
    }
    std::string String() const {   // parse.go:113-117
        return "{Time:" + time_layout(false) + " Offset:" + std::to_string(Offset) + " Length:" + std::to_string(Length) + " " +
               Message->MsgType() + ":" + Message->String() + "}";
    }
    std::string StringNoOffset() const {   // parse.go:119-121
        return "{Time:" + time_layout(false) + " " + Message->MsgType() + ":" + Message->String() + "}";
    }
    std::vector<std::string> Record() const {   // parse.go:123-129, then the signal report's five fields (-signal)
        std::vector<std::string> r = {time_layout(true), std::to_string(Offset), std::to_string(Length)};
        for (auto& f : Message->Record()) r.push_back(f);
        if (Message->Signal) {
            const protocol::SignalReport& s = *Message->Signal;
            if (s.Valid)
                for (auto& f : {std::to_string(s.Channel), std::to_string(s.Freq), Decibels(s.Level), Decibels(s.Noise), Decibels(s.SNR)})
                    r.push_back(f);
            else
                r.insert(r.end(), 5, "");
        }
        return r;
    }
    // A level in dB with two decimals, as the signal report prints it.
    static std::string Decibels(double v) {
        char b[32];
        snprintf(b, sizeof(b), "%.2f", v);
        return b;
    }
};

// ertgpu_decode_file's plain line: {Block:B Idx:I TYPE:{...}}, with -signal {Block:B Idx:I Channel:C Freq:F Level:L
// Noise:N SNR:S TYPE:{...}} ("-" for each of the five when the packet has no summary).
inline std::string BlockLine(const protocol::Message& m) {
    std::string s = "{Block:" + std::to_string(m.Block) + " Idx:" + std::to_string(m.Idx) + " ";
    if (m.Signal) {
        const protocol::SignalReport& r = *m.Signal;
        if (r.Valid)
            s += "Channel:" + std::to_string(r.Channel) + " Freq:" + std::to_string(r.Freq) + " Level:" + LogMessage::Decibels(r.Level) +
                 " Noise:" + LogMessage::Decibels(r.Noise) + " SNR:" + LogMessage::Decibels(r.SNR) + " ";
        else
            s += "Channel:- Freq:- Level:- Noise:- SNR:- ";
    }
    return s + m.MsgType() + ":" + m.String() + "}";
}

// flags.go:261-272: StringNoOffset when the sample file is os.DevNull (the default), String otherwise
inline std::string PlainLine(const LogMessage& m, bool sample_file_is_devnull) {
    return sample_file_is_devnull ? m.StringNoOffset() : m.String();
}

// One record in Go's encoding/csv writer format (Comma = ',', UseCRLF = false), csv/csv.go:36: a field is quoted when it
// is `\.`, contains the delimiter, a quote, CR or LF, or starts with a space; quotes are doubled; "" stays unquoted.
inline std::string CsvLine(const std::vector<std::string>& fields) {
    std::string out;
    for (size_t n = 0; n < fields.size(); n++) {
        const std::string& f = fields[n];
        if (n) out += ',';
        bool quote = false;
        if (!f.empty()) {
            quote = f == "\\." || f.find_first_of(",\"\r\n") != std::string::npos || f[0] == ' ' || f[0] == '\t';
        }
        if (!quote) {
            out += f;
            continue;
        }
        out += '"';
        for (char c : f) {
            if (c == '"') out += "\"\"";
            else out += c;   // UseCRLF = false: CR and LF are written as they are
        }
        out += '"';
    }
    return out + "\n";
}

// A JSON string as encoding/json writes it.  Every string the encoders produce (RFC3339 time, message type, standard
// base64) is plain ASCII without `"`, `\`, control characters or the `<`, `>`, `&` that Go's HTML escaping would rewrite:
// anything else is a programming error here, not something to escape.
inline std::string JsonString(const std::string& s) {
    for (unsigned char c : s)
        if (c < 0x20 || c >= 0x7F || c == '"' || c == '\\' || c == '<' || c == '>' || c == '&')
            throw std::logic_error("JsonString: \"" + s + "\" would need escaping");
    return "\"" + s + "\"";
}

// encoding/base64.StdEncoding, which encoding/json uses for a []byte
inline std::string Base64(const std::vector<uint8_t>& b) {
    static const char* A = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
    std::string out;
    for (size_t i = 0; i < b.size(); i += 3) {
        const uint32_t v = (uint32_t)b[i] << 16 | (i + 1 < b.size() ? (uint32_t)b[i + 1] << 8 : 0) | (i + 2 < b.size() ? b[i + 2] : 0);
        out += A[v >> 18];
        out += A[(v >> 12) & 63];
        out += i + 1 < b.size() ? A[(v >> 6) & 63] : '=';
        out += i + 2 < b.size() ? A[v & 63] : '=';
    }
    return out;
}

// json.NewEncoder(os.Stdout).Encode(logMsg), flags.go:147-148: one compact object per line, keys in struct order.  The
// embedded Message is an interface, which encoding/json does not flatten, so the message is a nested object.
inline std::string JsonLine(const LogMessage& m) {
    std::string s = "{\"Time\":" + JsonString(m.time_layout(true)) + ",\"Offset\":" + std::to_string(m.Offset) +
                    ",\"Length\":" + std::to_string(m.Length) + ",\"Type\":" + JsonString(m.Message->MsgType()) + ",\"Message\":{";
    bool first = true;
    for (const protocol::Field& f : m.Message->Fields()) {
        s += (first ? "\"" : ",\"") + std::string(f.Name) + "\":";
        first = false;
        if (f.kind == protocol::Field::UINT) {
            s += std::to_string(f.Uint);
        } else if (f.kind == protocol::Field::BYTES) {
            s += JsonString(Base64(f.Bytes));
        } else {
            s += '[';
            for (size_t i = 0; i < f.Uint16s.size(); i++) s += (i ? "," : "") + std::to_string(f.Uint16s[i]);
            s += ']';
        }
    }
    s += '}';
    if (m.Message->Signal) {   // -signal: the report after the message, null without a summary
        const protocol::SignalReport& r = *m.Message->Signal;
        s += ",\"Signal\":";
        s += r.Valid ? "{\"Channel\":" + std::to_string(r.Channel) + ",\"Freq\":" + std::to_string(r.Freq) + ",\"Level\":" +
                           LogMessage::Decibels(r.Level) + ",\"Noise\":" + LogMessage::Decibels(r.Noise) + ",\"SNR\":" +
                           LogMessage::Decibels(r.SNR) + "}"
                     : "null";
    }
    return s + "}\n";
}

// xml.EscapeText / printer.EscapeString: the five markup characters, tab, LF and CR become character references; a byte
// that does not start valid UTF-8, and a rune outside XML's Char production, become U+FFFD.  Runes are decoded the way
// utf8.DecodeRune does: an invalid sequence consumes one byte.
inline std::string XmlEscape(const uint8_t* p, size_t n) {
    std::string out;
    size_t i = 0;
    while (i < n) {
        const uint8_t c = p[i];
        uint32_t r = 0xFFFD;
        size_t w = 1;
        if (c < 0x80) {
            r = c;
        } else {
            const size_t need = c >= 0xC2 && c <= 0xDF ? 2 : c >= 0xE0 && c <= 0xEF ? 3 : c >= 0xF0 && c <= 0xF4 ? 4 : 0;
            if (need && i + need <= n) {
                // second byte's range depends on the lead byte (no overlong forms, no surrogates, nothing above U+10FFFF)
                const uint8_t lo = c == 0xE0 ? 0xA0 : c == 0xF0 ? 0x90 : 0x80;
                const uint8_t hi = c == 0xED ? 0x9F : c == 0xF4 ? 0x8F : 0xBF;
                bool ok = p[i + 1] >= lo && p[i + 1] <= hi;
                for (size_t k = 2; ok && k < need; k++) ok = (p[i + k] & 0xC0) == 0x80;
                if (ok) {
                    r = need == 2 ? (c & 0x1Fu) : need == 3 ? (c & 0x0Fu) : (c & 0x07u);
                    for (size_t k = 1; k < need; k++) r = r << 6 | (p[i + k] & 0x3Fu);
                    w = need;
                }
            }
        }
        const bool valid = w > 1 || c < 0x80;
        switch (r) {
        case '"': out += "&#34;"; break;
        case '\'': out += "&#39;"; break;
        case '&': out += "&amp;"; break;
        case '<': out += "&lt;"; break;
        case '>': out += "&gt;"; break;
        case '\t': out += "&#x9;"; break;
        case '\n': out += "&#xA;"; break;
        case '\r': out += "&#xD;"; break;
        default: {
            const bool in_char = r >= 0x20 && (r <= 0xD7FF || (r >= 0xE000 && r <= 0xFFFD) || r >= 0x10000);
            if (valid && in_char) out.append((const char*)p + i, w);
            else out += "\xEF\xBF\xBD";
        }
        }
        i += w;
    }
    return out;
}

// NewLineEncoder{xml.NewEncoder(os.Stdout)}.Encode(logMsg), flags.go:149-170, then the newline it prints.  The embedded
// Message interface is not flattened: it is a child element named after the field.  A field tagged `,attr` is an
// attribute; an untagged one is a child element, once per item for an array; a []byte is character data.  Go never
// writes a self-closing tag.
inline std::string XmlLine(const LogMessage& m) {
    const auto esc = [](const std::string& s) { return XmlEscape((const uint8_t*)s.data(), s.size()); };
    std::string s = "<LogMessage Time=\"" + esc(m.time_layout(true)) + "\" Offset=\"" + std::to_string(m.Offset) + "\" Length=\"" +
                    std::to_string(m.Length) + "\" Type=\"" + esc(m.Message->MsgType()) + "\"><Message";
    const std::vector<protocol::Field> fields = m.Message->Fields();
    for (const protocol::Field& f : fields)
        if (f.XmlAttr) s += " " + std::string(f.XmlAttr) + "=\"" + std::to_string(f.Uint) + "\"";
    s += '>';
    for (const protocol::Field& f : fields) {
        if (f.XmlAttr) continue;
        const std::string open = "<" + std::string(f.Name) + ">", close = "</" + std::string(f.Name) + ">";
        if (f.kind == protocol::Field::UINT) s += open + std::to_string(f.Uint) + close;
        else if (f.kind == protocol::Field::BYTES) s += open + XmlEscape(f.Bytes.data(), f.Bytes.size()) + close;
        else
            for (uint16_t v : f.Uint16s) s += open + std::to_string(v) + close;
    }
    s += "</Message>";
    if (m.Message->Signal) {   // -signal: a child element after the message, without attributes when there is no summary
        const protocol::SignalReport& r = *m.Message->Signal;
        s += "<Signal";
        if (r.Valid)
            s += " Channel=\"" + std::to_string(r.Channel) + "\" Freq=\"" + std::to_string(r.Freq) + "\" Level=\"" +
                 LogMessage::Decibels(r.Level) + "\" Noise=\"" + LogMessage::Decibels(r.Noise) + "\" SNR=\"" +
                 LogMessage::Decibels(r.SNR) + "\"";
        s += "></Signal>";
    }
    return s + "</LogMessage>\n";
}

// -format (flags.go:140-170), with erthost_encode's values; a fixed underlying type, so that any other int the C surface
// is given converts to a value that is none of the four and is encoded as plain.
enum Format : int { PLAIN = 0, CSV = 1, JSON = 2, XML = 3 };

// The csv, json or xml line of a message.  The plain line is not here: each caller has its own (PlainLine, BlockLine).
inline std::string Line(Format f, const LogMessage& m) {
    switch (f) {
    case CSV: return CsvLine(m.Record());
    case JSON: return JsonLine(m);
    case XML: return XmlLine(m);
    default: throw std::logic_error("Line: the plain line is the caller's");
    }
}

}  // namespace receiver
