// sigmf.cpp -- see sigmf.hpp.
#include "sigmf.hpp"

#include <sys/stat.h>

#include <cerrno>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <memory>
#include <sstream>
#include <stdexcept>
#include <utility>

#include "../../include/ertgpu.h"
#include "protocol.hpp"

namespace sigmf {

namespace {

[[noreturn]] void bad(const std::string& what) { throw std::runtime_error("SigMF: " + what); }

// ---- JSON (RFC 8259) ----
struct Value {
    enum Kind { kNull, kBool, kNumber, kString, kArray, kObject } kind = kNull;
    bool b = false;
    double num = 0;
    std::string str;                                  // a string, or a number's text
    std::vector<Value> items;                         // array
    std::vector<std::pair<std::string, Value>> members;   // object, in order

    const Value* get(const char* key) const {         // the last member of that name
        const Value* v = nullptr;
        for (const auto& m : members)
            if (m.first == key) v = &m.second;
        return v;
    }
};

class Parser {
public:
    explicit Parser(const std::string& s) : s_(s) {}

    Value document() {
        Value v = value(0);
        ws();
        if (i_ != s_.size()) fail("text after the top-level value");
        return v;
    }

private:
    static constexpr int kMaxDepth = 64;
    const std::string& s_;
    size_t i_ = 0;

    [[noreturn]] void fail(const std::string& what) const {
        bad("malformed metadata at byte " + std::to_string(i_) + ": " + what);
    }
    void ws() {
        while (i_ < s_.size() && (s_[i_] == ' ' || s_[i_] == '\t' || s_[i_] == '\n' || s_[i_] == '\r')) i_++;
    }
    bool eat(char c) {
        ws();
        if (i_ < s_.size() && s_[i_] == c) {
            i_++;
            return true;
        }
        return false;
    }
    void literal(const char* word) {
        const size_t n = strlen(word);
        if (s_.compare(i_, n, word) != 0) fail("invalid literal");
        i_ += n;
    }

    Value value(int depth) {
        if (depth > kMaxDepth) fail("nesting deeper than " + std::to_string(kMaxDepth));
        ws();
        if (i_ >= s_.size()) fail("unexpected end of text");
        Value v;
        const char c = s_[i_];
        if (c == '{') {
            i_++;
            v.kind = Value::kObject;
            if (eat('}')) return v;
            do {
                ws();
                if (i_ >= s_.size() || s_[i_] != '"') fail("expected a member name");
                std::string key = string();
                if (!eat(':')) fail("expected ':'");
                v.members.emplace_back(std::move(key), value(depth + 1));
            } while (eat(','));
            if (!eat('}')) fail("expected ',' or '}'");
        } else if (c == '[') {
            i_++;
            v.kind = Value::kArray;
            if (eat(']')) return v;
            do v.items.push_back(value(depth + 1));
            while (eat(','));
            if (!eat(']')) fail("expected ',' or ']'");
        } else if (c == '"') {
            v.kind = Value::kString;
            v.str = string();
        } else if (c == 't' || c == 'f') {
            literal(c == 't' ? "true" : "false");
            v.kind = Value::kBool;
            v.b = c == 't';
        } else if (c == 'n') {
            literal("null");
        } else if (c == '-' || (c >= '0' && c <= '9')) {
            v.kind = Value::kNumber;
            number(v);
        } else {
            fail(std::string("unexpected character '") + c + "'");
        }
        return v;
    }

    bool digit() const { return i_ < s_.size() && s_[i_] >= '0' && s_[i_] <= '9'; }

    // -?(0|[1-9][0-9]*)(.[0-9]+)?([eE][+-]?[0-9]+)?
    void number(Value& v) {
        const size_t start = i_;
        if (s_[i_] == '-') i_++;
        if (!digit()) fail("invalid number");
        if (s_[i_] == '0') i_++;
        else while (digit()) i_++;
        if (i_ < s_.size() && s_[i_] == '.') {
            i_++;
            if (!digit()) fail("invalid number");
            while (digit()) i_++;
        }
        if (i_ < s_.size() && (s_[i_] == 'e' || s_[i_] == 'E')) {
            i_++;
            if (i_ < s_.size() && (s_[i_] == '+' || s_[i_] == '-')) i_++;
            if (!digit()) fail("invalid number");
            while (digit()) i_++;
        }
        v.str = s_.substr(start, i_ - start);
        v.num = strtod(v.str.c_str(), nullptr);
    }

    unsigned hex4() {
        if (i_ + 4 > s_.size()) fail("truncated \\u escape");
        unsigned u = 0;
        for (int k = 0; k < 4; k++) {
            const char c = s_[i_++];
            u <<= 4;
            if (c >= '0' && c <= '9') u |= c - '0';
            else if (c >= 'a' && c <= 'f') u |= c - 'a' + 10;
            else if (c >= 'A' && c <= 'F') u |= c - 'A' + 10;
            else fail("invalid \\u escape");
        }
        return u;
    }

    static void utf8(std::string& out, unsigned cp) {
        if (cp < 0x80) {
            out += (char)cp;
        } else if (cp < 0x800) {
            out += (char)(0xC0 | cp >> 6);
            out += (char)(0x80 | (cp & 0x3F));
        } else if (cp < 0x10000) {
            out += (char)(0xE0 | cp >> 12);
            out += (char)(0x80 | (cp >> 6 & 0x3F));
            out += (char)(0x80 | (cp & 0x3F));
        } else {
            out += (char)(0xF0 | cp >> 18);
            out += (char)(0x80 | (cp >> 12 & 0x3F));
            out += (char)(0x80 | (cp >> 6 & 0x3F));
            out += (char)(0x80 | (cp & 0x3F));
        }
    }

    std::string string() {   // at the opening quote
        i_++;
        std::string out;
        for (;;) {
            if (i_ >= s_.size()) fail("unterminated string");
            const unsigned char c = (unsigned char)s_[i_];
            if (c == '"') {
                i_++;
                return out;
            }
            if (c < 0x20) fail("control character in a string");
            if (c != '\\') {
                out += (char)c;
                i_++;
                continue;
            }
            if (++i_ >= s_.size()) fail("unterminated string");
            const char e = s_[i_++];
            switch (e) {
                case '"': out += '"'; break;
                case '\\': out += '\\'; break;
                case '/': out += '/'; break;
                case 'b': out += '\b'; break;
                case 'f': out += '\f'; break;
                case 'n': out += '\n'; break;
                case 'r': out += '\r'; break;
                case 't': out += '\t'; break;
                case 'u': {
                    unsigned cp = hex4();
                    if (cp >= 0xDC00 && cp <= 0xDFFF) fail("unpaired low surrogate");
                    if (cp >= 0xD800 && cp <= 0xDBFF) {
                        if (s_.compare(i_, 2, "\\u") != 0) fail("unpaired high surrogate");
                        i_ += 2;
                        const unsigned lo = hex4();
                        if (lo < 0xDC00 || lo > 0xDFFF) fail("high surrogate without a low surrogate");
                        cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
                    }
                    utf8(out, cp);
                    break;
                }
                default: i_--; fail(std::string("invalid escape '\\") + e + "'");
            }
        }
    }
};

// A whole number >= min from a JSON number (2.4e6 is one, 2048000.5 is not).
int64_t whole(const Value* v, const std::string& field, int64_t min) {
    if (!v || v->kind != Value::kNumber) bad(field + " is not a number");
    if (!std::isfinite(v->num) || v->num != std::floor(v->num) || v->num < (double)min || v->num > 9.0e18)
        bad(field + " " + v->str + " is not a whole number" + (min > 0 ? " > 0" : " >= 0"));
    return (int64_t)v->num;
}

int64_t days_from_civil(int64_t y, int64_t m, int64_t d) {   // proleptic Gregorian, 1970-01-01 = 0
    y -= m <= 2;
    const int64_t era = (y >= 0 ? y : y - 399) / 400;
    const int64_t yoe = y - era * 400;
    const int64_t doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
    const int64_t doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
    return era * 146097 + doe - 719468;
}

int64_t floor_div(__int128 a, __int128 b) {   // b > 0
    __int128 q = a / b;
    if (a % b != 0 && a < 0) q--;
    return (int64_t)q;
}

// The data file's bytes without the segments' header bytes, for fopencookie.
struct SampleReader {
    FILE* f;
    std::vector<std::pair<int64_t, int64_t>> ext;   // (sample-byte position where an extent starts, file offset - position)
    int64_t pos = 0;                                // sample-byte position of the next read
    size_t k = 0;                                   // the extent pos is in

    static ssize_t read(void* cookie, char* buf, size_t n) {
        auto* r = static_cast<SampleReader*>(cookie);
        size_t got = 0;
        while (got < n) {
            while (r->k + 1 < r->ext.size() && r->pos >= r->ext[r->k + 1].first) {
                r->k++;
                if (fseeko(r->f, (off_t)(r->pos + r->ext[r->k].second), SEEK_SET) != 0) return got ? (ssize_t)got : -1;
            }
            size_t want = n - got;
            if (r->k + 1 < r->ext.size()) want = (size_t)std::min<int64_t>((int64_t)want, r->ext[r->k + 1].first - r->pos);
            const size_t m = fread(buf + got, 1, want, r->f);
            got += m;
            r->pos += (int64_t)m;
            if (m < want) break;
        }
        return (ssize_t)got;
    }
    static int close(void* cookie) {
        auto* r = static_cast<SampleReader*>(cookie);
        const int rc = fclose(r->f);
        delete r;
        return rc;
    }
};

}  // namespace

int32_t FormatOf(const std::string& t) {
    static const std::pair<const char*, int32_t> names[] = {
        {"cu8", ERTGPU_FORMAT_CU8},         {"ci8", ERTGPU_FORMAT_CS8},         {"ci16_le", ERTGPU_FORMAT_CS16},
        {"cf32_le", ERTGPU_FORMAT_CF32},    {"ci16_be", ERTGPU_FORMAT_CS16BE},  {"cf32_be", ERTGPU_FORMAT_CF32BE},
        {"cu16_le", ERTGPU_FORMAT_CU16},    {"cu16_be", ERTGPU_FORMAT_CU16BE},  {"ci32_le", ERTGPU_FORMAT_CS32},
        {"ci32_be", ERTGPU_FORMAT_CS32BE},  {"cu32_le", ERTGPU_FORMAT_CU32},    {"cu32_be", ERTGPU_FORMAT_CU32BE},
        {"cf64_le", ERTGPU_FORMAT_CF64},    {"cf64_be", ERTGPU_FORMAT_CF64BE}};
    for (const auto& n : names)
        if (t == n.first) return n.second;
    return -1;
}

const char* FormatName(int32_t f) {
    switch (f) {
        case ERTGPU_FORMAT_CU8: return "cu8";
        case ERTGPU_FORMAT_CS8: return "cs8";
        case ERTGPU_FORMAT_CS16: return "cs16";
        case ERTGPU_FORMAT_CF32: return "cf32";
        case ERTGPU_FORMAT_CS16BE: return "ci16_be";
        case ERTGPU_FORMAT_CF32BE: return "cf32_be";
        case ERTGPU_FORMAT_CU16: return "cu16_le";
        case ERTGPU_FORMAT_CU16BE: return "cu16_be";
        case ERTGPU_FORMAT_CS32: return "ci32_le";
        case ERTGPU_FORMAT_CS32BE: return "ci32_be";
        case ERTGPU_FORMAT_CU32: return "cu32_le";
        case ERTGPU_FORMAT_CU32BE: return "cu32_be";
        case ERTGPU_FORMAT_CF64: return "cf64_le";
        case ERTGPU_FORMAT_CF64BE: return "cf64_be";
        default: return "?";
    }
}

int64_t ParseDatetime(const std::string& s) {
    const auto fail = [&s]() { bad("core:datetime \"" + s + "\" is not ISO 8601 YYYY-MM-DDTHH:MM:SS[.fraction](Z|+HH:MM)"); };
    size_t i = 0;
    const auto num = [&](int n) {
        int64_t v = 0;
        for (int k = 0; k < n; k++, i++) {
            if (i >= s.size() || s[i] < '0' || s[i] > '9') fail();
            v = v * 10 + (s[i] - '0');
        }
        return v;
    };
    const auto sep = [&](char c) {
        if (i >= s.size() || s[i] != c) fail();
        i++;
    };
    const int64_t Y = num(4);
    sep('-');
    const int64_t Mo = num(2);
    sep('-');
    const int64_t D = num(2);
    sep('T');
    const int64_t h = num(2);
    sep(':');
    const int64_t mi = num(2);
    sep(':');
    const int64_t sec = num(2);
    int64_t frac = 0;
    if (i < s.size() && s[i] == '.') {
        i++;
        int digits = 0;
        while (i < s.size() && s[i] >= '0' && s[i] <= '9') {
            if (digits < 9) frac = frac * 10 + (s[i] - '0');
            digits++;
            i++;
        }
        if (!digits) fail();
        for (int k = digits; k < 9; k++) frac *= 10;
    }
    int64_t off = 0;
    if (i < s.size() && s[i] == 'Z') {
        i++;
    } else if (i < s.size() && (s[i] == '+' || s[i] == '-')) {
        const int64_t sign = s[i++] == '-' ? -1 : 1;
        const int64_t oh = num(2);
        sep(':');
        const int64_t om = num(2);
        if (oh > 23 || om > 59) fail();
        off = sign * (oh * 3600 + om * 60);
    } else {
        fail();
    }
    if (i != s.size()) fail();
    static const int mdays[12] = {31, 29, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31};
    const bool leap = (Y % 4 == 0 && Y % 100 != 0) || Y % 400 == 0;
    if (Mo < 1 || Mo > 12 || D < 1 || D > mdays[Mo - 1] || (Mo == 2 && D == 29 && !leap) || h > 23 || mi > 59 || sec > 59)
        fail();
    const __int128 secs = (__int128)days_from_civil(Y, Mo, D) * 86400 + h * 3600 + mi * 60 + sec - off;
    const __int128 ns = secs * 1000000000 + frac;
    if (ns > INT64_MAX || ns < INT64_MIN) bad("core:datetime \"" + s + "\" is outside the years 1678 ... 2262");
    return (int64_t)ns;
}

Recording Parse(const std::string& json, const std::string& data_path) {
    const Value doc = Parser(json).document();
    if (doc.kind != Value::kObject) bad("the metadata is not a JSON object");
    const Value* g = doc.get("global");
    if (!g || g->kind != Value::kObject) bad("global is missing or not an object");
    Recording r;
    r.data_path = data_path;
    const Value* dt = g->get("core:datatype");
    if (!dt) bad("global core:datatype is missing");
    if (dt->kind != Value::kString) bad("core:datatype is not a string");
    r.format = FormatOf(dt->str);
    if (r.format < 0) {
        if (!dt->str.empty() && dt->str[0] == 'r') bad("core:datatype \"" + dt->str + "\" is real-valued: IQ needs a complex (c...) type");
        bad("core:datatype \"" + dt->str + "\" is not a complex SigMF datatype");
    }
    if (!g->get("core:sample_rate")) bad("global core:sample_rate is missing");
    r.rate = whole(g->get("core:sample_rate"), "core:sample_rate", 1);
    if (const Value* nc = g->get("core:num_channels"))
        if (whole(nc, "core:num_channels", 0) != 1) bad("core:num_channels " + nc->str + ": one channel only");
    if (g->get("core:dataset")) bad("core:dataset (a non-conforming dataset file) is not supported");
    if (g->get("core:metadata_only")) bad("core:metadata_only: the recording has no samples");
    const Value* caps = doc.get("captures");
    if (caps && caps->kind != Value::kArray) bad("captures is not an array");
    bool have_freq = false;
    std::string freq_text;
    if (caps)
        for (size_t k = 0; k < caps->items.size(); k++) {
            const Value& c = caps->items[k];
            const std::string at = "captures[" + std::to_string(k) + "] ";
            if (c.kind != Value::kObject) bad(at + "is not an object");
            Segment sg;
            if (const Value* v = c.get("core:sample_start")) sg.sample_start = whole(v, at + "core:sample_start", 0);
            else if (k) bad(at + "core:sample_start is missing");
            if (!r.segments.empty() && sg.sample_start <= r.segments.back().sample_start)
                bad(at + "core:sample_start " + std::to_string(sg.sample_start) + " does not ascend");
            if (const Value* v = c.get("core:header_bytes")) sg.header_bytes = whole(v, at + "core:header_bytes", 0);
            if (const Value* v = c.get("core:datetime")) {
                if (v->kind != Value::kString) bad(at + "core:datetime is not a string");
                sg.datetime_ns = ParseDatetime(v->str);
                sg.dated = true;
            }
            if (const Value* v = c.get("core:frequency")) {
                if (v->kind != Value::kNumber || !std::isfinite(v->num) || v->num != std::floor(v->num) || v->num <= 0 || v->num > 9.0e18)
                    bad(at + "core:frequency " + v->str + " is not a whole number of Hz > 0");
                const int64_t f = (int64_t)v->num;
                if (have_freq && f != r.frequency)
                    bad(at + "core:frequency " + v->str + " differs from " + freq_text + ": a recording that retunes is not supported");
                have_freq = true;
                r.frequency = f;
                freq_text = v->str;
            }
            r.segments.push_back(sg);
        }
    if (r.segments.empty()) r.segments.emplace_back();
    return r;
}

Recording Read(const std::string& path) {
    std::string name = path;
    for (const char* ext : {".sigmf-meta", ".sigmf-data"})
        if (name.size() > strlen(ext) && name.compare(name.size() - strlen(ext), std::string::npos, ext) == 0)
            name.resize(name.size() - strlen(ext));
    const std::string meta = name + ".sigmf-meta";
    std::ifstream in(meta, std::ios::binary);
    if (!in) bad(meta + ": " + strerror(errno));
    std::stringstream ss;
    ss << in.rdbuf();
    Recording r = Parse(ss.str(), name + ".sigmf-data");
    struct stat st;
    if (stat(r.data_path.c_str(), &st) != 0) bad(r.data_path + ": " + strerror(errno));
    int64_t headers = 0;
    for (const Segment& s : r.segments) headers += s.header_bytes;
    const int64_t S = protocol::FormatBytes(r.format), data = (int64_t)st.st_size - headers;
    if (data < 0 || data % S)
        bad("core:header_bytes: the data file's " + std::to_string((long long)st.st_size) + " bytes less " + std::to_string(headers) +
            " header bytes are not a whole number of " + std::to_string(S) + "-byte " + FormatName(r.format) + " samples");
    r.samples = data / S;
    if (r.segments.back().sample_start > r.samples)
        bad("core:sample_start " + std::to_string(r.segments.back().sample_start) + " is past the data file's " +
            std::to_string(r.samples) + " samples");
    return r;
}

bool Dated(const Recording& r) {
    for (const Segment& s : r.segments)
        if (s.dated) return true;
    return false;
}

int64_t BlockTime(const Recording& r, int64_t block, int64_t block_size, int64_t rate_out) {
    const __int128 n_in = (__int128)(block + 1) * block_size * r.rate;   // n * R_in
    const Segment *k = nullptr, *first = nullptr;   // the segments ascend
    for (const Segment& s : r.segments) {
        if (!s.dated) continue;
        if (!first) first = &s;
        if ((__int128)s.sample_start * rate_out <= n_in) k = &s;
    }
    if (!first) bad("no capture segment has a core:datetime");
    if (!k) k = first;
    const __int128 num = (n_in - (__int128)k->sample_start * rate_out) * 1000000000;
    return k->datetime_ns + floor_div(num, (__int128)r.rate * rate_out);
}

FILE* OpenSamples(const Recording& r) {
    FILE* f = fopen(r.data_path.c_str(), "rb");
    if (!f) bad(r.data_path + ": " + strerror(errno));
    auto* rd = new SampleReader{f, {}};
    const int64_t S = protocol::FormatBytes(r.format);
    int64_t h = 0;
    rd->ext.emplace_back(0, 0);
    for (const Segment& s : r.segments) {
        h += s.header_bytes;
        rd->ext.emplace_back(s.sample_start * S, h);
    }
    if (fseeko(f, (off_t)rd->ext[0].second, SEEK_SET) != 0) {
        SampleReader::close(rd);
        bad(r.data_path + ": seek failed");
    }
    cookie_io_functions_t io{};
    io.read = &SampleReader::read;
    io.close = &SampleReader::close;
    FILE* out = fopencookie(rd, "r", io);
    if (!out) {
        SampleReader::close(rd);
        bad("fopencookie failed");
    }
    return out;
}

}  // namespace sigmf
