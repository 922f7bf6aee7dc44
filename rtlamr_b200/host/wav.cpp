// wav.cpp -- see wav.hpp.
#include "wav.hpp"

#include <sys/stat.h>

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/ertgpu.h"

namespace wav {

namespace {

struct Reader {
    FILE* in;
    int64_t pos = 0;
    // n bytes or an error naming what was being read
    void get(void* dst, size_t n, const char* what) {
        if (fread(dst, 1, n, in) != n) throw std::runtime_error(std::string("WAV: truncated header (") + what + ")");
        pos += (int64_t)n;
    }
    void skip(uint64_t n, const char* what) {
        char buf[4096];
        while (n) {
            const size_t k = (size_t)std::min<uint64_t>(n, sizeof(buf));
            get(buf, k, what);
            n -= k;
        }
    }
};

uint16_t u16(const uint8_t* p) { return (uint16_t)(p[0] | p[1] << 8); }
uint32_t u32(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
uint64_t u64(const uint8_t* p) { return (uint64_t)u32(p) | (uint64_t)u32(p + 4) << 32; }

[[noreturn]] void bad(const std::string& what) { throw std::runtime_error("WAV: " + what); }

// The format of a "fmt " chunk's body (n bytes).
int32_t parse_fmt(const uint8_t* f, uint32_t n, int64_t* rate) {
    if (n < 16) bad("fmt chunk of " + std::to_string(n) + " bytes (at least 16)");
    uint32_t tag = u16(f);
    const int channels = u16(f + 2), align = u16(f + 12), bits = u16(f + 14);
    if (tag == 0xFFFE) {   // WAVE_FORMAT_EXTENSIBLE: the sub-format GUID is the tag followed by a fixed tail
        static const uint8_t tail[14] = {0x00, 0x00, 0x00, 0x00, 0x10, 0x00, 0x80, 0x00, 0x00, 0xAA, 0x00, 0x38, 0x9B, 0x71};
        if (n < 40) bad("extensible fmt chunk of " + std::to_string(n) + " bytes (at least 40)");
        if (memcmp(f + 26, tail, sizeof(tail)) != 0) bad("extensible sub-format GUID (PCM or IEEE float)");
        tag = u16(f + 24);
    }
    if (channels != 2) bad("channels " + std::to_string(channels) + " (IQ needs 2: I left, Q right)");
    int32_t format;
    if (tag == 1 && bits == 8) format = ERTGPU_FORMAT_CU8;
    else if (tag == 1 && bits == 16) format = ERTGPU_FORMAT_CS16;
    else if (tag == 3 && bits == 32) format = ERTGPU_FORMAT_CF32;
    else if (tag == 1 || tag == 3) bad("bits per sample " + std::to_string(bits) + " (8 or 16 for PCM, 32 for float)");
    else {
        char s[64];
        snprintf(s, sizeof(s), "format tag 0x%04X (PCM 1 or IEEE float 3)", tag);
        bad(s);
    }
    if (align != 2 * bits / 8) bad("block align " + std::to_string(align) + " (" + std::to_string(2 * bits / 8) + " for 2 channels)");
    *rate = u32(f + 4);
    if (*rate == 0) bad("sample rate 0");
    return format;
}

}  // namespace

Header ReadHeader(FILE* in) {
    Reader r{in};
    uint8_t h[12];
    r.get(h, 12, "RIFF");
    const bool rf64 = !memcmp(h, "RF64", 4);
    if ((!rf64 && memcmp(h, "RIFF", 4)) || memcmp(h + 8, "WAVE", 4)) bad("not a RIFF/WAVE or RF64 file");
    Header out;
    bool have_fmt = false, have_ds64 = false;
    uint64_t ds64_data = 0;
    for (;;) {
        uint8_t c[8];
        r.get(c, 8, "chunk header: no data chunk");
        const uint32_t size = u32(c + 4);
        if (!memcmp(c, "ds64", 4)) {
            if (size < 24 || size > (1u << 20)) bad("ds64 chunk of " + std::to_string(size) + " bytes (at least 24)");
            std::vector<uint8_t> b(size);
            r.get(b.data(), size, "ds64");
            ds64_data = u64(b.data() + 8);
            have_ds64 = true;
        } else if (!memcmp(c, "fmt ", 4)) {
            if (size > 1024) bad("fmt chunk of " + std::to_string(size) + " bytes");
            std::vector<uint8_t> b(size);
            r.get(b.data(), size, "fmt");
            out.format = parse_fmt(b.data(), size, &out.rate);
            have_fmt = true;
        } else if (!memcmp(c, "data", 4)) {
            if (!have_fmt) bad("data chunk before the fmt chunk");
            uint64_t n = size;
            if (rf64 && size == 0xFFFFFFFFu) {
                if (!have_ds64) bad("RF64 data size without a ds64 chunk");
                n = ds64_data;
            }
            out.data_offset = r.pos;
            out.data_size = (n == 0 || n == 0xFFFFFFFFu || n > (uint64_t)INT64_MAX) ? -1 : (int64_t)n;
            struct stat st;
            if (out.data_size > 0 && fstat(fileno(in), &st) == 0 && S_ISREG(st.st_mode) &&
                out.data_offset + out.data_size > (int64_t)st.st_size)
                out.data_size = -1;
            return out;
        } else {
            r.skip((uint64_t)size + (size & 1), "chunk body");   // an odd-sized chunk is followed by a pad byte
            continue;
        }
        if (size & 1) r.skip(1, "pad byte");
    }
}

}  // namespace wav
