// wav.hpp -- the header of a baseband WAV recording (SDR#, SDR++, SDRuno, HDSDR): RIFF/WAVE or RF64, two channels
// (I left, Q right) of 8-bit unsigned PCM, 16-bit signed PCM or 32-bit float, plain or WAVE_FORMAT_EXTENSIBLE.
// The header is read from the stream in order, never seeking, so a pipe or stdin works; the stream is left at the
// first byte of the samples.
#pragma once

#include <cstdint>
#include <cstdio>

namespace wav {

struct Header {
    int32_t format = 0;        // ERTGPU_FORMAT_CU8 (8-bit PCM), _CS16 (16-bit PCM) or _CF32 (float32)
    int64_t rate = 0;          // samples per second
    int64_t data_offset = 0;   // bytes before the first sample
    int64_t data_size = -1;    // bytes of samples; -1: to the end of the stream
};

// Parse the header; throws std::runtime_error naming the field that cannot be decoded (mono, 24-bit, A-law, a
// truncated header, ...).  A data size of 0 or 0xFFFFFFFF, or one that runs past the end of a regular file, reads
// to the end of the stream: a recording that was cut off, or that passed 4 GiB without RF64, leaves such a size.
Header ReadHeader(FILE* in);

}  // namespace wav
