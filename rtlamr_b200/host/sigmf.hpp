// sigmf.hpp -- the metadata of a SigMF recording (NAME.sigmf-meta, JSON, beside the samples in NAME.sigmf-data): the
// sample format, rate and capture frequency the decoder's input needs, the capture segments' header bytes in the data
// file, and the segments' start times, from which a decoded block gets the time it was received at.  One channel of
// complex samples; `.sigmf` archives, multi-channel datasets, retuning recordings, core:dataset and
// core:metadata_only are not taken.  Errors are std::runtime_error naming the field.
#pragma once

#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

namespace sigmf {

struct Segment {
    int64_t sample_start = 0;   // core:sample_start: the segment's first sample in the data file
    int64_t header_bytes = 0;   // core:header_bytes: skipped in the data file before that sample
    bool dated = false;         // core:datetime given
    int64_t datetime_ns = 0;    // ... as nanoseconds since 1970-01-01T00:00:00Z
};

struct Recording {
    int32_t format = 0;          // ERTGPU_FORMAT_* of core:datatype
    int64_t rate = 0;            // core:sample_rate, whole Hz
    int64_t frequency = 0;       // the segments' core:frequency in whole Hz, 0 when none gives one
    std::string data_path;       // NAME.sigmf-data
    std::vector<Segment> segments;   // ascending sample_start; at least one
    int64_t samples = 0;         // IQ samples in the data file
};

// The recording named by `path`: NAME.sigmf-meta, NAME.sigmf-data or NAME.  Checks the data file's size too.
Recording Read(const std::string& path);

// The same from the metadata's text; data_path is stored, and the data file is not opened.
Recording Parse(const std::string& json, const std::string& data_path);

// ISO 8601 as SigMF writes it, YYYY-MM-DDTHH:MM:SS[.fraction](Z|+HH:MM|-HH:MM), in nanoseconds since the Unix epoch;
// the fraction may have any number of digits and is truncated to nanoseconds.
int64_t ParseDatetime(const std::string& s);

// The ERTGPU_FORMAT_* of a complex SigMF datatype name (cu8, ci8, ci16_le, ..., cf64_be), or -1.
int32_t FormatOf(const std::string& datatype);

// The name of a format: its SigMF datatype, or cu8 / cs8 / cs16 / cf32 for the first four.
const char* FormatName(int32_t format);

// Whether any segment carries a core:datetime.
bool Dated(const Recording& r);

// The time, in nanoseconds since the Unix epoch, at which a live receiver would have finished decoder block `block`:
// the end of its last sample.  With n = (block + 1) * block_size samples at the decoder's rate rate_out and the
// recording's rate R_in, segment k is the last dated one with sample_start * rate_out <= n * R_in (the first dated one
// if there is none) and the time is datetime_k + floor((n * R_in - sample_start_k * rate_out) * 10^9 / (R_in * rate_out)),
// in exact integers.  Throws when no segment is dated.
int64_t BlockTime(const Recording& r, int64_t block, int64_t block_size, int64_t rate_out);

// A FILE that reads the recording's samples: the data file without its segments' header bytes.  fclose releases it.
FILE* OpenSamples(const Recording& r);

}  // namespace sigmf
