/*
 * ertgpu_format.h -- the input sample formats (ERTGPU_FORMAT_*, ertgpu_set_input_format) as one table shared by
 * libertgpu.so, the host mirror, ertgpu_decode_file and the CPU test harness.  Per format: bytes per IQ sample, its
 * complex SigMF datatype, the short name kernel labels and messages use (cu8, cs8, cs16, cf32; the SigMF datatype for
 * the others), and the default gain, which maps full scale to full scale (0 for cu8, which is not scaled).
 */
#ifndef ERTGPU_FORMAT_H
#define ERTGPU_FORMAT_H

#include <stdint.h>
#include <string.h>

#include "ertgpu.h"

#if defined(__CUDACC__)
#define ERTFMT_HD __host__ __device__ constexpr
#elif defined(__cplusplus)
#define ERTFMT_HD constexpr
#else
#define ERTFMT_HD static inline
#endif

/* X(format, bytes per sample, SigMF datatype, short name, default gain) */
#define ERTFMT_TABLE(X)                                                      \
    X(ERTGPU_FORMAT_CU8, 2, "cu8", "cu8", 0.0f)                              \
    X(ERTGPU_FORMAT_CS8, 2, "ci8", "cs8", 1.0f)                              \
    X(ERTGPU_FORMAT_CS16, 4, "ci16_le", "cs16", 1.0f / 256.0f)               \
    X(ERTGPU_FORMAT_CF32, 8, "cf32_le", "cf32", 128.0f)                      \
    X(ERTGPU_FORMAT_CS16BE, 4, "ci16_be", "ci16_be", 1.0f / 256.0f)          \
    X(ERTGPU_FORMAT_CF32BE, 8, "cf32_be", "cf32_be", 128.0f)                 \
    X(ERTGPU_FORMAT_CU16, 4, "cu16_le", "cu16_le", 1.0f / 256.0f)            \
    X(ERTGPU_FORMAT_CU16BE, 4, "cu16_be", "cu16_be", 1.0f / 256.0f)          \
    X(ERTGPU_FORMAT_CS32, 8, "ci32_le", "ci32_le", 1.0f / 16777216.0f)       \
    X(ERTGPU_FORMAT_CS32BE, 8, "ci32_be", "ci32_be", 1.0f / 16777216.0f)     \
    X(ERTGPU_FORMAT_CU32, 8, "cu32_le", "cu32_le", 1.0f / 16777216.0f)       \
    X(ERTGPU_FORMAT_CU32BE, 8, "cu32_be", "cu32_be", 1.0f / 16777216.0f)     \
    X(ERTGPU_FORMAT_CF64, 16, "cf64_le", "cf64_le", 128.0f)                  \
    X(ERTGPU_FORMAT_CF64BE, 16, "cf64_be", "cf64_be", 128.0f)

#define ERTFMT_BYTES_(F, B, S, N, G) f == F ? B:
#define ERTFMT_SIGMF_(F, B, S, N, G) f == F ? S:
#define ERTFMT_NAME_(F, B, S, N, G) f == F ? N:
#define ERTFMT_SCALE_(F, B, S, N, G) f == F ? G:
#define ERTFMT_FROM_SIGMF_(F, B, S, N, G) !strcmp(s, S) ? F:
#define ERTFMT_FROM_NAME_(F, B, S, N, G) !strcmp(s, N) || !strcmp(s, S) ? F:

/* Bytes per IQ sample of a format; 0 for an unknown one. */
ERTFMT_HD int ertfmt_bytes(int32_t f) { return ERTFMT_TABLE(ERTFMT_BYTES_) 0; }

/* The SigMF datatype of a format; NULL for an unknown one. */
static inline const char *ertfmt_sigmf(int32_t f) { return ERTFMT_TABLE(ERTFMT_SIGMF_) NULL; }

/* The short name of a format; NULL for an unknown one. */
static inline const char *ertfmt_name(int32_t f) { return ERTFMT_TABLE(ERTFMT_NAME_) NULL; }

/* The default gain of a format. */
static inline float ertfmt_default_scale(int32_t f) { return ERTFMT_TABLE(ERTFMT_SCALE_) 0.0f; }

/* The format of a complex SigMF datatype; -1 for any other string. */
static inline int32_t ertfmt_from_sigmf(const char *s) { return ERTFMT_TABLE(ERTFMT_FROM_SIGMF_) - 1; }

/* The format of a -sampleformat name: a short name or a SigMF datatype; -1 for any other string. */
static inline int32_t ertfmt_from_name(const char *s) { return ERTFMT_TABLE(ERTFMT_FROM_NAME_) - 1; }

#undef ERTFMT_BYTES_
#undef ERTFMT_SIGMF_
#undef ERTFMT_NAME_
#undef ERTFMT_SCALE_
#undef ERTFMT_FROM_SIGMF_
#undef ERTFMT_FROM_NAME_

#endif
