/* The format table of include/ertgpu_format.h as exported symbols, for tests/test_format_table.py. */
#include "ertgpu_format.h"

int fmtref_bytes(int32_t f) { return ertfmt_bytes(f); }
const char *fmtref_sigmf(int32_t f) { return ertfmt_sigmf(f); }
const char *fmtref_name(int32_t f) { return ertfmt_name(f); }
float fmtref_default_scale(int32_t f) { return ertfmt_default_scale(f); }
int32_t fmtref_from_sigmf(const char *s) { return ertfmt_from_sigmf(s); }
int32_t fmtref_from_name(const char *s) { return ertfmt_from_name(s); }
