/* The gain rule of include/ertgpu_level.h as an exported symbol, for tests/test_input_level.py. */
#include "ertgpu_level.h"

int32_t lvref_exponent(const int64_t *bins, int64_t components, int64_t zeros, int64_t nans, int32_t default_k) {
    return ertlv_exponent(bins, components, zeros, nans, default_k);
}

int32_t lvref_window(void) { return ERTLV_WINDOW; }
