/* signal_ref.c -- include/ertgpu_signal.h's host half for ctypes (tests/signal_ref.py): the summary of a record and the
 * choice of the protocol whose span is measured. */
#include <string.h>

#include "ertgpu_signal.h"

int sigref_summary(const ertgpu_signal* r, int64_t channel_hz, int64_t rate_out, ertsig_summary_t* s) {
    return ertsig_summary(r, channel_hz, rate_out, s);
}

int32_t sigref_protocol(int32_t nproto, const int32_t* preamble_id, int32_t pid, uint32_t check_mask) {
    ertsig_geometry g;
    memset(&g, 0, sizeof(g));
    g.nproto = nproto;
    for (int32_t i = 0; i < nproto; i++) g.preamble_id[i] = preamble_id[i];
    return ertsig_protocol(&g, pid, check_mask);
}
