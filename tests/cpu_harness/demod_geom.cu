// Host-only harness for tests/test_search_params.py: compile-time geometry of demod_fast_kernel for every
// specialised chip length (rtlamr_b200/csrc/demod_fast.cuh).  No kernel is launched.
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "../../rtlamr_b200/csrc/demod_fast.cuh"

template <int CL>
void row(bool first) {
    using G = ert::FastGeom<CL>;
    const int W = ert::fast_warps<CL>();
    printf("%s{\"CL\":%d,\"L\":%d,\"pad\":%d,\"row_bytes\":%d,\"stages\":%d,\"warps\":%d,\"tail_bits\":%d,"
           "\"smem\":%d,\"smem7\":%d,\"variant\":%d}",
           first ? "" : ",", CL, G::L, G::kPad, G::kRowBytes, G::kStages, W, G::kTailBits,
           ert::fast_smem_bytes<G>(W, 1024), ert::fast_smem_bytes<G>(W == 8 ? 7 : W, 1024),
           ert::demod_fast_variant(CL, 4096));
}

// work-tile plan of a launch: "plan NTILES SMS W" prints how many tiles go out dynamically and checks that the
// pre-assigned rest covers every remaining tile exactly once with at most one tile per (SM, scheduler)
int plan(long long ntiles, long long sms, int W) {
    long long grid = (ntiles + W - 1) / W;
    if (grid > sms) grid = sms;
    const long long dyn = ert::fast_dynamic_tiles(ntiles, grid, W);
    long long covered = 0, per_sched_max = 0;
    bool dup = false;
    if (dyn < ntiles) {
        std::vector<char> seen((size_t)(ntiles - dyn), 0);
        for (long long cta = 0; cta < grid; cta++)
            for (int w = 0; w < 4 && w < W; w++) {   // the kernel: warp w < 4 of CTA cta takes tile dyn + cta + grid * w
                const long long s = dyn + cta + grid * w;
                if (s < ntiles) {
                    if (seen[(size_t)(s - dyn)]) dup = true;
                    seen[(size_t)(s - dyn)] = 1;
                    covered++;
                    per_sched_max = 1;
                }
            }
    }
    printf("{\"ntiles\":%lld,\"grid\":%lld,\"W\":%d,\"dyn\":%lld,\"static_covered\":%lld,\"dup\":%s,\"per_sched_max\":%lld,"
           "\"cost7\":%.3f,\"cost8\":%.3f}\n",
           ntiles, grid, W, dyn, covered, dup ? "true" : "false", per_sched_max, ert::fast_round_cost(ntiles, sms, 7),
           ert::fast_round_cost(ntiles, sms, 8));
    return 0;
}

int main(int argc, char** argv) {
    if (argc == 5 && std::string(argv[1]) == "plan") return plan(atoll(argv[2]), atoll(argv[3]), atoi(argv[4]));
    printf("[");
    row<32>(true); row<40>(false); row<48>(false); row<56>(false); row<64>(false);
    row<72>(false); row<78>(false); row<80>(false); row<88>(false); row<96>(false);
    printf("]\n");
    return 0;
}
