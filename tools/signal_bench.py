"""Cost of per-packet signal reports (ertgpu_enable_signal): the device-resident step of bench.py (reset, one
ertgpu_decode_device_async over the resident synthetic IQ, the counters read back) on two handles of the same geometry,
one with reports and one without, alternated in one run.

Cases: scm at 1 GiB with 512 injected packets (BASELINE configs[1]), scm,scm+,idm at 8 GiB (configs[2]), and the same
1 GiB scm,scm+,idm stream with every candidate returned (flags 0), which adds the noise hits to the records.  Prints one
JSON line with the card's name and power limit (read in the same run) and, per case, the candidates per step, the median
step time of each handle over --reps alternated runs of --steps steps, and packet_signal_kernel's time per step from
torch.profiler in a run of its own.
Usage: python tools/signal_bench.py [--reps 5] [--steps 10] [--only NAME]"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from rtlamr_b200 import capi, synth  # noqa: E402
from resample_bench import power_limit_w  # noqa: E402

CL = 72
CASES = [("scm_1GiB", "scm", 1 << 30, 512, capi.DECODE_ONLY_VALID),
         ("scm_scmplus_idm_8GiB", "scm,scm+,idm", 8 << 30, 4096, capi.DECODE_ONLY_VALID),
         ("scm_scmplus_idm_1GiB_all_candidates", "scm,scm+,idm", 1 << 30, 512, 0)]


def step(h, d, nbytes, flags, st):
    h.reset()
    h.decode_device_async(d.data_ptr(), nbytes, flags, st.cuda_stream)
    return h.last_counts()


def run_case(name, mt, nbytes, npk, flags, reps, steps):
    probe = capi.new_decoder(mt, CL, max_blocks_per_call=1)
    bs, bs2 = probe.cfg.block_size, probe.cfg.block_size2
    probe.close()
    nbytes = nbytes // bs2 * bs2
    nblocks, nsamples = nbytes // bs2, nbytes // 2
    pk, _ = synth.make_packets(mt, CL, nsamples, seed=1, spacing=nsamples // npk)
    d = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    capi.synth_fill(0, d.data_ptr(), 0, nsamples, 0x5EED0001, pk)
    hs = {False: capi.new_decoder(mt, CL, max_blocks_per_call=nblocks, max_candidates=1 << 20),
          True: capi.new_decoder(mt, CL, max_blocks_per_call=nblocks, max_candidates=1 << 20, signal=True)}
    st = torch.cuda.Stream()
    for h in hs.values():
        for _ in range(2):
            step(h, d, nbytes, flags, st)
    assert hs[True].fetch(1 << 20).tobytes() == hs[False].fetch(1 << 20).tobytes()
    cands = step(hs[True], d, nbytes, flags, st)[0]
    times = {False: [], True: []}
    for r in range(reps):
        for sig in ((False, True) if r % 2 == 0 else (True, False)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                step(hs[sig], d, nbytes, flags, st)
            times[sig].append((time.perf_counter() - t0) / steps * 1e3)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step(hs[True], d, nbytes, flags, st)
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "packet_signal_kernel" in e.key) / steps
    for h in hs.values():
        h.close()
    base, with_sig = statistics.median(times[False]), statistics.median(times[True])
    return {"case": name, "msgtype": mt, "bytes": nbytes, "flags": flags, "candidates": int(cands),
            "step_ms_without": round(base, 4), "step_ms_with": round(with_sig, 4),
            "ratio": round(with_sig / base, 4), "steps_ms_without": [round(t, 4) for t in times[False]],
            "steps_ms_with": [round(t, 4) for t in times[True]], "packet_signal_kernel_us": round(us, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--only", default="")
    a = ap.parse_args()
    out = [run_case(*c, a.reps, a.steps) for c in CASES if not a.only or c[0] == a.only]
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "cases": out}))


if __name__ == "__main__":
    main()
