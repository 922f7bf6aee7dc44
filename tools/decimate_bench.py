"""Throughput of the decimating tuned input: scm, the channel 2.4 MHz below the capture's centre, fed about 1 GiB of
cs16 at 30.72 and 61.44 MS/s (chip length 72, D = 4 and 7) and cs8 at 20 MS/s (chip length 32, D = 5), with the
one-stage tuned resampler on cs8 at 10:1 (23.59 MS/s, chip length 72) measured in the same run for comparison.

Prints one JSON line with the card's name and power limit (read in the same run) and, per case,
  - decimate_kernel's and resample_kernel's own times (torch.profiler), and the input Gsamples/s of the two together,
  - the whole device-resident step (CUDA events),
  - end to end from pinned host memory.
Usage: python tools/decimate_bench.py [--gib 1] [--reps 5]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from rtlamr_b200 import capi  # noqa: E402
from resample_bench import power_limit_w  # noqa: E402

CAPTURE, OFFSET = 915_000_000, -2_400_000


def run_case(name, rate_in, cl, fmt, nbytes, reps):
    flags = capi.DECODE_ONLY_VALID
    s = capi.FORMAT_BYTES[fmt]
    nbytes = nbytes // (8192 * s) * (8192 * s)
    nsamples = nbytes // s
    g = torch.Generator(device="cuda").manual_seed(1)
    d = torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device="cuda", generator=g)
    host = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
    host.copy_(d)
    torch.cuda.synchronize()
    out_blocks = int(nsamples * 32768 * cl / rate_in) // 2048 + 2
    h = capi.new_decoder("scm", cl, max_blocks_per_call=out_blocks, max_candidates=1 << 20, input_rate=rate_in,
                         input_format=fmt, capture_freq=CAPTURE, center_freq=CAPTURE + OFFSET)
    st = torch.cuda.Stream()

    def device_step():
        h.reset()
        h.decode_device_async(d.data_ptr(), nbytes, flags, st.cuda_stream)
        h.fetch(cap=1 << 20)

    for _ in range(2):
        device_step()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        h.reset()
        e0.record(st)
        h.decode_device_async(d.data_ptr(), nbytes, flags, st.cuda_stream)
        e1.record(st)
        h.fetch(cap=1 << 20)
        ms.append(e0.elapsed_time(e1))
    kernels = h.last_kernels()
    from torch.profiler import ProfilerActivity, profile
    dc_us, rs_us = [], []
    for _ in range(reps):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            device_step()
            torch.cuda.synchronize()
        dc_us.append(sum(e.device_time for e in prof.events() if "decimate_kernel" in e.name))
        rs_us.append(sum(e.device_time for e in prof.events() if "resample_kernel" in e.name))

    def e2e_once():
        h.reset()
        t0 = time.perf_counter()
        h.decode((host.data_ptr(), nbytes), flags, 1 << 20)
        return time.perf_counter() - t0

    e2e_once()
    te = [e2e_once() for _ in range(reps)]
    dec, _ = h.decimator()
    info, _ = h.resampler()
    step_ms = float(np.median(ms))
    dc_ms, rs_ms = float(np.median(dc_us)) / 1e3, float(np.median(rs_us)) / 1e3
    res = {
        "case": name, "input_rate": rate_in, "chip_length": cl, "format": fmt, "input_bytes": nbytes,
        "D": dec["D"], "T1": dec["T1"], "T": info["T"], "P": info["P"],
        "decimate_kernel_ms": dc_ms, "resample_kernel_ms": rs_ms,
        "input_stage_gsps": nsamples / ((dc_ms + rs_ms) * 1e6),
        "device_step_ms": step_ms, "device_step_gsps": nsamples / (step_ms * 1e6),
        "e2e_pinned_s": float(np.median(te)), "e2e_pinned_gsps": nsamples / float(np.median(te)) / 1e9,
        "kernels": kernels,
    }
    h.close()
    del d, host
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    nb = int(args.gib * (1 << 30))
    cases = [run_case("tuned_cs8_10to1", 10 * 32768 * 72, 72, capi.FORMAT_CS8, nb, args.reps),
             run_case("decimated_cs16_30.72MSps", 30_720_000, 72, capi.FORMAT_CS16, nb, args.reps),
             run_case("decimated_cs16_61.44MSps", 61_440_000, 72, capi.FORMAT_CS16, nb, args.reps),
             run_case("decimated_cs8_20MSps_cl32", 20_000_000, 32, capi.FORMAT_CS8, nb, args.reps)]
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "offset_hz": OFFSET,
                      "cases": cases}))


if __name__ == "__main__":
    main()
