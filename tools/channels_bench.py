"""Several channels of one capture: one ertgpu_decode_channels group against C separate handles, each fed the same bytes
with its own upload.  scm at chip length 72 on cs16 at 30.72 and 61.44 MS/s (D = 4 and 7), and at chip length 32 on cs8
at 20 MS/s (D = 5), about 1 GiB each, C = 1, 4 and 16 channels spread across the capture.

Prints one JSON line with the card's name and power limit (read in the same run) and, per case and C, for the group and
for the separate handles:
  - the device-resident step over the whole input (CUDA events),
  - the first stage's kernel time (decimate_channels_kernel or decimate_kernel, torch.profiler in runs of its own),
  - end to end from pinned host memory (input Gsamples/s of the capture, whatever C).
Usage: python tools/channels_bench.py [--gib 1] [--reps 3] [--channels 1,4,16]"""
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

CAPTURE = 915_000_000
CAP = 1 << 18


def offsets(rate_in, rate_out, c):
    w = (rate_in // 2 - 4 * rate_out // 10) * 9 // 10   # every channel inside the capture
    return [-2_400_000] if c == 1 else [int(o) for o in np.linspace(-w, w, c)]


def run_case(name, rate_in, cl, fmt, nbytes, counts, reps):
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
    st = torch.cuda.Stream()
    rows = []
    for c in counts:
        hs = [capi.new_decoder("scm", cl, max_blocks_per_call=out_blocks, max_candidates=CAP, input_rate=rate_in,
                               input_format=fmt, capture_freq=CAPTURE, center_freq=CAPTURE + o)
              for o in offsets(rate_in, 32768 * cl, c)]

        def reset():
            for h in hs:
                h.reset()

        def dev_group():
            capi.decode_channels_device_async(hs, d.data_ptr(), nbytes, flags, st.cuda_stream)

        def dev_separate():
            for h in hs:
                h.decode_device_async(d.data_ptr(), nbytes, flags, st.cuda_stream)

        def fetch():
            for h in hs:
                h.fetch(cap=CAP)

        res = {"channels": c}
        for label, step in (("group", dev_group), ("separate", dev_separate)):
            for _ in range(2):
                reset()
                step()
                fetch()
            ms = []
            for _ in range(reps):
                reset()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                step()
                e1.record(st)
                fetch()
                ms.append(e0.elapsed_time(e1))
            res[f"{label}_device_step_ms"] = float(np.median(ms))
        for label, step in (("group", dev_group), ("separate", dev_separate)):
            from torch.profiler import ProfilerActivity, profile
            us = []
            for _ in range(reps):
                reset()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    step()
                    fetch()
                    torch.cuda.synchronize()
                us.append(sum(e.device_time for e in prof.events() if "decimate" in e.name))
            res[f"{label}_stage1_ms"] = float(np.median(us)) / 1e3
        for label in ("group", "separate"):
            def e2e():
                reset()
                t0 = time.perf_counter()
                if label == "group":
                    capi.decode_channels(hs, (host.data_ptr(), nbytes), flags, CAP)
                else:
                    for h in hs:
                        h.decode((host.data_ptr(), nbytes), flags, CAP)
                return time.perf_counter() - t0
            e2e()
            t = float(np.median([e2e() for _ in range(reps)]))
            res[f"{label}_e2e_pinned_s"] = t
            res[f"{label}_e2e_pinned_gsps"] = nsamples / t / 1e9
        res["kernels_group"] = hs[0].last_kernels()
        res["stage1_per_channel_gain"] = 1 - res["group_stage1_ms"] / res["separate_stage1_ms"]
        res["e2e_speedup"] = res["separate_e2e_pinned_s"] / res["group_e2e_pinned_s"]
        rows.append(res)
        for h in hs:
            h.close()
        torch.cuda.empty_cache()
    dec, _ = capi.new_decoder("scm", cl, input_rate=rate_in, input_format=fmt, capture_freq=CAPTURE,
                              center_freq=CAPTURE - 2_400_000).decimator()
    del d, host
    torch.cuda.empty_cache()
    return {"case": name, "input_rate": rate_in, "chip_length": cl, "format": fmt, "input_bytes": nbytes,
            "D": dec["D"], "T1": dec["T1"], "results": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--channels", default="1,4,16")
    args = ap.parse_args()
    nb = int(args.gib * (1 << 30))
    counts = [int(x) for x in args.channels.split(",")]
    cases = [run_case("cs16_30.72MSps", 30_720_000, 72, capi.FORMAT_CS16, nb, counts, args.reps),
             run_case("cs16_61.44MSps", 61_440_000, 72, capi.FORMAT_CS16, nb, counts, args.reps),
             run_case("cs8_20MSps_cl32", 20_000_000, 32, capi.FORMAT_CS8, nb, counts, args.reps)]
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "cases": cases}))


if __name__ == "__main__":
    main()
