"""The wide channel path (ertgpu_set_channel_gain) against today's narrow tuned path, alternated in one run on the same
device-resident bytes: cs16 at 10 MS/s and cs8 at 20 MS/s (one stage), cs16 at 30.72 and 61.44 MS/s (two stages) with
C = 1 and 4 channels, scm at chip length 72.

Prints one JSON line with the card's name and power limit (read in the same run) and, per case, C and path:
  - the device-resident step over the whole input (CUDA events, median of --reps, narrow and wide alternated),
  - the input stage's kernel time (resample_* and decimate_* kernels, torch.profiler in runs of its own).
Usage: python tools/channel_gain_bench.py [--gib 1] [--reps 3]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from rtlamr_b200 import capi  # noqa: E402
from resample_bench import power_limit_w  # noqa: E402

CAPTURE = 915_000_000
CAP = 1 << 18
K = 4


def offsets(rate_in, rate_out, c):
    w = (rate_in // 2 - 4 * rate_out // 10) * 9 // 10
    return [-2_400_000] if c == 1 else [int(o) for o in np.linspace(-w, w, c)]


def run_case(name, rate_in, fmt, nbytes, counts, reps):
    cl, flags = 72, capi.DECODE_ONLY_VALID
    s = capi.FORMAT_BYTES[fmt]
    nbytes = nbytes // (8192 * s) * (8192 * s)
    g = torch.Generator(device="cuda").manual_seed(1)
    d = torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device="cuda", generator=g)
    out_blocks = int(nbytes // s * 32768 * cl / rate_in) // 2048 + 2
    st = torch.cuda.Stream()
    rows = []
    for c in counts:
        paths = {}
        for label, k in (("narrow", None), ("wide", K)):
            paths[label] = [capi.new_decoder("scm", cl, max_blocks_per_call=out_blocks, max_candidates=CAP, input_rate=rate_in,
                                             input_format=fmt, capture_freq=CAPTURE, center_freq=CAPTURE + o, channel_gain=k)
                            for o in offsets(rate_in, 32768 * cl, c)]

        def step(hs):
            for h in hs:
                h.reset()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            if len(hs) == 1:
                hs[0].decode_device_async(d.data_ptr(), nbytes, flags, st.cuda_stream)
            else:
                capi.decode_channels_device_async(hs, d.data_ptr(), nbytes, flags, st.cuda_stream)
            e1.record(st)
            for h in hs:
                h.fetch(cap=CAP)
            return e0.elapsed_time(e1)

        res = {"channels": c}
        for hs in paths.values():
            step(hs)
            step(hs)
        ms = {label: [] for label in paths}
        for _ in range(reps):
            for label, hs in paths.items():   # alternated
                ms[label].append(step(hs))
        from torch.profiler import ProfilerActivity, profile
        for label, hs in paths.items():
            res[f"{label}_device_step_ms"] = float(np.median(ms[label]))
            us = []
            for _ in range(reps):
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    step(hs)
                    torch.cuda.synchronize()
                us.append(sum(e.device_time for e in prof.events() if "resample" in e.name or "decimate" in e.name))
            res[f"{label}_input_kernels_ms"] = float(np.median(us)) / 1e3
            res[f"{label}_kernels"] = hs[0].last_kernels().split(";", 1)[1]
        res["wide_over_narrow_input_kernels"] = res["wide_input_kernels_ms"] / res["narrow_input_kernels_ms"]
        res["wide_over_narrow_device_step"] = res["wide_device_step_ms"] / res["narrow_device_step_ms"]
        rows.append(res)
        for hs in paths.values():
            for h in hs:
                h.close()
        torch.cuda.empty_cache()
    del d
    torch.cuda.empty_cache()
    return {"case": name, "input_rate": rate_in, "format": fmt, "input_bytes": nbytes, "k": K, "results": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    nb = int(args.gib * (1 << 30))
    cases = [run_case("cs16_10MSps", 10_000_000, capi.FORMAT_CS16, nb, [1], args.reps),
             run_case("cs8_20MSps", 20_000_000, capi.FORMAT_CS8, nb, [1], args.reps),
             run_case("cs16_30.72MSps", 30_720_000, capi.FORMAT_CS16, nb, [1, 4], args.reps),
             run_case("cs16_61.44MSps", 61_440_000, capi.FORMAT_CS16, nb, [1, 4], args.reps)]
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "cases": cases}))


if __name__ == "__main__":
    main()
