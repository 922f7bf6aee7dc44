"""Cost of the input spectrum (ertgpu_enable_spectrum): the device-resident step (reset, one ertgpu_decode_device_async
over resident input, the counters read back) of two handles of one geometry, one with a spectrum and one without,
alternated in one run; spectrum_kernel's time per step from torch.profiler in a run of its own; and the end-to-end rate
of ertgpu_decode from pinned host memory with and without the spectrum, alternated.

Cases: cu8 at the decoder's rate (1 GiB), cs16 at 10 MS/s tuned 2 MHz off centre (1 GiB) and cs16 at 61.44 MS/s
decimated (1 GiB), each at N = 1024, 4096 and 16384 with F = ceil(2^18 / N).  Prints one JSON line with the card's name
and power limit (read in the same run) and, per case, the step times, the kernel time, its rate in input Gsamples/s, and
its share of HBM bandwidth (input bytes over kernel time, of 3.35 TB/s) and of FP32 peak (5 N log2 N flops per frame
over kernel time, of 67 TFLOP/s), naming the larger as the bound.
Usage: python tools/spectrum_bench.py [--reps 5] [--steps 10] [--only NAME]"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from rtlamr_b200 import capi  # noqa: E402
from resample_bench import power_limit_w  # noqa: E402

CL = 72
CAPTURE = 915_000_000
HBM_BPS, FP32_FLOPS = 3.35e12, 67e12
INPUTS = [("cu8_native", capi.FORMAT_CU8, 0, None), ("cs16_10M_tuned", capi.FORMAT_CS16, 10_000_000, -2_000_000),
          ("cs16_61M44_decimated", capi.FORMAT_CS16, 61_440_000, 2_400_000)]
CASES = [(f"{name}_N{1 << n}", name, fmt, rate, off, n) for name, fmt, rate, off in INPUTS for n in (10, 12, 14)]


def make(fmt, rate, off, nblocks, spectrum):
    kw = {"max_blocks_per_call": nblocks, "max_candidates": 1 << 20, "spectrum": spectrum}
    if fmt != capi.FORMAT_CU8:
        kw["input_format"] = fmt
    if rate:
        kw.update(input_rate=rate, capture_freq=CAPTURE, center_freq=CAPTURE + off)
    return capi.new_decoder("scm", CL, **kw)


def step(h, d, nbytes, st):
    h.reset()
    h.decode_device_async(d.data_ptr(), nbytes, 0, st.cuda_stream)
    return h.last_counts()


def run_case(name, inp, fmt, rate, off, log2n, reps, steps):
    nbytes = 1 << 30
    s = capi.FORMAT_BYTES[fmt]
    probe = make(fmt, rate, off, 1, None)
    bs = probe.cfg.block_size
    probe.close()
    nbytes = nbytes // (bs * s) * (bs * s)
    nsamples = nbytes // s
    out_rate = 32768 * CL
    nblocks = nsamples * out_rate // (rate or out_rate) // bs + 2
    g = torch.Generator(device="cuda").manual_seed(1)
    d = torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device="cuda", generator=g)
    if fmt == capi.FORMAT_CS16:   # 8-bit noise in the top byte: cs16 at the default gain maps it to full scale
        d.view(torch.int16).copy_((d.view(torch.int16) >> 4))
    F = -(-(1 << 18) >> log2n)
    hs = {False: make(fmt, rate, off, nblocks, None), True: make(fmt, rate, off, nblocks, (log2n, F))}
    st = torch.cuda.Stream()
    for h in hs.values():
        for _ in range(2):
            step(h, d, nbytes, st)
    assert hs[True].fetch(1 << 20).tobytes() == hs[False].fetch(1 << 20).tobytes()
    times = {False: [], True: []}
    for r in range(reps):
        for sp in ((False, True) if r % 2 == 0 else (True, False)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                step(hs[sp], d, nbytes, st)
            times[sp].append((time.perf_counter() - t0) / steps * 1e3)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step(hs[True], d, nbytes, st)
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "spectrum_kernel" in e.key) / steps
    # end to end from pinned host memory, the handles alternated
    host = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    host.copy_(d)
    e2e = {False: [], True: []}
    for r in range(reps):
        for sp in ((False, True) if r % 2 == 0 else (True, False)):
            hs[sp].reset()
            t0 = time.perf_counter()
            hs[sp].decode((host.data_ptr(), nbytes), cap=1 << 20)
            e2e[sp].append(nsamples / (time.perf_counter() - t0) / 1e9)
    for h in hs.values():
        h.close()
    frames = nsamples >> log2n
    t = us * 1e-6
    hbm = nbytes / t / HBM_BPS if t else 0.0
    fp32 = frames * 5 * (1 << log2n) * log2n / t / FP32_FLOPS if t else 0.0
    base, with_sp = statistics.median(times[False]), statistics.median(times[True])
    return {"case": name, "input": inp, "N": 1 << log2n, "F": F, "bytes": nbytes, "samples": nsamples,
            "step_ms_without": round(base, 4), "step_ms_with": round(with_sp, 4),
            "steps_ms_without": [round(x, 4) for x in times[False]], "steps_ms_with": [round(x, 4) for x in times[True]],
            "spectrum_kernel_ms": round(us / 1e3, 4), "kernel_gsamples_per_s": round(nsamples / t / 1e9, 2) if t else 0,
            "hbm_share": round(hbm, 4), "fp32_share": round(fp32, 4), "bound": "fp32" if fp32 > hbm else "hbm",
            "e2e_gsamples_per_s_without": round(statistics.median(e2e[False]), 3),
            "e2e_gsamples_per_s_with": round(statistics.median(e2e[True]), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--only", default="")
    a = ap.parse_args()
    out = [run_case(*c, a.reps, a.steps) for c in CASES if not a.only or a.only in c[0]]
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "cases": out}))


if __name__ == "__main__":
    main()
