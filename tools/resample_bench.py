"""Throughput of the input-rate resampler: scm at chip length 72 fed 1 GiB of 2.4 MS/s uint8 IQ.

Prints one JSON line with
  - the card's name and power limit (read in the same run),
  - resample_kernel's own time (torch.profiler) and the whole device-resident step (CUDA events), as input
    Gsamples/s,
  - end to end from pinned host memory with resampling, next to the native end to end of the same bytes.
Usage: python tools/resample_bench.py [--gib 1] [--reps 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rtlamr_b200 import capi, synth  # noqa: E402


def power_limit_w():
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        return pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
    except Exception:
        try:
            out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                 capture_output=True, text=True, timeout=30).stdout.strip()
            return float(out.splitlines()[0])
        except Exception:
            return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rate", type=int, default=2_400_000)
    args = ap.parse_args()
    cl, rate_in = 72, args.rate
    nbytes = int(args.gib * (1 << 30)) // 8192 * 8192
    nsamples = nbytes // 2
    flags = capi.DECODE_ONLY_VALID

    d = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    pk, _ = synth.make_packets("scm", cl, nsamples, seed=1, spacing=1 << 20)
    capi.synth_fill(0, d.data_ptr(), 0, nsamples, 2, pk)
    host = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
    host.copy_(d)
    torch.cuda.synchronize()

    native = capi.new_decoder("scm", cl, max_blocks_per_call=nbytes // 8192 + 1, max_candidates=1 << 20)
    bs = native.cfg.block_size
    out_blocks = int(nsamples * native.cfg.sample_rate / rate_in) // bs + 2
    rs = capi.new_decoder("scm", cl, max_blocks_per_call=max(out_blocks, 1), max_candidates=1 << 20, input_rate=rate_in)
    st = torch.cuda.Stream()  # a real stream: a null handle would mean the decoder's own stream

    def device_step():
        rs.reset()
        rs.decode_device_async(d.data_ptr(), nbytes, flags, st.cuda_stream)
        rs.fetch(cap=1 << 20)

    for _ in range(2):
        device_step()
    ms = []
    for _ in range(args.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        rs.reset()
        e0.record(st)
        rs.decode_device_async(d.data_ptr(), nbytes, flags, st.cuda_stream)
        e1.record(st)
        rs.fetch(cap=1 << 20)
        ms.append(e0.elapsed_time(e1))
    kernels = rs.last_kernels()

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        device_step()
        torch.cuda.synchronize()
    rs_us = [e.device_time for e in prof.events() if "resample_kernel" in e.name]
    demod_us = [e.device_time for e in prof.events() if "demod_" in e.name]

    def e2e_once(h):
        h.reset()
        t0 = time.perf_counter()
        h.decode((host.data_ptr(), nbytes), flags, 1 << 20)
        return time.perf_counter() - t0

    for h in (native, rs, native, rs):  # warm-up
        e2e_once(h)
    tn, tr = [], []
    for _ in range(args.reps):  # the two arms alternate, so drift of the link or the clocks hits both alike
        tn.append(e2e_once(native))
        tr.append(e2e_once(rs))
    t_native, t_rs = float(np.median(tn)), float(np.median(tr))
    step_ms = float(np.median(ms))
    res = {
        "gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(),
        "input_rate": rate_in, "output_rate": native.cfg.sample_rate, "input_bytes": nbytes,
        "resample_kernel_ms": (float(np.median(rs_us)) / 1e3) if rs_us else None,
        "resample_kernel_gsps": (nsamples / (np.median(rs_us) * 1e3)) if rs_us else None,
        "demod_kernel_ms": (float(np.median(demod_us)) / 1e3) if demod_us else None,
        "device_step_ms": step_ms, "device_step_ms_all": ms, "device_step_gsps": nsamples / (step_ms * 1e6),
        "e2e_pinned_resampled_gsps": nsamples / t_rs / 1e9, "e2e_pinned_native_gsps": nsamples / t_native / 1e9,
        "e2e_native_s_all": tn, "e2e_resampled_s_all": tr, "kernels": kernels,
    }
    res["e2e_ratio"] = res["e2e_pinned_resampled_gsps"] / res["e2e_pinned_native_gsps"]
    res["step_over_e2e"] = res["device_step_gsps"] / res["e2e_pinned_resampled_gsps"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
