"""Cost of the input-format conversion: scm at chip length 72 on about 1 GiB of decoder-rate uint8 IQ (512 Mi samples),
fed in each format of --formats (cs16 and cf32 by default, or any complex SigMF datatype name) at the decoder's rate
(convert_kernel) and at 2.4 MS/s (resample_kernel<F>), each arm alternated with the same samples as uint8 (cu8).

Prints one JSON line with the card's name and power limit (read in the same run) and, per arm:
  - the conversion kernel's time (torch.profiler) and, natively, its read + write bytes/s as a fraction of the H100 SXM
    data sheet's 3.35 TB/s;
  - the device-resident step (CUDA events around ertgpu_decode_device_async);
  - end to end from pinned host memory (ertgpu_decode), unless --no-e2e.
Usage: python tools/format_bench.py [--reps 5] [--formats cs16,cf32,ci16_be,...,cf64_be] [--samples N] [--no-e2e]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rtlamr_b200 import capi, synth  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from resample_bench import power_limit_w  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
FORMATS = {"cs16": capi.FORMAT_CS16, "cf32": capi.FORMAT_CF32, "ci16_be": capi.FORMAT_CS16BE, "cf32_be": capi.FORMAT_CF32BE,
           "cu16_le": capi.FORMAT_CU16, "cu16_be": capi.FORMAT_CU16BE, "ci32_le": capi.FORMAT_CS32,
           "ci32_be": capi.FORMAT_CS32BE, "cu32_le": capi.FORMAT_CU32, "cu32_be": capi.FORMAT_CU32BE,
           "cf64_le": capi.FORMAT_CF64, "cf64_be": capi.FORMAT_CF64BE}
BIG_ENDIAN = {capi.FORMAT_CS16BE, capi.FORMAT_CF32BE, capi.FORMAT_CU16BE, capi.FORMAT_CS32BE, capi.FORMAT_CU32BE,
              capi.FORMAT_CF64BE}


def encode_on_device(u8: torch.Tensor, fmt: int) -> torch.Tensor:
    """The exact encoding of uint8 IQ in fmt (the default scale maps it back to the same bytes)."""
    v = u8.to(torch.int16) - 128
    if fmt == capi.FORMAT_CS16:
        return (v * 256).view(torch.uint8)
    if fmt == capi.FORMAT_CF32:
        return (v.to(torch.float32) / 128).view(torch.uint8)
    k = capi.FORMAT_BYTES[fmt] // 2   # bytes per component
    if fmt in (capi.FORMAT_CF32BE, capi.FORMAT_CF64, capi.FORMAT_CF64BE):
        b = (v.to(torch.float32 if k == 4 else torch.float64) / 128).view(torch.uint8).view(-1, k)
    else:
        x = v.to(torch.int64) * (1 << (8 * k - 8))
        if fmt in (capi.FORMAT_CU16, capi.FORMAT_CU16BE, capi.FORMAT_CU32, capi.FORMAT_CU32BE):
            x += 1 << (8 * k - 1)
        b = x.view(torch.uint8).view(-1, 8)[:, :k]   # the low k bytes, little-endian
    return (b.flip(1) if fmt in BIG_ENDIAN else b).contiguous().view(-1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--samples", type=int, default=1 << 29, help="decoder-rate IQ samples (2^29 = 1 GiB of uint8)")
    ap.add_argument("--formats", default="cs16,cf32")
    ap.add_argument("--no-e2e", action="store_true", help="skip the end-to-end arms from pinned host memory")
    args = ap.parse_args()
    cl, flags = 72, capi.DECODE_ONLY_VALID
    rate_out = 32768 * cl
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "arms": []}

    for rate_in in (rate_out, 2_400_000):
        n = args.samples * rate_in // rate_out // 4096 * 4096   # input samples: a whole number of decoder blocks
        u8 = torch.empty(2 * n, dtype=torch.uint8, device="cuda")
        pk, _ = synth.make_packets("scm", cl, n, seed=1, spacing=1 << 20)
        capi.synth_fill(0, u8.data_ptr(), 0, n, 2, pk)
        out_blocks = int(n * rate_out / rate_in) // 4096 + 2
        base = capi.new_decoder("scm", cl, max_blocks_per_call=out_blocks, max_candidates=1 << 20, input_rate=rate_in)
        for name in args.formats.split(","):
            fmt = FORMATS[name]
            d = encode_on_device(u8, fmt)
            host = host_u8 = None
            if not args.no_e2e:
                host = torch.empty(d.numel(), dtype=torch.uint8).pin_memory()
                host.copy_(d)
                host_u8 = torch.empty(u8.numel(), dtype=torch.uint8).pin_memory()
                host_u8.copy_(u8)
            torch.cuda.synchronize()
            h = capi.new_decoder("scm", cl, max_blocks_per_call=out_blocks, max_candidates=1 << 20, input_rate=rate_in,
                                 input_format=fmt)
            st = torch.cuda.Stream()
            arms = {"cu8": (base, u8, host_u8), name: (h, d, host)}

            def step(dec, buf):
                dec.reset()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                dec.decode_device_async(buf.data_ptr(), buf.numel(), flags, st.cuda_stream)
                e1.record(st)
                rows = dec.fetch(cap=1 << 20)
                return e0.elapsed_time(e1), rows

            def e2e(dec, hbuf):
                dec.reset()
                t0 = time.perf_counter()
                dec.decode((hbuf.data_ptr(), hbuf.numel()), flags, 1 << 20)
                return time.perf_counter() - t0

            ms = {k: [] for k in arms}
            same = True
            for _ in range(2):
                for k, (dec, buf, _h) in arms.items():
                    step(dec, buf)
            for _ in range(args.reps):   # the arms alternate, so drift of the clocks or the link hits both alike
                outs = {}
                for k, (dec, buf, _h) in arms.items():
                    t, rows = step(dec, buf)
                    ms[k].append(t)
                    outs[k] = rows.tobytes()
                same = same and outs["cu8"] == outs[name]
            labels = {k: a[0].last_kernels() for k, a in arms.items()}

            kern_us = {}
            from torch.profiler import ProfilerActivity, profile
            for k, (dec, buf, _h) in arms.items():
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    step(dec, buf)
                    torch.cuda.synchronize()
                want = "convert_kernel" if (k != "cu8" and rate_in == rate_out) else "resample_kernel"
                us = [e.device_time for e in prof.events() if want in e.name]
                kern_us[k] = float(np.sum(us)) if us else None

            t_e2e = {k: [float("nan")] for k in arms}
            if not args.no_e2e:
                for k, (dec, _b, hbuf) in arms.items():
                    e2e(dec, hbuf)
                t_e2e = {k: [] for k in arms}
            for _ in range(0 if args.no_e2e else args.reps):
                for k, (dec, _b, hbuf) in arms.items():
                    t_e2e[k].append(e2e(dec, hbuf))

            arm = {"format": name, "input_rate": rate_in, "input_samples": n, "input_bytes": d.numel(),
                   "candidates_identical_to_cu8": same, "kernels": labels}
            for k in arms:
                s = np.median(ms[k])
                arm[k] = {"step_ms": float(s), "step_ms_all": ms[k], "step_gsps": n / (s * 1e6),
                          "e2e_s": float(np.median(t_e2e[k])), "e2e_s_all": t_e2e[k],
                          "e2e_gsps": n / np.median(t_e2e[k]) / 1e9,
                          "front_kernel_ms": kern_us[k] / 1e3 if kern_us[k] is not None else None}
            if rate_in == rate_out and kern_us[name]:
                moved = n * (capi.FORMAT_BYTES[fmt] + 2)   # read the format, write uint8
                arm["convert_bytes_per_s"] = moved / (kern_us[name] * 1e-6)
                arm["convert_fraction_of_3p35TBps"] = arm["convert_bytes_per_s"] / HBM_BYTES_PER_S
            elif kern_us[name] and kern_us["cu8"]:
                arm["resample_time_ratio_to_cu8"] = kern_us[name] / kern_us["cu8"]
            res["arms"].append(arm)
            h.close()
            del d, host, host_u8, arms
            torch.cuda.empty_cache()
        base.close()
        del u8
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
