"""scratch: device-resident stage times of the decode pipeline for a list of ERTGPU_FAST_WARPS knobs
(100 * VAR + W, see launch_demod_fast).  usage: sweep.py MSGTYPE GIB knob[,knob...] [reps]"""
import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from rtlamr_b200 import capi, synth

mt = sys.argv[1] if len(sys.argv) > 1 else "scm"
gib = float(sys.argv[2]) if len(sys.argv) > 2 else 1.0
knobs = sys.argv[3].split(",") if len(sys.argv) > 3 else ["0"]
reps = int(sys.argv[4]) if len(sys.argv) > 4 else 10
cl = 72
nbytes = int(gib * (1 << 30))
probe = capi.new_decoder(mt, cl, max_blocks_per_call=1)
bs2 = probe.cfg.block_size2
probe.close()
nbytes = nbytes // bs2 * bs2
nsamples = nbytes // 2
pk, truth = synth.make_packets(mt, cl, nsamples, seed=1, spacing=1 << 20)
d = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
capi.synth_fill(0, d.data_ptr(), 0, nsamples, 0x5EED0002, pk)
ts = torch.cuda.Stream()
torch.cuda.set_stream(ts)
st = ts.cuda_stream
peak = 3350.0   # GB/s, H100 SXM data sheet (HBM3)
ref = None
for k in knobs:
    if k == "0":
        os.environ.pop("ERTGPU_FAST_WARPS", None)
    else:
        os.environ["ERTGPU_FAST_WARPS"] = k
    h = capi.new_decoder(mt, cl, max_blocks_per_call=nbytes // bs2, max_candidates=1 << 20)
    for _ in range(3):
        h.reset(); h.decode_device_async(d.data_ptr(), nbytes, capi.DECODE_ONLY_VALID, st); c = h.last_counts()
    if ref is None:
        ref = c
    assert c == ref, (k, c, ref)
    def loop():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(ts)
        for _ in range(reps):
            h.reset(); h.decode_device_async(d.data_ptr(), nbytes, capi.DECODE_ONLY_VALID, st); h.last_counts()
        e1.record(ts); torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps
    ms = loop()                 # no events inside a step (programmatic dependent launches active)
    h.set_stage_timing(True)
    ms_staged = loop()
    sm, n = h.stage_ms_mean()
    print(json.dumps({"mt": mt, "gib": gib, "knob": k, "kernels": h.last_kernels(), "ms_per_step": round(ms, 4), "ms_staged": round(ms_staged, 4),
                      "stage_ms": {a: round(b, 4) for a, b in sm.items()}, "demod_frac": round(2 * nsamples / (sm["demod"] * 1e-3) / 1e9 / peak, 4),
                      "step_frac": round(2 * nsamples / (ms * 1e-3) / 1e9 / peak, 4), "counts": c}), flush=True)
    h.close()
