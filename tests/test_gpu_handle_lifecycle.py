"""GPU test (-m gpu) of a handle's allocation life cycle: an allocation the device cannot hold is refused with
ERTGPU_ENOMEM and leaves the handle unallocated, and the same handle, allocated again, decodes exactly what a fresh handle
decodes: candidates, signal records and spectrum rows."""
import pytest

import tune_ref
from rtlamr_b200 import capi

pytestmark = pytest.mark.gpu

CAPTURE = 915_000_000
RATE = 30_720_000   # 13 times the decoder's rate at chip length 72: the tuned handle decimates first
OFFSET = 300_000
SPECTRUM = (12, 64)


def configure() -> capi.Handle:
    """A tuned, decimating cs16 handle with signal reports and a spectrum, configured as capi.new_decoder does it and not
    allocated."""
    h = capi.Handle()
    h.register(capi.stock_protocol("scm", 72))
    h.set_input_tuning(CAPTURE, CAPTURE + OFFSET)
    h.allow_input_decimation()
    h.set_input_rate(RATE)
    h.set_input_format(capi.FORMAT_CS16)
    h.enable_signal()
    h.enable_spectrum(*SPECTRUM)
    return h


def outputs(h, raw):
    cands = h.decode(raw, cap=1 << 16)
    rows, mean, peak = h.fetch_spectrum(partial=True)
    return {"candidates": cands.tobytes(), "signal": h.fetch_signal().tobytes(), "rows": rows.tobytes(),
            "mean": mean.tobytes(), "peak": peak.tobytes()}


def test_allocate_again_after_a_refused_allocation(built):
    z, _ = tune_ref.wideband([("scm", OFFSET, 11, 0)], RATE, 4_000_000, 5)
    raw = tune_ref.quantize(z, capi.FORMAT_CS16)
    fresh = configure()
    fresh.allocate()
    want = outputs(fresh, raw)
    fresh.close()
    assert want["candidates"] and want["signal"] and want["rows"]

    h = configure()
    assert h.decimator()[0]["D"] > 1
    with pytest.raises(capi.ErtGpuError) as e:
        h.allocate(max_candidates=1 << 40)   # terabytes of hit records: cudaMalloc refuses them
    assert e.value.code == capi.ENOMEM and "out of memory" in str(e.value)
    with pytest.raises(capi.ErtGpuError) as e:
        h.decode(raw)
    assert e.value.code == capi.EINVAL
    h.allocate()
    assert outputs(h, raw) == want
    h.close()
