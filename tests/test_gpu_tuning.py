"""GPU tests (-m gpu) of the tuned input resampler (ertgpu_set_input_tuning): resample_kernel<F,tuned> against the CPU
restatement (tests/cpu_harness/tune_ref.c) byte for byte, the zero offset as the untuned handle, off-centre packets of
wideband captures recovered next to interferers, two channels on two handles, call splitting, a large device call,
reset, sharding, the allocation sweep and the file receiver."""
import os
import subprocess

import numpy as np
import pytest

from rtlamr_b200 import capi

import format_ref
import tune_ref
from test_gpu_resample import _cuts, keys, native_of, out_end, tap_resampled
from test_gpu_resample import stream as native_stream

pytestmark = pytest.mark.gpu

DATA_RATE = 32768
FMT = {"cu8": capi.FORMAT_CU8, "cs8": capi.FORMAT_CS8, "cs16": capi.FORMAT_CS16}
CAPTURE = 915_000_000


def _u8(raw, fmt):
    return format_ref.convert(raw, FMT[fmt])


def _render(msgtypes, rate_in, n, seed, off, fmt, other_off=None, other=None):
    """(raw capture bytes, truth of the wanted channel, truth of the interferers)."""
    ch = [(msgtypes, off, seed, 0)]
    if other_off is not None:
        ch.append((other or msgtypes, other_off, seed + 1000, 40_000))
    z, truths = tune_ref.wideband(ch, rate_in, n, seed)
    if fmt == "cu8":
        raw = np.empty(2 * n, dtype=np.uint8)
        raw[0::2] = np.clip(np.round(z.real + 127.5), 0, 255)
        raw[1::2] = np.clip(np.round(z.imag + 127.5), 0, 255)
    else:
        raw = tune_ref.quantize(z, FMT[fmt])
    return raw, truths[0], truths[1] if len(truths) > 1 else []


def _decoder(msgtypes, cl, rate_in, off, fmt, **kw):
    center = CAPTURE + off
    return capi.new_decoder(msgtypes, cl, input_rate=rate_in, input_format=FMT[fmt], capture_freq=CAPTURE,
                            center_freq=center, **kw)


KERNEL_CASES = [(2_400_000, 72, "cu8", 200_000), (DATA_RATE * 72, 72, "cu8", -200_000), (8_000_000, 72, "cs8", -2_400_000),
                (9_437_184, 72, "cs8", 3_000_000), (10_000_000, 72, "cs16", -2_400_000), (16_000_000, 72, "cs8", 2_000_000),
                (20_000_000, 72, "cs8", 5_000_000), (8_000_000, 32, "cs8", -2_400_000)]


@pytest.mark.parametrize("rate_in,cl,fmt,off", KERNEL_CASES)
@pytest.mark.parametrize("kind", ["random", "synthetic"])
def test_kernel_equals_cpu_restatement(built, rate_in, cl, fmt, off, kind):
    rate_out = DATA_RATE * cl
    n = 1_200_000
    if kind == "random":
        raw = np.random.default_rng(rate_in ^ cl).integers(0, 256, 2 * n * (2 if fmt == "cs16" else 1), dtype=np.uint8)
    else:
        raw, _, _ = _render("scm", rate_in, n, 11, off, fmt, other_off=0)
    ref = tune_ref.tune(_u8(raw, fmt), rate_in, rate_out, off)
    h = _decoder("scm", cl, rate_in, off, fmt)
    info, _ = h.resampler()
    assert info["P"] == tune_ref.plan(rate_in, rate_out, off)["P"]
    got = h.decode(raw, cap=1 << 16)
    bs = h.cfg.block_size
    nblocks = (ref.size // 2) // bs
    assert nblocks > 4
    assert f"resample_kernel<{fmt},tuned>" in h.last_kernels().split(";")
    assert np.array_equal(tap_resampled(h, 0, nblocks), ref[:2 * nblocks * bs])
    assert keys(got) == keys(native_of("scm", cl, ref))
    h.close()


def test_zero_offset_is_the_untuned_handle(built):
    rate_in, cl = 2_400_000, 72
    iq, _ = native_stream("scm", rate_in, 1_500_000, seed=7)
    a = capi.new_decoder("scm", cl, input_rate=rate_in)
    b = capi.new_decoder("scm", cl, input_rate=rate_in, capture_freq=912_600_155)   # the channel is the centre
    ga, gb = a.decode(iq, cap=1 << 16), b.decode(iq, cap=1 << 16)
    assert ga.tobytes() == gb.tobytes() and len(ga) > 0
    assert a.last_kernels() == b.last_kernels() and "resample_kernel" in b.last_kernels().split(";")
    nb = (out_end(a.resampler()[0], iq.size // 2)) // a.cfg.block_size
    assert np.array_equal(tap_resampled(a, 0, nb), tap_resampled(b, 0, nb))
    a.close()
    b.close()


def _found(rows, truth, msgtype):
    valid = [r for r in rows if r["check_mask"]]
    if msgtype == "r900":
        return [any([d[2 * k] * 6 + d[2 * k + 1] for k in range(21)] == list(t.data) for d in (r["r900_digits"] for r in valid))
                for t in truth]
    return [any(r["bytes"][:len(t.data)].tobytes() == t.data for r in valid) for t in truth]


@pytest.mark.parametrize("rate_in,fmt", [(8_000_000, "cs8"), (10_000_000, "cs16")])
@pytest.mark.parametrize("msgtype", ["scm", "scm+", "idm", "r900"])
def test_off_centre_packets_are_recovered(built, msgtype, rate_in, fmt):
    n = 8_000_000
    raw, want, other = _render(msgtype, rate_in, n, 61, -2_400_000, fmt, other_off=1_500_000)
    assert len(want) >= 10 and other
    h = _decoder(msgtype, 72, rate_in, -2_400_000, fmt)
    s = capi.FORMAT_BYTES[FMT[fmt]]
    rows, off = [], 0
    for c in (123_457, 700_001, 77, 1_500_000):
        rows.extend(h.decode(raw[off:off + s * c], cap=1 << 16))
        off += s * c
    rows.extend(h.decode(raw[off:], cap=1 << 16))
    assert all(_found(rows, want, msgtype)), msgtype
    assert not any(_found(rows, other, msgtype))
    h.close()
    if rate_in == 8_000_000 and fmt == "cs8":   # an untuned handle at 3.39:1 decodes the centre, not the channel
        u = capi.new_decoder(msgtype, 72, input_rate=rate_in, input_format=FMT[fmt])
        assert not any(_found(u.decode(raw, cap=1 << 16), want, msgtype))
        u.close()


def test_two_handles_two_channels(built):
    rate_in, fmt = 8_000_000, "cs8"
    raw, a_truth, b_truth = _render("scm", rate_in, 4_000_000, 71, -2_400_000, fmt, other_off=1_500_000)
    ha = _decoder("scm", 72, rate_in, -2_400_000, fmt)
    hb = _decoder("scm", 72, rate_in, 1_500_000, fmt)
    ra, rb = ha.decode(raw, cap=1 << 16), hb.decode(raw, cap=1 << 16)
    assert all(_found(ra, a_truth, "scm")) and not any(_found(ra, b_truth, "scm"))
    assert all(_found(rb, b_truth, "scm")) and not any(_found(rb, a_truth, "scm"))
    ha.close()
    hb.close()


def test_call_splitting_host_and_device_at_10_to_1(built):
    import torch
    cl, fmt, off = 72, "cs16", -2_400_000
    rate_in = 10 * DATA_RATE * cl
    raw, _, _ = _render("scm", rate_in, 3_000_000, 31, off, fmt)
    ref = tune_ref.tune(_u8(raw, fmt), rate_in, DATA_RATE * cl, off)
    want = keys(native_of("scm", cl, ref))
    rng = np.random.default_rng(77)
    sizes = [4 * (s // 2) for s in _cuts(rng, raw.size // 2, 40)]
    sizes[-1] += raw.size - sum(sizes)
    # the host path with max_blocks_per_call = 3 cuts every call into many pipelines (the taps see only the last one)
    for path, max_blocks in (("host", 0), ("device", 0), ("host", 3)):
        h = _decoder("scm", cl, rate_in, off, fmt, max_blocks_per_call=max_blocks)
        info, _ = h.resampler()
        assert info["P"] == 64
        bs = h.cfg.block_size
        rows, res, o, done = [], [], 0, 0
        for s in sizes:
            part = raw[o:o + s]
            o += s
            if path == "host":
                rows.extend(h.decode(part, cap=1 << 16))
            else:
                d = torch.from_numpy(part.copy()).cuda()
                h.decode_device_async(d.data_ptr(), d.numel(), 0, torch.cuda.current_stream().cuda_stream)
                rows.extend(h.fetch(cap=1 << 16))
                del d
            nb = out_end(info, o // 4) // bs
            if not max_blocks:
                res.append(tap_resampled(h, done, nb))
            done = nb
        assert keys(rows) == want, (path, max_blocks)
        if not max_blocks:
            allb = np.concatenate(res)
            assert np.array_equal(allb, ref[:allb.size]) and allb.size == 2 * done * bs, path
        h.reset()   # the mixer's phase restarts with the stream
        assert keys(h.decode(raw, cap=1 << 16)) == want
        h.close()


def test_64mib_device_resident_call(built):
    import torch
    cl, fmt, off, rate_in = 72, "cs16", -2_400_000, 10_000_000
    n = 16 << 20   # 64 MiB of cs16
    raw, _, _ = _render("scm", rate_in, n, 81, off, fmt)
    ref = tune_ref.tune(_u8(raw, fmt), rate_in, DATA_RATE * cl, off)
    h = _decoder("scm", cl, rate_in, off, fmt)
    d = torch.from_numpy(raw).cuda()
    h.decode_device_async(d.data_ptr(), d.numel(), 0, torch.cuda.current_stream().cuda_stream)
    got = h.fetch(cap=1 << 16)
    bs = h.cfg.block_size
    nblocks = (ref.size // 2) // bs
    assert keys(got) == keys(native_of("scm", cl, ref))
    for b in sorted(set(np.random.default_rng(3).integers(0, nblocks, 24).tolist()) | {0, nblocks - 1}):
        assert np.array_equal(h.tap(capi.TAP_RESAMPLED, b), ref[2 * b * bs:2 * (b + 1) * bs]), b
    h.close()


def test_reset_and_sharding(built):
    rate_in, fmt, off = 8_000_000, "cs8", -2_400_000
    raw, _, _ = _render("scm", rate_in, 1_500_000, 91, off, fmt)
    h = _decoder("scm", 72, rate_in, off, fmt)
    first = h.decode(raw, cap=1 << 16)
    t0 = h.tap(capi.TAP_RESAMPLED, 3)
    h.reset()
    again = h.decode(raw, cap=1 << 16)
    assert first.tobytes() == again.tobytes() and np.array_equal(t0, h.tap(capi.TAP_RESAMPLED, 3))
    h.close()
    for kw in ({"input_rate": rate_in}, {}):   # tuned, also at the decoder's own rate
        hh = capi.new_decoder("scm", 72, capture_freq=912_600_155 - 100_000, **kw)
        with pytest.raises(capi.ErtGpuError) as e:
            capi.decode_sharded([hh], np.zeros(8192 * 2, dtype=np.uint8))
        assert e.value.code == capi.EINVAL
        hh.close()


def test_allocation_sweep(built):
    rate_out = DATA_RATE * 72
    """Tuned handles allocate and run across the whole ratio range (50 kHz off: every one runs the tuned instance), so
    the shared-memory sizing of every P holds."""
    for rate_in in sorted(set(np.linspace(rate_out // 4, rate_out * 10, 25).astype(np.int64).tolist()) | {rate_out * 10}):
        h = capi.new_decoder("scm", 72, input_rate=int(rate_in), capture_freq=912_600_155 - 50_000)
        assert h.resampler()[0]["P"] == tune_ref.plan(int(rate_in), rate_out, 50_000)["P"]
        h.decode(np.full(2 * 200_000, 128, dtype=np.uint8), cap=1 << 10)
        assert "tuned>" in h.last_kernels()
        h.close()


CLI = os.path.join(tune_ref.ROOT, "rtlamr_b200", "ertgpu_decode_file")


def test_cli_capturefreq(built, tmp_path):
    rate_in = 10_000_000
    raw, want, other = _render("scm", rate_in, 5_000_000, 101, -2_399_845, "cs16", other_off=1_500_000)
    path = tmp_path / "wide.cs16"
    raw.tofile(path)
    from test_gpu_resample import _scm_fields
    base = [CLI, "-msgtype=scm", "-sampleformat=cs16", f"-samplerate={rate_in}", "-capturefreq=915000000", "-format=json"]
    out = subprocess.run(base + [str(path)], capture_output=True, text=True, timeout=300, check=True)
    import json
    ids = {json.loads(l)["Message"]["ID"] for l in out.stdout.splitlines()}
    assert {_scm_fields(t.data)[0] for t in want} <= ids
    assert not ({_scm_fields(t.data)[0] for t in other} & ids)
    out = subprocess.run(base + [f"-centerfreq={915_000_000 + 1_500_000}", str(path)], capture_output=True, text=True,
                         timeout=300, check=True)
    ids = {json.loads(l)["Message"]["ID"] for l in out.stdout.splitlines()}
    assert {_scm_fields(t.data)[0] for t in other} <= ids
    assert not ({_scm_fields(t.data)[0] for t in want} & ids)


def test_cli_capturefreq_at_the_channel_is_a_no_op(built, tmp_path):
    iq, _ = native_stream("scm", DATA_RATE * 72, 1 << 21, seed=5)
    path = tmp_path / "native.bin"
    iq.tofile(path)
    a = subprocess.run([CLI, "-msgtype=scm", str(path)], capture_output=True, text=True, timeout=300, check=True)
    b = subprocess.run([CLI, "-msgtype=scm", "-capturefreq=912600155", str(path)], capture_output=True, text=True,
                       timeout=300, check=True)
    assert a.stdout == b.stdout and a.stdout


def test_host_receiver_binding_takes_the_tuning(built):
    from rtlamr_b200 import host
    from test_gpu_resample import _scm_fields
    rate_in = 8_000_000
    raw, want, _ = _render("scm", rate_in, 3_000_000, 111, -2_399_845, "cs8")
    r = host.Receiver("scm", 72, input_rate=rate_in, input_format=capi.FORMAT_CS8, capture_freq=CAPTURE)
    assert "CaptureFreq: 915000000" in r.log()
    msgs = r.decode(raw[:2 * 1_000_001]) + r.decode(raw[2 * 1_000_001:])
    assert {_scm_fields(t.data)[0] for t in want} <= {m.meter_id for m in msgs}
    r.close()
