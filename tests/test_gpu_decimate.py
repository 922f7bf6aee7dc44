"""GPU tests (-m gpu) of the decimating tuned input (ertgpu_allow_input_decimation): decimate_kernel<F> into
resample_kernel<cu8> against the CPU restatement (tests/cpu_harness/decimate_ref.c into resample_ref.c) byte for byte in
every block, every format, the opted-in handle at 10:1 as today's tuned handle, off-centre packets next to an
interferer, three channels of one capture on three handles, call splitting, chunking, reset, a large device call and
the file receiver."""
import json
import os
import re
import subprocess

import numpy as np
import pytest

from rtlamr_b200 import capi

import decimate_ref
import tune_ref
from test_gpu_resample import _cuts, _scm_fields, keys, native_of, out_end, tap_resampled
from test_sigmf import NAME, SIGMF, convert, encode, write_recording

pytestmark = pytest.mark.gpu

DATA_RATE = 32768
CAPTURE = 915_000_000
ALL_FORMATS = [capi.FORMAT_CU8, capi.FORMAT_CS8, capi.FORMAT_CS16, capi.FORMAT_CF32] + list(SIGMF)
CLI = os.path.join(tune_ref.ROOT, "rtlamr_b200", "ertgpu_decode_file")


def _raw(z, fmt):
    """Capture bytes of the complex signal z (8-bit units) in format fmt."""
    if fmt in (capi.FORMAT_CS8, capi.FORMAT_CS16):
        return tune_ref.quantize(z, fmt)
    u8 = np.empty(2 * z.size, dtype=np.uint8)
    u8[0::2] = np.clip(np.round(z.real + 127.5), 0, 255)
    u8[1::2] = np.clip(np.round(z.imag + 127.5), 0, 255)
    return encode(u8, fmt)


def _decoder(msgtypes, cl, rate_in, off, fmt, **kw):
    return capi.new_decoder(msgtypes, cl, input_rate=rate_in, input_format=fmt, capture_freq=CAPTURE,
                            center_freq=CAPTURE + off, **kw)


def _check_blocks(h, ref, cl, rows):
    """Every block's ERTGPU_TAP_RESAMPLED bytes equal the restatement's, and the candidates the native decode's."""
    bs = h.cfg.block_size
    nblocks = (ref.size // 2) // bs
    assert nblocks > 4
    assert np.array_equal(tap_resampled(h, 0, nblocks), ref[:2 * nblocks * bs])
    assert keys(rows) == keys(native_of("scm", cl, ref))


KERNEL_CASES = [(20_000_000, 32, capi.FORMAT_CS8, -2_400_000), (30_720_000, 72, capi.FORMAT_CS16, -2_400_000),
                (56_000_000, 72, capi.FORMAT_CS16, 6_000_000), (61_440_000, 72, capi.FORMAT_CS16, -2_400_000),
                (61_440_000, 72, capi.FORMAT_CF32, 12_000_000), (20_000_000, 8, capi.FORMAT_CS8, -2_400_000),
                (256 * DATA_RATE * 8, 8, capi.FORMAT_CS16, 30_000_000)]


@pytest.mark.parametrize("rate_in,cl,fmt,off", KERNEL_CASES)
@pytest.mark.parametrize("kind", ["random", "synthetic"])
def test_kernel_equals_cpu_restatement(built, rate_in, cl, fmt, off, kind):
    rate_out = DATA_RATE * cl
    n = 12 * (rate_in // rate_out) * (16384 * cl // 72)   # about 12 decoder blocks
    if kind == "random":
        u8 = np.random.default_rng(rate_in ^ cl).integers(0, 256, 2 * n, dtype=np.uint8)
        raw = encode(u8, fmt)
    else:
        z, _ = tune_ref.wideband([("scm", off, 11, 0), ("scm", 0, 12, 40_000)], rate_in, n, 11)
        raw = _raw(z, fmt)
    ref = decimate_ref.decimate(convert(raw, fmt), rate_in, rate_out, off)
    h = _decoder("scm", cl, rate_in, off, fmt)
    dec, _ = h.decimator()
    assert dec["D"] == decimate_ref.plan(rate_in, rate_out, off)[0]["D"] >= 3
    rows = h.decode(raw, cap=1 << 16)
    ks = h.last_kernels().split(";")
    assert ks[0].startswith("demod_") and ks[-2:] == [f"decimate_kernel<{NAME[fmt]}>", "resample_kernel<cu8>"]
    _check_blocks(h, ref, cl, rows)
    h.close()


@pytest.mark.parametrize("fmt", ALL_FORMATS)
def test_every_format(built, fmt):
    rate_in, cl, off = 30_720_000, 72, -2_400_000
    u8 = np.random.default_rng(fmt + 7).integers(0, 256, 2 * 1_200_000, dtype=np.uint8)
    raw = encode(u8, fmt)
    ref = decimate_ref.decimate(convert(raw, fmt), rate_in, DATA_RATE * cl, off)
    h = _decoder("scm", cl, rate_in, off, fmt)
    rows = h.decode(raw, cap=1 << 16)
    assert f"decimate_kernel<{NAME[fmt]}>" in h.last_kernels().split(";")
    _check_blocks(h, ref, cl, rows)
    h.close()


@pytest.mark.parametrize("rate_in,off", [(10 * DATA_RATE * 72, -2_400_000), (8_000_000, -2_400_000), (DATA_RATE * 72, 200_000)])
def test_opted_in_handle_up_to_10_to_1_is_todays_tuned_handle(built, rate_in, off):
    z, _ = tune_ref.wideband([("scm", off, 21, 0)], rate_in, 3_000_000, 21)
    raw = tune_ref.quantize(z, capi.FORMAT_CS16)
    hs = []
    for allow in (False, True):
        h = capi.Handle()
        h.register(capi.stock_protocol("scm", 72))
        h.set_input_tuning(CAPTURE, CAPTURE + off)
        if allow:
            h.allow_input_decimation()
        h.set_input_rate(rate_in)
        h.set_input_format(capi.FORMAT_CS16)
        h.allocate(0)
        hs.append((h, h.decode(raw, cap=1 << 16)))
    (a, ra), (b, rb) = hs
    assert ra.tobytes() == rb.tobytes() and a.last_kernels() == b.last_kernels() and "decimate" not in b.last_kernels()
    assert b.decimator()[0]["D"] == 1 and a.resampler()[0] == b.resampler()[0]
    nb = out_end(a.resampler()[0], raw.size // 4) // a.cfg.block_size
    assert nb > 4 and np.array_equal(tap_resampled(a, 0, nb), tap_resampled(b, 0, nb))
    a.close()
    b.close()


def _found(rows, truth, msgtype):
    valid = [r for r in rows if r["check_mask"]]
    if msgtype == "r900":
        return [any([d[2 * k] * 6 + d[2 * k + 1] for k in range(21)] == list(t.data) for d in (r["r900_digits"] for r in valid))
                for t in truth]
    return [any(r["bytes"][:len(t.data)].tobytes() == t.data for r in valid) for t in truth]


@pytest.mark.parametrize("rate_in", [30_720_000, 61_440_000])
@pytest.mark.parametrize("msgtype", ["scm", "scm+", "idm", "r900"])
def test_off_centre_packets_are_recovered(built, msgtype, rate_in):
    off, other_off = -2_400_000, 1_500_000
    spacing = 1 << 22 if msgtype == "idm" else 1 << 21   # an idm packet at 61.44 MS/s is 2.8 million samples long
    n = 7 * spacing
    z, (want, other) = decimate_ref.wideband([(msgtype, off, 61, 0), (msgtype, other_off, 1061, 40_000)], rate_in, n, 61,
                                         spacing=spacing)
    raw = tune_ref.quantize(z, capi.FORMAT_CS16)
    assert len(want) >= 3 and other
    h = _decoder(msgtype, 72, rate_in, off, capi.FORMAT_CS16)
    rows, o = [], 0
    for c in (123_457, 3_700_001, 77):
        rows.extend(h.decode(raw[o:o + 4 * c], cap=1 << 16))
        o += 4 * c
    rows.extend(h.decode(raw[o:], cap=1 << 16))
    assert all(_found(rows, want, msgtype)), msgtype
    assert not any(_found(rows, other, msgtype))
    h.close()


def test_three_channels_of_one_capture(built):
    rate_in, offs = 32_000_000, (-2_400_000, 2_000_000, 5_200_000)
    z, truths = decimate_ref.wideband([("scm", o, 71 + i, 30_000 * i) for i, o in enumerate(offs)], rate_in, 12_000_000, 71,
                                  spacing=1 << 20)
    raw = tune_ref.quantize(z, capi.FORMAT_CS8)
    for i, o in enumerate(offs):
        h = _decoder("scm", 72, rate_in, o, capi.FORMAT_CS8)
        assert h.decimator()[0]["D"] == 4
        rows = h.decode(raw, cap=1 << 16)
        for j, t in enumerate(truths):
            found = _found(rows, t, "scm")
            assert all(found) if i == j else not any(found), (i, j)
        h.close()


@pytest.mark.parametrize("rate_in,cl,fmt,off", [(61_440_000, 72, capi.FORMAT_CS16, -2_400_000),
                                                (20_000_000, 32, capi.FORMAT_CS8, 3_000_000)])
def test_call_splitting_chunking_and_reset(built, rate_in, cl, fmt, off):
    import torch
    s = capi.FORMAT_BYTES[fmt]
    z, _ = decimate_ref.wideband([("scm", off, 31, 0)], rate_in, 8_000_003, 31, spacing=1 << 20)
    raw = _raw(z, fmt)
    ref = decimate_ref.decimate(convert(raw, fmt), rate_in, DATA_RATE * cl, off)
    want = keys(native_of("scm", cl, ref))
    assert len(want) > 0
    D = decimate_ref.plan(rate_in, DATA_RATE * cl, off)[0]["D"]
    rng = np.random.default_rng(77)
    sizes = [s * (c // 2) for c in _cuts(rng, raw.size // s * 2, 40)]
    sizes[-1] += raw.size - sum(sizes)
    assert any((c // s) % D for c in sizes)
    for path, max_blocks in (("host", 0), ("device", 0), ("host", 3)):
        h = _decoder("scm", cl, rate_in, off, fmt, max_blocks_per_call=max_blocks)
        bs = h.cfg.block_size
        rows, res, o, done = [], [], 0, 0
        for c in sizes:
            part = raw[o:o + c]
            o += c
            if path == "host":
                rows.extend(h.decode(part, cap=1 << 16))
            else:
                d = torch.from_numpy(part.copy()).cuda()
                h.decode_device_async(d.data_ptr(), d.numel(), 0, torch.cuda.current_stream().cuda_stream)
                rows.extend(h.fetch(cap=1 << 16))
                del d
            if not max_blocks:
                nb = _blocks_after(o // s, rate_in, DATA_RATE * cl, off, bs)
                res.append(tap_resampled(h, done, nb))
                done = nb
        assert keys(rows) == want, (path, max_blocks)
        if not max_blocks:
            allb = np.concatenate(res)
            assert np.array_equal(allb, ref[:allb.size]) and allb.size == 2 * done * bs, path
        h.reset()   # both stages and the mixer's phase restart with the stream
        again = h.decode(raw, cap=1 << 16)
        assert keys(again) == want
        fresh = _decoder("scm", cl, rate_in, off, fmt)
        assert fresh.decode(raw, cap=1 << 16).tobytes() == again.tobytes()
        last = _blocks_after(raw.size // s, rate_in, DATA_RATE * cl, off, h.cfg.block_size) - 1   # in the last pipeline
        assert np.array_equal(h.tap(capi.TAP_RESAMPLED, last), fresh.tap(capi.TAP_RESAMPLED, last))
        fresh.close()
        h.close()
    hh = _decoder("scm", cl, rate_in, off, fmt)
    with pytest.raises(capi.ErtGpuError) as e:
        capi.decode_sharded([hh], np.zeros(8192 * s, dtype=np.uint8))
    assert e.value.code == capi.EINVAL
    hh.close()


def _blocks_after(x, rate_in, rate_out, off, bs):
    """Whole output blocks once x input samples are in: the first stage's complete outputs, then the second's."""
    dec, info = decimate_ref.plan(rate_in, rate_out, off)
    a = x - dec["T1"] // 2
    return out_end(info, -(-a // dec["D"]) if a > 0 else 0) // bs


def test_256mib_device_resident_call(built):
    import torch
    cl, fmt, off, rate_in = 72, capi.FORMAT_CS16, -2_400_000, 61_440_000
    n = 64 << 20   # 256 MiB of cs16
    raw = np.random.default_rng(81).integers(0, 256, 4 * n, dtype=np.uint8)
    ref = decimate_ref.decimate(convert(raw, fmt), rate_in, DATA_RATE * cl, off)
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


def _ids(stdout):
    return {json.loads(l)["Message"]["ID"] for l in stdout.splitlines()}


def test_cli_decodes_wide_captures(built, tmp_path):
    off = -2_399_845   # scm's 912.6 MHz channel of a 915 MHz capture
    common = ["-msgtype=scm", "-format=json"]
    # raw cs16 at 61.44 MS/s
    z, (want, other) = decimate_ref.wideband([("scm", off, 101, 0), ("scm", 1_500_000, 1101, 40_000)], 61_440_000,
                                         10_000_000, 101, spacing=1 << 20)
    path = tmp_path / "wide.cs16"
    tune_ref.quantize(z, capi.FORMAT_CS16).tofile(path)
    args = common + ["-sampleformat=cs16", "-samplerate=61440000", "-capturefreq=915000000"]
    r = subprocess.run([CLI] + args + [str(path)], capture_output=True, text=True, timeout=600, check=True)
    assert "Decimation: 7\nIntermediateRate: 8777142.857\n" in r.stderr
    ids = _ids(r.stdout)
    assert {_scm_fields(t.data)[0] for t in want} <= ids and not ({_scm_fields(t.data)[0] for t in other} & ids)
    auto = subprocess.run([CLI] + args + ["-samplescale=auto", str(path)], capture_output=True, text=True, timeout=600,
                          check=True)
    g = re.search(r"-samplescale=auto: 2\^(-?\d+) = (\S+) from", auto.stderr).group(2)
    fixed = subprocess.run([CLI] + args + [f"-samplescale={g}", str(path)], capture_output=True, text=True, timeout=600,
                           check=True)
    strip = lambda s: [json.dumps({k: v for k, v in json.loads(l).items() if k != "Time"}) for l in s.splitlines()]
    assert strip(auto.stdout) == strip(fixed.stdout) and auto.stdout
    # a SigMF recording at 30.72 MS/s: format, rate and capture frequency from the metadata
    z, (want,) = decimate_ref.wideband([("scm", off, 111, 0)], 30_720_000, 6_000_000, 111, spacing=1 << 20)
    base = write_recording(tmp_path / "rec", tune_ref.quantize(z, capi.FORMAT_CS16).tobytes(), "ci16_le", 30_720_000,
                           captures=[{"core:sample_start": 0, "core:frequency": CAPTURE}])
    r = subprocess.run([CLI] + common + ["-sampleformat=sigmf", base], capture_output=True, text=True, timeout=600,
                       check=True)
    assert "Decimation: 4\nIntermediateRate: 7680000.000\n" in r.stderr
    assert {_scm_fields(t.data)[0] for t in want} <= _ids(r.stdout)


def test_host_receiver_decimates(built):
    from rtlamr_b200 import host
    rate_in = 30_720_000
    z, (want,) = decimate_ref.wideband([("scm", -2_399_845, 121, 0)], rate_in, 5_000_000, 121, spacing=1 << 20)
    raw = tune_ref.quantize(z, capi.FORMAT_CS8)
    r = host.Receiver("scm", 72, input_rate=rate_in, input_format=capi.FORMAT_CS8, capture_freq=CAPTURE)
    assert "Decimation: 4" in r.log()
    msgs = r.decode(raw[:2 * 1_000_001]) + r.decode(raw[2 * 1_000_001:])
    assert {_scm_fields(t.data)[0] for t in want} <= {m.meter_id for m in msgs}
    r.close()
