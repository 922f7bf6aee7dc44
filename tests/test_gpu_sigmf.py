"""GPU tests (-m gpu) of SigMF input: convert_kernel and the resample_kernel instances of the ten SigMF formats after
cf32 against the restatement in tests/test_sigmf.py byte for byte (at the decoder's rate, resampled, and tuned), call
splitting and chunking with up to 16-byte samples, the golden capture as raw samples of every new format and as a
SigMF recording of every datatype (with capture segments and header bytes too), the Time fields of a dated recording,
an off-centre ci16_be recording, and the host binding fed from host.sigmf_probe."""
import json
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from rtlamr_b200 import capi, host

import resample_ref
import tune_ref
from test_gpu_input_format import _cuts, _scm_fields, keys, native_keys, taps, u8_stream
from test_sigmf import DATATYPES, NAME, NEW_FORMATS, SIGMF, _ns_ref, convert, encode, with_headers, write_recording

pytestmark = pytest.mark.gpu

DATA_RATE = 32768
CLI = os.path.join(ROOT, "rtlamr_b200", "ertgpu_decode_file")
GOLDEN_RATE = 2_555_904   # tests/golden/sample_cl78.bin: uint8 IQ at 32768 * 78 S/s


def random_raw(fmt, nsamples, seed):
    """Random raw IQ of format fmt: every stored value of an integer format, floats around full scale with specials."""
    rng = np.random.default_rng(seed)
    s = capi.FORMAT_BYTES[fmt]
    if SIGMF[fmt][1][1] != "f":
        return rng.integers(0, 256, s * nsamples, dtype=np.uint8)
    x = rng.standard_normal(2 * nsamples) * 0.7
    sp = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 5e-324, -1e-310, 0.5 / 128, 1.5 / 128, 127.5 / 128, -128.5 / 128,
                   126.5 / 128, 1e30, -1e30])
    at = rng.choice(x.size, min(4096, x.size // 4), replace=False)
    x[at] = sp[rng.integers(0, sp.size, at.size)]
    with np.errstate(over="ignore"):
        return x.astype(SIGMF[fmt][1]).view(np.uint8)


@pytest.mark.parametrize("fmt", NEW_FORMATS)
def test_native_kernel_equals_restatement(built, fmt):
    cl = 72
    h = capi.new_decoder("scm", cl, input_format=fmt)
    bs = h.cfg.block_size
    nblocks = 40
    raw = random_raw(fmt, nblocks * bs, seed=fmt)
    got = h.decode(raw, cap=1 << 16)
    want = convert(raw, fmt)
    assert np.array_equal(taps(h, 0, nblocks), want)
    assert h.last_kernels().split(";")[-1] == f"convert_kernel<{NAME[fmt]}>"
    assert keys(got) == native_keys("scm", cl, want)
    h.close()


@pytest.mark.parametrize("fmt", NEW_FORMATS)
def test_resampling_kernel_equals_restatement(built, fmt):
    rate_in, cl, n = 2_400_000, 72, 300_000
    raw = random_raw(fmt, n, seed=100 + fmt)
    ref = resample_ref.resample(convert(raw, fmt), rate_in, DATA_RATE * cl)
    h = capi.new_decoder("scm", cl, input_rate=rate_in, input_format=fmt)
    got = h.decode(raw, cap=1 << 16)
    nblocks = (ref.size // 2) // h.cfg.block_size
    assert nblocks > 4
    assert np.array_equal(taps(h, 0, nblocks), ref[:2 * nblocks * h.cfg.block_size])
    assert h.last_kernels().split(";")[-1] == f"resample_kernel<{NAME[fmt]}>"
    assert keys(got) == native_keys("scm", cl, ref)
    h.close()


@pytest.mark.parametrize("fmt", NEW_FORMATS)
def test_tuned_kernel_equals_restatement(built, fmt):
    rate_in, cl, off, capture = 10_000_000, 72, -2_400_000, 915_000_000
    n = 1_000_000
    raw = random_raw(fmt, n, seed=200 + fmt)
    ref = tune_ref.tune(convert(raw, fmt), rate_in, DATA_RATE * cl, off)
    h = capi.new_decoder("scm", cl, input_rate=rate_in, input_format=fmt, capture_freq=capture, center_freq=capture + off)
    got = h.decode(raw, cap=1 << 16)
    nblocks = (ref.size // 2) // h.cfg.block_size
    assert nblocks > 4
    assert f"resample_kernel<{NAME[fmt]},tuned>" in h.last_kernels().split(";")
    assert np.array_equal(taps(h, 0, nblocks), ref[:2 * nblocks * h.cfg.block_size])
    assert keys(got) == native_keys("scm", cl, ref)
    h.close()


@pytest.mark.parametrize("fmt", [capi.FORMAT_CS16BE, capi.FORMAT_CU32BE, capi.FORMAT_CF64, capi.FORMAT_CF64BE])
@pytest.mark.parametrize("rate_in", [DATA_RATE * 72, 2_400_000])
def test_call_splitting_host_and_device(built, fmt, rate_in):
    import torch
    cl, msgtypes = 72, "scm,r900"
    u8, _ = u8_stream(msgtypes, rate_in, 1_200_000, seed=31)
    s = capi.FORMAT_BYTES[fmt]
    native = rate_in == DATA_RATE * cl
    whole = capi.new_decoder(msgtypes, cl, input_rate=rate_in, input_format=fmt)
    bs = whole.cfg.block_size
    nsamples = (u8.size // 2) // bs * bs if native else u8.size // 2
    raw = encode(u8, fmt)[:nsamples * s]
    want = keys(whole.decode(raw, cap=1 << 16))
    whole.close()
    assert want
    rng = np.random.default_rng(rate_in + fmt)
    sizes = _cuts(rng, nsamples // bs, bs, (4, 16, 64)) if native else _cuts(rng, nsamples, 1, (64, 5000, 200_000))
    assert len(sizes) >= 8
    for path in ("host", "device"):
        h = capi.new_decoder(msgtypes, cl, input_rate=rate_in, input_format=fmt)
        rows, off = [], 0
        for n in sizes:
            part = raw[off * s:(off + n) * s]
            off += n
            if path == "host":
                rows.extend(h.decode(part, cap=1 << 16))
            else:
                d = torch.from_numpy(part.copy()).cuda()
                h.decode_device_async(d.data_ptr(), d.numel(), 0, torch.cuda.current_stream().cuda_stream)
                rows.extend(h.fetch(cap=1 << 16))
                del d
        assert keys(rows) == want, path
        h.close()


@pytest.mark.parametrize("rate_in", [DATA_RATE * 72, 1_024_000])
def test_host_chunking_respects_max_blocks_with_16_byte_samples(built, rate_in):
    import torch
    cl, fmt = 72, capi.FORMAT_CF64BE
    u8, _ = u8_stream("scm", rate_in, 400_000, seed=41)
    raw = encode(u8, fmt)
    h = capi.new_decoder("scm", cl, input_rate=rate_in, input_format=fmt, max_blocks_per_call=3)
    bs = h.cfg.block_size
    if rate_in == DATA_RATE * cl:
        raw = raw[:(u8.size // 2) // bs * bs * 16]
        want = native_keys("scm", cl, convert(raw, fmt))
    else:
        want = native_keys("scm", cl, resample_ref.resample(convert(raw, fmt), rate_in, DATA_RATE * cl))
    assert keys(h.decode(raw, cap=1 << 16)) == want
    h.reset()
    d = torch.from_numpy(raw).cuda()
    with pytest.raises(capi.ErtGpuError) as e:
        h.decode_device_async(d.data_ptr(), d.numel(), 0, torch.cuda.current_stream().cuda_stream)
    assert e.value.code == capi.ESIZE
    rows, step = [], 16 * 2 * bs if rate_in == DATA_RATE * cl else 16 * 4096
    for off in range(0, raw.size, step):
        h.decode_device_async(d.data_ptr() + off, min(step, raw.size - off), 0, torch.cuda.current_stream().cuda_stream)
        rows.extend(h.fetch(cap=1 << 16))
    assert keys(rows) == want
    h.close()


def _run_cli(*args, ok=True):
    r = subprocess.run([CLI, *map(str, args)], capture_output=True, text=True, timeout=300)
    if ok:
        assert r.returncode == 0, r.stderr
    return r.stdout.splitlines()


COMMON = ["-msgtype=scm", "-symbollength=78", "-blocks=7"]


def _golden():
    src = os.path.join(GOLDEN, "sample_cl78.bin")
    want = _run_cli(*COMMON, src)
    assert len(want) >= 10
    return np.fromfile(src, dtype=np.uint8), want


def test_golden_capture_raw_in_every_new_format(built, tmp_path):
    u8, want = _golden()
    for fmt in NEW_FORMATS:
        p = tmp_path / f"in.{NAME[fmt]}"
        encode(u8, fmt).tofile(p)
        assert _run_cli(*COMMON, f"-sampleformat={NAME[fmt]}", p) == want, NAME[fmt]


def test_golden_capture_as_sigmf_of_every_datatype(built, tmp_path):
    u8, want = _golden()
    for name, fmt in DATATYPES.items():
        base = write_recording(tmp_path / name, encode(u8, fmt).tobytes(), name, GOLDEN_RATE)
        assert _run_cli(*COMMON, "-sampleformat=sigmf", base + ".sigmf-meta") == want, name
    # capture segments with junk header bytes: the same samples, the same lines; the stream carries on across segments
    n = u8.size // 2
    starts, headers = [0, 12_345, 200_001, n - 1000], [7, 33, 1, 4096]
    for name in ("cu8", "ci16_be", "cf64_le"):
        fmt = DATATYPES[name]
        data = with_headers(encode(u8, fmt).tobytes(), capi.FORMAT_BYTES[fmt], starts, headers)
        caps = [{"core:sample_start": s, "core:header_bytes": h} for s, h in zip(starts, headers)]
        base = write_recording(tmp_path / f"seg_{name}", data, name, GOLDEN_RATE, captures=caps)
        assert _run_cli(*COMMON, "-sampleformat=sigmf", base + ".sigmf-data") == want, name
        assert _run_cli(*COMMON, "-sampleformat=sigmf", base, base) == want + want, name   # a batch of two


def _times(lines, fmt):
    if fmt == "json":
        return [_ns_ref(json.loads(l)["Time"]) for l in lines]
    if fmt == "xml":
        return [_ns_ref(re.search(r'Time="([^"]*)"', l).group(1)) for l in lines]
    return [_ns_ref(l.split(",")[0]) for l in lines]


@pytest.mark.parametrize("rate", [GOLDEN_RATE, 2_400_000])
def test_times_come_from_block_time(built, tmp_path, rate):
    """A dated recording's csv, json and xml Time fields are sigmf::BlockTime of the message's block, at the decoder's
    rate and resampled."""
    if rate == GOLDEN_RATE:
        u8, _ = _golden()
        cl = 78
    else:
        u8, _ = u8_stream("scm", rate, 3_000_000, seed=5)
        cl = 72
    common = ["-msgtype=scm", f"-symbollength={cl}", "-blocks=7"]
    n = u8.size // 2
    caps = [{"core:sample_start": 0}, {"core:sample_start": 1000, "core:datetime": "2025-06-01T12:00:00.123456789Z"},
            {"core:sample_start": n // 2, "core:datetime": "2025-06-01T13:00:00-02:30"}]
    base = write_recording(tmp_path / "t", u8.tobytes(), "cu8", rate, captures=caps)
    plain = _run_cli(*common, "-sampleformat=sigmf", base)
    assert len(plain) >= 10
    blocks = [int(re.match(r"\{Block:(\d+) ", l).group(1)) for l in plain]
    h = capi.new_decoder("scm", cl)
    bs, rate_out = h.cfg.block_size, DATA_RATE * cl
    h.close()
    want = [host.sigmf_block_time(base, b, bs, rate_out) for b in blocks]
    assert len(set(want)) > 1
    for fmt in ("json", "csv", "xml"):
        lines = _run_cli(*common, "-sampleformat=sigmf", f"-format={fmt}", base)
        assert _times(lines, fmt) == want, fmt
    # an undated recording keeps the wall clock
    und = write_recording(tmp_path / "u", u8.tobytes(), "cu8", rate)
    assert all(t > want[-1] for t in _times(_run_cli(*common, "-sampleformat=sigmf", "-format=json", und), "json"))


def test_off_centre_ci16_be_recording(built, tmp_path):
    rate_in, n, off, capture = 10_000_000, 8_000_000, -2_400_000, 915_000_000
    z, truths = tune_ref.wideband([("scm,idm", off, 61, 0)], rate_in, n, 61)
    cs16 = tune_ref.quantize(z, capi.FORMAT_CS16)
    raw = tmp_path / "cap.cs16"
    cs16.tofile(raw)
    base = write_recording(tmp_path / "cap", cs16.view("<i2").astype(">i2").tobytes(), "ci16_be", rate_in,
                           captures=[{"core:sample_start": 0, "core:frequency": capture}])
    common = ["-msgtype=scm,idm", "-symbollength=72", "-format=json", f"-centerfreq={capture + off}"]
    got = _run_cli(*common, "-sampleformat=sigmf", base)
    ref = _run_cli(*common, "-sampleformat=cs16", f"-samplerate={rate_in}", f"-capturefreq={capture}", raw)
    strip = lambda lines: [json.dumps({k: v for k, v in json.loads(l).items() if k != "Time"}) for l in lines]
    assert strip(got) == strip(ref)
    msgs = [json.loads(l)["Message"] for l in got]
    truth = truths[0]
    assert len(truth) >= 10
    for t in truth:
        if t.msgtype == "scm":
            mid, cons = _scm_fields(t.data)
            assert any(m.get("ID") == mid and m.get("Consumption") == cons for m in msgs), mid
        else:
            assert any(m.get("ERTSerialNumber") == t.meter_id for m in msgs), t.meter_id


def test_host_receiver_fed_from_the_probe(built, tmp_path):
    u8, truth = u8_stream("scm", 2_400_000, 1_000_000, seed=111)
    base = write_recording(tmp_path / "p", encode(u8, capi.FORMAT_CU32BE).tobytes(), "cu32_be", 2.4e6)
    p = host.sigmf_probe(base)
    assert p["format"] == capi.FORMAT_CU32BE and p["rate"] == 2_400_000
    r = host.Receiver("scm", 72, input_rate=p["rate"], input_format=p["format"], capture_freq=p["frequency"] or 0)
    raw = np.fromfile(p["data_path"], dtype=np.uint8)
    s = capi.FORMAT_BYTES[p["format"]]
    msgs = r.decode(raw[:s * 333_333]) + r.decode(raw[s * 333_333:])
    ids = {_scm_fields(t.data)[0] for t in truth}
    assert ids and ids <= {m.meter_id for m in msgs}
    r.close()
