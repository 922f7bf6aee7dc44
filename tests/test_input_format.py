"""CPU tests of the input-format conversion: the numpy restatement (tests/format_ref.py) against independent
statements of the formula, the exact round trips the GPU tests rely on, the WAV header reader, the argument checks of
ertgpu_set_input_format that need no GPU, and the file receiver's usage errors."""
import os
import struct
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from rtlamr_b200 import capi, host

import format_ref
from format_ref import DEFAULT_SCALE, to_u8, wav_bytes

CLI = os.path.join(ROOT, "rtlamr_b200", "ertgpu_decode_file")


def _exact(x: float, g: float) -> int:
    """The formula from exact arithmetic: the double product of two float32 values is exact, its conversion to
    float32 rounds to nearest even, round() rounds half to even."""
    p = float(np.float32(float(x) * float(np.float32(g))))
    if p != p:
        return 128
    if p in (float("inf"), float("-inf")):
        return 255 if p > 0 else 0
    return min(127, max(-128, round(p))) + 128


@pytest.mark.parametrize("g", [2.0 ** -8, 2.0 ** -4, 0.3])
def test_every_int16_value(g):
    x = np.arange(-32768, 32768, dtype=np.int16)
    want = np.array([_exact(v, g) for v in x.tolist()], dtype=np.uint8)
    assert np.array_equal(to_u8(x, g), want)


@pytest.mark.parametrize("g", [1.0, 0.3, 1.7])
def test_every_int8_value(g):
    x = np.arange(-128, 128, dtype=np.int8)
    want = np.array([_exact(v, g) for v in x.tolist()], dtype=np.uint8)
    assert np.array_equal(to_u8(x, g), want)
    if g == 1.0:
        assert np.array_equal(to_u8(x, g), (x.astype(np.int32) + 128).astype(np.uint8))


def test_float_specials():
    f32 = np.float32
    up, down = (lambda v: np.nextafter(f32(v), f32(np.inf))), (lambda v: np.nextafter(f32(v), f32(-np.inf)))
    cases = {  # x at g = 1: u
        0.0: 128, -0.0: 128, np.inf: 255, -np.inf: 0, np.nan: 128, -np.nan: 128,
        1e-45: 128, -1e-45: 128, 1.1754942e-38: 128,          # denormals
        0.5: 128, -0.5: 128, 1.5: 130, -1.5: 126, 2.5: 130,    # half-way: to even
        126.5: 254, 127.5: 255, 128.5: 255, -127.5: 0, -128.5: 0, -129.5: 0, 1e30: 255, -1e30: 0,
        float(up(0.5)): 129, float(down(0.5)): 128, float(up(1.5)): 130, float(down(1.5)): 129,
        float(up(126.5)): 255, float(down(126.5)): 254, float(down(127.5)): 255, float(up(-128.5)): 0,
        float(up(-127.5)): 1, float(down(-127.5)): 0, float(up(-126.5)): 2, float(down(-126.5)): 1,
    }
    x = np.array(list(cases), dtype=np.float32)
    assert np.array_equal(to_u8(x, 1.0), np.array(list(cases.values()), dtype=np.uint8))
    for v, u in cases.items():
        assert _exact(v, 1.0) == u, v
    # at the default 2^7 the same values, divided by 128 (exact), give the same bytes
    assert np.array_equal(to_u8(x / np.float32(128), DEFAULT_SCALE[capi.FORMAT_CF32])[np.isfinite(x) & (np.abs(x) > 1e-30)],
                          to_u8(x, 1.0)[np.isfinite(x) & (np.abs(x) > 1e-30)])
    # fl32(0.3) * 5 lies exactly half-way between two float32 values: the product rounds to even, 1.5, then to 2
    assert to_u8(np.float32(5), 0.3)[()] == _exact(5, 0.3) == 130


@pytest.mark.parametrize("fmt", [capi.FORMAT_CS8, capi.FORMAT_CS16, capi.FORMAT_CF32])
def test_round_trip_is_exact(fmt):
    u = np.arange(256, dtype=np.uint8)
    raw = format_ref.encode(np.repeat(u, 2), fmt)
    assert raw.size == 256 * capi.FORMAT_BYTES[fmt]
    assert np.array_equal(format_ref.convert(raw, fmt), np.repeat(u, 2))


def _probe(tmp_path, data: bytes, name="x.wav"):
    p = tmp_path / name
    p.write_bytes(data)
    return host.wav_probe(str(p))


def test_wav_probe_encodings(built, tmp_path):
    pay = bytes(range(256)) * 4
    for kw, fmt in [(dict(bits=8), capi.FORMAT_CU8), (dict(bits=16), capi.FORMAT_CS16),
                    (dict(bits=32, tag=3), capi.FORMAT_CF32), (dict(bits=16, extensible=True), capi.FORMAT_CS16),
                    (dict(bits=32, tag=3, extensible=True), capi.FORMAT_CF32), (dict(bits=8, extensible=True), capi.FORMAT_CU8)]:
        w = wav_bytes(pay, rate=2_400_000, **kw)
        got = _probe(tmp_path, w)
        assert got == {"format": fmt, "rate": 2_400_000, "data_offset": len(w) - len(pay), "data_size": len(pay)}, kw
    # RF64: the data size comes from ds64
    w = wav_bytes(pay, bits=32, tag=3, rate=2_359_296, rf64=True)
    assert _probe(tmp_path, w) == {"format": capi.FORMAT_CF32, "rate": 2_359_296, "data_offset": len(w) - len(pay),
                                   "data_size": len(pay)}


def test_wav_probe_chunks_and_sizes(built, tmp_path):
    pay = bytes(1000)
    auxi = b"auxi" + struct.pack("<I", 5) + b"abcde" + b"\0"   # odd size: one pad byte
    w = wav_bytes(pay, bits=16, rate=2_048_000, before_data=auxi + b"LIST" + struct.pack("<I", 4) + b"INFO")
    assert _probe(tmp_path, w) == {"format": capi.FORMAT_CS16, "rate": 2_048_000, "data_offset": len(w) - len(pay),
                                   "data_size": len(pay)}
    for size in (0, 0xFFFFFFFF, len(pay) + 2):   # unknown, or running past the end of the file: read to the end
        assert _probe(tmp_path, wav_bytes(pay, bits=16, rate=2_048_000, data_size=size))["data_size"] == -1, size
    # an RF64 file with an unknown size in ds64
    assert _probe(tmp_path, wav_bytes(pay, bits=16, rate=2_048_000, rf64=True, data_size=0))["data_size"] == -1


@pytest.mark.parametrize("kw,field", [(dict(bits=16, channels=1), "channels"), (dict(bits=24), "bits per sample"),
                                      (dict(bits=8, tag=6), "format tag 0x0006"), (dict(bits=64, tag=3), "bits per sample")])
def test_wav_probe_rejects(built, tmp_path, kw, field):
    with pytest.raises(ValueError) as e:
        _probe(tmp_path, wav_bytes(bytes(64), rate=2_400_000, **kw))
    assert field in str(e.value)


def test_wav_probe_rejects_truncated_and_foreign(built, tmp_path):
    w = wav_bytes(bytes(64), bits=16, rate=2_400_000)
    for cut in (6, 20, 30, 40):
        with pytest.raises(ValueError) as e:
            _probe(tmp_path, w[:cut])
        assert "truncated" in str(e.value), cut
    with pytest.raises(ValueError) as e:
        _probe(tmp_path, b"\x80" * 64)
    assert "RIFF" in str(e.value)


def test_format_checks_without_gpu(built):
    h = capi.Handle()
    h.register(capi.stock_protocol("scm", 72))
    for fmt, scale in [(4, 0.0), (-1, 0.0), (capi.FORMAT_CS16, -1.0), (capi.FORMAT_CS16, float("nan")),
                       (capi.FORMAT_CF32, float("inf")), (capi.FORMAT_CS8, -float("inf")), (capi.FORMAT_CU8, 1.0),
                       (capi.FORMAT_CU8, 2.0 ** -8)]:
        with pytest.raises(capi.ErtGpuError) as e:
            h.set_input_format(fmt, scale)
        assert e.value.code == capi.EINVAL, (fmt, scale)
    assert h.input_format() == (capi.FORMAT_CU8, 0.0)   # a rejected call changes nothing
    for fmt, g in DEFAULT_SCALE.items():
        h.set_input_format(fmt)
        assert h.input_format() == (fmt, g)
    h.set_input_format(capi.FORMAT_CS16, 0.0625)
    assert h.input_format() == (capi.FORMAT_CS16, 0.0625)
    h.set_input_rate(2_400_000)   # the rate after the format: the order is free
    # a resampling cs16 handle takes whole 4-byte samples
    with pytest.raises(capi.ErtGpuError) as e:
        h.decode(np.zeros(4098, dtype=np.uint8))
    assert e.value.code == capi.ESIZE
    h.set_input_format(capi.FORMAT_CU8)
    assert h.input_format() == (capi.FORMAT_CU8, 0.0)
    h.close()


def _cli(*args, stdin=None):
    r = subprocess.run([CLI, *args], capture_output=True, timeout=60, input=stdin)
    r.stderr = r.stderr.decode(errors="replace")
    return r


def test_cli_usage_errors(built, tmp_path):
    raw = tmp_path / "in.bin"
    np.zeros(1 << 14, dtype=np.uint8).tofile(raw)
    w8 = tmp_path / "a8.wav"
    w8.write_bytes(wav_bytes(bytes(1 << 14), bits=8, rate=2_359_296))
    w8b = tmp_path / "b8.wav"
    w8b.write_bytes(wav_bytes(bytes(1 << 14), bits=8, rate=2_400_000))
    w16 = tmp_path / "a16.wav"
    w16.write_bytes(wav_bytes(bytes(1 << 14), bits=16, rate=2_359_296))
    sf = f"-samplefile={tmp_path / 's.bin'}"
    cases = [
        (["-sampleformat=cs12", str(raw)], "-sampleformat"),
        (["-sampleformat=WAV", str(raw)], "-sampleformat"),
        (["-samplescale=0.5", str(raw)], "-samplescale"),
        (["-sampleformat=cu8", "-samplescale=2", str(raw)], "-samplescale"),
        (["-sampleformat=cs16", "-samplescale=-1", str(raw)], "-samplescale"),
        (["-sampleformat=cs16", "-samplescale=nan", str(raw)], "-samplescale"),
        (["-sampleformat=cs16", "-samplescale=x", str(raw)], "-samplescale"),
        (["-sampleformat=wav", "-samplescale=0.5", str(w8)], "-samplescale"),   # an 8-bit WAV is cu8
        (["-sampleformat=wav", "-samplerate=2400000", str(w8)], "-samplerate"),
        (["-sampleformat=wav", str(w8), str(w8b)], "batch"),
        (["-sampleformat=wav", str(w8), str(w16)], "batch"),
        (["-sampleformat=cs8", sf, str(raw)], "-samplefile"),
        (["-sampleformat=cf32", sf, str(raw)], "-samplefile"),
        (["-sampleformat=wav", sf, str(w16)], "-samplefile"),
        (["-sampleformat=wav", "-symbollength=72", sf, str(w8b)], "-samplefile"),
    ]
    for args, word in cases:
        r = _cli(*args)
        assert r.returncode == 2 and word in r.stderr, (args, r.returncode, r.stderr)
        assert "CenterFreq" not in r.stderr, args   # no decoder was set up
    assert not (tmp_path / "s.bin").exists()
    # a WAV header that cannot be decoded is an error naming the field, also before any device
    mono = tmp_path / "mono.wav"
    mono.write_bytes(wav_bytes(bytes(64), bits=16, channels=1, rate=2_400_000))
    r = _cli("-sampleformat=wav", str(mono))
    assert r.returncode == 1 and "channels" in r.stderr and "CenterFreq" not in r.stderr
    r = _cli("-sampleformat=wav", "-", stdin=wav_bytes(bytes(64), bits=24, rate=2_400_000))
    assert r.returncode == 1 and "bits per sample" in r.stderr
