"""CPU tests of SigMF input: a numpy restatement of the ten SigMF sample formats' conversion against exact integer and
Fraction arithmetic, their identity encodings, the SigMF metadata reader and its JSON parser (host.sigmf_probe), the
block times of sigmf::BlockTime against Fraction, the new ertgpu_set_input_format constants, and the file receiver's
SigMF usage errors.  The restatement and the recording writer are shared with tests/test_gpu_sigmf.py."""
from __future__ import annotations

import datetime as dt
import json
import os
import struct
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from conftest import ROOT
from rtlamr_b200 import capi, host

import format_ref

CLI = os.path.join(ROOT, "rtlamr_b200", "ertgpu_decode_file")

# the ten formats after cf32: SigMF name, numpy dtype of one component, offset subtracted, default gain
SIGMF = {
    capi.FORMAT_CS16BE: ("ci16_be", ">i2", 0, 2.0 ** -8),
    capi.FORMAT_CF32BE: ("cf32_be", ">f4", 0, 2.0 ** 7),
    capi.FORMAT_CU16: ("cu16_le", "<u2", 2 ** 15, 2.0 ** -8),
    capi.FORMAT_CU16BE: ("cu16_be", ">u2", 2 ** 15, 2.0 ** -8),
    capi.FORMAT_CS32: ("ci32_le", "<i4", 0, 2.0 ** -24),
    capi.FORMAT_CS32BE: ("ci32_be", ">i4", 0, 2.0 ** -24),
    capi.FORMAT_CU32: ("cu32_le", "<u4", 2 ** 31, 2.0 ** -24),
    capi.FORMAT_CU32BE: ("cu32_be", ">u4", 2 ** 31, 2.0 ** -24),
    capi.FORMAT_CF64: ("cf64_le", "<f8", 0, 2.0 ** 7),
    capi.FORMAT_CF64BE: ("cf64_be", ">f8", 0, 2.0 ** 7),
}
NEW_FORMATS = list(SIGMF)
# every complex SigMF datatype and its format
DATATYPES = {"cu8": capi.FORMAT_CU8, "ci8": capi.FORMAT_CS8, "ci16_le": capi.FORMAT_CS16, "cf32_le": capi.FORMAT_CF32,
             **{v[0]: f for f, v in SIGMF.items()}}
NAME = {**format_ref.NAME, **{f: v[0] for f, v in SIGMF.items()}}


def components(raw, fmt) -> np.ndarray:
    """x of every component: the stored value less the offset, int64 or float64 (float32 for cf32_be)."""
    name, dtype, off, _ = SIGMF[fmt]
    v = np.ascontiguousarray(raw, dtype=np.uint8).view(dtype)
    if dtype[1] == "f":
        return v.astype(v.dtype.newbyteorder("="))
    return v.astype(np.int64) - off


def convert(raw, fmt: int, scale: float = 0.0) -> np.ndarray:
    """The uint8 IQ bytes the decoder reads for raw bytes of format fmt (any format)."""
    if fmt not in SIGMF:
        return format_ref.convert(raw, fmt, scale)
    g = np.float32(scale or SIGMF[fmt][3])
    x = components(raw, fmt)
    if fmt in (capi.FORMAT_CS16BE, capi.FORMAT_CU16, capi.FORMAT_CU16BE, capi.FORMAT_CF32BE):   # exact in float32
        return format_ref.to_u8(x.astype(np.float32), float(g))
    with np.errstate(invalid="ignore", over="ignore"):
        p = x.astype(np.float64) * np.float64(g)   # one double multiply, round to nearest even
        v = np.where(np.isnan(p), 0.0, np.clip(np.rint(p), -128, 127))
    return (v + 128).astype(np.uint8)


def encode(u8, fmt: int) -> np.ndarray:
    """uint8 IQ as raw bytes of format fmt that convert() at the default gain maps back exactly."""
    if fmt not in SIGMF:
        return format_ref.encode(u8, fmt)
    name, dtype, off, _ = SIGMF[fmt]
    v = np.asarray(u8, dtype=np.int64) - 128
    if dtype[1] == "f":
        return (v.astype(np.float64) / 128).astype(dtype).view(np.uint8)
    bits = np.dtype(dtype).itemsize * 8
    return (v * 2 ** (bits - 8) + off).astype(dtype).view(np.uint8)


def write_recording(base, data: bytes, datatype: str, rate, *, captures=None, glob_extra=None, meta_text=None):
    """base.sigmf-meta and base.sigmf-data; captures defaults to one segment at sample 0."""
    meta = {"global": {"core:datatype": datatype, "core:sample_rate": rate, "core:version": "1.0.0", **(glob_extra or {})},
            "captures": captures if captures is not None else [{"core:sample_start": 0}], "annotations": []}
    with open(f"{base}.sigmf-meta", "w") as f:
        f.write(meta_text if meta_text is not None else json.dumps(meta))
    with open(f"{base}.sigmf-data", "wb") as f:
        f.write(data)
    return str(base)


def with_headers(raw: bytes, sample_bytes: int, starts, headers, junk=0xA5):
    """raw samples laid out with headers[k] junk bytes before sample starts[k]."""
    out, prev = bytearray(), 0
    for s, h in zip(starts, headers):
        out += raw[prev * sample_bytes:s * sample_bytes] + bytes([junk]) * h
        prev = s
    return bytes(out + raw[prev * sample_bytes:])


def block_time_ref(segs, rate_in, block, block_size, rate_out):
    """sigmf::BlockTime from its definition, in Fraction."""
    n = (block + 1) * block_size
    dated = [s for s in segs if s["datetime_ns"] is not None]
    before = [s for s in dated if s["start"] * rate_out <= n * rate_in]
    k = before[-1] if before else dated[0]
    t = Fraction(n, rate_out) - Fraction(k["start"], rate_in)   # seconds after the segment's first sample
    return k["datetime_ns"] + (t * 10 ** 9).__floor__()


# ---- the conversion ----

def _exact(x, g, double: bool) -> int:
    """The formula from exact arithmetic: Fraction product, rounded to float32 (16-bit and cf32_be) or float64 (Python's
    int / int is correctly rounded), clamped, rounded half to even by round()."""
    if isinstance(x, float) and x != x:
        return 128
    if isinstance(x, float) and x in (float("inf"), float("-inf")):
        return 255 if (x > 0) == (g > 0) else 0
    prod = Fraction(x) * Fraction(float(np.float32(g)))
    p = prod.numerator / prod.denominator if prod.numerator.bit_length() < 1100 else float("inf") * (1 if prod > 0 else -1)
    if not double:
        p = float(np.float32(p)) if abs(p) < 3.4e38 else p   # the double product of x and g is exact here
    if p in (float("inf"), float("-inf")):
        return 255 if p > 0 else 0
    return min(127, max(-128, round(p))) + 128


@pytest.mark.parametrize("fmt", [capi.FORMAT_CS16BE, capi.FORMAT_CU16, capi.FORMAT_CU16BE])
@pytest.mark.parametrize("g", [2.0 ** -8, 0.3])
def test_every_16bit_value(fmt, g):
    name, dtype, off, _ = SIGMF[fmt]
    v = np.arange(65536, dtype=np.uint32)
    raw = v.astype(dtype).view(np.uint8)                     # every stored value in the format's byte order
    assert np.array_equal(components(raw, fmt), v.astype(np.int64) - off if off else v.astype(np.uint16).view(np.int16))
    want = np.array([_exact(int(x), g, False) for x in components(raw, fmt).tolist()], dtype=np.uint8)
    assert np.array_equal(convert(raw, fmt, g), want)
    # the byte order matters: the same bytes read little-endian give other values
    if dtype[0] == ">":
        assert not np.array_equal(raw.view(dtype), raw.view("<" + dtype[1:]))


def _half_steps(g):
    """int32 x whose product with fl32(g) lies on or next to a half-integer step, and the extremes."""
    gf = Fraction(float(np.float32(g)))
    xs = {0, 1, -1, 2 ** 31 - 1, -2 ** 31, 2 ** 30, -2 ** 30}
    for k in [0, 1, 2, 62, 125, 126, 127, 128, 200]:
        for sgn in (1, -1):
            x0 = (sgn * (Fraction(2 * k + 1, 2)) / gf).__floor__()
            xs.update(x for x in (x0 - 1, x0, x0 + 1, x0 + 2) if -2 ** 31 <= x < 2 ** 31)
    return sorted(xs)


@pytest.mark.parametrize("fmt", [capi.FORMAT_CS32, capi.FORMAT_CS32BE, capi.FORMAT_CU32, capi.FORMAT_CU32BE])
@pytest.mark.parametrize("g", [2.0 ** -24, 3 * 2.0 ** -25, 0.3 * 2.0 ** -20, 1.0, 5 * 2.0 ** -30])
def test_32bit_extremes_and_half_steps(fmt, g):
    name, dtype, off, _ = SIGMF[fmt]
    xs = _half_steps(g)
    stored = np.array([x + off for x in xs], dtype=np.int64).astype(dtype)
    raw = stored.view(np.uint8)
    assert components(raw, fmt).tolist() == xs
    want = np.array([_exact(x, g, True) for x in xs], dtype=np.uint8)
    assert np.array_equal(convert(raw, fmt, g), want)
    if g == 2.0 ** -24:   # exact half steps at the default: to even
        half = [(2 * k + 1) * 2 ** 23 for k in (0, 1, 126, 127, -1, -2, -128)]
        got = convert(np.array([x + off for x in half], dtype=np.int64).astype(dtype).view(np.uint8), fmt)
        assert got.tolist() == [128, 130, 254, 255, 128, 126, 0]


@pytest.mark.parametrize("fmt", [capi.FORMAT_CF64, capi.FORMAT_CF64BE, capi.FORMAT_CF32BE])
def test_float_specials(fmt):
    f64 = fmt != capi.FORMAT_CF32BE
    tiny = [5e-324, -5e-324, 2.2250738585072014e-308 / 3, 1e-300] if f64 else [1e-45, -1e-45, 1.1754942e-38]
    cases = {0.0: 128, -0.0: 128, float("inf"): 255, float("-inf"): 0, float("nan"): 128, -float("nan"): 128,
             **{t: 128 for t in tiny}, 0.5: 128, -0.5: 128, 1.5: 130, -1.5: 126, 127.5: 255, -127.5: 0, 128.5: 255,
             -128.5: 0, 126.5: 254, -126.5: 2, 1e300 if f64 else 1e30: 255, -1e300 if f64 else -1e30: 0}
    if f64:   # the neighbours of the half steps, which float32 could not tell apart from them
        for h in (0.5, 126.5, -127.5):
            cases[float(np.nextafter(h, np.inf))] = round(h) + 129 if h > 0 else 1
            cases[float(np.nextafter(h, -np.inf))] = round(h) + 128 if h > 0 else 0
    dtype = SIGMF[fmt][1]
    xs = list(cases)
    raw = np.array(xs, dtype=np.float64).astype(dtype).view(np.uint8)
    got = convert(raw, fmt, 1.0)
    assert got.tolist() == list(cases.values())
    for x, u in cases.items():
        assert _exact(x, 1.0, f64) == u, x
    # at the default 2^7, the same values over 128 (exact) give the same bytes
    raw128 = (np.array(xs, dtype=np.float64) / 128).astype(dtype).view(np.uint8)
    norm = [i for i, x in enumerate(xs) if x == x and abs(x) > 1e-30]
    assert convert(raw128, fmt)[norm].tolist() == [list(cases.values())[i] for i in norm]


@pytest.mark.parametrize("fmt", NEW_FORMATS)
def test_identity_encodings_round_trip(fmt):
    u = np.repeat(np.arange(256, dtype=np.uint8), 2)
    raw = encode(u, fmt)
    assert raw.size == 256 * capi.FORMAT_BYTES[fmt]
    assert np.array_equal(convert(raw, fmt), u)
    name, dtype, off, g = SIGMF[fmt]
    x = components(raw, fmt)
    v = u.astype(np.int64) - 128
    if dtype[1] == "f":
        assert np.array_equal(x, v / 128)
    else:
        assert np.array_equal(x, v * 2 ** (np.dtype(dtype).itemsize * 8 - 8))


# ---- ertgpu_set_input_format ----

def test_set_input_format_takes_the_new_constants(built):
    h = capi.Handle()
    h.register(capi.stock_protocol("scm", 72))
    for fmt, (name, dtype, off, g) in SIGMF.items():
        h.set_input_format(fmt)
        assert h.input_format() == (fmt, g), name
        h.set_input_format(fmt, 0.125)
        assert h.input_format() == (fmt, 0.125), name
    for bad in (4, 15, 26, 100, -1):
        with pytest.raises(capi.ErtGpuError) as e:
            h.set_input_format(bad)
        assert e.value.code == capi.EINVAL
    h.set_input_format(capi.FORMAT_CF64)
    h.set_input_rate(2_400_000)
    with pytest.raises(capi.ErtGpuError) as e:   # a resampling cf64 handle takes whole 16-byte samples
        h.decode(np.zeros(4104, dtype=np.uint8))
    assert e.value.code == capi.ESIZE
    h.close()


# ---- the metadata reader ----

def _rec(tmp_path, datatype="ci16_le", rate=2_400_000, nbytes=4096, **kw):
    return write_recording(tmp_path / "r", bytes(nbytes), datatype, rate, **kw)


def _err(base) -> str:
    with pytest.raises(ValueError) as e:
        host.sigmf_probe(base)
    return str(e.value)


def test_every_datatype_and_the_file_names(built, tmp_path):
    for name, fmt in DATATYPES.items():
        base = _rec(tmp_path, name, 2.4e6, nbytes=16 * 64)
        for arg in (base, base + ".sigmf-meta", base + ".sigmf-data"):
            p = host.sigmf_probe(arg)
            assert p["format"] == fmt and p["rate"] == 2_400_000 and p["frequency"] is None, (name, arg)
            assert p["data_path"] == base + ".sigmf-data"
            assert p["samples"] == 16 * 64 // capi.FORMAT_BYTES[fmt]
            assert p["segments"] == [{"start": 0, "header_bytes": 0, "datetime_ns": None}]
    for name in ("rf32_le", "ri16_le", "ru8"):
        assert "real-valued" in _err(_rec(tmp_path, name)) and name in _err(_rec(tmp_path, name))
    for name in ("ci12_le", "CI16_LE", "ci16", "cs16", ""):
        msg = _err(_rec(tmp_path, name))
        assert "core:datatype" in msg and f'"{name}"' in msg


@pytest.mark.parametrize("glob,field", [
    ({"core:sample_rate": 2048000.5}, "core:sample_rate"), ({"core:sample_rate": 0}, "core:sample_rate"),
    ({"core:sample_rate": "2400000"}, "core:sample_rate"), ({"core:sample_rate": -1}, "core:sample_rate"),
    ({"core:num_channels": 2}, "core:num_channels"), ({"core:dataset": "x.bin"}, "core:dataset"),
    ({"core:metadata_only": True}, "core:metadata_only"), ({"core:datatype": 16}, "core:datatype")])
def test_global_field_errors(built, tmp_path, glob, field):
    base = _rec(tmp_path, glob_extra=glob)
    assert field in _err(base)


def test_global_fields_accepted(built, tmp_path):
    base = _rec(tmp_path, rate=2.4e6, glob_extra={"core:num_channels": 1, "core:sha512": "ab", "ext:thing": {"a": [1, {}]},
                                                  "core:extensions": [{"name": "x", "version": "1", "optional": True}]})
    assert host.sigmf_probe(base)["rate"] == 2_400_000
    base = write_recording(tmp_path / "m", bytes(64), "cf32_le", 1e7,
                           meta_text='{"global":{"core:datatype":"ci16_le","core:sample_rate":10e6}}')
    p = host.sigmf_probe(base)   # no captures: one segment at sample 0
    assert p["rate"] == 10_000_000 and p["segments"] == [{"start": 0, "header_bytes": 0, "datetime_ns": None}]
    with open(base + ".sigmf-meta", "w") as f:   # missing fields
        f.write('{"global":{"core:sample_rate":1}}')
    assert "core:datatype" in _err(base)
    with open(base + ".sigmf-meta", "w") as f:
        f.write('{"global":{"core:datatype":"cu8"}}')
    assert "core:sample_rate" in _err(base)
    os.remove(base + ".sigmf-data")
    with open(base + ".sigmf-meta", "w") as f:
        f.write('{"global":{"core:datatype":"cu8","core:sample_rate":1}}')
    assert ".sigmf-data" in _err(base)
    assert ".sigmf-meta" in _err(tmp_path / "nothing")


def test_captures_and_header_bytes(built, tmp_path):
    caps = [{"core:sample_start": 0, "core:header_bytes": 12, "core:frequency": 915e6},
            {"core:sample_start": 100, "core:header_bytes": 3},
            {"core:sample_start": 250, "core:frequency": 915000000, "core:global_index": 7}]
    base = _rec(tmp_path, "ci16_be", nbytes=12 + 3 + 4 * 400, captures=caps)
    p = host.sigmf_probe(base)
    assert p["format"] == capi.FORMAT_CS16BE and p["frequency"] == 915_000_000 and p["samples"] == 400
    assert [(s["start"], s["header_bytes"]) for s in p["segments"]] == [(0, 12), (100, 3), (250, 0)]
    # header bytes that leave a partial sample, a last segment past the data
    assert "core:header_bytes" in _err(_rec(tmp_path, "ci16_be", nbytes=12 + 4 * 400, captures=caps))
    assert "core:header_bytes" in _err(_rec(tmp_path, "cf64_le", nbytes=1000))
    assert "core:sample_start" in _err(_rec(tmp_path, nbytes=4 * 10, captures=[{"core:sample_start": 0},
                                                                                {"core:sample_start": 11}]))
    for bad, field in [
            ([{"core:sample_start": 5}, {"core:sample_start": 5}], "core:sample_start"),
            ([{"core:sample_start": 5}, {"core:sample_start": 2}], "core:sample_start"),
            ([{"core:sample_start": 0}, {}], "core:sample_start"),
            ([{"core:sample_start": -1}], "core:sample_start"),
            ([{"core:sample_start": 0, "core:header_bytes": 1.5}], "core:header_bytes"),
            ([{"core:sample_start": 0, "core:frequency": 9e8}, {"core:sample_start": 1, "core:frequency": 9.1e8}], "retunes"),
            ([{"core:sample_start": 0, "core:frequency": 915000000.5}], "core:frequency"),
            ([{"core:sample_start": 0, "core:datetime": 5}], "core:datetime"),
            ([7], "captures[0]")]:
        assert field in _err(_rec(tmp_path, captures=bad)), bad
    with open(tmp_path / "r.sigmf-meta", "w") as f:
        f.write('{"global":{"core:datatype":"cu8","core:sample_rate":1},"captures":{}}')
    assert "captures" in _err(tmp_path / "r")


def test_json_escapes_surrogates_and_errors(built, tmp_path):
    text = ('{"global":{"core:datatype":"\\u0063i16\\u005f\\u0062e","core:sample_rate":2.4E+6,'
            '"core:description":"tab\\t nl\\n q\\" bs\\\\ sl\\/ \\b\\f\\r \\u00e9 \\u20ac \\ud83d\\ude00 \\uD834\\uDD1E",'
            '"core:author":"é€\U0001F600", "x":[true,false,null,-0,0.5e-3,1E2,[[[]]],{}]},'
            ' "captures" : [ ] , "annotations":[{"core:sample_start":0,"core:comment":"\\ud83d\\ude00"}] }\r\n\t ')
    base = write_recording(tmp_path / "j", bytes(64), "", 0, meta_text=text)
    p = host.sigmf_probe(base)
    assert p["format"] == capi.FORMAT_CS16BE and p["rate"] == 2_400_000
    good = '{"global":{"core:datatype":"cu8","core:sample_rate":1}}'
    cases = [good[:-1], good + "x", good.replace(":1", ":01"), good.replace(":1", ":1."), good.replace(":1", ":-"),
             good.replace(":1", ":.5"), good.replace(":1", ":1e"), good.replace(":1", ":+1"), good.replace('"cu8"', '"cu8'),
             good.replace('"cu8"', '"c\\x"'), good.replace('"cu8"', '"\\ud83d"'), good.replace('"cu8"', '"\\ude00"'),
             good.replace('"cu8"', '"\\ud83d\\u0041"'), good.replace('"cu8"', '"\\u12G4"'), good.replace('"cu8"', '"c\tu8"'),
             good.replace('"cu8"', "'cu8'"), good.replace(",", ",,"), good.replace("}}", ",}}"), good.replace("1", "tru"),
             good.replace("1", "nul"), "[" * 100 + "]" * 100, "", "  ", good.replace(":1", ":1}")]
    for t in cases:
        with open(base + ".sigmf-meta", "w") as f:
            f.write(t)
        msg = _err(base)
        assert "malformed metadata at byte " in msg or "not a JSON object" in msg, t
    # the byte offset is where the parser stopped
    text = '{"global": {"core:datatype": "cu8", "core:sample_rate": 1,, }}'
    with open(base + ".sigmf-meta", "w") as f:
        f.write(text)
    assert f"at byte {text.index(',,') + 1}:" in _err(base)   # the second comma
    for depth, ok in [(60, True), (70, False)]:   # bounded nesting
        with open(base + ".sigmf-meta", "w") as f:
            f.write('{"global":{"core:datatype":"cu8","core:sample_rate":1,"x":' + "[" * depth + "]" * depth + "}}")
        if ok:
            host.sigmf_probe(base)
        else:
            assert "nesting" in _err(base)


def _ns_ref(text: str) -> int:
    """A SigMF datetime through Python's datetime: whole seconds from datetime, the fraction truncated to ns."""
    head, zone = (text[:-1], "+00:00") if text.endswith("Z") else (text[:-6], text[-6:])
    frac = ""
    if "." in head:
        head, frac = head.split(".")
    d = dt.datetime.fromisoformat(head + zone)
    return int(d.timestamp()) * 10 ** 9 + int((frac + "000000000")[:9])


def test_datetime_parsing(built, tmp_path):
    texts = ["2024-02-29T23:59:59.123456789123Z", "1970-01-01T00:00:00Z", "1969-12-31T23:59:59.5Z",
             "2026-10-16T05:14:25+05:30", "2026-10-16T05:14:25.000001-08:00", "2000-03-01T00:00:00.9999999999Z",
             "1678-01-01T00:00:00Z", "2262-04-11T23:47:16.854775807Z", "2100-02-28T12:00:00.1+00:00"]
    for t in texts:
        base = _rec(tmp_path, captures=[{"core:sample_start": 0, "core:datetime": t}])
        assert host.sigmf_probe(base)["segments"][0]["datetime_ns"] == _ns_ref(t), t
    for t in ["2024-02-30T00:00:00Z", "2023-02-29T00:00:00Z", "2024-13-01T00:00:00Z", "2024-01-01T24:00:00Z",
              "2024-01-01T00:60:00Z", "2024-01-01T00:00:60Z", "2024-01-01T00:00:00", "2024-01-01 00:00:00Z",
              "2024-01-01T00:00:00.Z", "2024-1-01T00:00:00Z", "2024-01-01T00:00:00+0530", "2024-01-01T00:00:00z",
              "2024-01-01T00:00:00Zx", "2024-01-01", "2262-04-11T23:47:16.854775808Z", "1677-09-21T00:00:00Z"]:
        base = _rec(tmp_path, captures=[{"core:sample_start": 0, "core:datetime": t}])
        assert "core:datetime" in _err(base), t


@pytest.mark.parametrize("rate_in", [32768 * 72, 2_400_000, 10_000_000])
def test_block_time_against_fraction(built, tmp_path, rate_in):
    rate_out, bs = 32768 * 72, 2 ** 14
    t0 = _ns_ref("2025-06-01T12:00:00.123456789Z")
    segs = [{"start": 0, "header_bytes": 0, "datetime_ns": None},
            {"start": 1000, "header_bytes": 0, "datetime_ns": t0},
            {"start": 700_001, "header_bytes": 0, "datetime_ns": None},
            {"start": 1_500_000, "header_bytes": 0, "datetime_ns": t0 + 10 ** 12 + 7},
            {"start": 4_000_003, "header_bytes": 0, "datetime_ns": t0 - 5 * 10 ** 9}]
    iso = lambda ns: dt.datetime.fromtimestamp(ns // 10 ** 9, dt.timezone.utc).strftime("%Y-%m-%dT%H:%M:%S.") + \
        f"{ns % 10 ** 9:09d}Z"
    caps = [{"core:sample_start": s["start"], **({"core:datetime": iso(s["datetime_ns"])} if s["datetime_ns"] else {})}
            for s in segs]
    base = _rec(tmp_path, "cu8", rate_in, nbytes=2 * 5_000_000, captures=caps)
    assert host.sigmf_probe(base)["segments"] == segs
    last = 5_000_000 * rate_out // rate_in // bs
    blocks = sorted({0, 1, 2, last - 1, last} | set(range(0, last, 7)))
    for b in blocks:
        assert host.sigmf_block_time(base, b, bs, rate_out) == block_time_ref(segs, rate_in, b, bs, rate_out), b
    # the first block ends before the first dated segment: that segment's time, counted backwards
    assert block_time_ref(segs, rate_in, 0, 16, rate_out) < t0
    assert host.sigmf_block_time(base, 0, 16, rate_out) == block_time_ref(segs, rate_in, 0, 16, rate_out)
    undated = _rec(tmp_path, "cu8", rate_in, nbytes=64)
    with pytest.raises(ValueError, match="core:datetime"):
        host.sigmf_block_time(undated, 0, bs, rate_out)


# ---- the file receiver ----

def _cli(*args):
    r = subprocess.run([CLI, *args], capture_output=True, timeout=60)
    r.stderr = r.stderr.decode(errors="replace")
    return r


def test_cli_usage_errors(built, tmp_path):
    a = write_recording(tmp_path / "a", bytes(4 << 12), "ci16_le", 2_400_000, captures=[{"core:sample_start": 0,
                                                                                         "core:frequency": 915e6}])
    b = write_recording(tmp_path / "b", bytes(4 << 12), "ci16_le", 2_400_000, captures=[{"core:sample_start": 0,
                                                                                         "core:frequency": 914e6}])
    c = write_recording(tmp_path / "c", bytes(8 << 12), "ci32_le", 2_400_000)
    d = write_recording(tmp_path / "d", bytes(4 << 12), "ci16_le", 2_000_000)
    u = write_recording(tmp_path / "u", bytes(2 << 12), "cu8", 32768 * 72)
    ut = write_recording(tmp_path / "ut", bytes(2 << 12), "cu8", 32768 * 72,
                         captures=[{"core:sample_start": 0, "core:frequency": 912600000}])
    sf = f"-samplefile={tmp_path / 's.bin'}"
    cases = [
        (["-sampleformat=sigmf", "-"], "stdin"),
        (["-sampleformat=sigmf", "-samplerate=2048000", a], "-samplerate"),
        (["-sampleformat=sigmf", "-capturefreq=912600000", a], "-capturefreq"),
        (["-sampleformat=sigmf", a, b], "batch"),
        (["-sampleformat=sigmf", a, c], "batch"),
        (["-sampleformat=sigmf", a + ".sigmf-meta", d], "batch"),
        (["-sampleformat=sigmf", sf, a], "-samplefile"),
        (["-sampleformat=sigmf", sf, c], "-samplefile"),
        (["-sampleformat=sigmf", sf, ut], "-samplefile"),
        (["-sampleformat=sigmf", "-samplescale=2", u], "-samplescale"),
        (["-sampleformat=sigmf", "-centerfreq=912600000", u], "-centerfreq"),
        (["-sampleformat=ci12_be", a], "-sampleformat"),
        (["-sampleformat=SIGMF", a], "-sampleformat"),
        (["-sampleformat=rf32_le", a], "-sampleformat"),
        (["-sampleformat=cf64", a], "-sampleformat"),
        (["-sampleformat=cu16_le", "-samplescale=-1", a], "-samplescale"),
        (["-sampleformat=cf64_be", sf, a], "-samplefile"),
    ]
    for args, word in cases:
        r = _cli(*args)
        assert r.returncode == 2 and word in r.stderr, (args, r.returncode, r.stderr)
        assert "CenterFreq" not in r.stderr, args   # no decoder was set up
    assert not (tmp_path / "s.bin").exists()
    # metadata that cannot be read is an error naming the field, also before any device
    bad = write_recording(tmp_path / "bad", bytes(64), "rf32_le", 2_400_000)
    r = _cli("-sampleformat=sigmf", bad)
    assert r.returncode == 1 and "core:datatype" in r.stderr and "CenterFreq" not in r.stderr
    r = _cli("-sampleformat=sigmf", str(tmp_path / "missing"))
    assert r.returncode == 1 and "missing.sigmf-meta" in r.stderr
