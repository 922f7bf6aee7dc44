"""GPU tests (-m gpu) of the automatic gain: level_kernel's histogram against NumPy for every converted format, the
stream state around ertgpu_measure_input and ertgpu_set_input_scale, -samplescale=auto against the gain it prints, weak
packets that only auto decodes, a loud packet that clips, and a batch of streams at different levels."""
import json
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from rtlamr_b200 import capi, host, synth

from format_ref import wav_bytes
from test_gpu_input_format import DATA_RATE, _scm_fields, add_packets, keys, u8_stream
from test_input_level import rule_ref
from test_sigmf import SIGMF, write_recording

pytestmark = pytest.mark.gpu

CLI = os.path.join(ROOT, "rtlamr_b200", "ertgpu_decode_file")
WINDOW = 1 << 22
# every converted format: (numpy dtype of a stored component, offset: x = stored - offset)
LAYOUT = {capi.FORMAT_CS8: ("i1", 0), capi.FORMAT_CS16: ("<i2", 0), capi.FORMAT_CF32: ("<f4", 0),
          **{f: (v[1], v[2]) for f, v in SIGMF.items()}}
DEFAULT_K = {capi.FORMAT_CS8: 0, capi.FORMAT_CS16: -8, capi.FORMAT_CF32: 7, **{f: int(np.log2(v[3])) for f, v in SIGMF.items()}}


def raw_with_specials(fmt, nsamples, seed):
    """Random stored components of fmt (every bit pattern for the floats, so every exponent, subnormals, infinities and
    NaNs of both signs) with 0, -0, the extremes, -2^15 / -2^31 of the unsigned formats, subnormals, +-inf and NaN
    written over a few of them.  Returns the raw bytes and x of every component (float64, NaN as NaN)."""
    dtype, off = LAYOUT[fmt]
    dt = np.dtype(dtype)
    rng = np.random.default_rng(seed)
    raw = rng.integers(0, 256, 2 * nsamples * dt.itemsize, dtype=np.uint8)
    v = raw.view(dt)
    if dt.kind == "f":
        fi = np.finfo(dt)
        sp = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, fi.max, -fi.max, fi.tiny, -fi.tiny,
                       fi.smallest_subnormal, -fi.smallest_subnormal, fi.tiny / 3, 1.0, -1.0, 127.5 / 128], dtype=dt)
        if fmt == capi.FORMAT_CF32:   # mostly ordinary levels as well
            v[: v.size // 2] = (rng.standard_normal(v.size // 2) * 0.01).astype(dt)
    else:
        lo, hi = -(1 << (8 * dt.itemsize - 1)), (1 << (8 * dt.itemsize - 1)) - 1   # x range
        sp = np.array([x + off for x in (0, 1, -1, lo, hi, lo + 1, 2, -2)]).astype(dt)
    at = rng.choice(v.size, min(v.size, 64 * sp.size), replace=False)
    v[at] = sp[np.arange(at.size) % sp.size]
    with np.errstate(invalid="ignore"):
        x = v.astype(np.float64) if dt.kind == "f" else v.astype(np.int64).astype(np.float64) - off   # exact: |x| <= 2^31
    return raw, x


def hist_ref(x):
    """zeros, NaNs and bins[e + 128] of e = floor(log2 |x|) clamped to [-128, 127], +-inf in the top bin."""
    nan = np.isnan(x)
    zero = x == 0
    inf = np.isinf(x)
    rest = x[~nan & ~zero & ~inf]
    _, ex = np.frexp(np.abs(rest))           # |x| = m * 2^ex, m in [0.5, 1): floor(log2 |x|) = ex - 1
    e = np.clip(ex.astype(np.int64) - 1, -128, 127)
    bins = np.bincount(e + 128, minlength=256).astype(np.int64)
    bins[255] += int(inf.sum())
    return int(zero.sum()), int(nan.sum()), bins


@pytest.mark.parametrize("fmt", list(LAYOUT), ids=lambda f: str(f))
def test_histogram_equals_numpy(built, fmt):
    """measure_input bin for bin against NumPy: an odd size that is no multiple of a CTA's work, one sample, none, and
    a size over three staging chunks of a handle with 64-block calls (pageable and pinned input)."""
    h = capi.new_decoder("scm", 72, input_format=fmt, max_blocks_per_call=64)
    chunk = 64 * h.cfg.block_size   # samples per staging chunk at the decoder's rate
    for n, seed in ((1_000_003, 1), (1, 2), (0, 3), (3 * chunk + 12_345, 4)):
        raw, x = raw_with_specials(fmt, n, seed + 100 * fmt)
        got = h.measure_input(raw)
        zeros, nans, bins = hist_ref(x)
        assert got["components"] == 2 * n
        assert (got["zeros"], got["nans"]) == (zeros, nans), n
        assert np.array_equal(got["bins"], bins), (n, np.nonzero(got["bins"] != bins))
        k = rule_ref(bins, 2 * n, zeros, nans, DEFAULT_K[fmt])
        assert got["exponent"] == k and got["scale"] == np.float32(2.0 ** k), n
    # pinned input gives the same counts
    raw, x = raw_with_specials(fmt, 2 * chunk + 3, 7)
    p = C_pinned(raw)
    assert np.array_equal(h.measure_input((p.addr, raw.size))["bins"], hist_ref(x)[2])
    p.free()
    h.close()


class C_pinned:
    def __init__(self, data):
        import ctypes as C
        ptr = C.c_void_p()
        assert capi.lib().ertgpu_host_alloc(C.byref(ptr), data.size) == capi.OK
        self.addr = ptr.value
        C.memmove(self.addr, data.ctypes.data, data.size)

    def free(self):
        capi.lib().ertgpu_host_free(self.addr)


def test_measure_leaves_the_stream_alone(built):
    """A measure between two decode calls changes nothing (resampling cs16 handle); set_input_scale is refused after
    a decode call and for cu8, accepted after reset, and the new gain survives the next reset."""
    rate = 2_400_000
    u8, truth = u8_stream("scm", rate, 1_500_000, seed=21)
    raw = (u8.astype(np.int16) - 128).astype("<i2") * 256
    raw = raw.view(np.uint8)
    cut = 4 * 700_001
    ref = capi.new_decoder("scm", 72, input_rate=rate, input_format=capi.FORMAT_CS16)
    want = keys(ref.decode(raw[:cut])) + keys(ref.decode(raw[cut:]))
    h = capi.new_decoder("scm", 72, input_rate=rate, input_format=capi.FORMAT_CS16)
    h.measure_input(raw[: 4 * 100_000])
    a = h.decode(raw[:cut])
    kern = h.last_kernels()
    h.measure_input(raw[4 * 300_000:])
    assert h.last_kernels() == kern
    b = h.decode(raw[cut:])
    assert keys(a) + keys(b) == want and want
    with pytest.raises(capi.ErtGpuError) as e:
        h.set_input_scale(0.5)
    assert e.value.code == capi.EINVAL
    with pytest.raises(capi.ErtGpuError) as e:
        h.measure_input(raw[:3])   # not a whole sample
    assert e.value.code == capi.ESIZE
    h.reset()
    h.set_input_scale(1.0)
    h.reset()
    assert h.input_format() == (capi.FORMAT_CS16, 1.0)
    with pytest.raises(capi.ErtGpuError):
        h.set_input_scale(float("nan"))
    h.set_input_scale(0.0)   # the default again
    assert h.input_format() == (capi.FORMAT_CS16, 2.0 ** -8)
    u = capi.new_decoder("scm", 72)
    for call in (lambda: u.set_input_scale(1.0), lambda: u.measure_input(u8[:1024])):
        with pytest.raises(capi.ErtGpuError) as e:
            call()
        assert e.value.code == capi.EINVAL
    for x in (h, ref, u):
        x.close()


def _cli(*args, stdin=None):
    r = subprocess.run([CLI, *args], capture_output=True, timeout=600, stdin=stdin)
    assert r.returncode == 0, r.stderr.decode(errors="replace")
    return r.stdout.decode(), r.stderr.decode()


def _gains(err):
    return [(int(k), float(g), int(n)) for k, g, n in re.findall(r"-samplescale=auto: 2\^(-?\d+) = (\S+) from (\d+) samples", err)]


def _no_time(out):
    rows = [json.loads(l) for l in out.splitlines()]
    for r in rows:
        r.pop("Time", None)
    return rows


def _stream(rate, n, seed, msgtypes="scm,idm"):
    """Complex baseband (float64 I and Q, zero mean) with packets: the synthetic uint8 stream less 127.5."""
    u8, truth = u8_stream(msgtypes, rate, n, seed=seed)
    return u8.astype(np.float64) - 127.5, truth


def _captures(tmp_path):
    out = []
    # cs16 at 2.4 MS/s as a 12-bit radio writes it, longer than the window
    x, _ = _stream(2_400_000, 5_000_000, 31)
    p = tmp_path / "a.cs16"
    np.rint(x * 12).astype("<i2").tofile(p)
    out.append(([f"-samplerate=2400000", "-sampleformat=cs16", str(p)], 5_000_000))
    # cf32 at the decoder's rate, normalised as gqrx writes it
    x, _ = _stream(32768 * 72, 2_000_000, 32)
    p = tmp_path / "b.cf32"
    (x / 2000).astype("<f4").tofile(p)
    out.append((["-sampleformat=cf32", str(p)], 2_000_000))
    # cs8 at 8 MS/s, the channel 1 MHz above the capture's centre
    x, _ = _stream(8_000_000, 3_000_000, 33)
    z = (x[0::2] + 1j * x[1::2]) * np.exp(2j * np.pi * 1e6 / 8e6 * np.arange(x.size // 2))
    p = tmp_path / "c.cs8"
    np.rint(np.stack([z.real, z.imag], 1).ravel() * 0.7).astype(np.int8).tofile(p)
    out.append((["-samplerate=8000000", "-sampleformat=cs8", "-capturefreq=911600155", str(p)], 3_000_000))
    # a float WAV
    x, _ = _stream(2_400_000, 2_000_000, 34)
    p = tmp_path / "d.wav"
    p.write_bytes(wav_bytes((x / 700).astype("<f4").tobytes(), bits=32, tag=3, rate=2_400_000))
    out.append((["-sampleformat=wav", str(p)], 2_000_000))
    # a SigMF cf32 recording with header bytes in front of the samples
    x, _ = _stream(2_400_000, 2_000_000, 35)
    data = b"\xa5" * 24 + (x / 90).astype("<f4").tobytes()
    base = write_recording(tmp_path / "e", data, "cf32_le", 2_400_000, captures=[{"core:sample_start": 0, "core:header_bytes": 24}])
    out.append((["-sampleformat=sigmf", base], 2_000_000))
    return out


def test_auto_equals_the_printed_gain(built, tmp_path):
    """-samplescale=auto prints 2^k = G and the samples measured, and its stdout is that of -samplescale=G, also with
    -blocks=1 and (raw input) from stdin."""
    common = ["-msgtype=scm,idm", "-symbollength=72", "-format=json"]
    for args, n in _captures(tmp_path):
        out, err = _cli(*common, "-samplescale=auto", *args)
        (k, g, m), = _gains(err)
        assert g == 2.0 ** k and m == min(n, WINDOW), (args, err)
        want, _ = _cli(*common, f"-samplescale={g!r}", *args)
        assert _no_time(out) == _no_time(want) and want, args
        out1, err1 = _cli(*common, "-samplescale=auto", "-blocks=1", *args)
        assert _gains(err1) == [(k, g, m)] and _no_time(out1) == _no_time(want), args
        if "-sampleformat=sigmf" not in args:
            with open(args[-1], "rb") as f:
                out2, err2 = _cli(*common, "-samplescale=auto", *args[:-1], "-", stdin=f)
            assert _gains(err2) == [(k, g, m)] and _no_time(out2) == _no_time(want), args


def _weak_cs16(tmp_path, loud=False):
    rate_in, n = 2_400_000, 6_000_000
    rng = np.random.default_rng(41)
    iq = np.rint(rng.standard_normal(2 * n) * 20).astype(np.int32)
    pk, truth = synth.make_packets("scm,idm", -(-rate_in // DATA_RATE), n - (1 << 18), seed=42, spacing=1 << 17,
                                   amplitude=(90, 90))
    if loud:   # one packet after the measured window, 30 dB above the others
        j = int(np.nonzero(pk["start_sample"] > WINDOW + 100_000)[0][0])
        pk["amp_i"][j] = np.int16(np.rint(pk["amp_i"][j] * 31.6))
        pk["amp_q"][j] = np.int16(np.rint(pk["amp_q"][j] * 31.6))
    add_packets(iq, pk, rate_in)
    p = tmp_path / ("loud.cs16" if loud else "weak.cs16")
    np.clip(iq, -32768, 32767).astype("<i2").tofile(p)
    return p, truth


def _found(out, truth):
    msgs = [json.loads(l)["Message"] for l in out.splitlines()]
    hit = 0
    for t in truth:
        if t.msgtype == "scm":
            mid, cons = _scm_fields(t.data)
            hit += any(m.get("ID") == mid and m.get("Consumption") == cons for m in msgs)
        else:
            hit += any(m.get("ERTSerialNumber") == t.meter_id for m in msgs)
    return hit


def test_weak_packets_need_auto(built, tmp_path):
    """A carrier of 90 over noise of sigma 20 as cs16: under half an LSB at the default 2^-8, so few packets (if any)
    are reported without a gain, and every one with -samplescale=auto.  host.Receiver(input_scale="auto") picks the
    same gain from the same window."""
    p, truth = _weak_cs16(tmp_path)
    common = ["-msgtype=scm,idm", "-symbollength=72", "-samplerate=2400000", "-sampleformat=cs16", "-format=json", str(p)]
    assert len(truth) >= 30
    out, _ = _cli(*common)
    assert _found(out, truth) < len(truth) / 2
    out, err = _cli("-samplescale=auto", *common)
    assert _found(out, truth) == len(truth)
    (k, g, m), = _gains(err)
    r = host.Receiver("scm,idm", 72, input_rate=2_400_000, input_format=capi.FORMAT_CS16, input_scale="auto")
    raw = np.fromfile(p, dtype=np.uint8)
    assert r.input_level() is None
    msgs = r.decode(raw[: 4 * WINDOW]) + r.decode(raw[4 * WINDOW:])
    lv = r.input_level()
    assert (lv["exponent"], lv["scale"], lv["components"]) == (k, g, 2 * WINDOW)
    assert {t.meter_id for t in truth if t.msgtype == "idm"} <= {m.meter_id for m in msgs}
    r.reset()
    assert r.input_level() is None
    r.close()


def test_a_loud_packet_clips_and_is_still_reported(built, tmp_path):
    """One packet 30 dB above everything in the measured window: the gain comes from the window, that packet clips at
    the byte's full scale, and the magnitude decoder still reports it and every other packet."""
    p, truth = _weak_cs16(tmp_path, loud=True)
    out, err = _cli("-samplescale=auto", "-msgtype=scm,idm", "-symbollength=72", "-samplerate=2400000",
                    "-sampleformat=cs16", "-format=json", str(p))
    (k, g, m), = _gains(err)
    assert 2800 * g > 4 * 128   # the loud packet's carrier is four times the byte's full scale
    assert _found(out, truth) == len(truth)


def test_batch_streams_get_their_own_gains(built, tmp_path):
    """Two files 24 dB apart: two different gains, and each file's lines equal its run alone."""
    x, _ = _stream(2_400_000, 2_500_000, 51)
    a, b = tmp_path / "a.cs16", tmp_path / "b.cs16"
    np.rint(x * 4).astype("<i2").tofile(a)
    np.rint(x * 64).astype("<i2").tofile(b)
    common = ["-msgtype=scm,idm", "-symbollength=72", "-samplerate=2400000", "-sampleformat=cs16", "-samplescale=auto"]
    out, err = _cli(*common, str(a), str(b))
    ga, gb = _gains(err)
    assert gb[0] == ga[0] - 4
    sa, ea = _cli(*common, str(a))
    sb, eb = _cli(*common, str(b))
    assert _gains(ea) == [ga] and _gains(eb) == [gb]
    assert out == sa + sb and sa
