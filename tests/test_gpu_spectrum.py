"""GPU tests (-m gpu) of the input spectrum (ertgpu_enable_spectrum, ertgpu_fetch_spectrum, spectrum_kernel<F>): rows
against the NumPy restatement (tests/spectrum_ref.py) over every input format and frame length; rows that do not depend
on the handle's path, the call split, the device path, reset, channel groups or signal reports; candidates and kernel
lists of a handle with a spectrum; where packets and carriers land; and the rules of the calls."""
import ctypes as C

import numpy as np
import pytest

import nearfar_ref
import signal_ref
import spectrum_ref
import tune_ref
from helpers import synth_stream
from rtlamr_b200 import capi

pytestmark = pytest.mark.gpu

DATA_RATE = 32768
CAPTURE = 915_000_000
FORMATS = [capi.FORMAT_CU8, capi.FORMAT_CS8, capi.FORMAT_CS16, capi.FORMAT_CF32, capi.FORMAT_CS16BE, capi.FORMAT_CF32BE,
           capi.FORMAT_CU16, capi.FORMAT_CU16BE, capi.FORMAT_CS32, capi.FORMAT_CS32BE, capi.FORMAT_CU32, capi.FORMAT_CU32BE,
           capi.FORMAT_CF64, capi.FORMAT_CF64BE]


def encode(z, fmt: int) -> np.ndarray:
    """Raw bytes of the complex signal z (8-bit units) in format fmt, full scale to full scale at the default gain."""
    v = np.empty(2 * z.size, dtype=np.float64)
    v[0::2], v[1::2] = z.real, z.imag
    if fmt == capi.FORMAT_CU8:
        return np.clip(np.round(v + 127.5), 0, 255).astype(np.uint8)
    if fmt == capi.FORMAT_CS8:
        return np.clip(np.round(v), -128, 127).astype(np.int8).view(np.uint8)
    ints = {capi.FORMAT_CS16: ("<i2", 8, 0), capi.FORMAT_CS16BE: (">i2", 8, 0), capi.FORMAT_CU16: ("<u2", 8, 1 << 15),
            capi.FORMAT_CU16BE: (">u2", 8, 1 << 15), capi.FORMAT_CS32: ("<i4", 24, 0), capi.FORMAT_CS32BE: (">i4", 24, 0),
            capi.FORMAT_CU32: ("<u4", 24, 1 << 31), capi.FORMAT_CU32BE: (">u4", 24, 1 << 31)}
    if fmt in ints:
        dt, sh, bias = ints[fmt]
        lim = (1 << (np.dtype(dt).itemsize * 8 - 1)) - 1
        x = np.clip(np.round(v * (1 << sh)), -lim - 1, lim) + bias
        return x.astype(dt).view(np.uint8)
    dt = {capi.FORMAT_CF32: "<f4", capi.FORMAT_CF32BE: ">f4", capi.FORMAT_CF64: "<f8", capi.FORMAT_CF64BE: ">f8"}[fmt]
    return (v / 128.0).astype(dt).view(np.uint8)


def tone_noise(n, seed, rel_freq=0.123, amp=90.0, noise=3.0):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    return amp * np.exp(2j * np.pi * rel_freq * t) + noise * (rng.standard_normal(n) + 1j * rng.standard_normal(n))


def least_f(log2n):
    return -(-(1 << 18) >> log2n)


def _check(h, raw, fmt, log2n, F, partial=True):
    rows, mean, peak = h.fetch_spectrum(partial=partial)
    want_rows, want_mean, want_peak = spectrum_ref.rows(raw, fmt, log2n, F, partial=partial)
    assert [tuple(int(x) for x in r) for r in rows] == want_rows
    spectrum_ref.assert_close(mean, want_mean, "mean")
    spectrum_ref.assert_close(peak, want_peak, "peak")
    return rows, mean, peak


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("log2n", [6, 10, 11, 12, 13, 14])
def test_rows_against_the_restatement(built, fmt, log2n):
    F = least_f(log2n) * (3 if log2n == 10 else 1)
    h = capi.new_decoder("scm", 72, input_format=fmt, spectrum=(log2n, F))
    bs = h.cfg.block_size
    n = (5 * (F << log2n) // 2) // bs * bs
    raw = encode(tone_noise(n, 7 + fmt), fmt)
    h.decode(raw, cap=1 << 16)
    rows, _, _ = _check(h, raw, fmt, log2n, F)
    assert len(rows) == 3 and rows[-1]["frames"] < F
    h.close()


@pytest.mark.parametrize("log2n", [10, 12])
def test_wideband_capture_against_the_restatement(built, log2n):
    rate_in, fmt = 10_000_000, capi.FORMAT_CS16
    z, _ = tune_ref.wideband([("scm", -2_000_000 + 90_000, 11, 0), ("scm", 3_000_000, 12, 0)], rate_in, 3_000_000, 11)
    raw = tune_ref.quantize(z, fmt)
    F = 2 * least_f(log2n)
    h = capi.new_decoder("scm", 72, input_rate=rate_in, input_format=fmt, capture_freq=CAPTURE,
                         center_freq=CAPTURE - 2_000_000, spectrum=(log2n, F))
    h.decode(raw, cap=1 << 16)
    _check(h, raw, fmt, log2n, F)
    h.close()


def _rows_of(h, parts, device=False):
    import torch
    out = []
    for p in parts:
        if device:
            d = torch.from_numpy(np.ascontiguousarray(p)).cuda()
            torch.cuda.synchronize()
            h.decode_device_async(d.data_ptr(), p.size)
            h.fetch(cap=1 << 16)
        else:
            h.decode(p, cap=1 << 16)
        out.append(h.fetch_spectrum())
    rows = np.concatenate([o[0] for o in out])
    return rows, np.concatenate([o[1] for o in out]), np.concatenate([o[2] for o in out])


def _same(a, b):
    assert a[0].tobytes() == b[0].tobytes()
    assert a[1].tobytes() == b[1].tobytes()
    assert a[2].tobytes() == b[2].tobytes()


def test_rows_do_not_depend_on_the_path(built):
    """The same cs16 bytes through an untuned, a resampled, a tuned, a decimated and a wide handle."""
    fmt, log2n, F = capi.FORMAT_CS16, 10, 300
    z, _ = tune_ref.wideband([("scm", 500_000, 11, 0)], 10_000_000, 2_000_000, 11)
    raw = tune_ref.quantize(z, fmt)
    kinds = [{}, {"input_rate": 5_000_000}, {"input_rate": 10_000_000, "capture_freq": CAPTURE, "center_freq": CAPTURE + 500_000},
             {"input_rate": 30_720_000, "capture_freq": CAPTURE, "center_freq": CAPTURE + 500_000},
             {"input_rate": 10_000_000, "capture_freq": CAPTURE, "center_freq": CAPTURE + 500_000, "channel_gain": 4}]
    got = []
    for kw in kinds:
        h = capi.new_decoder("scm", 72, input_format=fmt, spectrum=(log2n, F), **kw)
        bs4 = h.cfg.block_size * 4
        got.append(_rows_of(h, [raw[:raw.size // bs4 * bs4]]))
        h.close()
    assert len(got[0][0]) >= 5
    for g in got[1:]:
        _same(g, got[0])


def test_call_splits_device_path_reset_and_signal(built):
    fmt, log2n, F = capi.FORMAT_CS16, 12, 70
    rate_in = 10_000_000
    z, _ = tune_ref.wideband([("scm", 300_000, 11, 0)], rate_in, 3_000_000, 5)
    raw = tune_ref.quantize(z, fmt)

    def mk(**kw):
        return capi.new_decoder("scm", 72, input_rate=rate_in, input_format=fmt, capture_freq=CAPTURE,
                                center_freq=CAPTURE + 300_000, spectrum=(log2n, F), **kw)
    h = mk()
    one = _rows_of(h, [raw])
    assert len(one[0]) >= 8
    rng = np.random.default_rng(3)
    for _ in range(3):   # cuts anywhere: inside frames, groups and rows
        h.reset()
        cuts = sorted(set(int(x) * 4 for x in rng.integers(1, raw.size // 4, 7)))
        _same(_rows_of(h, [raw[a:b] for a, b in zip([0] + cuts, cuts + [raw.size])]), one)
    h.reset()
    step = 4 * 200_000 + 4 * 37
    _same(_rows_of(h, [raw[a:a + step] for a in range(0, raw.size, step)], device=True), one)
    h.close()
    s = mk(signal=True)
    _same(_rows_of(s, [raw]), one)
    s.close()


def test_native_cu8_splits(built):
    log2n, F = 14, 16
    h = capi.new_decoder("scm", 72, spectrum=(log2n, F))
    bs2 = h.cfg.block_size2
    iq, _, _ = synth_stream("scm", 72, 1 << 22, spacing=1 << 18)
    iq = iq[:iq.size // bs2 * bs2]
    one = _rows_of(h, [iq])
    want = spectrum_ref.rows(iq, capi.FORMAT_CU8, log2n, F)
    spectrum_ref.assert_close(one[1], want[1])
    spectrum_ref.assert_close(one[2], want[2])
    h.reset()
    cuts = [bs2 * 3, bs2 * 100, bs2 * 101, bs2 * 700]
    _same(_rows_of(h, [iq[a:b] for a, b in zip([0] + cuts, cuts + [iq.size])]), one)
    h.close()


@pytest.mark.parametrize("flags", [0, capi.DECODE_ONLY_VALID])
def test_candidates_signal_and_kernels_unchanged(built, flags):
    cl, mt = 72, "scm,scm+,idm,r900"
    a = capi.new_decoder(mt, cl, signal=True)
    b = capi.new_decoder(mt, cl, signal=True, spectrum=(10, 256))
    bs2 = a.cfg.block_size2
    iq, _, _ = synth_stream(mt, cl, 1 << 21, spacing=1 << 18)
    iq = iq[:iq.size // bs2 * bs2]
    for part in (iq[:iq.size // 2], iq[iq.size // 2:]):
        ca, cb = a.decode(part, flags=flags, cap=1 << 16), b.decode(part, flags=flags, cap=1 << 16)
        assert ca.tobytes() == cb.tobytes()
        assert a.fetch_signal().tobytes() == b.fetch_signal().tobytes()
        assert b.last_kernels() == a.last_kernels() + ";spectrum_kernel<cu8>"
        assert b.last_launches() == a.last_launches() + 1
    plain = capi.new_decoder(mt, cl)
    plain.decode(iq[:iq.size // 2], flags=flags, cap=1 << 16)
    assert "spectrum" not in plain.last_kernels()
    for x in (a, b, plain):
        x.close()


@pytest.mark.parametrize("nch", [3, 8])
def test_channel_groups_equal_a_lone_handle(built, nch):
    cl, rate_in, fmt, log2n, F = 72, 10_000_000, capi.FORMAT_CS16, 11, 200
    offs = [-3_000_000 + 800_000 * k for k in range(nch)]
    z, _ = tune_ref.wideband([("scm", offs[1] + 300_000, 11, 0)], rate_in, 3_000_000, 11)
    raw = tune_ref.quantize(z, fmt)

    def mk(off, spec):
        return capi.new_decoder("scm", cl, input_rate=rate_in, input_format=fmt, capture_freq=CAPTURE,
                                center_freq=CAPTURE + off, spectrum=(log2n, F) if spec else None)
    lone = mk(offs[0], True)
    want = _rows_of(lone, [raw])
    for who in (0, nch - 1):
        group = [mk(o, k == who) for k, o in enumerate(offs)]
        capi.decode_channels(group, raw, cap=1 << 16)
        _same(group[who].fetch_spectrum(), want)
        assert group[who].last_kernels().endswith(";spectrum_kernel<cs16>")
        for h in group:
            h.close()
    lone.close()


def _bin_hz(log2n, k, rate_in=10_000_000, centre=CAPTURE):
    return spectrum_ref.lib().specref_bin_hz(centre, rate_in, log2n, int(k))


def test_packets_land_on_their_carriers_and_signal_freqs(built):
    """scm packets at -700, -150, +90 and +620 kHz from a channel 2 MHz off the centre of a 10 MS/s capture, decoded with
    signal reports: for every message, the strongest bin of the peak-hold rows over its packet is within one bin of the
    injected carrier, and the message's Freq within one bin of that maximum."""
    rate_in, fmt, log2n, cl = 10_000_000, capi.FORMAT_CS16, 10, 72
    F, n_bins = least_f(log2n), 1 << log2n
    binw, r_out, channel = rate_in / n_bins, DATA_RATE * cl, CAPTURE - 2_000_000
    for d in (-700_000, -150_000, 90_000, 620_000):
        carrier = channel + d
        z, _ = tune_ref.wideband([("scm", carrier - CAPTURE, 11, 0)], rate_in, 3_000_000, 11)
        raw = tune_ref.quantize(z, fmt)
        h = capi.new_decoder("scm", cl, input_rate=rate_in, input_format=fmt, capture_freq=CAPTURE, center_freq=channel,
                             signal=True, spectrum=(log2n, F))
        cands = h.decode(raw, flags=capi.DECODE_ONLY_VALID, cap=1 << 16)
        sig = h.fetch_signal()
        rows, _, peak = h.fetch_spectrum(partial=True)
        c = h.cfg
        checked = 0
        for cand, s in zip(cands, sig):
            sm = signal_ref.summary({f: int(s[f]) for f in signal_ref.FIELDS}, channel, r_out)
            if sm is None:
                continue
            a0 = (int(cand["block"]) + 1) * c.block_size - c.buffer_length + int(cand["idx"]) - c.symbol_length
            s0, s1 = a0 * rate_in // r_out, (a0 + c.packet_length) * rate_in // r_out
            over = [i for i, r in enumerate(rows) if r["first_sample"] < s1 and r["first_sample"] + r["frames"] * n_bins > s0]
            f = _bin_hz(log2n, np.argmax(peak[over].max(axis=0)))
            assert abs(f - carrier) <= binw, (d, f - carrier)
            assert abs(sm["freq"] - f) <= binw, (d, sm["freq"] - f)
            checked += 1
        assert checked >= 2, d
        h.close()


def test_near_far_capture(built):
    """tests/nearfar_ref.py's capture: the mean rows put the strong carrier 3.5 MHz below the meter channel in its bin,
    at the restatement's level; the peak-hold rows show the scm packets in their channel, far below the carrier."""
    nf = nearfar_ref
    raw, truth = nf.capture(3)
    fmt, log2n, F = capi.FORMAT_CS16, 10, 256
    n_bins = 1 << log2n
    binw = nf.RATE / n_bins
    h = capi.new_decoder("scm", 72, input_rate=nf.RATE, input_format=fmt, capture_freq=nf.CAPTURE,
                         center_freq=nf.CAPTURE + nf.OFFSET, spectrum=(log2n, F))
    h.decode(raw, cap=1 << 16)
    rows, mean, peak = h.fetch_spectrum()
    _, want_mean, want_peak = spectrum_ref.rows(raw, fmt, log2n, F)
    spectrum_ref.assert_close(mean, want_mean, "mean")
    spectrum_ref.assert_close(peak, want_peak, "peak")
    strong = [int(np.argmax(m)) for m in mean]
    assert all(abs(_bin_hz(log2n, k, nf.RATE, nf.CAPTURE) - (nf.CAPTURE + nf.STRONG_OFFSET)) <= binw for k in strong)
    kc = n_bins // 2 + round(nf.OFFSET / binw)
    chan = peak[:, kc - 20:kc + 21]
    at = np.argmax(chan, axis=1) + kc - 20
    hot = [r for r in range(len(rows)) if abs(_bin_hz(log2n, at[r], nf.RATE, nf.CAPTURE) - (nf.CAPTURE + nf.OFFSET)) <= binw]
    floor = chan.max(axis=1).min()
    assert len(hot) >= len(truth) // 2, (len(hot), len(truth))
    for r in hot:
        assert chan[r].max() > 30 * floor                 # the packet stands out of the channel's floor
        assert chan[r].max() < peak[r][strong[r]] / 100   # and lies far below the carrier
    h.close()


def test_largest_device_call(built):
    """A device call of the most input samples a decimating handle accepts, with no rows waiting, is taken whole and
    measured as the restatement measures it."""
    import torch
    rate_in, fmt, log2n, F = 30_720_000, capi.FORMAT_CS16, 6, 4096
    z, _ = tune_ref.wideband([("scm", 2_400_000, 11, 0)], rate_in, 4_500_000, 11)
    raw = tune_ref.quantize(z, fmt)
    h = capi.new_decoder("scm", 72, input_rate=rate_in, input_format=fmt, capture_freq=CAPTURE,
                         center_freq=CAPTURE + 2_400_000, max_blocks_per_call=64, spectrum=(log2n, F))
    d = torch.from_numpy(raw).cuda()
    torch.cuda.synchronize()
    lo, hi = 1, raw.size // 4   # the largest n the input stage's rule accepts
    while lo < hi:
        mid = (lo + hi + 1) // 2
        h.reset()
        try:
            h.decode_device_async(d.data_ptr(), 4 * mid)
            h.fetch(cap=1 << 16)
            lo = mid
        except capi.ErtGpuError as e:
            assert e.code == capi.ESIZE, e
            hi = mid - 1
    assert lo < raw.size // 4
    h.reset()
    h.fetch_spectrum()
    h.decode_device_async(d.data_ptr(), 4 * lo)
    h.fetch(cap=1 << 16)
    got = h.fetch_spectrum(partial=True)
    want = spectrum_ref.rows(raw[:4 * lo], fmt, log2n, F, partial=True)
    assert [tuple(int(x) for x in r) for r in got[0]] == want[0]
    spectrum_ref.assert_close(got[1], want[1])
    spectrum_ref.assert_close(got[2], want[2])
    h.close()


def test_long_device_call_is_cut_the_same(built):
    """A device call longer than one launch takes (2^24 samples) gives the rows of the host path's staging chunks."""
    import torch
    log2n, F = 10, 256
    a = capi.new_decoder("scm", 72, spectrum=(log2n, F))
    b = capi.new_decoder("scm", 72, spectrum=(log2n, F))
    plain = capi.new_decoder("scm", 72)
    iq = np.random.default_rng(5).integers(0, 256, 2 << 25, dtype=np.uint8)   # 2^25 samples
    host = _rows_of(a, [iq])
    d = torch.from_numpy(iq).cuda()
    torch.cuda.synchronize()
    b.decode_device_async(d.data_ptr(), iq.size)
    b.fetch(cap=1 << 16)
    plain.decode_device_async(d.data_ptr(), iq.size)
    plain.fetch(cap=1 << 16)
    assert b.last_launches() == plain.last_launches() + 2
    _same(b.fetch_spectrum(), host)
    for x in (a, b, plain):
        x.close()


def test_rules(built):
    h = capi.new_decoder("scm", 72, spectrum=(10, 256))
    with pytest.raises(capi.ErtGpuError) as e:
        h.enable_spectrum(10, 256)
    assert e.value.code == capi.EINVAL
    for n, f in ((5, 1 << 13), (15, 16), (10, 255), (14, 15), (6, 0)):
        x = capi.Handle()
        x.register(capi.stock_protocol("scm", 72))
        with pytest.raises(capi.ErtGpuError) as e:
            x.enable_spectrum(n, f)
        assert e.value.code == capi.EINVAL
        x.close()
    plain = capi.new_decoder("scm", 72)
    with pytest.raises(capi.ErtGpuError) as e:
        plain.fetch_spectrum()
    assert e.value.code == capi.EINVAL
    bs2 = h.cfg.block_size2
    with pytest.raises(capi.ErtGpuError) as e:
        capi.decode_sharded([h], np.zeros(bs2 * 4, np.uint8))
    assert e.value.code == capi.EINVAL
    assert "spectrum" in capi.lib().ertgpu_last_error(h._h).decode()
    # capacity of the fetch: ertgpu_fetch's rules, nothing consumed
    iq = np.full(bs2 * 160, 127, np.uint8)   # 655 360 samples: 2 rows of 2^18 samples
    h.decode(iq, cap=16)
    n = C.c_size_t(0)
    rows = np.zeros(1, capi.SPECTRUM_ROW_DTYPE)
    buf = np.zeros((1, 1024), np.float32)
    rc = capi.lib().ertgpu_fetch_spectrum(h._h, 1, rows.ctypes.data, buf.ctypes.data, buf.ctypes.data, 1, C.byref(n))
    assert rc == capi.ECAPACITY and n.value == 3
    r, m, p = h.fetch_spectrum(partial=True)
    assert len(r) == 3 and r[2]["frames"] == 640 - 512
    r, m, p = h.fetch_spectrum(partial=True)
    assert len(r) == 1 and r[0]["first_sample"] == 2 * (1 << 18)
    # decode overflow: rows left unfetched and a call that would not fit -> ECAPACITY before anything is enqueued
    cap_rows = None
    k = 0
    while True:
        try:
            h.decode(iq, cap=16)
        except capi.ErtGpuError as err:
            assert err.code == capi.ECAPACITY
            cap_rows = k
            break
        k += 1
        assert k < 10000
    r, _, _ = h.fetch_spectrum()
    assert len(r) >= cap_rows
    h.decode(iq, cap=16)   # fits again
    # two spectra in one channel group
    def mk(off, spec):
        return capi.new_decoder("scm", 72, input_rate=10_000_000, input_format=capi.FORMAT_CS16, capture_freq=CAPTURE,
                                center_freq=CAPTURE + off, spectrum=(10, 256) if spec else None)
    g = [mk(0, True), mk(500_000, True)]
    with pytest.raises(capi.ErtGpuError) as e:
        capi.decode_channels(g, np.zeros(4 * 100_000, np.uint8))
    assert e.value.code == capi.EINVAL
    for x in g + [h, plain]:
        x.close()


def test_cli_spectrum_file(built, tmp_path):
    """ertgpu_decode_file -spectrum=FILE on a three-channel cs16 capture: rtl_power's layout, the rows of
    ertgpu_fetch_spectrum in dB to two decimals, stdout unchanged; -spectrumpeak; a dated SigMF recording's times."""
    import json
    import os
    import subprocess
    from conftest import ROOT
    rate_in, chans = 10_000_000, [CAPTURE - 3_000_000, CAPTURE - 1_000_000, CAPTURE + 2_000_000]
    z, _ = tune_ref.wideband([("scm", chans[1] + 250_000 - CAPTURE, 11, 0)], rate_in, 3_000_000, 11)
    raw = tune_ref.quantize(z, capi.FORMAT_CS16)
    path = tmp_path / "cap.cs16"
    raw.tofile(path)
    cli = os.path.join(ROOT, "rtlamr_b200", "ertgpu_decode_file")
    base = ["-msgtype=scm", "-sampleformat=cs16", f"-samplerate={rate_in}", f"-capturefreq={CAPTURE}",
            "-centerfreq=" + ",".join(map(str, chans))]
    run = lambda *a: subprocess.run([cli, *a], capture_output=True, text=True, timeout=300, check=True).stdout  # noqa: E731
    out = tmp_path / "s.csv"
    plain = run(*base, str(path))
    assert run(f"-spectrum={out}", "-spectrumint=50ms", *base, str(path)) == plain
    log2n, F = 10, 488   # -spectrumbin 10 kHz at 10 MS/s: N = 1024; 50 ms: round(0.05 * 10^7 / 1024) frames
    h = capi.new_decoder("scm", 72, input_rate=rate_in, input_format=capi.FORMAT_CS16, capture_freq=CAPTURE,
                         center_freq=chans[0], spectrum=(log2n, F))
    h.decode(raw, cap=1 << 16)
    rows, mean, peak = h.fetch_spectrum(partial=True)
    h.close()

    def parse(p):
        lines = [ln.split(", ") for ln in open(p).read().splitlines()]
        assert len(lines) == len(rows) == 7
        for i, f in enumerate(lines):
            assert f[0] == "1970-01-01" and f[1] == "00:00:00"
            assert (int(f[2]), int(f[3]), f[4]) == (CAPTURE - rate_in // 2, CAPTURE + rate_in // 2, "9765.62")
            assert int(f[5]) == int(rows[i]["frames"]) << log2n
            assert len(f) == 6 + (1 << log2n)
        return lines
    for f, w in zip(parse(out), mean):
        assert f[6:] == [f"{spectrum_ref.lib().specref_db(float(x)):.2f}" for x in w]
    run(f"-spectrum={out}", "-spectrumint=50ms", "-spectrumpeak", *base, str(path))
    for f, w in zip(parse(out), peak):
        assert f[6:] == [f"{spectrum_ref.lib().specref_db(float(x)):.2f}" for x in w]
    # a dated SigMF recording: the recording time of each row's first sample
    (tmp_path / "rec.sigmf-data").write_bytes(raw.tobytes())
    (tmp_path / "rec.sigmf-meta").write_text(json.dumps({
        "global": {"core:datatype": "ci16_le", "core:sample_rate": rate_in, "core:version": "1.0.0"},
        "captures": [{"core:sample_start": 0, "core:frequency": CAPTURE, "core:datetime": "2024-05-01T12:00:59.8Z"}],
        "annotations": []}))
    run(f"-spectrum={out}", "-spectrumint=50ms", "-msgtype=scm", "-sampleformat=sigmf", str(tmp_path / "rec"))
    times = [ln.split(", ")[:2] for ln in open(out).read().splitlines()]
    want = ["12:00:59" if 59.8 + r[0] / rate_in < 60 else "12:01:00" for r in rows]
    assert times == [["2024-05-01", t] for t in want]


def test_host_receiver_spectrum(built):
    from rtlamr_b200 import host
    rate_in, off, log2n, F = 10_000_000, -2_000_000, 11, 200
    z, _ = tune_ref.wideband([("scm", off + 90_000, 11, 0)], rate_in, 3_000_000, 11)
    raw = tune_ref.quantize(z, capi.FORMAT_CS16)
    kw = dict(input_rate=rate_in, input_format=capi.FORMAT_CS16, capture_freq=CAPTURE, center_freq=CAPTURE + off)
    r = host.Receiver("scm", 72, spectrum=(log2n, F), **kw)
    plain = host.Receiver("scm", 72, **kw)
    msgs = []
    for a in range(0, raw.size, 4 * 700_001):
        msgs += r.decode(raw[a:a + 4 * 700_001])
    assert [(m.block, m.idx, m.text) for m in msgs] == [(m.block, m.idx, m.text) for m in plain.decode(raw)]
    h = capi.new_decoder("scm", 72, spectrum=(log2n, F), **kw)
    h.decode(raw, cap=1 << 16)
    _same(r.spectrum(partial=True), h.fetch_spectrum(partial=True))
    r.reset()
    assert len(r.spectrum()[0]) == 0
    for x in (r, plain, h):
        x.close()
