"""CPU tests of the decimating tuned input (ertgpu_allow_input_decimation): the plan rule of
include/ertgpu_resample.h at its boundaries, the first stage's taps, the shared memory of both kernels over the ratio
range, the quality of the two-stage cascade through its CPU restatement (tests/cpu_harness/decimate_ref.c into
resample_ref.c), and the argument checks that need no GPU."""
import numpy as np
import pytest

from rtlamr_b200 import capi

import decimate_ref
import resample_ref
import tune_ref

DATA_RATE = 32768
R72, R32, R8 = DATA_RATE * 72, DATA_RATE * 32, DATA_RATE * 8


def test_rule_boundaries():
    for rate_out in (R72, R32, R8):
        dec, info = decimate_ref.plan(10 * rate_out, rate_out, 0)
        assert dec["D"] == 1 and dec["T1"] == 0 and info == tune_ref.plan(10 * rate_out, rate_out, 0)
        dec, info = decimate_ref.plan(10 * rate_out + 1, rate_out, 0)
        assert dec["D"] == 3 and info["rate_out"] == 3 * rate_out and info["P"] == 256 and info["T"] <= 88
        dec, _ = decimate_ref.plan(256 * rate_out, rate_out, 0)
        assert dec["D"] == 64
        assert decimate_ref.plan(256 * rate_out + 1, rate_out, 0) is None
        # inside the range, R_mid = R_in / D lies in (3 R_out, 4 R_out] and the second stage is the untuned plan
        for rate_in in np.linspace(10 * rate_out + 1, 256 * rate_out, 200).astype(np.int64):
            dec, info = decimate_ref.plan(int(rate_in), rate_out, 0)
            D = dec["D"]
            assert D == -(-int(rate_in) // (4 * rate_out)) and 3 * rate_out * D < rate_in <= 4 * rate_out * D
            assert info == resample_ref.Resampler(int(rate_in), D * rate_out).info


@pytest.mark.parametrize("rate_in,rate_out", [(30_720_000, R72), (61_440_000, R72), (20_000_000, R32), (61_440_000, R8)])
def test_channel_inside_rule_at_both_signs(rate_in, rate_out):
    # 10 |offset| + 4 R_out <= 5 R_in
    edge = (5 * rate_in - 4 * rate_out) // 10
    for sign in (1, -1):
        assert decimate_ref.plan(rate_in, rate_out, sign * edge) is not None
        assert decimate_ref.plan(rate_in, rate_out, sign * (edge + 1)) is None


@pytest.mark.parametrize("rate_in,rate_out", [(10 * R72 + 1, R72), (30_720_000, R72), (56_000_000, R72), (61_440_000, R72),
                                              (20_000_000, R32), (256 * R8, R8), (40 * R72 + 7, R72)])
def test_stage1_taps(rate_in, rate_out):
    s = decimate_ref.Stage1(rate_in, rate_out, -2_400_000 if rate_in > 20_000_000 else 0)
    h = s.taps().astype(np.int64)
    T1 = s.dec["T1"]
    assert T1 % 2 == 0 and h[T1 - 1] == 0
    assert np.array_equal(h[:T1 - 1], h[:T1 - 1][::-1])       # symmetric about tap T1/2 - 1
    assert h.sum() == 1 << 14 and np.abs(h).max() <= 32767
    # about 4.3 R_mid / (R_mid - R_out) taps per input sample
    mid = rate_in / s.dec["D"]
    assert T1 / s.dec["D"] <= 4.33 * mid / (mid - rate_out) + 2 / s.dec["D"]
    # the filter itself: flat to 0.4 R_out, and from R_mid - 0.6 R_out down by the 70 dB design less what rounding the
    # taps to 2^-14 costs (most at D = 64, whose taps peak near 240)
    H = np.abs(np.fft.rfft(h / (1 << 14), 1 << 20))
    f = np.arange(H.size) / (1 << 20) * rate_in
    assert np.all(np.abs(20 * np.log10(H[f <= 0.4 * rate_out])) <= 0.05)
    assert np.all(20 * np.log10(np.maximum(H[f >= mid - 0.6 * rate_out], 1e-12)) <= -55.0)


def _dc_smem(D, T1):
    """dc_smem_bytes of csrc/decimate.cuh with dc_per_thread's tile."""
    per = min(16, max(1, (20480 - T1) // (256 * D)))
    span = (256 * per - 1) * D + T1
    assert span <= 20480
    return (4096 + T1 // 2 + span + (span >> 5) + 1) * 4


def test_shared_memory_fits_over_the_ratio_range():
    worst1 = worst2 = 0
    for rate_out in (R72, R32, R8):
        for rate_in in np.unique(np.linspace(10 * rate_out + 1, 256 * rate_out, 3000).astype(np.int64)):
            dec, info = decimate_ref.plan(int(rate_in), rate_out, 0)
            worst1 = max(worst1, _dc_smem(dec["D"], dec["T1"]))
            T, P, L, M = info["T"], info["P"], info["L"], info["M"]
            worst2 = max(worst2, P * T * 6 + (((2047 * M + L - 1) // L) + 1 + T + 1) * 4)   # rs_smem_bytes, untuned
    assert worst1 <= 227 * 1024 and worst2 <= 227 * 1024, (worst1, worst2)


def _settled(out, skip=64):
    x = out.reshape(-1, 2).astype(np.float64)[skip:] - 127.5
    return x[:, 0] + 1j * x[:, 1]


def _band_db(z, k=None):
    """Power in dB (8-bit units squared) of the strongest tone of z, or of the one at bin k, after removing the mean."""
    z = z - z.mean()
    w = np.hanning(z.size)
    spec = np.abs(np.fft.fft(z * w)) ** 2
    if k is None:
        k = int(np.argmax(spec))
    band = spec[np.arange(k - 4, k + 5) % z.size].sum()
    return 10 * np.log10(band / (w ** 2).sum() / z.size), k


CASCADES = [(20_000_000, R32, -2_400_000), (30_720_000, R72, -2_400_000), (61_440_000, R72, 5_000_000),
            (56_000_000, R72, -12_600_000)]


def _alias_bin(f_hz, rate_in, rate_out, D, n):
    """The output bin a tone f_hz from the channel lands in: folded at R_mid by stage 1, then at R_out by stage 2."""
    mid = rate_in / D
    f1 = f_hz - np.round(f_hz / mid) * mid
    f2 = f1 - np.round(f1 / rate_out) * rate_out
    return int(np.round(f2 / rate_out * n)) % n


def _tone(n, f_cyc, amp=60.0, noise=4.0):
    """uint8 IQ of a complex tone at f_cyc cycles per sample in Gaussian noise of sigma `noise` per component, as a
    capture carries it.  Without noise, a leak far below one LSB sits at the intermediate bytes' rounding threshold
    (s' = 0 is u = 127.5) and comes out as half-LSB switching about 10 dB above the filter's own leak."""
    rng = np.random.default_rng(int(f_cyc * 1e9) & 0xFFFF)
    z = amp * np.exp(2j * np.pi * f_cyc * np.arange(n)) + noise * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    iq = np.empty(2 * n, dtype=np.uint8)
    iq[0::2] = np.clip(np.round(127.5 + z.real), 0, 255)
    iq[1::2] = np.clip(np.round(127.5 + z.imag), 0, 255)
    return iq


def _out(rate_in, rate_out, off, f_hz, n_out=1 << 16):
    n = (n_out + 256) * rate_in // rate_out + 4096
    return _settled(decimate_ref.decimate(_tone(n, (off + f_hz) / rate_in), rate_in, rate_out, off))[:n_out]


@pytest.mark.parametrize("rate_in,rate_out,off", CASCADES)
def test_cascade_passband(rate_in, rate_out, off):
    """A tone of amplitude 60 anywhere within 0.4 R_out of the channel comes out at 60 within +-0.5 dB."""
    want = 20 * np.log10(60.0)
    for frac in (-0.4, -0.3, -0.2, -0.1, 0.03, 0.1, 0.2, 0.3, 0.4):   # not 0: _band_db removes the mean
        z = _out(rate_in, rate_out, off, frac * rate_out)
        p, k = _band_db(z)
        assert abs(((k / z.size + 0.5) % 1.0 - 0.5) - frac) <= 2.0 / z.size, frac
        assert abs(p - want) <= 0.5, (frac, p - want)


@pytest.mark.parametrize("rate_in,rate_out,off", CASCADES)
def test_cascade_stopband_and_aliases(rate_in, rate_out, off):
    """Tones at |f| >= 0.62 R_out from the channel, those near multiples of R_mid (which stage 1 folds onto the
    channel) among them, come out at least 50 dB below a passband tone."""
    p_ref, _ = _band_db(_out(rate_in, rate_out, off, 0.1 * rate_out))
    D = decimate_ref.plan(rate_in, rate_out, off)[0]["D"]
    mid = rate_in / D
    fs = [s * a * rate_out for s in (1, -1) for a in (0.62, 0.8, 1.3, 2.5)]
    fs += [s * (k * mid + d * rate_out) for s in (1, -1) for k in (1, 2) for d in (-0.3, 0.15, 0.35)]
    tested = 0
    for f in fs:
        if abs(off + f) >= 0.5 * rate_in - 0.02 * rate_out:
            continue
        z = _out(rate_in, rate_out, off, f)
        p, _ = _band_db(z, _alias_bin(f, rate_in, rate_out, D, z.size))
        assert p_ref - p >= 50.0, (f, p_ref - p)
        tested += 1
    assert tested >= 10


@pytest.mark.parametrize("rate_in,rate_out,off", [(20_000_000, R32, 2_000_000), (30_720_000, R72, -2_400_000),
                                                  (61_440_000, R72, 1_500_000), (61_440_000, R8, -300_000)])
def test_dc_spike_is_removed(rate_in, rate_out, off):
    """A constant input (the capture's DC spike) with |offset| >= 0.62 R_out comes out within +-1 of 127.5.  The levels
    keep |s| below 255 after the mix: a larger spike close enough to the channel to pass stage 1 clips in the
    intermediate bytes, and its harmonics can fold into the channel."""
    assert abs(off) >= 0.62 * rate_out
    for u in (64, 100, 160, 200):
        out = decimate_ref.decimate(np.full(2 * (400 * rate_in // rate_out + 50_000), u, dtype=np.uint8), rate_in,
                                    rate_out, off)
        settled = out[2 * 64:].astype(np.int32)
        assert settled.size > 500 and np.all(np.abs(2 * settled - 255) <= 2), (u, np.unique(settled))


def test_restatement_is_split_invariant():
    rate_in, rate_out, off = 61_440_000, R72, -2_400_000
    rng = np.random.default_rng(5)
    n = 1_000_003
    iq = rng.integers(0, 256, 2 * n, dtype=np.uint8)
    whole = decimate_ref.decimate(iq, rate_in, rate_out, off)
    c = decimate_ref.Cascade(rate_in, rate_out, off)
    cuts = np.sort(rng.choice(np.arange(1, n), 60, replace=False))
    parts, prev = [], 0
    for cut in list(cuts) + [n]:
        parts.append(c.feed(iq[2 * prev:2 * cut]))
        prev = cut
    assert np.array_equal(np.concatenate(parts), whole) and whole.size > 2 * 30_000


def _einval(fn, *args):
    with pytest.raises(capi.ErtGpuError) as e:
        fn(*args)
    assert e.value.code == capi.EINVAL


def test_decimation_argument_checks_without_gpu():
    h = capi.Handle()
    _einval(h.allow_input_decimation)                          # no protocol, no tuning
    h.register(capi.stock_protocol("scm", 72))
    _einval(h.allow_input_decimation)                          # untuned
    h.set_input_tuning(915_000_000)
    _einval(h.decimator)                                       # not allowed yet
    h.allow_input_decimation()
    _einval(h.decimator)                                       # no rate yet
    _einval(h.set_input_rate, 256 * R72 + 1)                   # above 256:1
    h.set_input_rate(61_440_000)
    h.close()
    h = capi.Handle()
    h.register(capi.stock_protocol("scm", 72))
    h.set_input_tuning(915_000_000, 935_000_000)
    h.allow_input_decimation()
    _einval(h.set_input_rate, 30_720_000)                      # 20 MHz off: outside a 30.72 MS/s capture
    h.set_input_rate(61_440_000)
    h.close()


def test_decimation_plans_through_the_abi_without_gpu():
    off = -2_399_845   # 915 MHz capture, scm's 912.6 MHz channel
    for rate_in in (10 * R72, 30_720_000, 61_440_000, 256 * R72):
        h = capi.Handle()
        h.register(capi.stock_protocol("scm", 72))
        h.set_input_tuning(915_000_000)
        h.allow_input_decimation()
        h.set_input_rate(rate_in)
        _einval(h.allow_input_decimation)                      # after the rate
        dec, taps = h.decimator()
        info, table = h.resampler()
        want_dec, want_info = decimate_ref.plan(rate_in, R72, off)
        assert dec == want_dec and info == want_info
        assert h.tuning()["nco_step"] == tune_ref.nco_step(off, rate_in)
        if dec["D"] == 1:
            assert taps.size == 0 and np.array_equal(table, tune_ref.Tuner(rate_in, R72, off).table())
        else:
            assert np.array_equal(taps, decimate_ref.Stage1(rate_in, R72, off).taps())
            assert np.array_equal(table, resample_ref.Resampler(rate_in, dec["D"] * R72).table())
        h.close()
    # without the call a tuned handle keeps [1/10, 4]
    h = capi.Handle()
    h.register(capi.stock_protocol("scm", 72))
    h.set_input_tuning(915_000_000)
    _einval(h.set_input_rate, 10 * R72 + 1)
    h.close()
