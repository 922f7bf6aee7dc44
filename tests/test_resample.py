"""CPU tests of the input-rate resampler: the prototype table libertgpu.so exports (include/ertgpu_resample.h),
the argument checks of ertgpu_set_input_rate / ertgpu_decode that need no GPU, and the CPU restatement
(tests/cpu_harness/resample_ref.c) the GPU tests compare the kernel with."""
import numpy as np
import pytest

from rtlamr_b200 import capi

import resample_ref

DATA_RATE = 32768
# (input rate, chip length): the common SDR rates against chip lengths 72 and 32, and 1.024 MS/s against 72
CASES = [(r, cl) for r in (2_048_000, 2_400_000, 2_560_000, 2_880_000, 3_200_000) for cl in (72, 32)] + [(1_024_000, 72)]


def _handle(rate_in, cl, msgtype="scm"):
    h = capi.Handle()
    h.register(capi.stock_protocol(msgtype, cl))
    h.set_input_rate(rate_in)
    return h


def _coefficients(info, table, phases):
    """Per-output integer coefficients of the given phases phi_n (before the DC correction)."""
    T, P, F = info["T"], info["P"], info["F"]
    tab = table.astype(np.int64).reshape(P + 1, T)
    q = (phases.astype(object) * (P << F) // info["L"]).astype(np.int64)
    p, w = q >> F, q & ((1 << F) - 1)
    h0, h1 = tab[p], tab[p + 1]
    return h0 + (((h1 - h0) * w[:, None] + (1 << (F - 1))) >> F), p


def _response_db(info, table, f):
    """|H(f)| in dB of the prototype (P sub-phases per input sample), f in cycles per input sample."""
    T, P, S = info["T"], info["P"], info["S"]
    tab = table.astype(np.float64).reshape(P + 1, T)[:P]
    tau = (np.arange(T)[None, :] - T // 2 + 1) - np.arange(P)[:, None] / P  # time of tab[p, t]
    order = np.argsort(tau.ravel())
    h, t0 = tab.ravel()[order], tau.ravel()[order][0]
    nfft = 1 << 21
    H = np.abs(np.fft.rfft(h, nfft)) / (P * (1 << S))
    grid = np.arange(H.size) * P / nfft
    return 20 * np.log10(np.maximum(np.interp(f, grid, H), 1e-12)), t0


@pytest.mark.parametrize("rate_in,cl", CASES)
def test_table_properties(built, rate_in, cl):
    h = _handle(rate_in, cl)
    info, table = h.resampler()
    h.close()
    rate_out = DATA_RATE * cl
    assert info["rate_out"] == rate_out and info["rate_in"] == rate_in
    assert info["L"] * rate_in == info["M"] * rate_out and np.gcd(info["L"], info["M"]) == 1
    T, P, S = info["T"], info["P"], info["S"]
    assert T % 2 == 0 and T <= 128 and table.size == (P + 1) * T
    tab = table.reshape(P + 1, T).astype(np.int64)
    # the CPU restatement builds the same table from the same header
    assert np.array_equal(resample_ref.Resampler(rate_in, rate_out).table(), table)
    # symmetry h(-d) = h(d): table[p][t] == table[P-p][T-1-t]
    assert np.array_equal(tab, tab[::-1, ::-1])
    # every row has DC gain exactly 2^S
    assert np.all(tab.sum(axis=1) == 1 << S)
    # passband and stopband, in cycles per input sample
    nu = min(rate_in, rate_out) / rate_in
    pas, _ = _response_db(info, table, np.linspace(0, 0.40 * nu, 400))
    assert np.max(np.abs(pas)) <= 0.1, np.max(np.abs(pas))
    stop, _ = _response_db(info, table, np.linspace(0.60 * nu, P / 2, 200_000))
    assert np.max(stop) <= -60.0, np.max(stop)
    # the gain error of the interpolated coefficients stays below 1/255 at every phase (all phases when L is small)
    phases = np.arange(info["L"]) if info["L"] <= 1 << 16 else \
        np.random.default_rng(1).integers(0, info["L"], 1 << 16)
    c, _ = _coefficients(info, table, phases)
    assert np.max(np.abs(c.sum(axis=1) - (1 << S))) < (1 << S) / 255


@pytest.mark.parametrize("rate_in,cl", CASES)
def test_constant_input_is_exact(built, rate_in, cl):
    """A constant u comes out as exactly u for every u once the window is full."""
    rate_out = DATA_RATE * cl
    T = resample_ref.Resampler(rate_in, rate_out).info["T"]
    for u in range(256):
        r = resample_ref.Resampler(rate_in, rate_out)
        out = r.feed(np.full(2 * (T + 4000), u, dtype=np.uint8)).reshape(-1, 2)
        L, M = r.info["L"], r.info["M"]
        full = np.arange(out.shape[0]) * M // L - T // 2 + 1 >= 0  # window inside the stream
        assert np.all(out[full] == u), (u, np.unique(out[full]))


def test_rate_checks_without_gpu(built):
    h = capi.Handle()
    with pytest.raises(capi.ErtGpuError) as e:  # no protocol yet: the decoder rate is unknown
        h.set_input_rate(2_400_000)
    assert e.value.code == capi.EINVAL
    h.register(capi.stock_protocol("scm", 72))
    rate_out = DATA_RATE * 72
    for bad in (0, -1, rate_out * 4 + 1, rate_out // 4 - 1, 10**12):
        with pytest.raises(capi.ErtGpuError) as e:
            h.set_input_rate(bad)
        assert e.value.code == capi.EINVAL
    h.set_input_rate(rate_out * 4)   # both bounds are inside
    h.set_input_rate(rate_out // 4)
    h.set_input_rate(2_400_000)
    with pytest.raises(capi.ErtGpuError) as e:  # protocols are registered before the rate
        h.register(capi.stock_protocol("idm", 72))
    assert e.value.code == capi.EINVAL
    # odd byte counts are not whole IQ samples
    odd = np.zeros(4097, dtype=np.uint8)
    with pytest.raises(capi.ErtGpuError) as e:
        h.decode(odd)
    assert e.value.code == capi.ESIZE
    with pytest.raises(capi.ErtGpuError) as e:
        h.decode_device_async(odd.ctypes.data, odd.size)
    assert e.value.code == capi.ESIZE
    h.close()
    # the decoder's own rate needs no resampler
    h = _handle(rate_out, 72)
    with pytest.raises(capi.ErtGpuError) as e:
        h.resampler()
    assert e.value.code == capi.EINVAL
    h.close()


def test_cli_rejects_samplefile_with_resampling(built, tmp_path):
    """-samplefile with a resampling -samplerate is a usage error (exit status 2), before any device is touched."""
    import os
    import subprocess
    cli = os.path.join(resample_ref.ROOT, "rtlamr_b200", "ertgpu_decode_file")
    f = tmp_path / "in.bin"
    np.zeros(4096, dtype=np.uint8).tofile(f)
    r = subprocess.run([cli, "-symbollength=72", "-samplerate=2400000", f"-samplefile={tmp_path / 's.bin'}", str(f)],
                       capture_output=True, text=True, timeout=60)
    assert r.returncode == 2 and "-samplefile" in r.stderr


def _tone(n, f_cyc, amp=60.0):
    """uint8 IQ of a complex tone at f_cyc cycles per sample (with a dither-free rounding)."""
    t = np.arange(n)
    z = amp * np.exp(2j * np.pi * f_cyc * t)
    iq = np.empty(2 * n, dtype=np.uint8)
    iq[0::2] = np.clip(np.round(127.5 + z.real), 0, 255)
    iq[1::2] = np.clip(np.round(127.5 + z.imag), 0, 255)
    return iq


def _tone_power_db(iq, f_cyc):
    x = iq.reshape(-1, 2).astype(np.float64) - 127.5
    z = x[:, 0] + 1j * x[:, 1]
    n = z.size
    w = np.hanning(n)
    spec = np.abs(np.fft.fft(z * w)) ** 2
    freqs = np.fft.fftfreq(n)
    k = np.argmin(np.abs(freqs - f_cyc))
    band = spec[max(0, k - 4):k + 5].sum()
    return 10 * np.log10(band / (w ** 2).sum() / n)


@pytest.mark.parametrize("rate_in,cl", [(2_400_000, 72), (2_048_000, 72), (3_200_000, 32), (1_024_000, 72)])
def test_oracle_keeps_passband_tone(rate_in, cl):
    rate_out = DATA_RATE * cl
    lo = min(rate_in, rate_out)
    for frac in (0.05, 0.2, 0.38):
        for sign in (1, -1):
            f_hz = sign * frac * lo
            iq = _tone(1 << 16, f_hz / rate_in)
            out = resample_ref.resample(iq, rate_in, rate_out)
            T = resample_ref.Resampler(rate_in, rate_out).info["T"]
            skip = 2 * (T * rate_out // rate_in + 8)
            out = out[skip: skip + 2 * (1 << 15)]
            p_in = _tone_power_db(iq[skip:skip + 2 * (1 << 15)], f_hz / rate_in)
            p_out = _tone_power_db(out, f_hz / rate_out)
            assert abs(p_out - p_in) <= 0.5, (f_hz, p_in, p_out)


@pytest.mark.parametrize("rate_in,cl", [(2_400_000, 72), (2_048_000, 72), (3_200_000, 32), (1_024_000, 72)])
def test_oracle_suppresses_stopband_tone(rate_in, cl):
    """A tone beyond 0.60 * min(R_in, R_out) comes out at least 50 dB below a passband tone of the same level
    (dBc), measured where it lands in the uint8 output: at its alias when decimating, at its own frequency when
    interpolating."""
    rate_out = DATA_RATE * cl
    lo = min(rate_in, rate_out)
    n = 1 << 16
    win = slice(4096, 4096 + 2 * (1 << 15))
    p_ref = _tone_power_db(resample_ref.resample(_tone(n, 0.1 * lo / rate_in), rate_in, rate_out)[win], 0.1 * lo / rate_out)
    for frac in (0.62, 0.75, 0.95):
        for sign in (1, -1):
            f_hz = sign * frac * lo
            if abs(f_hz) >= rate_in / 2:
                continue
            out = resample_ref.resample(_tone(n, f_hz / rate_in), rate_in, rate_out)[win]
            f_out = (f_hz / rate_out + 0.5) % 1.0 - 0.5  # where it lands at the output rate
            assert p_ref - _tone_power_db(out, f_out) >= 50.0, (f_hz, p_ref)


@pytest.mark.parametrize("rate_in,cl", [(2_400_000, 72), (2_048_000, 72), (3_200_000, 32), (1_024_000, 72)])
def test_oracle_is_split_invariant(rate_in, cl):
    rate_out = DATA_RATE * cl
    rng = np.random.default_rng(rate_in + cl)
    iq = rng.integers(0, 256, 2 * 200_003, dtype=np.uint8)
    whole = resample_ref.resample(iq, rate_in, rate_out)
    r = resample_ref.Resampler(rate_in, rate_out)
    cuts = np.sort(rng.choice(np.arange(1, 200_003), 40, replace=False))
    parts, prev = [], 0
    for c in list(cuts) + [200_003]:
        parts.append(r.feed(iq[2 * prev:2 * c]))
        prev = c
    parts.append(r.feed(iq[:0]))
    assert np.array_equal(np.concatenate(parts), whole)
    # every output whose window is inside the input has been produced
    T = r.info["T"]
    assert whole.size // 2 == -(-(200_003 - T // 2) * r.info["L"] // r.info["M"])
