"""CPU tests of the input spectrum's definitions (include/ertgpu_spectrum.h): the header's helpers against NumPy, the
NumPy restatement's own known answers (tests/spectrum_ref.py), the CSV line, and the CLI's usage errors."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import spectrum_ref
from spectrum_ref import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "rtlamr_b200", "ertgpu_decode_file")


@pytest.mark.parametrize("log2n", range(6, 15))
def test_window_and_scale(log2n):
    n = 1 << log2n
    w = np.empty(n, np.float32)
    lib().specref_window(log2n, w.ctypes.data)
    assert w.tobytes() == spectrum_ref.window(log2n).tobytes()
    assert lib().specref_power_scale(log2n) == np.float32(1.0 / (16320.0 * n / 2) ** 2)


def test_frame_length_from_bin_width_and_rows():
    for rate in (2_359_296, 2_400_000, 10_000_000, 61_440_000, 1000):
        for hz in (100.0, 1e3, 1e4, 3e4, 1e6):
            n = lib().specref_log2_for_bin(rate, hz)
            want = 6
            while want < 14 and rate / (1 << want) > hz:
                want += 1
            assert n == want
    assert lib().specref_log2_for_bin(10_000_000, 1e4) == 10
    assert lib().specref_log2_for_bin(61_440_000, 1e4) == 13
    assert lib().specref_frames_per_row(10, 1_000_000_000, 10_000_000) == 9766
    assert lib().specref_frames_per_row(10, 1_000_000, 10_000_000) == 256   # at least 2^18 samples
    assert lib().specref_frames_per_row(13, 0, 61_440_000) == 32


def test_bin_frequencies_and_db_floor():
    for log2n in (6, 10, 14):
        n = 1 << log2n
        f = [lib().specref_bin_hz(915_000_000, 10_000_000, log2n, k) for k in range(n)]
        want = 915_000_000 + np.fft.fftshift(np.fft.fftfreq(n, 1 / 10_000_000))
        assert np.allclose(f, want, rtol=0, atol=1e-6)
    assert lib().specref_db(0.0) == -200.0
    assert lib().specref_db(1e-30) == -200.0
    assert lib().specref_db(1.0) == 0.0
    assert abs(lib().specref_db(0.5) - 10 * np.log10(0.5)) < 1e-12


def _cu8_tone(n, k, frac=0.0):
    t = np.arange(n)
    z = 127.5 * np.exp(2j * np.pi * (k + frac) * t / n)
    raw = np.empty(2 * n, np.uint8)
    raw[0::2] = np.clip(np.round(z.real + 127.5), 0, 255)
    raw[1::2] = np.clip(np.round(z.imag + 127.5), 0, 255)
    return raw


def test_full_scale_tone_reads_zero_db():
    log2n = 10
    n = 1 << log2n
    p = spectrum_ref.frame_powers(_cu8_tone(n, 100), 0, log2n)[0]
    assert f"{spectrum_ref.db(p[n // 2 + 100]):.2f}" in ("0.00", "-0.00")
    assert int(np.argmax(p)) == n // 2 + 100


def test_half_bin_off_reads_the_scalloping_loss():
    log2n = 12
    n = 1 << log2n
    t = np.arange(n)
    z = 16320 / 16384 * np.exp(2j * np.pi * (300.5) * t / n)   # cf32 at the default gain 128: s_w = 16320 z
    raw = np.empty(2 * n, np.float32)
    raw[0::2], raw[1::2] = z.real, z.imag
    p = spectrum_ref.frame_powers(raw.view(np.uint8), 3, log2n)[0]
    assert f"{spectrum_ref.db(p[n // 2 + 300]):.2f}" == "-1.42"
    assert f"{spectrum_ref.db(p[n // 2 + 301]):.2f}" == "-1.42"


def test_constant_input():
    log2n = 8
    n = 1 << log2n
    # cs16 zeros: P = 0 everywhere
    p = spectrum_ref.frame_powers(np.zeros(4 * n, np.uint8), 2, log2n)[0]
    assert (spectrum_ref.db(p) == -200.0).all()
    # all-128 cu8 is s_w = 64 (2u - 255 is odd): DC at 20 log10(64 / 16320), its Hann neighbours 6.02 dB lower
    p = spectrum_ref.frame_powers(np.full(2 * n, 128, np.uint8), 0, log2n)[0]
    d = spectrum_ref.db(p)
    assert f"{d[n // 2]:.2f}" == f"{20 * np.log10(64 * (1 + 1j).__abs__() / 16320):.2f}"
    assert abs(d[n // 2 + 1] - (d[n // 2] - 6.0206)) < 1e-3 and abs(d[n // 2 - 1] - (d[n // 2] - 6.0206)) < 1e-3
    assert (d[np.r_[0:n // 2 - 1, n // 2 + 2:n]] == -200.0).all()


def test_white_noise_floor():
    log2n, frames = 10, 400
    n = 1 << log2n
    sigma = 4000.0 / 16320 / np.sqrt(2)   # per component, in units of full scale
    rng = np.random.default_rng(1)
    x = np.round(rng.standard_normal(2 * n * frames) * sigma * 16320 / 128 * 256)   # cs16 at the default gain
    raw = np.clip(x, -32768, 32767).astype("<i2").view(np.uint8)
    p = spectrum_ref.frame_powers(raw, 2, log2n)
    want = 2 * sigma ** 2 * 1.5 / n            # sum w^2 / (sum w)^2 = 1.5 / N for the periodic Hann window
    got = p.mean()
    assert abs(got / want - 1) < 5 / np.sqrt(n * frames / 2)


def test_csv_line():
    n = 64
    p = np.full(n, 1e-3, np.float32)
    p[5] = 0.0
    buf = C.create_string_buffer(8192)
    k = lib().specref_csv_line(buf, 8192, 1_700_000_000, 915_000_000, 10_000_000, 6, 64 * 4096, p.ctypes.data)
    line = buf.value.decode()
    assert k == len(line) and line.endswith("\n")
    f = line.rstrip("\n").split(", ")
    assert f[:6] == ["2023-11-14", "22:13:20", "910000000", "920000000", "156250.00", "262144"]
    assert len(f) == 6 + n and f[6 + 5] == "-200.00" and f[6] == "-30.00"
    # the needed length comes back when the buffer is too small, as snprintf does
    assert lib().specref_csv_line(None, 0, 0, 915_000_000, 10_000_000, 6, 64, p.ctypes.data) == len(
        "1970-01-01, 00:00:00, 910000000, 920000000, 156250.00, 64") + len(line) - len(", ".join(f[:6]))


@pytest.mark.parametrize("args", [["-spectrumbin=1000"], ["-spectrumint=2s"], ["-spectrumpeak"],
                                  ["-spectrum=/nonexistent/dir/out.csv"], ["-spectrum=x.csv", "-spectrumbin=abc"],
                                  ["-spectrum=x.csv", "-spectrumint=fast"]])
def test_cli_usage_errors(tmp_path, args):
    if not os.path.exists(CLI):
        pytest.skip("ertgpu_decode_file is not built")
    args = [a.replace("x.csv", str(tmp_path / "x.csv")) for a in args]
    r = subprocess.run([CLI] + args + [str(tmp_path / "none.cu8")], capture_output=True, text=True, timeout=60)
    assert r.returncode == 2, r.stderr
    assert "spectrum" in r.stderr
