"""CPU tests of the tuned input resampler (ertgpu_set_input_tuning): the mixer table E and the NCO step of
include/ertgpu_resample.h, the tuned plans and their tables, the CPU restatement (tests/cpu_harness/tune_ref.c) the
GPU tests compare the kernel with, the argument checks that need no GPU, and the file receiver's flags."""
import os
import subprocess

import numpy as np
import pytest

from rtlamr_b200 import capi

import resample_ref
import tune_ref
from test_resample import _coefficients, _response_db, _tone, _tone_power_db

DATA_RATE = 32768
RATES = [(2_048_000, 72), (2_400_000, 72), (2_560_000, 72), (2_880_000, 72), (3_200_000, 72), (1_024_000, 72),
         (2_400_000, 32), (3_200_000, 32)]   # test_gpu_resample.RATES
WIDE = [(8_000_000, 72, 256), (10_000_000, 72, 256), (16_000_000, 72, 128), (20_000_000, 72, 64), (8_000_000, 32, 64)]
CLI = os.path.join(tune_ref.ROOT, "rtlamr_b200", "ertgpu_decode_file")


def test_nco_table():
    E = tune_ref.nco_table()
    assert tuple(E[0]) == (16384, 0) and tuple(E[1024]) == (0, 16384)
    k = np.arange(4096)
    C, S = E[:, 0], E[:, 1]
    assert np.array_equal(C[(k + 1024) % 4096], -S) and np.array_equal(S[(k + 1024) % 4096], C)  # quarter turn
    assert np.array_equal(C[(4096 - k) % 4096], C) and np.array_equal(S[(4096 - k) % 4096], -S)  # conjugate
    assert np.array_equal(C[(2048 - k) % 4096], -C) and np.array_equal(S[(2048 - k) % 4096], S)
    mag = C.astype(np.int64) ** 2 + S.astype(np.int64) ** 2
    assert np.max(np.abs(mag - (1 << 28))) <= 1 << 15
    want = np.round(16384 * np.exp(2j * np.pi * k / 4096))
    assert np.max(np.abs(C - want.real)) <= 1 and np.max(np.abs(S - want.imag)) <= 1


def test_nco_step():
    for r in (2_359_296, 8_000_000, 9_437_184, 10_000_000, 20_000_000):
        assert tune_ref.nco_step(0, r) == 0
        for d in (1, 12_345, 200_000, -2_399_845, 3_000_000, r // 3, -(r // 2 - 1)):
            if abs(d) >= r // 2:   # the offset of a channel inside the capture is below Nyquist
                continue
            w, wn = tune_ref.nco_step(d, r), tune_ref.nco_step(-d, r)
            assert (w + wn) % (1 << 32) == 0
            ws = w - (1 << 32) if w >= 1 << 31 else w
            assert abs(ws * r / 2**32 - d) <= r / 2**33, (d, r)
    # 915 MHz capture, 912.6 MHz channel, 8 MS/s: W = round(-2399845 * 2^32 / 8e6)
    assert tune_ref.nco_step(-2_399_845, 8_000_000) == (-round(2_399_845 * 2**32 / 8_000_000)) % (1 << 32)


@pytest.mark.parametrize("rate_in,cl", RATES)
def test_tuned_plan_equals_untuned_in_the_old_range(rate_in, cl):
    rate_out = DATA_RATE * cl
    t = tune_ref.Tuner(rate_in, rate_out, 0)
    r = resample_ref.Resampler(rate_in, rate_out)
    assert t.info == r.info and t.info["P"] == 256
    assert np.array_equal(t.table(), r.table())


@pytest.mark.parametrize("rate_in,cl,P", WIDE)
def test_wide_plans(rate_in, cl, P):
    rate_out = DATA_RATE * cl
    info = tune_ref.plan(rate_in, rate_out, -2_400_000 if rate_in >= 8_000_000 else 0)
    assert info is not None and info["P"] == P and info["T"] <= 224
    assert info["P"] == (256 if info["T"] <= 96 else 128 if info["T"] <= 160 else 64)
    t = tune_ref.Tuner(rate_in, rate_out, -2_400_000)
    table = t.table()
    T, S = info["T"], info["S"]
    tab = table.reshape(P + 1, T).astype(np.int64)
    assert np.array_equal(tab, tab[::-1, ::-1]) and np.all(tab.sum(axis=1) == 1 << S)
    nu = min(rate_in, rate_out) / rate_in
    pas, _ = _response_db(info, table, np.linspace(0, 0.40 * nu, 400))
    assert np.max(np.abs(pas)) <= 0.1, np.max(np.abs(pas))
    stop, _ = _response_db(info, table, np.linspace(0.60 * nu, P / 2, 100_000))
    assert np.max(stop) <= -60.0, np.max(stop)
    phases = np.arange(info["L"]) if info["L"] <= 1 << 16 else np.random.default_rng(1).integers(0, info["L"], 1 << 16)
    c, _ = _coefficients(info, table, phases)
    assert np.max(np.abs(c.sum(axis=1) - (1 << S))) < (1 << S) / 255


def test_p_rule_boundaries_fit_shared_memory():
    """The largest shared memory of any tuned plan (table, one tile's input span and E, as rs_smem_bytes counts it)
    stays within the 227 KiB a CTA may have, across the whole ratio range and at every T boundary of the P rule."""
    rate_out = DATA_RATE * 72
    worst = 0
    for rate_in in np.unique(np.linspace(rate_out // 4, rate_out * 10, 3000).astype(np.int64)):
        info = tune_ref.plan(int(rate_in), rate_out, 0)
        assert info is not None
        T, P, L, M = info["T"], info["P"], info["L"], info["M"]
        span = ((2047 * M + L - 1) // L) + 1 + T + 1
        worst = max(worst, P * T * 6 + span * 4 + 4096 * 4)
    assert worst <= 227 * 1024, worst
    assert tune_ref.plan(rate_out * 10, rate_out, 0) is not None and tune_ref.plan(rate_out * 10 + 1, rate_out, 0) is None
    assert tune_ref.plan(rate_out // 4, rate_out, 0) is not None and tune_ref.plan(rate_out // 4 - 1, rate_out, 0) is None


def test_zero_offset_is_the_untuned_restatement():
    for rate_in, cl in RATES[:4]:
        iq = np.random.default_rng(rate_in).integers(0, 256, 2 * 50_001, dtype=np.uint8)
        assert np.array_equal(tune_ref.tune(iq, rate_in, DATA_RATE * cl, 0), resample_ref.resample(iq, rate_in, DATA_RATE * cl))


@pytest.mark.parametrize("rate_in,off", [(8_000_000, -2_400_000), (10_000_000, 3_000_000), (2_400_000, 200_000)])
def test_tone_is_translated_and_neighbours_rejected(rate_in, off):
    rate_out = DATA_RATE * 72
    lo = min(rate_in, rate_out)
    n = 1 << 18
    win = slice(2 * 4096, 2 * (4096 + (1 << 14)))
    f0 = 0.1 * lo
    out = tune_ref.tune(_tone(n, (off + f0) / rate_in), rate_in, rate_out, off)[win]
    z = out.reshape(-1, 2).astype(np.float64) - 127.5
    spec = np.abs(np.fft.fft((z[:, 0] + 1j * z[:, 1]) * np.hanning(z.shape[0])))
    peak = np.fft.fftfreq(z.shape[0])[np.argmax(spec)]
    assert abs(peak - f0 / rate_out) <= 1.0 / z.shape[0]
    p_ref = _tone_power_db(out, f0 / rate_out)
    for frac in (0.62, 0.8):
        for sign in (1, -1):
            f = off + sign * frac * lo
            if abs(f) >= rate_in / 2:
                continue
            o = tune_ref.tune(_tone(n, f / rate_in), rate_in, rate_out, off)[win]
            f_out = ((sign * frac * lo) / rate_out + 0.5) % 1.0 - 0.5
            assert p_ref - _tone_power_db(o, f_out) >= 50.0, (f, p_ref)


@pytest.mark.parametrize("rate_in,off", [(8_000_000, -2_400_000), (10_000_000, 1_500_000), (20_000_000, 5_000_000)])
def test_dc_spike_is_removed(rate_in, off):
    """A constant input (the capture's DC spike) with |offset| >= 0.6 R_out comes out within +-1 of 127.5."""
    rate_out = DATA_RATE * 72
    assert abs(off) >= 0.6 * rate_out
    T = tune_ref.plan(rate_in, rate_out, off)["T"]
    for u in (0, 37, 200, 255):
        out = tune_ref.tune(np.full(2 * 200_000, u, dtype=np.uint8), rate_in, rate_out, off)
        settled = out[2 * (T + 16):].astype(np.int32)
        assert np.all(np.abs(2 * settled - 255) <= 2), (u, np.unique(settled))


def test_restatement_is_split_invariant():
    rate_in, rate_out, off = 10_000_000, DATA_RATE * 72, -2_400_000
    rng = np.random.default_rng(5)
    iq = rng.integers(0, 256, 2 * 300_007, dtype=np.uint8)
    whole = tune_ref.tune(iq, rate_in, rate_out, off)
    t = tune_ref.Tuner(rate_in, rate_out, off)
    cuts = np.sort(rng.choice(np.arange(1, 300_007), 50, replace=False))
    parts, prev = [], 0
    for c in list(cuts) + [300_007]:
        parts.append(t.feed(iq[2 * prev:2 * c]))
        prev = c
    assert np.array_equal(np.concatenate(parts), whole)


def _handle(msgtype="scm", cl=72):
    h = capi.Handle()
    h.register(capi.stock_protocol(msgtype, cl))
    return h


def _einval(fn, *args):
    with pytest.raises(capi.ErtGpuError) as e:
        fn(*args)
    assert e.value.code == capi.EINVAL


def test_tuning_argument_checks_without_gpu():
    rate_out = DATA_RATE * 72
    h = capi.Handle()
    _einval(h.set_input_tuning, 915_000_000)                 # no protocol yet
    h.register(capi.stock_protocol("scm", 72))
    _einval(h.set_input_tuning, 0)
    _einval(h.set_input_tuning, -915_000_000)
    _einval(h.set_input_tuning, 915_000_000, -1)
    _einval(h.tuning)                                        # not tuned yet
    h.set_input_tuning(915_000_000)
    t = h.tuning()
    assert t["center_hz"] == 912_600_155 and t["offset_hz"] == -2_399_845 and t["nco_bits"] == 12
    _einval(h.register, capi.stock_protocol("idm", 72))      # protocols come before the tuning
    _einval(h.set_input_rate, rate_out * 10 + 1)             # ratio above 10
    _einval(h.set_input_rate, rate_out // 4 - 1)             # below 1/4
    _einval(h.set_input_rate, 4_000_000)                     # channel 2.4 MHz off: outside +-2 MHz
    h.set_input_rate(rate_out * 10)                          # 10:1 is accepted
    assert h.tuning()["nco_step"] == tune_ref.nco_step(-2_399_845, rate_out * 10)
    h.set_input_rate(8_000_000)
    _einval(h.set_input_tuning, 915_000_000)                 # the tuning comes before the rate
    h.close()
    # an untuned handle keeps [1/4, 4]
    h = _handle()
    _einval(h.set_input_rate, rate_out * 4 + 1)
    h.close()
    # a tuned handle at the native rate is checked at allocate (before any device is touched)
    h = _handle()
    h.set_input_tuning(915_000_000)
    _einval(h.allocate)
    h.close()


def _cli(*args, tmp_path):
    f = tmp_path / "in.bin"
    np.zeros(1 << 16, dtype=np.uint8).tofile(f)
    return subprocess.run([CLI, *args, str(f)], capture_output=True, text=True, timeout=60)


def test_cli_usage_errors(tmp_path):
    r = _cli("-centerfreq=912600155", tmp_path=tmp_path)
    assert r.returncode == 2 and "-capturefreq" in r.stderr
    r = _cli("-capturefreq=915000000", "-samplerate=8000000", f"-samplefile={tmp_path / 's.bin'}", tmp_path=tmp_path)
    assert r.returncode == 2 and "-samplefile" in r.stderr
    r = _cli("-capturefreq=-5", tmp_path=tmp_path)
    assert r.returncode == 2
