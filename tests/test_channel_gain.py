"""CPU tests of the wide channel path (ertgpu_set_channel_gain, include/ertgpu_resample.h) through its restatement
(tests/cpu_harness/wide_ref.c, tests/wide_ref.py): the overflow bounds over the plan sweeps, the wide component of
every format, constants, passband gain, the channel gain's scaling, the auto rule and split invariance."""
import numpy as np
import pytest

from rtlamr_b200 import capi

import decimate_ref
import tune_ref
import wide_ref
from test_gpu_decimate import ALL_FORMATS

DATA_RATE = 32768
R72, R32, R8 = DATA_RATE * 72, DATA_RATE * 32, DATA_RATE * 8
S_MAX = 23170            # |s'| after the mixer (header)
I32 = 2 ** 31


def test_mixer_bound():
    e = tune_ref.nco_table()
    worst = int((np.abs(e[:, 0]) + np.abs(e[:, 1])).max())
    assert worst == 23171
    assert max(abs((sg * 16383 * worst + (1 << 13)) >> 14) for sg in (1, -1)) == S_MAX
    assert tuple(e[0]) == (1 << 14, 0)   # stage 2 at W = 0 mixes s to itself


def _table_l1(table, T, P):
    """sum_t max(|table[p][t]|, |table[p+1][t]|) + 2T over every row pair: a bound of sum_t |c_t| + |delta|."""
    t = np.abs(table.reshape(P + 1, T).astype(np.int64))
    return int((np.maximum(t[:-1], t[1:]).sum(axis=1)).max()) + 2 * T


def test_accumulator_bounds_over_the_plan_sweeps():
    """(taps' L1 bound) * max |s'| < 2^31 for every plan of the tuned sweep (1/10 ... 4) and of the decimated sweep
    (10 ... 256), stage-1 taps included (folded pairs are bounded by the same |h| (|x0| + |x1|))."""
    worst = 0
    for rate_out in (R72, R32, R8):
        for rate_in in np.unique(np.linspace(rate_out // 4, rate_out * 10, 160).astype(np.int64)):
            w = wide_ref.Wide(int(rate_in), rate_out, 0)
            worst = max(worst, _table_l1(w.table(), w.info["T"], w.info["P"]))
        for rate_in in np.unique(np.linspace(10 * rate_out + 1, 256 * rate_out, 160).astype(np.int64)):
            w = wide_ref.Wide(int(rate_in), rate_out, 0)
            assert w.dec["D"] >= 2
            worst = max(worst, _table_l1(w.table(), w.info["T"], w.info["P"]), int(np.abs(w.taps().astype(np.int64)).sum()))
    assert worst * S_MAX < I32, worst


@pytest.mark.parametrize("rate_in,rate_out,off", [(R72, R72, 0), (10_000_000, R72, 1_500_000), (61_440_000, R72, -12_000_000),
                                                  (256 * R8, R8, 30_000_000)])
def test_full_scale_infinities_and_nan_stay_in_int32(rate_in, rate_out, off):
    """Input at +-full scale in the worst sign pattern for the centre taps, with +-inf and NaN: every accumulator of
    every stage fits int32, and NaN reads as 0."""
    rng = np.random.default_rng(rate_in)
    n = 40_000
    x = np.where(rng.integers(0, 2, 2 * n) > 0, np.float32(np.inf), np.float32(-np.inf))
    x[rng.integers(0, 2 * n, n // 4)] = np.nan
    x[: 2000] = np.float32(1.0)
    raw = x.astype("<f4").view(np.uint8)
    sw = wide_ref.wide_components(raw, capi.FORMAT_CF32)
    assert np.all(sw[np.isnan(x)] == 0) and np.abs(sw).max() == 16383
    w = wide_ref.Wide(rate_in, rate_out, off)
    w.feed(sw)
    assert 0 < w.max_acc() < I32


def test_wide_components_of_every_format():
    """cu8 is exactly 64 (2u - 255); every other format rint(x g 2^7) clamped to +-16383, its default g mapping full
    scale to full scale; NaN 0 and infinities clamp."""
    u = np.arange(256, dtype=np.uint8)
    assert np.array_equal(wide_ref.wide_components(u, capi.FORMAT_CU8), 64 * (2 * u.astype(np.int32) - 255))
    cs16 = np.array([0, 1, -1, 2, 127, -128, 32767, -32768, 12345, -257], dtype="<i2")
    assert np.array_equal(wide_ref.wide_components(cs16.view(np.uint8), capi.FORMAT_CS16),
                          np.clip(np.rint(cs16.astype(np.float64) / 2), -16383, 16383))
    f = np.array([0.5, -0.5, 1 / 256, 3 / 512, np.nan, np.inf, -np.inf, 200.0], dtype="<f4")
    assert list(wide_ref.wide_components(f.view(np.uint8), capi.FORMAT_CF32)) == [8192, -8192, 64, 96, 0, 16383, -16383, 16383]
    from test_sigmf import encode
    for fmt in ALL_FORMATS:   # a byte encoded at the default scale comes back as 128 (u - 128), -128 clamped
        raw = encode(u, fmt)
        want = 64 * (2 * u.astype(np.int32) - 255) if fmt == capi.FORMAT_CU8 else \
            np.clip(128 * (u.astype(np.int32) - 128), -16383, 16383)
        assert np.array_equal(wide_ref.wide_components(raw, fmt), want), fmt


@pytest.mark.parametrize("rate_in,off", [(R72, 0), (10_000_000, 0), (30_720_000, 0)])
@pytest.mark.parametrize("k", [0, 3, 7])
def test_constant_input_comes_out_as_the_constant(rate_in, off, k):
    """A constant s = 128 v (v in byte units) comes out as v 2^k + 128 once the filter has settled; cu8 u as u at k = 0."""
    for v in (-3, 0, 1, 5):
        sw = np.tile(np.array([128 * v, -128 * v], dtype=np.int32), 200_000)
        out, acc = wide_ref.Wide(rate_in, R72, off, k).feed(sw)
        tail = out[-2000:].astype(np.int32) - 128
        assert np.all(tail[0::2] == np.clip(v << k, -128, 127)) and np.all(tail[1::2] == np.clip(-v << k, -128, 127))
    for u in (0, 77, 127, 128, 255):
        sw = wide_ref.wide_components(np.full(400_000, u, dtype=np.uint8), capi.FORMAT_CU8)
        out, _ = wide_ref.Wide(rate_in, R72, off, 0).feed(sw)
        assert np.all(out[-2000:] == u)


def _tone_sw(n, f_cyc, amp, seed=1, noise=0.5):
    rng = np.random.default_rng(seed)
    z = amp * np.exp(2j * np.pi * f_cyc * np.arange(n)) + noise * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    sw = np.empty(2 * n, dtype=np.int32)
    sw[0::2], sw[1::2] = np.rint(128 * z.real), np.rint(128 * z.imag)
    return sw


def _db(out, k=None):
    z = (out.reshape(-1, 2).astype(np.float64) - 127.5) @ np.array([1, 1j])
    z = z[64:] - z[64:].mean()
    w = np.hanning(z.size)
    spec = np.abs(np.fft.fft(z * w)) ** 2
    k = int(np.argmax(spec)) if k is None else k
    return 10 * np.log10(spec[np.arange(k - 4, k + 5) % z.size].sum() / (w ** 2).sum() / z.size)


@pytest.mark.parametrize("rate_in,rate_out,off", [(R72, R72, 0), (10_000_000, R72, 2_000_000), (30_720_000, R72, -2_400_000),
                                                  (61_440_000, R72, 5_000_000), (20_000_000, R32, -2_400_000)])
def test_passband_tones_within_half_a_db(rate_in, rate_out, off):
    """A tone of amplitude A anywhere in +-0.35 R_out of the channel comes out at A 2^k within +-0.5 dB."""
    amp, k = 12.0, 3
    n_out = 1 << 15
    n = (n_out + 256) * rate_in // rate_out + 4096
    for f in (-0.35, -0.1, 0.02, 0.2, 0.35):
        out, _ = wide_ref.Wide(rate_in, rate_out, off, k).feed(_tone_sw(n, (off + f * rate_out) / rate_in, amp))
        got = _db(out[: 2 * n_out])
        assert abs(got - 20 * np.log10(amp * 2 ** k)) < 0.5, (f, got)


@pytest.mark.parametrize("rate_in,off", [(10_000_000, 1_000_000), (61_440_000, -7_000_000)])
def test_gain_scales_the_accumulators_output(rate_in, off):
    """The accumulators do not depend on k, and the bytes at k are the bytes at 0 scaled by 2^k (to the rounding of
    each) wherever nothing clips."""
    sw = _tone_sw(400_000, off / rate_in + 0.01, 3.0, noise=1.0)
    out0, acc0 = wide_ref.Wide(rate_in, R72, off, 0).feed(sw)
    for k in (1, 4, 5):
        out, acc = wide_ref.Wide(rate_in, R72, off, k).feed(sw)
        assert np.array_equal(acc, acc0)
        v0, v = out0.astype(np.int64) - 128, out.astype(np.int64) - 128
        ok = (v > -128) & (v < 127)
        assert ok.mean() > 0.9
        assert np.all(np.abs(v[ok] - (v0[ok] << k)) <= (1 << (k - 1)) + 1)
        exact = np.floor(acc.astype(np.float64) * 2.0 ** k / 2 ** 21 + 0.5 - 2.0 ** -40)   # half down
        assert np.array_equal(v, np.clip(exact, -128, 127).astype(np.int64))


def test_auto_rule_against_numpy():
    rng = np.random.default_rng(7)
    L = wide_ref.lib()
    for trial in range(400):
        bins = np.zeros(32, dtype=np.int64)
        top = int(rng.integers(0, 32))
        bins[: top + 1] = rng.integers(0, 1 << int(rng.integers(1, 20)), top + 1)
        if trial % 7 == 0:
            bins[:] = 0
        comps = int(bins.sum() + rng.integers(0, 1 << 20))
        want = wide_ref.channel_gain(bins, comps)
        assert L.wideref_channel_gain(bins.ctypes.data, comps) == want
        if bins.sum():   # the rule's definition: largest k whose clipping count is within the allowance
            over = [int(bins[28 - k:].sum()) for k in range(15)]
            ok = [k for k in range(15) if over[k] <= comps >> 16]
            assert want == (max(ok) if ok else 0)
        else:
            assert want == 0
    acc = np.array([0, 1, -1, 2, 3, 4, 2 ** 20 - 1, 2 ** 20, -(2 ** 30), 2 ** 31 - 1], dtype=np.int32)
    lv = wide_ref.level(acc)
    assert lv["zeros"] == 1 and lv["components"] == 10
    assert list(np.nonzero(lv["bins"])[0]) == [0, 1, 2, 19, 20, 30]
    assert lv["bins"][0] == 2 and lv["bins"][30] == 2


@pytest.mark.parametrize("rate_in,off", [(10_000_000, 1_500_000), (30_720_000, -2_400_000)])
def test_restatement_is_split_invariant(rate_in, off):
    rng = np.random.default_rng(rate_in)
    n = 300_007
    sw = rng.integers(-16383, 16384, 2 * n).astype(np.int32)
    whole, acc = wide_ref.Wide(rate_in, R72, off, 4).feed(sw)
    cuts = np.concatenate([[0], np.sort(rng.choice(np.arange(1, n), 60, replace=False)), [n]])
    w = wide_ref.Wide(rate_in, R72, off, 4)
    parts = [w.feed(sw[2 * a:2 * b]) for a, b in zip(cuts[:-1], cuts[1:])]
    assert np.array_equal(np.concatenate([p[0] for p in parts]), whole)
    assert np.array_equal(np.concatenate([p[1] for p in parts]), acc)


def test_one_stage_plan_and_cascade_stage_two():
    """At R_in = R_out and offset 0 the wide path filters with L = M = 1, T = 22; above 10:1 its second stage is the
    decimated plan's."""
    w = wide_ref.Wide(R72, R72, 0)
    assert (w.info["L"], w.info["M"], w.info["T"], w.dec["D"]) == (1, 1, 22, 1)
    w = wide_ref.Wide(61_440_000, R72, 0)
    dec, info = decimate_ref.plan(61_440_000, R72, 0)
    assert w.dec == dec and w.info == info


def test_channel_gain_argument_checks_without_gpu(built):
    h = capi.Handle()
    h.register(capi.stock_protocol("scm", 72))
    with pytest.raises(capi.ErtGpuError) as e:   # untuned
        h.set_channel_gain(2)
    assert e.value.code == capi.EINVAL and "untuned" in str(e.value)
    with pytest.raises(capi.ErtGpuError):
        h.channel_gain()
    h.set_input_tuning(915_000_000, 915_000_000)
    for k in (-1, 15):
        with pytest.raises(capi.ErtGpuError) as e:
            h.set_channel_gain(k)
        assert "0 ... 14" in str(e.value)
    h.set_channel_gain(9)
    assert h.channel_gain() == 9
    with pytest.raises(capi.ErtGpuError):   # not allocated
        h.measure_channel(np.zeros(64, np.uint8))
    h.close()
