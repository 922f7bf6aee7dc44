"""GPU tests (-m gpu) of the wide channel path (ertgpu_set_channel_gain): resample_wide_kernel<F>, and
decimate_wide_kernel<F> into resample_wide_kernel<mid16>, against the CPU restatement (tests/cpu_harness/wide_ref.c) byte
for byte in every block, every format, several rates and gains; candidates against the oracle on the restatement's
bytes; groups of channels against lone handles; call splits on the host and device paths and reset; the channel
measurement against the numpy histogram of the restatement's accumulators; and the rules of the C ABI."""
import numpy as np
import pytest

import oracle
from rtlamr_b200 import capi

import tune_ref
import wide_ref
from test_gpu_decimate import ALL_FORMATS, _raw
from test_gpu_resample import _cuts, keys, tap_resampled
from test_sigmf import NAME

pytestmark = pytest.mark.gpu

DATA_RATE = 32768
CAPTURE = 915_000_000


def _decoder(rate_in, off, fmt, k, cl=72, msgtypes="scm", **kw):
    return capi.new_decoder(msgtypes, cl, input_rate=rate_in, input_format=fmt, capture_freq=CAPTURE,
                            center_freq=CAPTURE + off, channel_gain=k, **kw)


def _capture(rate_in, off, fmt, nblocks=12, cl=72, seed=11, amp=1.0):
    """raw bytes of about nblocks decoder blocks: scm packets in the channel and beside it, over noise."""
    n = nblocks * -(-rate_in // (DATA_RATE * cl)) * (16384 * cl // 72)
    z, _ = tune_ref.wideband([("scm", off, seed, 0), ("scm", off + 700_000 if rate_in > 4_000_000 else 0, seed + 1, 40_000)],
                             rate_in, n, seed, noise=3.0)
    return _raw(z * amp, fmt)


def _check(h, ref, cl):
    """Every block's ERTGPU_TAP_RESAMPLED bytes equal the restatement's; returns the number of blocks."""
    bs = h.cfg.block_size
    nblocks = (ref.size // 2) // bs
    assert nblocks > 4
    assert np.array_equal(tap_resampled(h, 0, nblocks), ref[:2 * nblocks * bs])
    return nblocks


def _oracle_keys(msgtype, cl, ref, nblocks, bs2):
    o = oracle.Oracle(msgtype, cl, oracle.SEARCH_GO)
    cands, _ = o.decode(ref[:nblocks * bs2])
    return sorted((c.block, c.preamble_id, c.idx, c.data[:12]) for c in cands)


def _keys12(rows):
    return sorted((int(r["block"]), int(r["preamble_id"]), int(r["idx"]), r["bytes"][:12].tobytes()) for r in rows)


R72 = DATA_RATE * 72
CASES = [(R72, 72, capi.FORMAT_CS16, 0, 2), (8_000_000, 72, capi.FORMAT_CS16, -2_000_000, 3),
         (10_000_000, 72, capi.FORMAT_CS16, 1_500_000, 5), (10_000_000, 72, capi.FORMAT_CS8, -1_000_000, 0),
         (20_000_000, 72, capi.FORMAT_CF32, 3_000_000, 4), (20_000_000, 32, capi.FORMAT_CS16, -2_400_000, 1),
         (30_720_000, 72, capi.FORMAT_CS16, -2_400_000, 6), (61_440_000, 72, capi.FORMAT_CS16, 5_000_000, 2),
         (61_440_000, 72, capi.FORMAT_CF32, -12_000_000, 8)]


@pytest.mark.parametrize("rate_in,cl,fmt,off,k", CASES)
def test_kernel_equals_cpu_restatement_and_oracle(built, rate_in, cl, fmt, off, k):
    raw = _capture(rate_in, off, fmt, cl=cl)
    ref, _ = wide_ref.wide(raw, fmt, rate_in, DATA_RATE * cl, off, k)
    h = _decoder(rate_in, off, fmt, k, cl=cl)
    assert h.channel_gain() == k
    rows = h.decode(raw, cap=1 << 16)
    D = wide_ref.Wide(rate_in, DATA_RATE * cl, off).dec["D"]
    want = [f"decimate_kernel<{NAME[fmt]},wide>", "resample_kernel<mid16,tuned,wide>"] if D > 1 else \
        [f"resample_kernel<{NAME[fmt]},tuned,wide>"]
    assert h.last_kernels().split(";")[-len(want):] == want
    nblocks = _check(h, ref, cl)
    assert _keys12(rows) == _oracle_keys("scm", cl, ref, nblocks, h.cfg.block_size2)
    h.close()


@pytest.mark.parametrize("fmt", ALL_FORMATS)
@pytest.mark.parametrize("rate_in,off,k", [(10_000_000, 1_500_000, 3), (30_720_000, -2_400_000, 5)])
def test_every_format(built, fmt, rate_in, off, k):
    raw = _capture(rate_in, off, fmt, nblocks=6, seed=fmt + 3)
    ref, _ = wide_ref.wide(raw, fmt, rate_in, R72, off, k)
    h = _decoder(rate_in, off, fmt, k)
    h.decode(raw, cap=1 << 16)
    _check(h, ref, 72)
    h.close()


@pytest.mark.parametrize("nch", [1, 3, 8])
def test_a_wide_group_equals_lone_wide_handles(built, nch):
    rate_in, fmt = 30_720_000, capi.FORMAT_CS16
    offs = [int(o) for o in np.linspace(-9_000_000, 9_000_000, nch)] if nch > 1 else [-2_400_000]
    raw = _capture(rate_in, offs[0], fmt, nblocks=8)
    group = [_decoder(rate_in, o, fmt, i % 7) for i, o in enumerate(offs)]
    got = capi.decode_channels(group, raw, cap=1 << 16)
    assert group[0].last_kernels().split(";")[-2:] == ["decimate_kernel<cs16,wide>", "resample_kernel<mid16,tuned,wide>"]
    for i, (o, hg, rows) in enumerate(zip(offs, group, got)):
        lone = _decoder(rate_in, o, fmt, i % 7)
        want = lone.decode(raw, cap=1 << 16)
        assert keys(rows) == keys(want)
        ref, _ = wide_ref.wide(raw, fmt, rate_in, R72, o, i % 7)
        nb = _check(hg, ref, 72)
        assert np.array_equal(tap_resampled(hg, 0, nb), tap_resampled(lone, 0, nb))
        lone.close()
    for h in group:
        h.close()


def test_a_mixed_group_is_rejected(built):
    rate_in, fmt = 30_720_000, capi.FORMAT_CS16
    a = _decoder(rate_in, -2_000_000, fmt, 3)
    b = capi.new_decoder("scm", 72, input_rate=rate_in, input_format=fmt, capture_freq=CAPTURE,
                         center_freq=CAPTURE + 2_000_000)
    with pytest.raises(capi.ErtGpuError) as e:
        capi.decode_channels([a, b], np.zeros(4 * 100_000, np.uint8))
    assert e.value.code == capi.EINVAL and "wide channel path" in str(e.value)
    with pytest.raises(capi.ErtGpuError) as e:   # allocated without the wide path
        b.set_channel_gain(2)
    assert "allocated without" in str(e.value)
    a.close()
    b.close()


@pytest.mark.parametrize("rate_in,fmt,off", [(61_440_000, capi.FORMAT_CS16, -2_400_000),
                                             (10_000_000, capi.FORMAT_CS8, 3_000_000)])
def test_call_splits_host_and_device_and_reset(built, rate_in, fmt, off):
    import torch
    s = capi.FORMAT_BYTES[fmt]
    k = 4
    raw = _capture(rate_in, off, fmt, nblocks=10, seed=31)
    ref, _ = wide_ref.wide(raw, fmt, rate_in, R72, off, k)
    whole = _decoder(rate_in, off, fmt, k)
    want = keys(whole.decode(raw, cap=1 << 16))
    nb = _check(whole, ref, 72)
    rng = np.random.default_rng(rate_in)
    sizes = [s * (c // 2) for c in _cuts(rng, raw.size // s * 2, 30)]
    sizes[-1] += raw.size - sum(sizes)
    for path in ("host", "device"):
        h = _decoder(rate_in, off, fmt, k)
        rows, o = [], 0
        for c in sizes:
            part = raw[o:o + c]
            o += c
            if path == "host":
                rows.extend(h.decode(part, cap=1 << 16))
            else:
                d = torch.from_numpy(part.copy()).cuda()
                h.decode_device_async(d.data_ptr(), d.numel(), 0, torch.cuda.current_stream().cuda_stream)
                rows.extend(h.fetch(cap=1 << 16))
                del d
        assert keys(rows) == want, path
        with pytest.raises(capi.ErtGpuError):   # k changes only at a stream start
            h.set_channel_gain(k + 1)
        h.reset()
        h.set_channel_gain(k)
        again = h.decode(raw, cap=1 << 16)
        assert keys(again) == want
        assert np.array_equal(tap_resampled(h, 0, nb), ref[:2 * nb * h.cfg.block_size])
        h.close()
    whole.close()


@pytest.mark.parametrize("rate_in,fmt,off", [(10_000_000, capi.FORMAT_CS16, 1_500_000),
                                             (61_440_000, capi.FORMAT_CF32, -7_000_000), (R72, capi.FORMAT_CU8, 0)])
def test_measure_channel_is_the_restatements_histogram_and_leaves_the_stream(built, rate_in, fmt, off):
    raw = _capture(rate_in, off, fmt, nblocks=8, seed=5, amp=0.05)
    s = capi.FORMAT_BYTES[fmt]
    n = raw.size // s
    win = raw[: s * (n * 3 // 5)]
    _, acc = wide_ref.wide(win, fmt, rate_in, R72, off, 0)
    lv = wide_ref.level(acc)
    h = _decoder(rate_in, off, fmt, 0)
    got = h.measure_channel(win)
    assert got["components"] == lv["components"] and got["zeros"] == lv["zeros"]
    assert np.array_equal(got["bins"], lv["bins"]) and got["k"] == lv["k"] > 0
    # measured mid-stream, nothing of the stream changes; k applied at a stream start equals the explicit gain
    half = s * (n // 2)
    r1 = h.decode(raw[:half], cap=1 << 16)
    assert h.measure_channel(win)["bins"].tolist() == got["bins"].tolist()
    r2 = h.decode(raw[half:], cap=1 << 16)
    plain = _decoder(rate_in, off, fmt, 0)
    assert keys(list(r1) + list(r2)) == keys(plain.decode(raw, cap=1 << 16))
    h.reset()
    h.set_channel_gain(got["k"])
    ref, _ = wide_ref.wide(raw, fmt, rate_in, R72, off, got["k"])
    h.decode(raw, cap=1 << 16)
    _check(h, ref, 72)
    for x in (h, plain):
        x.close()
