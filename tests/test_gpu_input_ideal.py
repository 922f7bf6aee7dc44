"""GPU tests (-m gpu) of the input stage's kernels against the float64 model of tests/ideal_ref.py: a seeded subset of
the CPU sweep (tests/test_input_ideal_cpu.py) in every mode, at its edges and in cu8, cs8, cs16, cf32 and a big-endian
SigMF format, decoded through the C ABI.  Every block of ERTGPU_TAP_RESAMPLED is compared sample by sample with the
model under the plan's error budget, and byte for byte with the composed restatement (combo_ref.decoder_bytes).  A
decimating channel group holds decimate_channels_kernel to the model too."""
import numpy as np
import pytest

import combo_ref
import ideal_ref as ir
import test_input_ideal_cpu as cpu
import wide_ref
from rtlamr_b200 import capi
from test_sigmf import convert, encode

pytestmark = pytest.mark.gpu

FORMATS = [capi.FORMAT_CU8, capi.FORMAT_CS8, capi.FORMAT_CS16, capi.FORMAT_CF32, capi.FORMAT_CS16BE]
WIDE_FORMATS = [capi.FORMAT_CS16, capi.FORMAT_CF32, capi.FORMAT_CS16BE]
COMBO_MODE = {"untuned": "resample", "tuned": "tuned", "decimating": "decimate", "wide": "wide", "wide_dec": "wide_dec"}
MAX_OUTPUTS = 250_000       # model outputs per plan


def _plans():
    """About 40 plans: per mode the first edges of the sweep (every chip length) and seeded draws from the rest."""
    rng = np.random.default_rng(0x6B1)
    out = []
    for mode in cpu.MODES:
        sw = cpu.sweep(mode)
        n_edges = len(cpu.edge_rates(mode, cpu.DATA_RATE * 72)) * len(cpu.CHIP_LENGTHS)
        picks = sorted(set(rng.choice(n_edges, 5, replace=False).tolist())
                       | set((n_edges + rng.choice(len(sw) - n_edges, 3, replace=False)).tolist()))
        out += [sw[i] for i in picks]
    return out


PLANS = _plans()


def _raw(plan, mp, fmt, z):
    """Capture bytes of z (in the path's units) in fmt, and the model's input s from those bytes."""
    if mp["k"] is None:
        raw = encode(cpu.narrow_bytes(z), fmt)
        return raw, cpu.s_of_bytes(convert(raw, fmt))
    iq = np.empty(2 * z.size)
    iq[0::2], iq[1::2] = z.real, z.imag
    if fmt == capi.FORMAT_CF32:
        raw = (iq / 2.0 ** 14).astype("<f4").view(np.uint8)    # g = 2^7: s_w = x 2^14
    else:
        v = np.clip(np.round(2 * iq), -32768, 32767)            # g = 2^-8: s_w = x / 2
        raw = v.astype(">i2" if fmt == capi.FORMAT_CS16BE else "<i2").view(np.uint8)
    sw = wide_ref.wide_components(raw, fmt)
    return raw, sw[0::2] + 1j * sw[1::2].astype(np.float64)


def _cfg(plan, fmt):
    """The combo_ref configuration fields decoder_bytes reads."""
    return {"fmt": fmt, "scale": 0.0, "mode": COMBO_MODE[plan["mode"]], "rate_in": plan["rate_in"], "cl": plan["cl"],
            "offsets": [plan["offset"] or 0], "allow_decimation": plan["mode"] in ("decimating", "wide_dec")}


def _blocks_after(h, mp, x):
    """Whole decoder blocks once x input samples are in."""
    return ir.out_end(mp, ir.stage1_outputs(mp, x) if mp["D"] > 1 else x) // h.cfg.block_size


def _taps(h, mp, calls):
    """Run calls [(end sample, fn)] in order and read each call's new blocks of ERTGPU_TAP_RESAMPLED after it."""
    out, done = [], 0
    for end, fn in calls:
        fn()
        nb = _blocks_after(h, mp, end)
        out += [h.tap(capi.TAP_RESAMPLED, b) for b in range(done, nb)]
        done = nb
    return np.concatenate(out) if out else np.zeros(0, np.uint8)


def _compare(got, plan, mp, fmt, raw, s, x_in):
    """The decoded blocks: equal to the restatement's bytes, and within the budget of the model."""
    want = combo_ref.decoder_bytes(_cfg(plan, fmt), raw, 0, mp["k"])
    assert got.size >= 2 * 3 * 4096, (plan, got.size)
    combo_ref.assert_bytes(got, want[:got.size], str(plan))
    m = ir.model(mp, s, x_in)[:got.size]
    err = ir.errors(got, m, ir.centre(mp), ir.single_tap(mp, got.size // 2))
    b = ir.budget(mp, s, x_in)
    assert not ir.failures(err, b), (plan, fmt, err, b, ir.failures(err, b))
    print(f"\nIDEAL {plan['mode']} rate_in={plan['rate_in']} offset={plan['offset']} k={plan['k']} fmt={fmt} "
          f"outputs={got.size // 2} max={err['max']:.4f} budget={b['total']:.4f}")
    return err, b


def _input(plan, mp, fmt):
    """The plan's input: MAX_OUTPUTS outputs' worth, at least four decoder blocks of 16384 samples, at most 2^23
    samples (32 MiB of cs16)."""
    ratio = plan["rate_in"] / (cpu.DATA_RATE * plan["cl"])
    x_in = min(1 << 23, max(int(MAX_OUTPUTS * ratio), int(4 * 16384 * ratio) + mp["D"] * mp["T1"] + 4 * mp["T"]))
    z = cpu.channel(plan, x_in, np.random.default_rng(plan["seed"]), cpu.amplitude_of(mp))
    raw, s = _raw(plan, mp, fmt, z)
    return raw, s, x_in


@pytest.mark.parametrize("i", range(len(PLANS)))
def test_kernels_against_the_model(built, i):
    """One device call of the whole input (up to 32 MiB); every eighth plan through the host path in three calls."""
    import torch
    plan = PLANS[i]
    fmts = WIDE_FORMATS if plan["k"] is not None else FORMATS
    fmt = fmts[i % len(fmts)]
    h = cpu.handle(plan, fmt)
    mp = ir.plan_from_handle(h, plan["k"])
    h.allocate(0)
    raw, s, x_in = _input(plan, mp, fmt)
    sb = capi.FORMAT_BYTES[fmt]
    if i % 8 == 0:   # the host path in three calls, one of them 4097 samples
        cuts = [0, x_in // 3, x_in // 3 + 4097, x_in]
        calls = [(b, lambda a=a, b=b: h.decode(raw[sb * a:sb * b], cap=1 << 16)) for a, b in zip(cuts, cuts[1:])]
    else:
        d = torch.from_numpy(raw).cuda()

        def device_call():
            h.decode_device_async(d.data_ptr(), d.numel(), 0, torch.cuda.current_stream().cuda_stream)
            h.fetch(cap=1 << 16)
        calls = [(x_in, device_call)]
    _compare(_taps(h, mp, calls), plan, mp, fmt, raw, s, x_in)
    h.close()


def test_channel_group_against_the_model(built):
    """Three decimating channels of one cs16 capture through ertgpu_decode_channels (decimate_channels_kernel)."""
    rate_in, cl, fmt = 30_720_000, 72, capi.FORMAT_CS16
    offs = (-2_400_000, 1_000_000, 6_000_000)
    plans = [{"mode": "decimating", "i": -1, "cl": cl, "rate_in": rate_in, "offset": o, "k": None, "seed": 5} for o in offs]
    hs = [cpu.handle(p, fmt) for p in plans]
    mps = [ir.plan_from_handle(h) for h in hs]
    assert all(m["D"] == 4 for m in mps)
    for h in hs:
        h.allocate(0)
    x_in = 1 << 20
    rng = np.random.default_rng(11)
    z = sum(cpu.channel(p, x_in, rng, 30.0) for p in plans)
    raw, s = _raw(plans[0], mps[0], fmt, z)
    capi.decode_channels(hs, raw, cap=1 << 16)
    assert "decimate_channels_kernel" in hs[0].last_kernels()
    for h, p, mp in zip(hs, plans, mps):
        _compare(_taps(h, mp, [(x_in, lambda: None)]), p, mp, fmt, raw, s, x_in)
        h.close()
