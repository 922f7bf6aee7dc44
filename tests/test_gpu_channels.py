"""GPU tests (-m gpu) of several channels of one capture in one pass (ertgpu_decode_channels): every handle of a group
equals a lone handle tuned to its channel and fed the same bytes (candidates, ERTGPU_TAP_RESAMPLED bytes, the kernels
from stage 2 on), across formats, rates with and without a decimating first stage, group sizes, call splits and input
paths; packets in five channels are each found in their own channel only; every rule of a group is enforced; and the
file receiver's -centerfreq list prints the single-channel runs merged by the cross-channel dedup."""
import os
import subprocess

import numpy as np
import pytest

from rtlamr_b200 import capi

import decimate_ref
import tune_ref
from test_gpu_resample import _cuts, keys, out_end, tap_resampled
from test_sigmf import encode

pytestmark = pytest.mark.gpu

DATA_RATE = 32768
CAPTURE = 915_000_000
CLI = os.path.join(tune_ref.ROOT, "rtlamr_b200", "ertgpu_decode_file")
SPREAD = {8_000_000: 2_800_000, 30_720_000: 12_000_000, 61_440_000: 25_000_000}   # |offset| that fits the capture


def _offsets(rate_in, n):
    w = SPREAD[rate_in]
    return [int(o) + 7 * k for k, o in enumerate(np.linspace(-w, w, n) if n > 1 else [-2_400_000])]


def _decoder(rate_in, off, fmt, msgtypes="scm", cl=72, **kw):
    return capi.new_decoder(msgtypes, cl, input_rate=rate_in, input_format=fmt, capture_freq=CAPTURE,
                            center_freq=CAPTURE + off, **kw)


def _blocks(h, nsamples):
    """Whole output blocks of h once nsamples input samples are in."""
    dec, _ = h.decimator()
    info, _ = h.resampler()
    x = nsamples
    if dec["D"] > 1:
        a = x - dec["T1"] // 2
        x = -(-a // dec["D"]) if a > 0 else 0
    return out_end(info, x) // h.cfg.block_size


def _stage2_on(kernels):
    return kernels.replace("decimate_channels_kernel<", "decimate_kernel<")


@pytest.mark.parametrize("n", [1, 3, 8])
@pytest.mark.parametrize("rate_in", [8_000_000, 30_720_000, 61_440_000])
@pytest.mark.parametrize("fmt", [capi.FORMAT_CU8, capi.FORMAT_CS8, capi.FORMAT_CS16, capi.FORMAT_CF32])
def test_each_channel_equals_a_lone_handle(built, fmt, rate_in, n):
    nsamples = 10 * (rate_in // (DATA_RATE * 72) + 1) * 16384
    raw = encode(np.random.default_rng(rate_in ^ fmt ^ n).integers(0, 256, 2 * nsamples, dtype=np.uint8), fmt)
    offs = _offsets(rate_in, n)
    group = [_decoder(rate_in, o, fmt) for o in offs]
    got = capi.decode_channels(group, raw, 0, 1 << 16)
    D = group[0].decimator()[0]["D"]
    assert (D > 1) == (rate_in > 10 * DATA_RATE * 72)
    for h, o, rows in zip(group, offs, got):
        lone = _decoder(rate_in, o, fmt)
        want = lone.decode(raw, 0, 1 << 16)
        assert rows.tobytes() == want.tobytes(), o
        ks = h.last_kernels()
        assert ("decimate_channels_kernel<" in ks) == (D > 1 and n > 1), ks
        assert _stage2_on(ks) == lone.last_kernels()
        nb = _blocks(h, nsamples)
        assert nb > 4 and np.array_equal(tap_resampled(h, 0, nb), tap_resampled(lone, 0, nb)), o
        lone.close()
    for h in group:
        h.close()


@pytest.mark.parametrize("rate_in,fmt,n", [(61_440_000, capi.FORMAT_CS16, 4), (30_720_000, capi.FORMAT_CS8, 3),
                                           (8_000_000, capi.FORMAT_CS8, 3)])
def test_call_splits_input_paths_and_reset(built, rate_in, fmt, n):
    import torch
    s = capi.FORMAT_BYTES[fmt]
    offs = _offsets(rate_in, n)
    z, _ = decimate_ref.wideband([("scm", o, 41 + i, 9_000 * i) for i, o in enumerate(offs)], rate_in, 6_000_001, 41,
                                 spacing=1 << 20)
    raw = tune_ref.quantize(z, fmt)
    want, lones = [], []
    for o in offs:   # each lone handle's whole stream is in its last call: every block can be tapped
        lones.append(_decoder(rate_in, o, fmt))
        want.append(keys(lones[-1].decode(raw, cap=1 << 16)))
    assert any(want)
    rng = np.random.default_rng(rate_in + n)
    sizes = [s * (c // 2) for c in _cuts(rng, raw.size // s * 2, 30)]
    sizes[-1] += raw.size - sum(sizes)
    pinned = torch.empty(raw.size, dtype=torch.uint8).pin_memory()
    pinned.numpy()[:] = raw
    for path in ("pageable", "pinned", "device", "mixed"):
        group = [_decoder(rate_in, o, fmt) for o in offs]
        rows = [[] for _ in offs]
        o, done = 0, [0] * n
        for i, c in enumerate(sizes):
            p = path if path != "mixed" else ("pageable", "pinned", "device")[i % 3]
            if p == "pageable":
                got = capi.decode_channels(group, raw[o:o + c], cap=1 << 16)
            elif p == "pinned":
                got = capi.decode_channels(group, (pinned.data_ptr() + o, c), cap=1 << 16)
            else:
                d = torch.from_numpy(raw[o:o + c].copy()).cuda()
                capi.decode_channels_device_async(group, d.data_ptr(), c, 0, torch.cuda.current_stream().cuda_stream)
                got = [h.fetch(cap=1 << 16) for h in group]
                del d
            for r, g in zip(rows, got):
                r.extend(g)
            o += c
            for k, (h, lone) in enumerate(zip(group, lones)):   # the bytes at every call seam, each channel's history
                nb = _blocks(h, o // s)
                assert np.array_equal(tap_resampled(h, done[k], nb), tap_resampled(lone, done[k], nb)), (path, i, k)
                done[k] = nb
        assert done[0] > 4
        assert [keys(r) for r in rows] == want, path
        for h in group:   # reset is per handle: reset together, the group starts a new stream
            h.reset()
        again = capi.decode_channels(group, raw, cap=1 << 16)
        assert [keys(r) for r in again] == want, path
        for h, lone in zip(group, lones):
            assert np.array_equal(tap_resampled(h, 0, done[0]), tap_resampled(lone, 0, done[0])), path
        for h in group:
            h.close()
    for lone in lones:
        lone.close()


@pytest.mark.parametrize("fmt", [capi.FORMAT_CU8, capi.FORMAT_CS16])
def test_capture_centre_at_the_decoders_rate_over_many_calls(built, fmt):
    """At the decoder's own rate the channel at the capture's centre is not resampled (pass-through or convert only) and
    takes whole blocks; the group still counts its stream position with the others', call after call."""
    import torch
    rate = DATA_RATE * 72
    offs = [0, -200_000, 150_000]   # |offset| <= 0.1 * the rate at the decoder's own rate
    z, _ = tune_ref.wideband([("scm", o, 71 + i, 0) for i, o in enumerate(offs)], rate, 40 * 16384, 71)
    raw = tune_ref.quantize(z, capi.FORMAT_CS16) if fmt == capi.FORMAT_CS16 else \
        np.clip(np.round(np.stack([z.real, z.imag], 1).ravel() + 127.5), 0, 255).astype(np.uint8)
    s = capi.FORMAT_BYTES[fmt]
    bs = 16384
    lones, want = [], []
    for o in offs:
        lones.append(_decoder(rate, o, fmt))
        want.append(lones[-1].decode(raw, 0, 1 << 16))
    with pytest.raises(capi.ErtGpuError):   # the centre channel is not resampled; the others are
        lones[0].resampler()
    assert "resample" not in lones[0].last_kernels() and all(h.resampler()[0]["L"] for h in lones[1:])
    blocks = [1, 3, 2, 7, 1, 5, 4, 9, 8]   # 40 blocks in calls of whole blocks
    for path in ("host", "device"):
        group = [_decoder(rate, o, fmt) for o in offs]
        rows, o = [[] for _ in offs], 0
        for nbk in blocks:
            part = raw[o:o + nbk * bs * s]
            if path == "host":
                got = capi.decode_channels(group, part, 0, 1 << 16)
            else:
                d = torch.from_numpy(part.copy()).cuda()
                capi.decode_channels_device_async(group, d.data_ptr(), part.size, 0, torch.cuda.current_stream().cuda_stream)
                got = [h.fetch(cap=1 << 16) for h in group]
                del d
            for r, g in zip(rows, got):
                r.extend(g)
            o += part.size
        assert o == raw.size
        for r, w in zip(rows, want):
            assert keys(r) == keys(w), path
        for h in group:
            h.close()
    for lone in lones:
        lone.close()


def _found(rows, truth):
    valid = [r for r in rows if r["check_mask"]]
    return [any(r["bytes"][:len(t.data)].tobytes() == t.data for r in valid) for t in truth]


def test_packets_in_five_channels_are_found_in_their_own(built):
    rate_in = 30_720_000
    offs = (-12_000_000, -6_000_000, -2_400_000, 3_000_000, 9_000_000)
    z, truths = decimate_ref.wideband([("scm", o, 51 + i, 25_000 * i) for i, o in enumerate(offs)], rate_in, 9_000_000, 51,
                                      spacing=1 << 20)
    raw = tune_ref.quantize(z, capi.FORMAT_CS16)
    group = [_decoder(rate_in, o, capi.FORMAT_CS16) for o in offs]
    got = capi.decode_channels(group, raw, capi.DECODE_ONLY_VALID, 1 << 16)
    for i, rows in enumerate(got):
        for j, t in enumerate(truths):
            assert len(t) >= 3
            found = _found(rows, t)
            assert all(found) if i == j else not any(found), (i, j)
    # the same at 8 MS/s, where every channel's one-stage tuned resampler reads the shared copy
    offs8 = (-2_400_000, -800_000, 900_000, 2_500_000)
    z, truths = tune_ref.wideband([("scm", o, 61 + i, 0) for i, o in enumerate(offs8)], 8_000_000, 4_000_000, 61)
    raw = tune_ref.quantize(z, capi.FORMAT_CS8)
    group8 = [_decoder(8_000_000, o, capi.FORMAT_CS8) for o in offs8]
    got = capi.decode_channels(group8, raw, capi.DECODE_ONLY_VALID, 1 << 16)
    for i, rows in enumerate(got):
        for j, t in enumerate(truths):
            found = _found(rows, t)
            assert all(found) if i == j else not any(found), (i, j)
    for h in group + group8:
        h.close()


def _rejected(handles, iq=None, match=""):
    iq = np.zeros(8192 * 4, dtype=np.uint8) if iq is None else iq
    with pytest.raises(capi.ErtGpuError) as e:
        capi.decode_channels(handles, iq)
    assert e.value.code == capi.EINVAL and match in str(e.value), str(e.value)


def test_every_rule_of_a_group(built):
    cs16, r = capi.FORMAT_CS16, 30_720_000
    a, b = _decoder(r, -2_400_000, cs16), _decoder(r, 2_000_000, cs16)
    _rejected([a, b, a], match="channel 2 is the handle of channel 0 again")
    _rejected([a] * 65, match="65 channels")
    unalloc = capi.Handle()
    unalloc.register(capi.stock_protocol("scm", 72))
    _rejected([a, unalloc], match="channel 1: the handle is not allocated")
    _rejected([a, _decoder(r, 0, cs16, msgtypes="idm")], match="other protocols")
    _rejected([a, _decoder(r, 0, cs16, cl=32)], match="other protocols")
    _rejected([a, _decoder(r, 0, capi.FORMAT_CS8)], match="input format or scale")
    scaled = capi.new_decoder("scm", 72, input_rate=r, input_format=cs16, input_scale=0.5, capture_freq=CAPTURE,
                              center_freq=CAPTURE + 1_000_000)
    _rejected([a, scaled], match="input format or scale")
    _rejected([a, _decoder(61_440_000, 0, cs16)], match="input rate or capture centre")
    other_capture = capi.new_decoder("scm", 72, input_rate=r, input_format=cs16, capture_freq=CAPTURE + 1,
                                     center_freq=CAPTURE)
    _rejected([a, other_capture], match="input rate or capture centre")
    untuned = capi.new_decoder("scm", 72, input_rate=3_200_000, input_format=cs16)
    _rejected([untuned], match="channel 0 is not tuned")
    with pytest.raises(capi.ErtGpuError) as e:   # each handle's own call rules still hold
        capi.decode_channels([a, b], np.zeros(6, dtype=np.uint8))
    assert e.value.code == capi.ESIZE
    ahead = _decoder(r, 1_000_000, cs16)
    ahead.decode(np.zeros(4 * 1000, dtype=np.uint8))
    _rejected([a, ahead], match="channel 1 is at input sample 1000")
    ahead.reset()
    capi.decode_channels([a, ahead], np.zeros(4 * 1000, dtype=np.uint8))   # reset together: accepted
    plain = capi.Handle()   # up to 10:1 a handle that does not allow decimation is the same as one that does
    plain.register(capi.stock_protocol("scm", 72))
    plain.set_input_tuning(CAPTURE, CAPTURE - 2_400_000)
    plain.set_input_rate(8_000_000)
    plain.set_input_format(cs16)
    plain.allocate(0)
    opted = _decoder(8_000_000, 1_000_000, cs16)
    capi.decode_channels([plain, opted], np.zeros(4 * 1000, dtype=np.uint8))
    plain.close()
    opted.close()
    with pytest.raises(capi.ErtGpuError):   # tuned handles are not sharded
        capi.decode_sharded([a], np.zeros(8192 * 4, dtype=np.uint8))
    for h in (a, b, unalloc, scaled, other_capture, untuned, ahead):
        h.close()


def _plain(stdout):
    """(block, digest, line) of each plain line; the message text after Idx stands for its digest."""
    out = []
    for line in stdout.splitlines():
        head, rest = line.split(" Idx:", 1)
        out.append((int(head[len("{Block:"):]), rest.split(" ", 1)[1], line))
    return out


def _merged(runs, block_dedup=True):
    """The single-channel runs' lines merged as the receiver prints a channel list (ascending block, then channel), with
    the cross-channel dedup: a digest seen for the previous block in any channel or for this block in an earlier one is
    dropped.  The single runs' own dedup only ever drops what this rule drops as well."""
    lines = [[(b, d, l) for b, d, l in r] for r in runs]
    out, prev, prev_block = [], set(), -2
    for b in sorted({b for r in lines for b, _, _ in r}):
        if b != prev_block + 1:
            prev = set()
        nxt = set()
        for r in lines:
            earlier = set(nxt)
            for bb, d, l in r:
                if bb != b:
                    continue
                nxt.add(d)
                if not block_dedup or (d not in prev and d not in earlier):
                    out.append(l)
        prev, prev_block = nxt, b
    return out


def test_cli_channel_list_prints_the_single_runs_merged(built, tmp_path):
    rate_in, chans = 30_720_000, [911_000_000, 912_600_155, 912_900_000]
    offs = [-4_000_000, -2_399_845, -2_250_000]   # the last packets lie inside both of the last two channels
    z, truths = decimate_ref.wideband([("scm", o, 131 + i, 33_000 * i) for i, o in enumerate(offs)], rate_in, 9_000_000,
                                      131, spacing=1 << 20)
    path = tmp_path / "band.cs16"
    tune_ref.quantize(z, capi.FORMAT_CS16).tofile(path)
    args = [CLI, "-msgtype=scm", "-sampleformat=cs16", f"-samplerate={rate_in}", "-capturefreq=915000000"]
    run = lambda extra: subprocess.run(args + extra + [str(path)], capture_output=True, text=True, timeout=600, check=True)
    singles = [run([f"-centerfreq={c}", "-blockdedup=false"]) for c in chans]
    multi = run(["-centerfreq=" + ",".join(map(str, chans))])
    assert multi.stdout.splitlines() == _merged([_plain(r.stdout) for r in singles])
    nodedup = run(["-centerfreq=" + ",".join(map(str, chans)), "-blockdedup=false"])
    assert nodedup.stdout.splitlines() == _merged([_plain(r.stdout) for r in singles], block_dedup=False)
    assert multi.stderr.startswith("CenterFreq: 911000000,912600155,912900000\nCaptureFreq: 915000000\n")
    for c in chans:
        assert f"{c} Hz: " in multi.stderr
    # the overlapping packets decode in both of the last two channels and are printed once
    ids = lambda out: [int(l.split("ID:")[1].split()[0]) for l in out.splitlines()]
    from test_gpu_resample import _scm_fields
    shared = {_scm_fields(t.data)[0] for t in truths[2]} & set(ids(singles[1].stdout)) & set(ids(singles[2].stdout))
    assert len(shared) >= 3
    for i in shared:
        assert 0 < ids(multi.stdout).count(i) < ids(singles[1].stdout).count(i) + ids(singles[2].stdout).count(i)


def test_cli_channel_list_at_the_decoders_rate(built, tmp_path):
    """The capture's centre and an off-centre channel of a uint8 capture at the decoder's own rate, read in several
    calls of 4 blocks and a partial last one."""
    rate, chans = DATA_RATE * 72, [912_600_000, 912_400_000]
    z, _ = tune_ref.wideband([("scm", c - 912_600_000, 141 + i, 0) for i, c in enumerate(chans)], rate, 30 * 16384 + 1000, 141)
    path = tmp_path / "native.cu8"
    np.clip(np.round(np.stack([z.real, z.imag], 1).ravel() + 127.5), 0, 255).astype(np.uint8).tofile(path)
    args = [CLI, "-msgtype=scm", "-blocks=4", "-capturefreq=912600000"]
    run = lambda extra: subprocess.run(args + extra + [str(path)], capture_output=True, text=True, timeout=600, check=True)
    singles = [run([f"-centerfreq={c}", "-blockdedup=false"]) for c in chans]
    multi = run(["-centerfreq=" + ",".join(map(str, chans))])
    assert singles[0].stdout and singles[1].stdout
    assert multi.stdout.splitlines() == _merged([_plain(r.stdout) for r in singles])
