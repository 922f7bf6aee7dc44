"""GPU tests (-m gpu) of per-packet signal reports (ertgpu_enable_signal, ertgpu_fetch_signal): every record against the
NumPy restatement (tests/signal_ref.py) int64 field for int64 field, over native, converted, resampled, tuned, decimated
and wide handles; call splits, the device path and reset; candidates and kernels of a handle with reports; channel
groups; and the rules of the calls."""
import numpy as np
import pytest

import signal_ref
import tune_ref
from helpers import synth_stream
from rtlamr_b200 import capi

pytestmark = pytest.mark.gpu

DATA_RATE = 32768
CAPTURE = 915_000_000


def _protos(msgtypes, cl):
    return [capi.stock_protocol(m, cl) for m in msgtypes.split(",")]


def _decoded_bytes(h):
    """The decoder's bytes of every block of the last call (a converting or resampling handle, one call from the stream
    start)."""
    out, b = [], 0
    while True:
        try:
            out.append(h.tap(capi.TAP_RESAMPLED, b))
        except capi.ErtGpuError:
            return np.concatenate(out) if out else np.zeros(0, np.uint8)
        b += 1


def _expect(u8, cands, protos):
    return [signal_ref.record(u8, int(c["block"]), int(c["idx"]), int(c["preamble_id"]), int(c["check_mask"]),
                              c["bytes"].tobytes(), protos) for c in cands]


def _assert_records(sig, want):
    assert len(sig) == len(want)
    for i, (g, w) in enumerate(zip(sig, want)):
        got = {f: int(g[f]) for f in signal_ref.FIELDS}
        assert got == w, (i, got, w)


def _check_native(h, iq, protos, flags=0):
    cands = h.decode(iq, flags=flags, cap=1 << 16)
    sig = h.fetch_signal()
    _assert_records(sig, _expect(iq, cands, protos))
    return cands, sig


def test_golden_sample_every_candidate(built, sample_iq):
    cl = 78
    for flags in (0, capi.DECODE_ONLY_VALID):
        h = capi.new_decoder("scm", cl, signal=True)
        bs2 = h.cfg.block_size2
        iq = sample_iq[:sample_iq.size // bs2 * bs2]
        cands, _ = _check_native(h, iq, _protos("scm", cl), flags)
        assert len(cands) > 0
        h.close()


@pytest.mark.parametrize("msgtype", ["scm", "scm+", "idm", "netidm", "r900", "r900bcd"])
@pytest.mark.parametrize("cl", [72, 32, 8])
def test_synthetic_protocols_and_chip_lengths(built, msgtype, cl):
    h = capi.new_decoder(msgtype, cl, signal=True)
    bs2 = h.cfg.block_size2
    spacing = 1 << 19 if msgtype in ("idm", "netidm") else 1 << 17
    iq, _, truth = synth_stream(msgtype, cl, 6 * spacing, spacing=spacing)
    iq = iq[:iq.size // bs2 * bs2]
    cands, sig = _check_native(h, iq, _protos(msgtype, cl))
    assert sum(1 for c in cands if c["check_mask"]) >= 1
    h.close()


def _converted_case(kind):
    """(handle with reports, input bytes)."""
    cl = 72
    if kind == "resampled":
        rate_in, fmt, off = 2_400_000, capi.FORMAT_CU8, None
    elif kind == "cs16":
        rate_in, fmt, off = DATA_RATE * cl, capi.FORMAT_CS16, None
    elif kind == "tuned":
        rate_in, fmt, off = 10_000_000, capi.FORMAT_CS16, -2_000_000
    else:   # decimated and wide
        rate_in, fmt, off = 30_720_000, capi.FORMAT_CS16, 2_400_000
    n = 4_000_000 if rate_in > 4_000_000 else 1_000_000
    z, _ = tune_ref.wideband([("scm", off or 0, 11, 0)], rate_in, n, 11)
    if fmt == capi.FORMAT_CU8:
        raw = np.empty(2 * n, dtype=np.uint8)
        raw[0::2], raw[1::2] = np.clip(np.round(z.real + 127.5), 0, 255), np.clip(np.round(z.imag + 127.5), 0, 255)
    else:
        raw = tune_ref.quantize(z, fmt)
    kw = {}
    if off is not None:
        kw = {"capture_freq": CAPTURE, "center_freq": CAPTURE + off}
    if kind == "wide":
        kw["channel_gain"] = 5
    h = capi.new_decoder("scm", cl, input_rate=rate_in, input_format=fmt, signal=True, **kw)
    return h, raw


@pytest.mark.parametrize("kind", ["resampled", "cs16", "tuned", "decimated", "wide"])
def test_converted_inputs_against_the_decoders_bytes(built, kind):
    h, raw = _converted_case(kind)
    if kind == "cs16":
        bs = h.cfg.block_size * 4
        raw = raw[:raw.size // bs * bs]
    cands = h.decode(raw, cap=1 << 16)
    sig = h.fetch_signal()
    u8 = _decoded_bytes(h)
    assert sum(1 for c in cands if c["check_mask"]) >= 2
    _assert_records(sig, _expect(u8, cands, _protos("scm", 72)))
    h.close()


def _keyed(cands, sig):
    return [(int(c["block"]), int(c["preamble_id"]), int(c["idx"]), tuple(int(s[f]) for f in signal_ref.FIELDS))
            for c, s in zip(cands, sig)]


def test_call_splits_device_path_and_reset(built):
    import torch
    cl, mt = 72, "scm,scm+,idm"
    h = capi.new_decoder(mt, cl, signal=True)
    bs2 = h.cfg.block_size2
    iq, _, _ = synth_stream(mt, cl, 1 << 21, spacing=1 << 18)
    iq = iq[:iq.size // bs2 * bs2]
    one = _keyed(h.decode(iq, cap=1 << 16), h.fetch_signal())
    assert one
    rng = np.random.default_rng(9)
    for _ in range(3):
        h.reset()
        cuts = sorted(set(int(x) * bs2 for x in rng.integers(1, iq.size // bs2, 5)))
        got = []
        for a, b in zip([0] + cuts, cuts + [iq.size]):
            got += _keyed(h.decode(iq[a:b], cap=1 << 16), h.fetch_signal())
        assert got == one
    h.reset()
    d = torch.from_numpy(iq).cuda()
    torch.cuda.synchronize()
    got = []
    step = 64 * bs2
    for a in range(0, iq.size, step):
        h.decode_device_async(d.data_ptr() + a, min(step, iq.size - a))
        got += _keyed(h.fetch(cap=1 << 16), h.fetch_signal())
    assert got == one
    h.close()


def test_packet_before_the_first_block_of_a_call(built):
    """A packet whose candidates have idx < SL in the first block of a call, with the call split exactly there: symbol 0
    lies before the kept history, every measured symbol inside it, so the records equal one call's."""
    cl, mt = 32, "scm"
    h = capi.new_decoder(mt, cl, signal=True)
    c = h.cfg
    bs, bs2 = c.block_size, c.block_size2
    geo = signal_ref.geometry(_protos(mt, cl))
    split_block = 40
    start = signal_ref.first_sample(geo, split_block, c.symbol_length // 2)   # idx = SL/2 in block split_block
    from rtlamr_b200 import synth
    pk, _ = synth.make_packets(mt, cl, 1 << 16, seed=3, spacing=1 << 16)
    pk = pk[:1].copy()
    pk["start_sample"] = start
    iq = synth.host_fill(0, 80 * bs, 0x5EED0001, pk)
    one = _keyed(h.decode(iq, cap=1 << 16), h.fetch_signal())
    assert any(k[0] == split_block and k[2] < c.symbol_length for k in one)
    h.reset()
    got = _keyed(h.decode(iq[:split_block * bs2], cap=1 << 16), h.fetch_signal())
    got += _keyed(h.decode(iq[split_block * bs2:], cap=1 << 16), h.fetch_signal())
    assert got == one
    _assert_records([s for s in h.fetch_signal()], _expect(iq, h.fetch(cap=1 << 16), _protos(mt, cl)))
    h.close()


@pytest.mark.parametrize("flags", [0, capi.DECODE_ONLY_VALID])
def test_candidates_launches_and_kernels_unchanged(built, flags):
    cl, mt = 72, "scm,scm+,idm,r900"
    a = capi.new_decoder(mt, cl)
    b = capi.new_decoder(mt, cl, signal=True)
    bs2 = a.cfg.block_size2
    iq, _, _ = synth_stream(mt, cl, 1 << 21, spacing=1 << 18)
    iq = iq[:iq.size // bs2 * bs2]
    for part in (iq[:iq.size // 2], iq[iq.size // 2:]):
        ca, cb = a.decode(part, flags=flags, cap=1 << 16), b.decode(part, flags=flags, cap=1 << 16)
        assert ca.tobytes() == cb.tobytes()
        assert b.last_kernels() == a.last_kernels() + ";packet_signal_kernel"
        assert b.last_launches() > a.last_launches()
        assert len(b.fetch_signal()) == len(cb)
    a.close()
    b.close()


@pytest.mark.parametrize("nch", [3, 8])
def test_channel_groups_equal_lone_handles(built, nch):
    cl, rate_in, fmt = 72, 10_000_000, capi.FORMAT_CS16
    offs = [-3_000_000 + 800_000 * k for k in range(nch)]
    z, _ = tune_ref.wideband([("scm", offs[1] + 300_000, 11, 0)], rate_in, 3_000_000, 11)
    raw = tune_ref.quantize(z, fmt)

    def mk(off):
        return capi.new_decoder("scm", cl, input_rate=rate_in, input_format=fmt, capture_freq=CAPTURE,
                                center_freq=CAPTURE + off, signal=True)
    group = [mk(o) for o in offs]
    cands = capi.decode_channels(group, raw, cap=1 << 16)
    freqs = {}
    for k, (h, cs) in enumerate(zip(group, cands)):
        sig = h.fetch_signal()
        lone = mk(offs[k])
        assert _keyed(cs, sig) == _keyed(lone.decode(raw, cap=1 << 16), lone.fetch_signal())
        lone.close()
        for c, s in zip(cs, sig):
            if c["check_mask"]:
                sm = signal_ref.summary({f: int(s[f]) for f in signal_ref.FIELDS}, CAPTURE + offs[k], DATA_RATE * cl)
                freqs.setdefault(k, []).append(sm["freq"])
    # the packet at offs[1] + 300 kHz lies in the passbands of channels 1 and 2 (+-0.4 R_out = +-944 kHz)
    assert 1 in freqs and 2 in freqs
    for k in (1, 2):
        assert abs(np.median(freqs[k]) - (CAPTURE + offs[1] + 300_000)) <= 2_000
    for h in group:
        h.close()


def test_rules(built):
    h = capi.new_decoder("scm", 72, signal=True, max_candidates=64)
    with pytest.raises(capi.ErtGpuError) as e:
        h.enable_signal()
    assert e.value.code == capi.EINVAL
    plain = capi.new_decoder("scm", 72)
    with pytest.raises(capi.ErtGpuError) as e:
        plain.fetch_signal()
    assert e.value.code == capi.EINVAL
    with pytest.raises(capi.ErtGpuError) as e:
        capi.decode_sharded([h], np.zeros(h.cfg.block_size2 * 4, np.uint8))
    assert e.value.code == capi.EINVAL
    assert "signal" in capi.lib().ertgpu_last_error(h._h).decode()
    # capacity: ertgpu_fetch's rules
    iq, _, _ = synth_stream("scm", 72, 1 << 20, spacing=1 << 17)
    bs2 = h.cfg.block_size2
    big = capi.new_decoder("scm", 72, signal=True)
    cands = big.decode(iq[:iq.size // bs2 * bs2], cap=1 << 16)
    assert len(cands) > 1
    import ctypes as C
    n = C.c_size_t(0)
    out = np.empty(1, dtype=capi.SIGNAL_DTYPE)
    rc = capi.lib().ertgpu_fetch_signal(big._h, out.ctypes.data, 1, C.byref(n))
    assert rc == capi.ECAPACITY and n.value == len(cands)
    assert len(big.fetch_signal(cap=len(cands))) == len(cands)
    for x in (h, plain, big):
        x.close()


def test_cli_channel_list_names_the_channel_and_freq(built, tmp_path):
    """ertgpu_decode_file -signal with -centerfreq=F1,F2,F3 on a cs16 capture: every message names a channel whose
    passband holds the packet, and a Freq near the injected carrier; without -signal the lines are those of today."""
    import os
    import re
    import subprocess
    from conftest import ROOT
    rate_in, chans = 10_000_000, [CAPTURE - 3_000_000, CAPTURE - 1_000_000, CAPTURE + 2_000_000]
    carrier = chans[1] + 250_000
    z, _ = tune_ref.wideband([("scm", carrier - CAPTURE, 11, 0)], rate_in, 3_000_000, 11)
    path = tmp_path / "cap.cs16"
    tune_ref.quantize(z, capi.FORMAT_CS16).tofile(path)
    cli = os.path.join(ROOT, "rtlamr_b200", "ertgpu_decode_file")
    base = ["-msgtype=scm", "-sampleformat=cs16", f"-samplerate={rate_in}", f"-capturefreq={CAPTURE}",
            "-centerfreq=" + ",".join(map(str, chans)), str(path)]
    run = lambda *a: subprocess.run([cli, *a], capture_output=True, text=True, timeout=300, check=True).stdout.splitlines()  # noqa: E731
    plain, sig = run(*base), run("-signal", *base)
    assert len(sig) == len(plain) >= 2
    pat = re.compile(r"\{Block:(\d+) Idx:(\d+) Channel:(\d+) Freq:(\d+) Level:(-?\d+\.\d\d) Noise:(-?\d+\.\d\d) "
                     r"SNR:(-?\d+\.\d\d) (SCM:.*)")
    for p, s in zip(plain, sig):
        m = pat.fullmatch(s)
        assert m, s
        assert p == f"{{Block:{m[1]} Idx:{m[2]} {m[8]}"
        assert int(m[3]) == chans[1]
        assert abs(int(m[4]) - carrier) <= 3_000
    js = [__import__("json").loads(ln) for ln in run("-signal", "-format=json", *base)]
    assert all(j["Signal"]["Channel"] == chans[1] and abs(j["Signal"]["Freq"] - carrier) <= 3_000 for j in js)


def test_host_receiver_signal(built):
    from rtlamr_b200 import host
    rate_in, off = 10_000_000, -2_000_000
    z, _ = tune_ref.wideband([("scm", off + 90_000, 11, 0)], rate_in, 3_000_000, 11)
    raw = tune_ref.quantize(z, capi.FORMAT_CS16)
    kw = dict(input_rate=rate_in, input_format=capi.FORMAT_CS16, capture_freq=CAPTURE, center_freq=CAPTURE + off)
    r = host.Receiver("scm", 72, signal=True, **kw)
    msgs = r.decode(raw)
    plain = host.Receiver("scm", 72, **kw).decode(raw)
    assert len(msgs) == len(plain) >= 2
    for m, p in zip(msgs, plain):
        assert (m.block, m.idx, m.text, m.record) == (p.block, p.idx, p.text, p.record) and p.signal is None
        assert m.signal["channel"] == CAPTURE + off
        assert abs(m.signal["freq"] - (CAPTURE + off + 90_000)) <= 3_000
        assert m.signal["snr"] > m.signal["noise"] - 100
    r.close()
