"""GPU tests (-m gpu) of the input-format conversion: convert_kernel and the converting resample_kernel instances
against the numpy restatement (tests/format_ref.py) byte for byte, their composition with today's uint8 path,
call-splitting invariance, the size rules, the cu8 no-op, the golden capture re-encoded in every format and WAV
container, and weak cs16 packets decoded with a gain."""
import json
import os
import subprocess
import wave

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from helpers import assert_check_masks_exact
from rtlamr_b200 import capi, synth

import resample_ref
from format_ref import NAME, convert, encode, wav_bytes

pytestmark = pytest.mark.gpu

DATA_RATE = 32768
FORMATS = [capi.FORMAT_CS8, capi.FORMAT_CS16, capi.FORMAT_CF32]
CLI = os.path.join(ROOT, "rtlamr_b200", "ertgpu_decode_file")


def keys(rows):
    return sorted((int(r["block"]), int(r["idx"]), int(r["preamble_id"]), r["bytes"].tobytes(), int(r["check_mask"]),
                   r["r900_digits"].tobytes() if int(r["flags"]) & capi.CAND_HAS_R900 else b"") for r in rows)


def random_raw(fmt, nsamples, seed, specials=True):
    """Random raw IQ of format fmt: the whole int range, or float32 around full scale with specials sprinkled in."""
    rng = np.random.default_rng(seed)
    if fmt == capi.FORMAT_CS8:
        return rng.integers(0, 256, 2 * nsamples, dtype=np.uint8)
    if fmt == capi.FORMAT_CS16:
        return rng.integers(-32768, 32768, 2 * nsamples).astype("<i2").view(np.uint8)
    x = (rng.standard_normal(2 * nsamples) * 0.7).astype(np.float32)
    if specials:
        sp = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-45, -1e-40, 0.5 / 128, 1.5 / 128, 127.5 / 128,
                       -128.5 / 128, 126.5 / 128, 1e30, -1e30], dtype=np.float32)
        at = rng.choice(x.size, 4096, replace=False)
        x[at] = sp[rng.integers(0, sp.size, at.size)]
    return x.astype("<f4").view(np.uint8)


def u8_stream(msgtypes, rate_in, nsamples, seed, spacing=1 << 17, amplitude=(24, 60)):
    """uint8 IQ at rate_in: synthetic noise plus packets whose chip c covers the input samples from c * rate_in / 32768."""
    iq = synth.host_fill(0, nsamples, 0x5EED0000 + seed, None).astype(np.int32)
    pk, truth = synth.make_packets(msgtypes, -(-rate_in // DATA_RATE), nsamples - 2 * spacing, seed=seed, spacing=spacing,
                                   amplitude=amplitude)
    add_packets(iq, pk, rate_in)
    return np.clip(iq, 0, 255).astype(np.uint8), truth


def add_packets(iq, pk, rate_in):
    n_all = iq.size // 2
    for row in pk:
        n_chips = int(row["n_chips"])
        chips = np.unpackbits(row["chips"])[:n_chips]
        n = -(-n_chips * rate_in // DATA_RATE)
        s = np.arange(n)
        c = s * DATA_RATE // rate_in
        hi = chips[np.minimum(c, n_chips - 1)].astype(bool) & (c < n_chips)
        idx = int(row["start_sample"]) + s[hi]
        idx = idx[idx < n_all]
        iq[2 * idx] += int(row["amp_i"])
        iq[2 * idx + 1] += int(row["amp_q"])


def jittered(u8, fmt, seed):
    """u8 encoded in fmt, with sub-LSB jitter for cs16 / cf32 so that the default scale has something to round."""
    raw = encode(u8, fmt)
    rng = np.random.default_rng(seed)
    if fmt == capi.FORMAT_CS16:
        v = raw.view("<i2").astype(np.int32) + rng.integers(-128, 128, u8.size)
        return np.clip(v, -32768, 32767).astype("<i2").view(np.uint8)
    if fmt == capi.FORMAT_CF32:
        return (raw.view("<f4") + rng.uniform(-0.5, 0.5, u8.size).astype(np.float32) / np.float32(128)).astype("<f4").view(np.uint8)
    return raw


def native_keys(msgtypes, cl, u8):
    h = capi.new_decoder(msgtypes, cl)
    bs2 = h.cfg.block_size2
    got = h.decode(u8[:(u8.size // bs2) * bs2], cap=1 << 16)
    h.close()
    return keys(got)


def taps(h, first, last):
    return np.concatenate([h.tap(capi.TAP_RESAMPLED, b) for b in range(first, last)]) if last > first else np.zeros(0, np.uint8)


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("scale", [0.0, 0.3, 3.0])
def test_native_kernel_equals_restatement(built, fmt, scale):
    """Every byte the decoder read (ERTGPU_TAP_RESAMPLED) equals the restatement's, and the candidates equal today's
    decode of those bytes."""
    cl = 72
    h = capi.new_decoder("scm", cl, input_format=fmt, input_scale=scale)
    bs = h.cfg.block_size
    nblocks = 150
    raw = random_raw(fmt, nblocks * bs, seed=fmt * 7 + int(scale * 10))
    got = h.decode(raw, cap=1 << 16)
    want = convert(raw, fmt, scale)
    assert np.array_equal(taps(h, 0, nblocks), want)
    assert h.last_kernels().split(";")[-1] == f"convert_kernel<{NAME[fmt]}>"
    assert h.last_kernels().split(";")[0].startswith("demod_")
    assert keys(got) == native_keys("scm", cl, want)
    h.close()


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("rate_in,cl,scale", [(2_400_000, 72, 0.0), (2_048_000, 72, 0.3), (3_200_000, 32, 0.0),
                                              (1_024_000, 72, 3.0)])
def test_resampling_kernel_equals_restatement(built, fmt, rate_in, cl, scale):
    n = 400_000
    raw = random_raw(fmt, n, seed=rate_in + fmt)
    ref = resample_ref.resample(convert(raw, fmt, scale), rate_in, DATA_RATE * cl)
    h = capi.new_decoder("scm", cl, input_rate=rate_in, input_format=fmt, input_scale=scale)
    got = h.decode(raw, cap=1 << 16)
    bs = h.cfg.block_size
    nblocks = (ref.size // 2) // bs
    assert np.array_equal(taps(h, 0, nblocks), ref[:2 * nblocks * bs])
    assert h.last_kernels().split(";")[-1] == f"resample_kernel<{NAME[fmt]}>"
    assert keys(got) == native_keys("scm", cl, ref)
    h.close()


@pytest.mark.parametrize("msgtypes", ["scm", "scm,scm+,idm", "r900"])
@pytest.mark.parametrize("rate_in", [DATA_RATE * 72, 2_400_000])
def test_composition_with_uint8_path(built, msgtypes, rate_in):
    """Format-F candidates equal the candidates today's uint8 path gives for the restated bytes."""
    cl = 72
    u8, truth = u8_stream(msgtypes, rate_in, 2_400_000, seed=21)
    for fmt in FORMATS:
        raw = jittered(u8, fmt, seed=fmt)
        h = capi.new_decoder(msgtypes, cl, input_rate=rate_in, input_format=fmt)
        b = capi.new_decoder(msgtypes, cl, input_rate=rate_in)
        if rate_in == DATA_RATE * cl:
            bs = h.cfg.block_size
            n = (u8.size // 2) // bs * bs
            raw, conv = raw[:n * capi.FORMAT_BYTES[fmt]], convert(raw[:n * capi.FORMAT_BYTES[fmt]], fmt)
        else:
            conv = convert(raw, fmt)
        got, want = h.decode(raw, cap=1 << 16), b.decode(conv, cap=1 << 16)
        assert keys(got) == keys(want), NAME[fmt]
        assert_check_masks_exact(got, msgtypes)
        assert sum(1 for r in got if r["check_mask"]) >= len(truth) > 0
        h.close()
        b.close()


def _cuts(rng, total, unit, spans):
    """Call sizes of whole units (samples or blocks) adding up to total units, each 1 or up to one of spans units."""
    sizes = []
    while sum(sizes) < total:
        sizes.append(int(rng.choice([1] + [int(rng.integers(1, m + 1)) for m in spans])))
    sizes[-1] -= sum(sizes) - total
    return [unit * s for s in sizes if s > 0]


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("rate_in", [DATA_RATE * 72, 2_400_000])
def test_call_splitting_host_and_device(built, fmt, rate_in):
    import torch
    cl, msgtypes = 72, "scm,r900"
    u8, _ = u8_stream(msgtypes, rate_in, 1_200_000, seed=31)
    s = capi.FORMAT_BYTES[fmt]
    native = rate_in == DATA_RATE * cl
    whole = capi.new_decoder(msgtypes, cl, input_rate=rate_in, input_format=fmt)
    bs = whole.cfg.block_size
    nsamples = (u8.size // 2) // bs * bs if native else u8.size // 2
    raw = jittered(u8, fmt, seed=3)[:nsamples * s]
    want = keys(whole.decode(raw, cap=1 << 16))
    whole.close()
    assert want
    rng = np.random.default_rng(rate_in + fmt)
    sizes = _cuts(rng, nsamples // bs, bs, (4, 16, 64)) if native else _cuts(rng, nsamples, 1, (64, 5000, 200_000))
    assert len(sizes) >= 8
    for path in ("host", "device"):
        h = capi.new_decoder(msgtypes, cl, input_rate=rate_in, input_format=fmt)
        rows, off = [], 0
        for n in sizes:
            part = raw[off * s:(off + n) * s]
            off += n
            if path == "host":
                rows.extend(h.decode(part, cap=1 << 16))
            else:
                d = torch.from_numpy(part.copy()).cuda()
                h.decode_device_async(d.data_ptr(), d.numel(), 0, torch.cuda.current_stream().cuda_stream)
                rows.extend(h.fetch(cap=1 << 16))
                del d
        assert keys(rows) == want, path
        h.close()


@pytest.mark.parametrize("rate_in", [DATA_RATE * 72, 1_024_000])
def test_host_chunking_respects_max_blocks(built, rate_in):
    import torch
    cl, fmt = 72, capi.FORMAT_CF32
    u8, _ = u8_stream("scm", rate_in, 400_000, seed=41)
    raw = jittered(u8, fmt, seed=4)
    h = capi.new_decoder("scm", cl, input_rate=rate_in, input_format=fmt, max_blocks_per_call=3)
    bs = h.cfg.block_size
    if rate_in == DATA_RATE * cl:
        raw = raw[:(u8.size // 2) // bs * bs * 8]
        want = native_keys("scm", cl, convert(raw, fmt))
    else:
        want = native_keys("scm", cl, resample_ref.resample(convert(raw, fmt), rate_in, DATA_RATE * cl))
    assert keys(h.decode(raw, cap=1 << 16)) == want
    h.reset()
    d = torch.from_numpy(raw).cuda()
    with pytest.raises(capi.ErtGpuError) as e:
        h.decode_device_async(d.data_ptr(), d.numel(), 0, torch.cuda.current_stream().cuda_stream)
    assert e.value.code == capi.ESIZE
    rows, step = [], 8 * 2 * bs if rate_in == DATA_RATE * cl else 8 * 4096
    for off in range(0, raw.size, step):
        h.decode_device_async(d.data_ptr() + off, min(step, raw.size - off), 0, torch.cuda.current_stream().cuda_stream)
        rows.extend(h.fetch(cap=1 << 16))
    assert keys(rows) == want
    h.close()


def test_sharded_rejects_converting_handles(built):
    h = capi.new_decoder("scm", 72, input_format=capi.FORMAT_CS16)
    with pytest.raises(capi.ErtGpuError) as e:
        capi.decode_sharded([h], np.zeros(8192 * 4, dtype=np.uint8))
    assert e.value.code == capi.EINVAL
    h.close()


def test_size_and_order_rules(built):
    import torch
    d = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    for fmt in FORMATS:
        s = capi.FORMAT_BYTES[fmt]
        nat = capi.new_decoder("scm", 72, input_format=fmt)
        bs = nat.cfg.block_size
        for n in (bs * 2, bs * s - s, bs * s + 2 * s):   # whole blocks of s-byte samples only (bs * 2 = one cu8 block)
            if n % (bs * s) == 0:
                continue
            for call in (lambda: nat.decode(np.zeros(n, np.uint8)), lambda: nat.decode_device_async(d.data_ptr(), n, 0, st)):
                with pytest.raises(capi.ErtGpuError) as e:
                    call()
                assert e.value.code == capi.ESIZE, (fmt, n)
        with pytest.raises(capi.ErtGpuError) as e:   # 16-byte aligned device input
            nat.decode_device_async(d.data_ptr() + 8, bs * s, 0, st)
        assert e.value.code == capi.EINVAL
        nat.decode_device_async(d.data_ptr() + 16, bs * s, 0, st)
        nat.fetch()
        with pytest.raises(capi.ErtGpuError) as e:
            nat.set_input_format(capi.FORMAT_CS16)
        assert e.value.code == capi.EINVAL and "after allocate" in str(e.value)
        nat.close()
        rs = capi.new_decoder("scm", 72, input_rate=2_400_000, input_format=fmt)
        for n in (s + 1, 3 * s - 1) if s > 2 else (3, 1001):
            for call in (lambda: rs.decode(np.zeros(n, np.uint8)), lambda: rs.decode_device_async(d.data_ptr(), n, 0, st)):
                with pytest.raises(capi.ErtGpuError) as e:
                    call()
                assert e.value.code == capi.ESIZE, (fmt, n)
        if s > 2:   # s-byte aligned device input
            with pytest.raises(capi.ErtGpuError) as e:
                rs.decode_device_async(d.data_ptr() + s // 2, 100 * s, 0, st)
            assert e.value.code == capi.EINVAL
        rs.decode_device_async(d.data_ptr() + s, 100 * s, 0, st)
        rs.fetch()
        rs.close()
    plain = capi.new_decoder("scm", 72)
    plain.decode(np.zeros(8192 * 4, np.uint8))
    with pytest.raises(capi.ErtGpuError) as e:   # no conversion, no resampling: no such tap
        plain.tap(capi.TAP_RESAMPLED, 0)
    assert e.value.code == capi.EINVAL
    plain.close()


@pytest.mark.parametrize("rate_in", [0, 2_400_000])
def test_explicit_cu8_is_a_no_op(built, rate_in):
    cl = 72
    u8, _ = u8_stream("scm,r900", rate_in or DATA_RATE * cl, 1 << 21, seed=51)
    a = capi.new_decoder("scm,r900", cl, input_rate=rate_in)
    b = capi.Handle()
    for m in ("scm", "r900"):
        b.register(capi.stock_protocol(m, cl))
    b.set_input_format(capi.FORMAT_CU8)
    if rate_in:
        b.set_input_rate(rate_in)
    b.allocate(0)
    bs2 = a.cfg.block_size2
    iq = u8 if rate_in else u8[:(u8.size // bs2) * bs2]
    ga, gb = a.decode(iq, cap=1 << 16), b.decode(iq, cap=1 << 16)
    assert ga.tobytes() == gb.tobytes() and len(ga) > 0
    assert a.last_launches() == b.last_launches()
    assert a.last_kernels() == b.last_kernels() and "convert" not in b.last_kernels() and "<c" not in b.last_kernels()
    a.close()
    b.close()


def _run_cli(path, *args):
    r = subprocess.run([CLI, *args, str(path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    return r.stdout.splitlines()


@pytest.mark.parametrize("cl,rate_args", [(78, []), (72, ["-samplerate=2555904"])])
def test_golden_capture_in_every_encoding(built, tmp_path, cl, rate_args):
    """tests/golden/sample_cl78.bin (uint8 at 2 555 904 S/s) re-encoded at the default scales prints exactly the
    lines of the raw uint8 run."""
    src = os.path.join(GOLDEN, "sample_cl78.bin")
    u8 = np.fromfile(src, dtype=np.uint8)
    common = ["-msgtype=scm", f"-symbollength={cl}", "-blocks=7", *rate_args]
    want = _run_cli(src, *common)
    assert len(want) >= 10
    rate = 2_555_904
    for fmt in FORMATS:
        p = tmp_path / f"in.{NAME[fmt]}"
        encode(u8, fmt).tofile(p)
        assert _run_cli(p, *common, f"-sampleformat={NAME[fmt]}") == want, NAME[fmt]
    p8 = tmp_path / "u8.wav"
    with wave.open(str(p8), "wb") as w:   # 8-bit WAV samples are unsigned: the capture's bytes as they are
        w.setnchannels(2), w.setsampwidth(1), w.setframerate(rate)
        w.writeframes(u8.tobytes())
    p16 = tmp_path / "s16.wav"
    with wave.open(str(p16), "wb") as w:
        w.setnchannels(2), w.setsampwidth(2), w.setframerate(rate)
        w.writeframes(encode(u8, capi.FORMAT_CS16).tobytes())
    pf = tmp_path / "f32.wav"
    auxi = b"auxi" + (3).to_bytes(4, "little") + b"SDR\0"
    pf.write_bytes(wav_bytes(encode(u8, capi.FORMAT_CF32).tobytes() + b"LIST\x04\0\0\0INFO", bits=32, tag=3, rate=rate,
                             rf64=True, data_size=u8.size * 4, before_data=auxi))
    for p in (p8, p16, pf):
        assert _run_cli(p, *common, "-sampleformat=wav") == want, p.name
    # from stdin too: the header is read without seeking
    r = subprocess.run([CLI, *common, "-sampleformat=wav", "-"], stdin=open(p16, "rb"), capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0 and r.stdout.splitlines() == want


def _scm_fields(data: bytes):
    bits = "".join(f"{b:08b}" for b in data)
    return int(bits[21:23] + bits[56:80], 2), int(bits[32:56], 2)


def test_weak_cs16_packets_with_a_gain(built, tmp_path):
    """scm and idm packets with a carrier of 1500 over Gaussian noise of sigma 300, as cs16 at 2.4 MS/s: every packet
    is reported with -samplescale=0.0625."""
    rate_in, n = 2_400_000, 3_000_000
    rng = np.random.default_rng(7)
    iq = np.rint(rng.standard_normal(2 * n) * 300).astype(np.int32)
    pk, truth = synth.make_packets("scm,idm", -(-rate_in // DATA_RATE), n - (1 << 18), seed=8, spacing=1 << 17,
                                   amplitude=(1500, 1500))
    add_packets(iq, pk, rate_in)
    p = tmp_path / "weak.cs16"
    np.clip(iq, -32768, 32767).astype("<i2").tofile(p)
    assert len(truth) >= 16
    lines = _run_cli(p, "-msgtype=scm,idm", "-symbollength=72", f"-samplerate={rate_in}", "-sampleformat=cs16",
                     "-samplescale=0.0625", "-format=json")
    msgs = [json.loads(l)["Message"] for l in lines]
    for t in truth:
        if t.msgtype == "scm":
            mid, cons = _scm_fields(t.data)
            assert any(m.get("ID") == mid and m.get("Consumption") == cons for m in msgs), mid
        else:
            assert any(m.get("ERTSerialNumber") == t.meter_id for m in msgs), t.meter_id


def test_host_receiver_binding_takes_the_format(built):
    from rtlamr_b200 import host
    u8, truth = u8_stream("scm", 2_400_000, 1_000_000, seed=111)
    raw = encode(u8, capi.FORMAT_CF32)
    r = host.Receiver("scm", 72, input_rate=2_400_000, input_format=capi.FORMAT_CF32)
    msgs = r.decode(raw[:8 * 333_333]) + r.decode(raw[8 * 333_333:])
    ids = {_scm_fields(t.data)[0] for t in truth}
    assert ids and ids <= {m.meter_id for m in msgs}
    r.close()
