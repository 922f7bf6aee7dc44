"""GPU tests (-m gpu) of the input-rate resampler: resample_kernel against the CPU restatement
(tests/cpu_harness/resample_ref.c) byte for byte, its composition with the native decoder, call-splitting
invariance on the host and device paths, the no-op rate, and packets rendered at a foreign rate."""
import json
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from helpers import assert_check_masks_exact
from rtlamr_b200 import capi, synth

import resample_ref

pytestmark = pytest.mark.gpu

DATA_RATE = 32768
RATES = [(2_048_000, 72), (2_400_000, 72), (2_560_000, 72), (2_880_000, 72), (3_200_000, 72), (1_024_000, 72),
         (2_400_000, 32), (3_200_000, 32)]


def out_end(info, x):
    """Outputs whose window lies inside the first x input samples."""
    a = x - info["T"] // 2
    return 0 if a <= 0 else -(-a * info["L"] // info["M"])


def key(r):
    return (int(r["block"]), int(r["idx"]), int(r["preamble_id"]), r["bytes"].tobytes(), int(r["check_mask"]),
            r["r900_digits"].tobytes() if int(r["flags"]) & capi.CAND_HAS_R900 else b"")


def keys(rows):
    return sorted(key(r) for r in rows)


def native_of(msgtypes, cl, ref):
    """The existing native decode of an already resampled stream (whole blocks)."""
    h = capi.new_decoder(msgtypes, cl)
    bs2 = h.cfg.block_size2
    got = h.decode(ref[:(ref.size // bs2) * bs2], cap=1 << 16)
    h.close()
    return got


def stream(msgtypes, rate_in, nsamples, seed, spacing=1 << 17, noise_only=False):
    """uint8 IQ at rate_in: the synthetic noise of include/ertgpu_synth.h plus packets whose chip c covers the input
    samples from c * rate_in / 32768 (carrier added on high chips, as in synth)."""
    iq = synth.host_fill(0, nsamples, 0x5EED0000 + seed, None).astype(np.int32)
    cl_guess = -(-rate_in // DATA_RATE)
    # packets start at least two windows before the end, so the longest (idm) one ends inside the stream
    pk, truth = synth.make_packets(msgtypes, cl_guess, nsamples - 2 * spacing, seed=seed, spacing=spacing)
    if noise_only:
        return iq.astype(np.uint8), []
    for row in pk:
        n_chips = int(row["n_chips"])
        chips = np.unpackbits(row["chips"])[:n_chips]
        start = int(row["start_sample"])
        n = -(-n_chips * rate_in // DATA_RATE)
        s = np.arange(n)
        c = s * DATA_RATE // rate_in
        hi = chips[np.minimum(c, n_chips - 1)].astype(bool) & (c < n_chips)
        idx = start + s[hi]
        idx = idx[idx < nsamples]
        iq[2 * idx] += int(row["amp_i"])
        iq[2 * idx + 1] += int(row["amp_q"])
    return np.clip(iq, 0, 255).astype(np.uint8), truth


def tap_resampled(h, first_block, last_block):
    return np.concatenate([h.tap(capi.TAP_RESAMPLED, b) for b in range(first_block, last_block)]) \
        if last_block > first_block else np.zeros(0, np.uint8)


@pytest.mark.parametrize("rate_in,cl", RATES)
@pytest.mark.parametrize("kind", ["random", "synthetic"])
def test_kernel_equals_cpu_restatement(built, rate_in, cl, kind):
    """Every resampled byte the decoder read (ERTGPU_TAP_RESAMPLED) equals the CPU restatement's, and the candidates
    equal the native decode of the restatement's stream."""
    rate_out = DATA_RATE * cl
    n = 600_000
    if kind == "random":
        iq = np.random.default_rng(rate_in ^ cl).integers(0, 256, 2 * n, dtype=np.uint8)
    else:
        iq, _ = stream("scm", rate_in, n, seed=11)
    ref = resample_ref.resample(iq, rate_in, rate_out)
    h = capi.new_decoder("scm", cl, input_rate=rate_in)
    got = h.decode(iq, cap=1 << 16)
    bs = h.cfg.block_size
    nblocks = (ref.size // 2) // bs
    assert "resample_kernel" in h.last_kernels().split(";")
    assert h.last_kernels().split(";")[0].startswith("demod_")
    assert np.array_equal(tap_resampled(h, 0, nblocks), ref[:2 * nblocks * bs])
    assert keys(got) == keys(native_of("scm", cl, ref))
    h.close()


@pytest.mark.parametrize("msgtypes,rate_in", [("scm", 2_400_000), ("scm,scm+,idm", 2_048_000), ("r900", 2_400_000),
                                              ("r900", 1_024_000), ("scm,scm+,idm", 3_200_000)])
def test_composition_with_native_decode(built, msgtypes, rate_in):
    cl = 72
    iq, truth = stream(msgtypes, rate_in, 3_000_000, seed=21)
    ref = resample_ref.resample(iq, rate_in, DATA_RATE * cl)
    h = capi.new_decoder(msgtypes, cl, input_rate=rate_in)
    got = h.decode(iq, cap=1 << 16)
    want = native_of(msgtypes, cl, ref)
    assert keys(got) == keys(want)
    assert_check_masks_exact(got, msgtypes)
    assert sum(1 for r in got if r["check_mask"]) >= len(truth) > 0
    h.close()


def _cuts(rng, nbytes, ncalls):
    """Even call sizes: some tiny (no whole output block), some large."""
    sizes = []
    while sum(sizes) < nbytes:
        sizes.append(int(rng.choice([2, 2 * int(rng.integers(1, 64)), 2 * int(rng.integers(1, 5000)),
                                     2 * int(rng.integers(1, 200_000))])))
    sizes[-1] -= sum(sizes) - nbytes
    return [s for s in sizes if s > 0]


@pytest.mark.parametrize("msgtypes,rate_in,cl", [("scm", 2_400_000, 72), ("scm,scm+,idm", 2_048_000, 72),
                                                 ("r900", 3_200_000, 72), ("scm", 3_200_000, 32)])
def test_call_splitting_host_and_device(built, msgtypes, rate_in, cl):
    import torch
    rate_out = DATA_RATE * cl
    iq, _ = stream(msgtypes, rate_in, 1_500_000, seed=31)
    ref = resample_ref.resample(iq, rate_in, rate_out)
    whole = capi.new_decoder(msgtypes, cl, input_rate=rate_in)
    want = keys(whole.decode(iq, cap=1 << 16))
    whole.close()
    assert want == keys(native_of(msgtypes, cl, ref))
    rng = np.random.default_rng(rate_in + cl)
    sizes = _cuts(rng, iq.size, 40)
    assert any(s < 64 for s in sizes)
    for path in ("host", "device"):
        h = capi.new_decoder(msgtypes, cl, input_rate=rate_in)
        info, _ = h.resampler()
        bs = h.cfg.block_size
        rows, resampled, off, blocks_done = [], [], 0, 0
        for s in sizes:
            part = iq[off:off + s]
            off += s
            if path == "host":
                got = h.decode(part, cap=1 << 16)
            else:
                d = torch.from_numpy(part.copy()).cuda()
                h.decode_device_async(d.data_ptr(), d.numel(), 0, torch.cuda.current_stream().cuda_stream)
                got = h.fetch(cap=1 << 16)
                del d
            rows.extend(got)
            nb = out_end(info, off // 2) // bs
            resampled.append(tap_resampled(h, blocks_done, nb))
            blocks_done = nb
        assert keys(rows) == want, path
        allb = np.concatenate(resampled)
        assert np.array_equal(allb, ref[:allb.size]) and allb.size == 2 * blocks_done * bs, path
        # ertgpu_reset clears the resampler too: the stream decodes again from the start
        h.reset()
        assert keys(h.decode(iq, cap=1 << 16)) == want
        h.close()


def test_host_chunking_respects_max_blocks(built):
    """The host path cuts its input so that no pipeline exceeds max_blocks_per_call; the device path refuses a call
    that would, without changing the stream."""
    import torch
    rate_in, cl = 1_024_000, 72   # interpolating: one input sample gives more than two outputs
    iq, _ = stream("scm", rate_in, 400_000, seed=41)
    ref = resample_ref.resample(iq, rate_in, DATA_RATE * cl)
    want = keys(native_of("scm", cl, ref))
    h = capi.new_decoder("scm", cl, input_rate=rate_in, max_blocks_per_call=3)
    assert keys(h.decode(iq, cap=1 << 16)) == want
    h.reset()
    d = torch.from_numpy(iq).cuda()
    with pytest.raises(capi.ErtGpuError) as e:
        h.decode_device_async(d.data_ptr(), d.numel(), 0, torch.cuda.current_stream().cuda_stream)
    assert e.value.code == capi.ESIZE
    rows, step = [], 2 * 4096
    for off in range(0, iq.size, step):
        h.decode_device_async(d.data_ptr() + off, min(step, iq.size - off), 0, torch.cuda.current_stream().cuda_stream)
        rows.extend(h.fetch(cap=1 << 16))
    assert keys(rows) == want
    h.close()


def test_sharded_rejects_resampling_handles(built):
    h = capi.new_decoder("scm", 72, input_rate=2_400_000)
    with pytest.raises(capi.ErtGpuError) as e:
        capi.decode_sharded([h], np.zeros(8192 * 2, dtype=np.uint8))
    assert e.value.code == capi.EINVAL
    h.close()


def test_native_rate_is_a_no_op(built):
    cl = 72
    iq, _ = stream("scm,r900", DATA_RATE * cl, 1 << 21, seed=51)
    a = capi.new_decoder("scm,r900", cl)
    b = capi.new_decoder("scm,r900", cl, input_rate=DATA_RATE * cl)
    bs2 = a.cfg.block_size2
    iqw = iq[:(iq.size // bs2) * bs2]
    ga, gb = a.decode(iqw, cap=1 << 16), b.decode(iqw, cap=1 << 16)
    assert ga.tobytes() == gb.tobytes() and len(ga) > 0
    assert a.last_kernels() == b.last_kernels() and "resample" not in b.last_kernels()
    with pytest.raises(capi.ErtGpuError):  # it has no resampler, and still wants whole blocks
        b.decode(iqw[:bs2 + 2])
    a.close()
    b.close()


@pytest.mark.parametrize("rate_in", [2_400_000, 2_048_000])
@pytest.mark.parametrize("msgtype", ["scm", "scm+", "idm", "r900"])
def test_foreign_rate_packets_are_recovered(built, msgtype, rate_in):
    """Packets rendered at rate_in, decoded at chip length 72 through the resampler in calls of odd sizes (some
    packets straddle a call boundary): every packet comes out with a passing integrity check."""
    cl, n = 72, 2_000_000
    iq, truth = stream(msgtype, rate_in, n, seed=61, spacing=1 << 17)
    assert len(truth) >= 10
    h = capi.new_decoder(msgtype, cl, input_rate=rate_in)
    rows, off = [], 0
    for s in (2 * 123_457, 2 * 300_001, 2 * 77, 2 * 500_000):
        rows.extend(h.decode(iq[off:off + s], cap=1 << 16))
        off += s
    rows.extend(h.decode(iq[off:], cap=1 << 16))
    valid = [r for r in rows if r["check_mask"]]
    for t in truth:
        if msgtype == "r900":
            hit = any([d[2 * k] * 6 + d[2 * k + 1] for k in range(21)] == list(t.data)
                      for d in (r["r900_digits"] for r in valid))
        else:
            hit = any(r["bytes"][:len(t.data)].tobytes() == t.data for r in valid)
        assert hit, (msgtype, t.start_sample, t.meter_id)
    h.close()


def test_64mib_device_resident_window(built):
    """One 64 MiB device-resident call at 2.4 MS/s: candidates equal the native decode of the CPU restatement's
    stream, and sampled blocks of resampled bytes are identical."""
    import torch
    rate_in, cl = 2_400_000, 72
    n = 32 << 20
    iq, _ = stream("scm", rate_in, n, seed=71, spacing=1 << 19)
    ref = resample_ref.resample(iq, rate_in, DATA_RATE * cl)
    h = capi.new_decoder("scm", cl, input_rate=rate_in)
    d = torch.from_numpy(iq).cuda()
    h.decode_device_async(d.data_ptr(), d.numel(), 0, torch.cuda.current_stream().cuda_stream)
    got = h.fetch(cap=1 << 16)
    bs = h.cfg.block_size
    nblocks = (ref.size // 2) // bs
    assert keys(got) == keys(native_of("scm", cl, ref))
    for b in sorted(set(np.random.default_rng(3).integers(0, nblocks, 24).tolist()) | {0, nblocks - 1}):
        assert np.array_equal(h.tap(capi.TAP_RESAMPLED, b), ref[2 * b * bs:2 * (b + 1) * bs]), b
    h.close()


def test_rate_after_allocate_is_rejected(built):
    h = capi.new_decoder("scm", 72)
    with pytest.raises(capi.ErtGpuError) as e:
        h.set_input_rate(2_400_000)
    assert e.value.code == capi.EINVAL and "after allocate" in str(e.value)
    h.close()


def test_sub_block_call_then_reused_buffers(built):
    """ertgpu_decode is synchronous even when a call completes no block: the caller may refill the very buffer at
    once (pinned and pageable).  The device path likewise lets the caller overwrite its input after ertgpu_fetch."""
    import torch
    rate_in, cl = 2_400_000, 72
    iq, _ = stream("scm", rate_in, 1_200_000, seed=81)
    h = capi.new_decoder("scm", cl, input_rate=rate_in)
    want = keys(h.decode(iq, cap=1 << 16))
    assert want
    sizes = [2 * 37, 2 * 1000, 2 * 3, 2 * 150_000, 2 * 5, 2 * 2047, 2 * 400_000]
    sizes.append(iq.size - sum(sizes))
    pinned = torch.empty(max(sizes), dtype=torch.uint8).pin_memory()
    pageable = np.empty(max(sizes), dtype=np.uint8)
    dev = torch.empty(max(sizes), dtype=torch.uint8, device="cuda")
    for path in ("pinned", "pageable", "device"):
        h.reset()
        rows, off = [], 0
        for s in sizes:
            part = iq[off:off + s]
            off += s
            if path == "pinned":
                pinned[:s].copy_(torch.from_numpy(part))
                rows.extend(h.decode((pinned.data_ptr(), s), cap=1 << 16))
                pinned.fill_(0xA5)   # the call has returned: the buffer is the caller's again
            elif path == "pageable":
                pageable[:s] = part
                rows.extend(h.decode((pageable.ctypes.data, s), cap=1 << 16))
                pageable.fill(0xA5)
            else:
                dev[:s].copy_(torch.from_numpy(part).cuda())
                torch.cuda.synchronize()
                st = torch.cuda.Stream()
                h.decode_device_async(dev.data_ptr(), s, 0, st.cuda_stream)
                rows.extend(h.fetch(cap=1 << 16))
                dev.fill_(0xA5)   # on another stream, after fetch
        assert keys(rows) == want, path
    h.close()


def test_two_handles_at_different_rates_alternate(built):
    """The kernel's shared-memory limit is not a property of one handle: a 4:1 decimator (the largest table) allocated
    before a 2.4 MS/s handle keeps working when the two are used alternately."""
    cl = 72
    rates = [4 * DATA_RATE * cl, 2_400_000]
    iqs = [stream("scm", r, 1_600_000, seed=91 + i)[0] for i, r in enumerate(rates)]
    hs = [capi.new_decoder("scm", cl, input_rate=r) for r in rates]
    want = [keys(native_of("scm", cl, resample_ref.resample(iq, r, DATA_RATE * cl))) for iq, r in zip(iqs, rates)]
    rows = [[], []]
    step = 2 * 100_001
    for off in range(0, max(x.size for x in iqs), step):
        for i in (0, 1):
            if off < iqs[i].size:
                rows[i].extend(hs[i].decode(iqs[i][off:off + step], cap=1 << 16))
    for i in (0, 1):
        assert keys(rows[i]) == want[i], rates[i]
        hs[i].close()


CLI = os.path.join(ROOT, "rtlamr_b200", "ertgpu_decode_file")


def run_cli(path, *args):
    out = subprocess.run([CLI, *args, path], capture_output=True, text=True, timeout=300, check=True)
    return out.stdout.splitlines(), out.stderr


# Golden messages (ID) that chip length 72 does not recover from the resampled capture.  No candidate of any kind lies
# within 400 samples of where they sit: the 21-bit preamble never matches in the quantized bit plane there, so the
# search has nothing to hand to the parser.  The other eleven come out bit-identical at the same place (within one
# sample of 72/78 of their chip-length-78 position).
GOLDEN_MISSING_AT_72 = {17564085, 17556728, 17556726}


def test_cli_golden_capture_at_chip_length_72(built):
    """tests/golden/sample_cl78.bin was recorded at 2 555 904 S/s (chip length 78).  Resampled to chip length 72, the
    file receiver reports eleven of the 14 meter messages of the exact search at chip length 78 (ID, type,
    consumption), and nothing else."""
    golden = json.load(open(os.path.join(GOLDEN, "sample_cl78_scm.json")))["exact"]["messages"]
    want = sorted({(m[3], m[4], m[5]) for m in golden if m[3] not in GOLDEN_MISSING_AT_72})
    assert len(want) == 11
    lines, err = run_cli(os.path.join(GOLDEN, "sample_cl78.bin"), "-msgtype=scm", "-symbollength=72",
                         "-samplerate=2555904", "-format=json")
    got = [(m["ID"], m["Type"], m["Consumption"]) for m in (json.loads(l)["Message"] for l in lines)]
    assert sorted(set(got)) == want


def _scm_fields(data: bytes):
    bits = "".join(f"{b:08b}" for b in data)
    return int(bits[21:23] + bits[56:80], 2), int(bits[32:56], 2)


@pytest.mark.parametrize("rate_in", [2_400_000, 2_048_000])
def test_cli_reports_foreign_rate_packets(built, tmp_path, rate_in):
    """Packets rendered at rate_in come out of ertgpu_decode_file -samplerate with their IDs (and, for scm,
    consumption), read in calls of a few blocks so that some packets straddle a call boundary."""
    for msgtype in ("scm", "scm+", "idm", "r900"):
        iq, truth = stream(msgtype, rate_in, 2_000_000, seed=101, spacing=1 << 17)
        path = tmp_path / f"{msgtype}.bin"
        iq.tofile(path)
        lines, err = run_cli(str(path), f"-msgtype={msgtype}", "-symbollength=72", f"-samplerate={rate_in}",
                             "-blocks=3", "-format=json")
        msgs = [json.loads(l)["Message"] for l in lines]
        assert "messages" in err and f"{iq.size / 1e6:.1f} MB" in err
        for t in truth:
            if msgtype == "scm":
                mid, cons = _scm_fields(t.data)
                assert any(m["ID"] == mid and m["Consumption"] == cons for m in msgs), (msgtype, mid)
            elif msgtype == "scm+":
                assert any(m["EndpointID"] == t.meter_id for m in msgs), (msgtype, t.meter_id)
            elif msgtype == "idm":
                assert any(m["ERTSerialNumber"] == t.meter_id for m in msgs), (msgtype, t.meter_id)
            else:
                assert any(m["ID"] == t.meter_id for m in msgs), (msgtype, t.meter_id)


def test_host_receiver_binding_takes_the_rate(built):
    from rtlamr_b200 import host
    rate_in = 2_400_000
    iq, truth = stream("scm", rate_in, 1_000_000, seed=111)
    r = host.Receiver("scm", 72, input_rate=rate_in)
    msgs = r.decode(iq[:2 * 333_333]) + r.decode(iq[2 * 333_333:])
    ids = {_scm_fields(t.data)[0] for t in truth}
    assert ids and ids <= {m.meter_id for m in msgs}
    r.close()
