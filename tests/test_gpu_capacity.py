"""GPU tests (-m gpu) of the candidate capacity, max_candidates, at its boundary.

A decode call runs in steps of max_blocks_per_call blocks, and every preamble match ("hit") of a step takes one of the
handle's max_candidates slots: Search reserves hit and word slots with two counters, and the r900 kernels, Slice and
the signal reports clip their work to the capacity.  A step with more hits than that makes the call return
ERTGPU_ECAPACITY with "internal" in the message and *n_out = the hits of the largest step.

Every case runs a handle at the boundary beside an unbounded twin with the same configuration and the same
max_blocks_per_call.  With flags 0 every hit is one candidate, so the twin's candidates counted by step give the need H;
for the stock protocols the twin itself is checked against the oracle once.  Covered:

  a. one step of several at H - 1, H and H + 1, for scm, scm,scm+,idm, r900 at two chip lengths, densely packed
     scm,scm+,idm,r900 (words of many hits) and an all-ones preamble on constant input (32 hits per word);
  b. the stream after an overflow: the next calls through pageable, pinned and device input, taps and reset;
  c. the r900 chain and replay paths under an overflow;
  d. ERTGPU_DECODE_ONLY_VALID, which does not lower the need;
  e. the output arrays of ertgpu_decode, ertgpu_fetch and ertgpu_fetch_signal;
  f. a channel group in which one handle overflows;
  g. sharded decodes, whose need is the largest of any shard's (halo included)."""
import ctypes as C
import functools

import numpy as np
import pytest

import tune_ref
from helpers import (cand_key_gpu, cand_key_oracle, make_protocol, merged_geometry, oracle_run, r900_preamble_id,
                     synth_stream)
from rtlamr_b200 import capi

pytestmark = pytest.mark.gpu

CAPTURE = 915_000_000

# name: (protocols, chip length, max_blocks_per_call, synth_stream spacing or None for constant input, blocks of the
# first call, blocks of each following call, packet types of the stream when not the protocols)
CONFIGS = {
    "scm@72": ("scm", 72, 8, 1 << 13, 28, 2, None),
    "scm,scm+,idm@72": ("scm,scm+,idm", 72, 8, 1 << 14, 28, 2, None),
    "r900@40": ("r900", 40, 8, 1 << 13, 28, 2, None),
    "r900@72": ("r900", 72, 8, 1 << 14, 28, 2, None),
    "dense@72": ("scm,scm+,idm,r900", 72, 16, 1 << 10, 56, 3, "r900,r900,scm,r900,r900,scm+,r900,r900,idm"),   # back to back
    "ones@72": ("ones", 72, 8, None, 28, 2, None),
}
ONES = make_protocol("1" * 21, 72, 21, 96, capi.CHECK_NONE, name="ones")


def protocols(mt, cl):
    return [ONES] if mt == "ones" else [capi.stock_protocol(m, cl) for m in mt.split(",")]


def new_handle(mt, cl, max_blocks, max_cands=0, signal=False):
    h = capi.Handle()
    for p in protocols(mt, cl):
        h.register(p)
    if signal:
        h.enable_signal()
    h.allocate(0, max_blocks, max_cands)
    return h


@functools.lru_cache(maxsize=None)
def stream(name):
    """(protocols, chip length, max_blocks_per_call, the whole stream, blocks of the first call, of each next call,
    BlockSize2); the stream holds the first call and three following ones."""
    mt, cl, m, spacing, n1, nf, kinds = CONFIGS[name]
    bs = merged_geometry(protocols(mt, cl))["BS"]
    bs2 = 2 * bs
    nblocks = n1 + 3 * nf
    if spacing is None:
        iq = np.zeros(nblocks * bs2, np.uint8)
    else:
        iq, _, _ = synth_stream(kinds or mt, cl, nblocks * bs, spacing=spacing, pkt_seed=cl + len(mt))
    return mt, cl, m, iq[: nblocks * bs2], n1, nf, bs2


def step_hits(cands, first_block, m):
    """Hits per step of m blocks of a call that starts at first_block (flags 0: one candidate per hit)."""
    steps = (cands["block"] - first_block) // m
    return np.bincount(steps.astype(np.int64), minlength=1)


def msg(h):
    return (h._L.ertgpu_last_error(h._h) or b"").decode()


def raw_decode(h, iq, flags=0, cap=0, out=None):
    n = C.c_size_t(0)
    rc = h._L.ertgpu_decode(h._h, iq.ctypes.data, iq.size, flags, None if out is None else out.ctypes.data, cap,
                            C.byref(n))
    return rc, n.value


def raw_fetch(h, out, cap):
    n = C.c_size_t(0)
    rc = h._L.ertgpu_fetch(h._h, None if out is None else out.ctypes.data, cap, C.byref(n))
    return rc, n.value


def raw_fetch_signal(h, out, cap):
    n = C.c_size_t(0)
    rc = h._L.ertgpu_fetch_signal(h._h, None if out is None else out.ctypes.data, cap, C.byref(n))
    return rc, n.value


def assert_overflow(h, need, want_hits, signal):
    """The call on h overflowed its max_candidates: fetch (and fetch_signal) say so, with the need, twice."""
    big = np.empty(need + 64, capi.CAND_DTYPE)
    for _ in range(2):
        assert raw_fetch(h, big, big.size) == (capi.ECAPACITY, need)
        assert "internal" in msg(h), msg(h)
        assert raw_fetch(h, None, 0) == (capi.ECAPACITY, need)
        if signal:
            sig = np.empty(need + 64, capi.SIGNAL_DTYPE)
            assert raw_fetch_signal(h, sig, sig.size) == (capi.ECAPACITY, need)
            assert "internal" in msg(h), msg(h)
    assert h.last_counts()[0] == want_hits


def boundary_handle(name, cap, signal=True):
    mt, cl, m = CONFIGS[name][:3]
    return new_handle(mt, cl, m, cap, signal)


@functools.lru_cache(maxsize=None)
def twin_first_call(name):
    """The unbounded twin's candidates and signal records of the first call, the need H, and the call's hits."""
    mt, cl, m, iq, n1, nf, bs2 = stream(name)
    tw = boundary_handle(name, 0)
    cands = tw.decode(iq[: n1 * bs2], cap=1 << 18)
    sig = tw.fetch_signal(cap=1 << 18)
    hits = tw.last_counts()
    tw.close()
    per_step = step_hits(cands, 0, m)
    return cands, sig, int(per_step.max()), per_step, hits


# ---------------------------------------------------------------- a. the boundary, per step
@pytest.mark.parametrize("name", list(CONFIGS))
def test_step_boundary(built, name):
    mt, cl, m, iq, n1, nf, bs2 = stream(name)
    call = iq[: n1 * bs2]
    want, want_sig, H, per_step, (hits, _) = twin_first_call(name)
    assert n1 >= 3 * m and H >= 32 and hits == len(want), (per_step, hits)
    if mt != "ones":   # H does not rest on the GPU alone
        o, cands, _ = oracle_run(mt, cl, call)
        nb, pks = o.cfg.packet_symbols + 7 >> 3, o.cfg.packet_symbols
        assert sorted(cand_key_gpu(r, nb, pks) for r in want) == sorted(cand_key_oracle(c, nb, pks) for c in cands)
        o.close()
    else:   # (nearly) every start a hit: 32 hits per word
        assert H >= m * bs2 // 4 and (per_step[1:3] == H).all(), per_step
    out = np.empty(len(want) + 64, capi.CAND_DTYPE)
    for cap in (H, H + 1):
        h = boundary_handle(name, cap)
        assert raw_decode(h, call, 0, out.size, out) == (capi.OK, len(want)), (cap, msg(h))
        got = out[: len(want)]
        assert got.tobytes() == want.tobytes(), cap
        assert got["r900_digits"].tobytes() == want["r900_digits"].tobytes()
        assert h.fetch_signal(cap=1 << 18).tobytes() == want_sig.tobytes(), cap
        h.close()
    h = boundary_handle(name, H - 1)
    rc, n = raw_decode(h, call, 0, out.size, out)
    assert (rc, n) == (capi.ECAPACITY, H), (rc, n, H, msg(h))
    assert f"({H} hits)" in msg(h), msg(h)
    assert_overflow(h, H, hits, signal=True)
    h.close()
    again = boundary_handle(name, n)   # the need reported is enough
    assert again.decode(call, cap=1 << 18).tobytes() == want.tobytes()
    again.close()


# ---------------------------------------------------------------- b. the stream after an overflow
def feed(h, part, path):
    """One call on part through pageable, pinned or device input; its candidates."""
    import torch
    if path == "pageable":
        return h.decode(part.copy(), cap=1 << 18)
    if path == "pinned":
        pinned = torch.from_numpy(part.copy()).pin_memory()
        return h.decode((pinned.data_ptr(), part.size), cap=1 << 18)
    d = torch.from_numpy(part.copy()).cuda()
    h.decode_device_async(d.data_ptr(), d.numel(), 0, torch.cuda.current_stream().cuda_stream)
    got = h.fetch(cap=1 << 18)
    del d
    return got


PATHS = ("pageable", "pinned", "device")


def taps(h, block, r900):
    out = [h.tap(capi.TAP_QUANTIZED, block), h.tap(capi.TAP_PACKED, block)]
    if r900:
        out.append(h.tap(capi.TAP_R900_QUANTIZED, block))
    return [t.tobytes() for t in out]


@pytest.mark.parametrize("name", list(CONFIGS))
def test_stream_after_overflow(built, name):
    mt, cl, m, iq, n1, nf, bs2 = stream(name)
    _, _, H, _, _ = twin_first_call(name)
    r900 = "r900" in mt
    h, tw = boundary_handle(name, H - 1, signal=False), boundary_handle(name, 0, signal=False)
    assert raw_decode(h, iq[: n1 * bs2], 0, 0, None) == (capi.ECAPACITY, H)
    tw.decode(iq[: n1 * bs2], cap=1 << 18)
    # A candidate of block b at idx starts at sample b*BS + idx - PacketLength: calls of at most PacketLength samples
    # hold only packets that began in front of them, across the seam.
    assert nf * h.cfg.block_size <= h.cfg.packet_length
    a, seen = n1, 0
    for path in PATHS:
        part = iq[a * bs2:(a + nf) * bs2]
        want = feed(tw, part, path)
        assert int(step_hits(want, a, m).max()) < H - 1, path   # the call itself fits
        got = feed(h, part, path)
        assert got.tobytes() == want.tobytes(), path
        seen += len(want)
        a += nf
    assert seen > 0
    assert taps(h, a - 1, r900) == taps(tw, a - 1, r900)
    # reset: the handle equals a fresh one
    h.reset()
    fresh = boundary_handle(name, 0, signal=False)
    part = iq[n1 * bs2:(n1 + nf) * bs2]
    assert h.decode(part, cap=1 << 18).tobytes() == fresh.decode(part, cap=1 << 18).tobytes()
    assert taps(h, nf - 1, r900) == taps(fresh, nf - 1, r900)
    for x in (h, tw, fresh):
        x.close()


# ---------------------------------------------------------------- c. the r900 paths under overflow
def test_r900_paths_under_overflow(built, monkeypatch):
    name = "dense@72"
    mt, cl, m, iq, n1, nf, bs2 = stream(name)
    want, _, H, _, _ = twin_first_call(name)
    r9 = want[want["preamble_id"] == r900_preamble_id(mt)]
    D = int(np.bincount(np.unique(r9["block"]) // m).max())   # most detecting blocks of a step
    assert len(r9) >= 32 and D >= 2, (len(r9), D)
    tw = boundary_handle(name, 0, signal=False)
    tw.decode(iq[: n1 * bs2], cap=1 << 18)
    rest = iq[n1 * bs2:]   # the three following calls as one
    nxt = tw.decode(rest, cap=1 << 18)
    assert len(nxt) > 0
    for slots in (None, 1, max(1, D // 2)):
        for cap in (H - 1, H // 2):
            if slots is not None:
                monkeypatch.setenv("ERTGPU_R900_SLOTS", str(slots))
            h = boundary_handle(name, cap, signal=False)
            monkeypatch.delenv("ERTGPU_R900_SLOTS", raising=False)
            assert raw_decode(h, iq[: n1 * bs2], 0, 0, None) == (capi.ECAPACITY, H), (slots, cap, msg(h))
            assert "internal" in msg(h)
            assert int(step_hits(nxt, n1, m).max()) < cap
            assert h.decode(rest, cap=1 << 18).tobytes() == nxt.tobytes(), (slots, cap)
            h.close()
    tw.close()


# ---------------------------------------------------------------- d. ERTGPU_DECODE_ONLY_VALID does not lower the need
def test_only_valid_needs_every_hit(built):
    mt, cl, _, iq, _, _, bs2 = stream("dense@72")
    m = 16
    iq = iq[: m * bs2]   # one step
    h0 = new_handle(mt, cl, m)
    every = h0.decode(iq, cap=1 << 18)
    H = len(every)
    h0.reset()
    valid = h0.decode(iq, flags=capi.DECODE_ONLY_VALID, cap=1 << 18)
    V = len(valid)
    assert 1 <= V < H and (valid["check_mask"] != 0).all(), (V, H)
    assert valid.tobytes() == every[every["check_mask"] != 0].tobytes()
    out = np.empty(H + 8, capi.CAND_DTYPE)
    for cap in (V, H - 1):
        h = new_handle(mt, cl, m, cap)
        assert raw_decode(h, iq, capi.DECODE_ONLY_VALID, out.size, out) == (capi.ECAPACITY, H), cap
        assert "internal" in msg(h)
        h.close()
    h = new_handle(mt, cl, m, H)
    assert h.decode(iq, flags=capi.DECODE_ONLY_VALID, cap=H).tobytes() == valid.tobytes()
    assert h.last_counts() == (H, V)
    h.close()
    h0.close()


# ---------------------------------------------------------------- e. the output arrays
def test_output_arrays(built):
    mt, cl = "scm", 72
    h = new_handle(mt, cl, 0, signal=True)
    bs, bs2 = h.cfg.block_size, h.cfg.block_size2
    iq, _, _ = synth_stream(mt, cl, 24 * bs, spacing=1 << 14, pkt_seed=5)
    iq = iq[: 24 * bs2]
    want = h.decode(iq, cap=1 << 16)
    want_sig = h.fetch_signal()
    n = len(want)
    assert n >= 8
    out, sig = np.empty(n, capi.CAND_DTYPE), np.empty(n, capi.SIGNAL_DTYPE)
    for first_cap in (n - 1, 0):
        h.reset()
        arr = out if first_cap else None
        assert raw_decode(h, iq, 0, first_cap, arr) == (capi.ECAPACITY, n)
        assert "output array" in msg(h)
        for cap, a in ((n - 1, out), (0, None), (0, out)):   # nothing is lost, however often it is asked
            assert raw_fetch(h, a, cap) == (capi.ECAPACITY, n)
            assert raw_fetch_signal(h, None if a is None else sig, cap) == (capi.ECAPACITY, n)
        for _ in range(2):   # a successful fetch may be repeated
            out.view(np.uint8)[:] = 0
            assert raw_fetch(h, out, n) == (capi.OK, n)
            assert out.tobytes() == want.tobytes()
            assert raw_fetch_signal(h, sig, n) == (capi.OK, n)
            assert sig.tobytes() == want_sig.tobytes()
    h.reset()
    assert raw_decode(h, iq, 0, n, out) == (capi.OK, n) and out.tobytes() == want.tobytes()
    h.close()


# ---------------------------------------------------------------- f. channel groups
RATE_IN = 8_000_000
OFFSETS = (-2_400_000, 7, 2_400_014)


def tuned(off, cap=0):
    return capi.new_decoder("scm", 72, input_rate=RATE_IN, input_format=capi.FORMAT_CS8, capture_freq=CAPTURE,
                            center_freq=CAPTURE + off, max_candidates=cap)


@pytest.mark.parametrize("path", ["host", "device"])
def test_channel_group_with_one_overflow(built, path):
    import torch
    z, _ = tune_ref.wideband([("scm", o, 61 + k, 0) for k, o in enumerate(OFFSETS)], RATE_IN, 3_000_000, 61)
    raw = tune_ref.quantize(z, capi.FORMAT_CS8)
    first, second = raw[: 2 * 2_400_000], raw[2 * 2_400_000:]
    lones = [tuned(o) for o in OFFSETS]
    want1, hits = [], []
    for t in lones:   # each call is one input-stage step: the twin's count is the need
        want1.append(t.decode(first, cap=1 << 16))
        hits.append(t.last_counts()[0])
        assert hits[-1] == len(want1[-1])
    want2 = [t.decode(second, cap=1 << 16) for t in lones]
    H = hits[1]
    assert H >= 32 and len(want2[1]) < H - 1, (hits, len(want2[1]))
    group = [tuned(OFFSETS[0]), tuned(OFFSETS[1], H - 1), tuned(OFFSETS[2])]
    if path == "host":
        capi._channel_call(group, lambda hs, n: capi.lib().ertgpu_decode_channels(hs, n, first.ctypes.data, first.size, 0))
    else:
        d = torch.from_numpy(first.copy()).cuda()
        capi.decode_channels_device_async(group, d.data_ptr(), d.numel(), 0, torch.cuda.current_stream().cuda_stream)
    for k in (0, 2):
        assert group[k].fetch(cap=1 << 16).tobytes() == want1[k].tobytes(), k
    assert_overflow(group[1], H, H, signal=False)
    if path == "device":
        del d
    got = capi.decode_channels(group, second, cap=1 << 16)
    for k in range(3):
        assert got[k].tobytes() == want2[k].tobytes(), k
    for x in lones + group:
        x.close()


# ---------------------------------------------------------------- g. sharded decodes
class CountingLib:
    """capi.lib() with a count of ertgpu_decode_sharded calls."""

    def __init__(self, real):
        self._real, self.sharded = real, 0

    def __getattr__(self, name):
        return getattr(self._real, name)

    def ertgpu_decode_sharded(self, *a):
        self.sharded += 1
        return self._real.ertgpu_decode_sharded(*a)


def test_sharded_overflow_reports_the_largest_need(built, monkeypatch):
    mt, cl, m, nshards = "scm", 72, 8, 3
    h0 = new_handle(mt, cl, m)
    bs, bs2, pkl = h0.cfg.block_size, h0.cfg.block_size2, h0.cfg.packet_length
    nblocks = 60
    iq, _, _ = synth_stream(mt, cl, nblocks * bs, spacing=1 << 13, pkt_seed=17)
    iq = iq[: nblocks * bs2]
    single = h0.decode(iq, cap=1 << 18)
    needs = []
    for first, last, fed in capi.plan_shards(nblocks, nshards, bs, pkl):   # a shard decodes its halo and its blocks
        h0.reset()
        needs.append(int(step_hits(h0.decode(iq[fed * bs2:last * bs2], cap=1 << 18), 0, m).max()))
    h0.close()
    need = max(needs)
    assert len(set(needs)) > 1 and min(needs) >= 32, needs
    handles = [new_handle(mt, cl, m, min(needs) - 1) for _ in range(nshards)]   # every shard overflows
    hs = (C.c_void_p * nshards)(*[h._h for h in handles])
    out = np.empty(len(single) + 64, capi.CAND_DTYPE)
    n = C.c_size_t(0)
    rc = capi.lib().ertgpu_decode_sharded(hs, nshards, iq.ctypes.data, iq.size, 0, out.ctypes.data, out.size, C.byref(n))
    assert (rc, n.value) == (capi.ECAPACITY, need), (rc, n.value, needs)
    for h, nd in zip(handles, needs):
        assert "internal" in msg(h) and f"({nd} hits)" in msg(h), msg(h)
    counting = CountingLib(capi.lib())
    monkeypatch.setattr(capi, "lib", lambda: counting)
    with pytest.raises(capi.ErtGpuError) as e:
        capi.decode_sharded(handles, iq, cap=1)
    assert e.value.code == capi.ECAPACITY and "internal" in str(e.value)
    assert counting.sharded == 1   # raised at once: no second decode
    for h in handles:
        h.close()
    handles = [new_handle(mt, cl, m, need) for _ in range(nshards)]
    counting.sharded = 0
    assert capi.decode_sharded(handles, iq, cap=1).tobytes() == single.tobytes()   # an array too small: decoded again
    assert counting.sharded == 2
    monkeypatch.undo()
    for h in handles:
        h.close()
