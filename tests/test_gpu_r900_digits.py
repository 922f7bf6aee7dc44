"""Every r900 payload digit the GPU writes against the CPU oracle's r900 parser (tests/helpers.py oracle_r900_digits).

The 42 digits of an r900 candidate come from r900_mark_kernel -> r900_chain2_kernel -> r900_digits_kernel (one running
sum per detecting block, built by producer / consumer warps) or, for blocks that found no scratch slot, from
r900_replay_kernel.  Here they are compared digit for digit, with the r900 check_mask bits recomputed from the oracle's
digits, at the shapes where those kernels go wrong:

  * chip lengths: every specialised one (each gives its own span and partial last hand-off unit), one without a fast
    demod kernel, r900bcd, and merged sets whose BufferLength puts a chain's start many blocks back;
  * call seams: calls shorter than BufferLength / BlockSize, so chains start in history assembled by several carries or
    before the stream, with packets across the seams and inside the first BufferLength samples;
  * scratch overflow: calls served by replay only, by chain and replay, by the chain only;
  * multi-pass chain schedule: more detecting blocks than one pass of the chain grid.

The CPU tests check the oracle helper itself.  The last test checks that every r900 path was seen."""
import os
import re

import numpy as np
import pytest

import oracle
from helpers import compare_r900_digits, oracle_r900_digits, r900_preamble_id, r900_symbols, whole_blocks
from rtlamr_b200 import capi, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu

FAST_CLS = [32, 40, 48, 56, 64, 72, 78, 80, 88, 96]
SEEN = set()   # r900 paths the GPU tests ran: chain_only, mixed, mostly_replay, multi_pass, carried_history
STRONG, WEAK = (24, 60), (3, 6)   # carrier amplitudes (noise: about 4.6 per component); weak digits fail the screen


def geometry(mt, cl):
    o = oracle.Oracle(mt, cl)
    c = o.cfg
    g = {"BS": c.block_size, "bs2": c.block_size2, "SL": c.symbol_length, "PL": c.preamble_length,
         "PKL": c.packet_length, "BUF": c.buffer_length}
    o.close()
    return g


def r900_rows(cl, starts, amplitude, seed):
    """r900 packets (random fields) starting at `starts`."""
    pk, _ = synth.make_packets("r900", cl, len(starts) << 16, seed=seed, spacing=1 << 16, amplitude=amplitude)
    pk["start_sample"] = starts
    return pk


def fill(nsamples, seed, *tables):
    pk = np.sort(np.concatenate(tables), order="start_sample")
    plen = 232 * int(pk["chip_length"][0])
    assert np.all(np.diff(pk["start_sample"]) > plen), "packets overlap"
    return synth.host_fill(0, nsamples, seed, pk)


def seam_sweep(mt, cl, nblocks, seed):
    """A stream of nblocks blocks with one r900 packet every few blocks.  A packet at sample s is found at
    idx ~ s - ((b+1)*BS - BUF) + SL +- CL of block b, so starts -BUF - SL + delta (mod BS), delta swept over [-CL, CL],
    put each packet's candidates on both sides of a block seam.  Strong and weak packets alternate."""
    g = geometry(mt, cl)
    BS, plen = g["BS"], 232 * cl
    step = -(-(plen + 2 * BS) // BS) + 1
    seams = np.arange(step, nblocks - step, step)
    delta = -cl + (np.arange(seams.size) * 2 * cl) // max(1, seams.size - 1)
    starts = (seams * BS - (g["BUF"] + g["SL"]) % BS + delta).astype(np.int64)
    strong = r900_rows(cl, starts[0::2], STRONG, seed)
    weak = r900_rows(cl, starts[1::2], WEAK, seed + 1)
    return fill(nblocks * BS, 0x5EED0700 + seed, strong, weak)[: nblocks * g["bs2"]]


def chain_grid():
    """(CTAs per SM, chains per CTA) of the r900_chain2_kernel launch, read from the source."""
    src = open(os.path.join(ROOT, "rtlamr_b200", "csrc", "ertgpu.cu")).read()
    per_sm = re.findall(r"r900_chain2_kernel<<<\(unsigned\)h->sm_count \* (\d+), \(kChainProducers \+ 1\) \* 32", src)
    src = open(os.path.join(ROOT, "rtlamr_b200", "csrc", "search.cuh")).read()
    per_cta = re.findall(r"constexpr int kChainsPerCta = (\d+);", src)
    assert len(per_sm) == 1 and len(per_cta) == 1, (per_sm, per_cta)
    return int(per_sm[0]), int(per_cta[0])


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def detecting_blocks(want):
    return len({b for b, _, _ in want})


def handle(mt, cl, max_blocks=0, max_cands=0, slots=None, monkeypatch=None):
    if slots is not None:
        monkeypatch.setenv("ERTGPU_R900_SLOTS", str(slots))
    h = capi.new_decoder(mt, cl, max_blocks_per_call=max_blocks, max_candidates=max_cands)
    if slots is not None:
        monkeypatch.delenv("ERTGPU_R900_SLOTS")
    return h


def kernels(h):
    k = h.last_kernels().split(";")
    assert "r900_replay_kernel" not in k, k     # the chain geometry: replay only serves blocks without a slot
    assert "r900_chain2_kernel" in k, k
    return k


# ---------------------------------------------------------------- CPU: the oracle helper
@pytest.mark.parametrize("mt,cl", [("r900", 32), ("r900bcd", 72), ("scm,r900", 40)])
def test_helper_digits_rebuild_the_oracle_messages(mt, cl):
    """For every r900 / r900bcd message the oracle's parsers emit, the helper's digits at its (block, idx) give its 21
    symbols, meter id and consumption (r900.go:199-227, r900bcd.go:63-65)."""
    g = geometry(mt, cl)
    iq = seam_sweep(mt, cl, 160, cl)
    want = oracle_r900_digits(mt, cl, iq)
    o = oracle.Oracle(mt, cl, oracle.SEARCH_GO)
    _, msgs = o.decode(whole_blocks(iq, g["bs2"]), cand_cap=1 << 16, msg_cap=1 << 12)
    pid = r900_preamble_id(mt)
    msgs = [m for m in msgs if oracle.PROTO_NAMES[m.proto] in ("r900", "r900bcd")]
    assert len(msgs) >= 8
    for m in msgs:
        sym = r900_symbols(want[(m.block, m.idx, pid)])
        assert sym is not None and bytes(sym) == m.data, m
        bits = "".join(format(s, "05b") for s in sym)
        assert int(bits[:32], 2) == m.meter_id
        cons = int(bits[48:72], 2)
        if oracle.PROTO_NAMES[m.proto] == "r900bcd":
            h = format(cons, "x")
            cons = int(h) if h.isdigit() else 0
        assert cons == m.consumption, m


def test_helper_is_independent_of_the_segment_cuts():
    """Segments cut at every block, at random blocks, and only at the detecting blocks give the same digits;
    first_block only renumbers the blocks."""
    mt, cl = "r900", 32
    iq = seam_sweep(mt, cl, 96, 5)
    nblk = iq.size // geometry(mt, cl)["bs2"]
    base = oracle_r900_digits(mt, cl, iq)
    assert len(base) > 100 and detecting_blocks(base) >= 10
    rng = np.random.default_rng(0)
    assert oracle_r900_digits(mt, cl, iq, cuts=range(nblk)) == base
    assert oracle_r900_digits(mt, cl, iq, cuts=rng.choice(nblk, 20, replace=False)) == base
    shifted = oracle_r900_digits(mt, cl, iq, first_block=7)
    assert shifted == {(b + 7, i, p): d for (b, i, p), d in base.items()}


# ---------------------------------------------------------------- 1. chip lengths and message sets
MATRIX = [("r900", cl) for cl in FAST_CLS + [16]] + [("r900bcd", 40), ("r900bcd", 88)] + \
         [(mt, cl) for mt in ("scm,r900", "scm+,idm,r900", "scm,scm+,idm,r900") for cl in (32, 56, 72, 96)]
COMPARED = {}   # case -> (records compared, failing the screen[, detecting blocks, chain grid capacity])


@gpu
@pytest.mark.parametrize("mt,cl", MATRIX)
def test_digits_by_chip_length(built, mt, cl):
    g = geometry(mt, cl)
    nblocks = 16 * 32 + 7                       # at least 16 demod work tiles
    iq = seam_sweep(mt, cl, nblocks, cl)
    h = handle(mt, cl, max_blocks=nblocks, max_cands=1 << 16)
    got = h.decode(iq, cap=1 << 16)
    k = kernels(h)
    if cl not in FAST_CLS:
        assert k[0] == "demod_generic_kernel", k
    want = oracle_r900_digits(mt, cl, iq)
    n, fails = compare_r900_digits(got, mt, want)
    COMPARED[(mt, cl)] = (n, fails)
    SEEN.add("chain_only")
    idx = {i for _, i, _ in want}
    assert 0 in idx and g["BS"] - 1 in idx, (min(idx), max(idx))
    assert n >= 500 and fails >= 30, (n, fails)
    assert n - fails >= 10          # the strong packets pass the screen
    h.close()


# ---------------------------------------------------------------- 2. call seams and the start of the stream
def rounding_probe(iq, g, start, cl):
    """The payload of the packet at `start` replaced by one random chip of IQ bytes repeated: every 4-chip correlator
    is zero in exact arithmetic, so the digits are decided by the float32 rounding of the running sum alone.  Where the
    sums cross a power of two that rounding depends on every sample added before, so a sample added to or dropped
    from the chain in front of them changes digits."""
    a, b = 2 * (start + g["PL"]), 2 * (start + 232 * cl + 4 * cl)
    chip = np.random.default_rng(start).integers(96, 160, 2 * cl, dtype=np.uint8)
    iq[a:b] = np.resize(chip, b - a)
    return iq


SEAM_CASES = [("r900", 32), ("scm,scm+,idm,r900", 32), ("scm,scm+,idm,r900", 72)]


@gpu
@pytest.mark.parametrize("mt,cl", SEAM_CASES)
def test_call_seams_and_stream_start(built, mt, cl):
    """Host-path calls of 1, 1, 2, 3, 5 and random block counts, chunked by max_blocks_per_call, against the oracle fed
    the same bytes as one stream.  Packets start inside the first BufferLength samples (chains that begin before the
    stream, while the carried history is still filling) and across call seams; the first ones carry rounding probes."""
    g = geometry(mt, cl)
    BS, plen = g["BS"], 232 * cl
    nblocks = max(160, 3 * g["BUF"] // BS)
    rng = np.random.default_rng(cl)
    sizes = [1, 1, 2, 3, 5]
    while sum(sizes) < nblocks:
        sizes.append(int(min(nblocks - sum(sizes), rng.integers(1, 24))))
    seams = np.cumsum(sizes)[:-1]
    starts = [100, 100 + plen + 4 * cl + 3 * BS // 5]
    for i, s in enumerate(seams[4:]):
        if i % 2:    # a packet across the call seam
            want = int(s) * BS - plen // 2 + int(rng.integers(-BS // 2, BS // 2))
        else:        # a packet of earlier calls whose candidates sit in the call's first block: its chain reads only history
            want = (int(s) + 1) * BS - g["BUF"] - g["SL"] + int(rng.integers(-cl, BS // 2))
        starts.append(want)
    kept = []
    for s in sorted(starts):
        if s >= 0 and (not kept or s > kept[-1] + plen + 4 * cl):
            kept.append(s)
    starts = kept
    starts = np.array([s for s in starts if s + plen + 8 * cl < nblocks * BS], dtype=np.int64)
    weak = np.zeros(starts.size, bool)
    weak[2::3] = True
    iq = fill(nblocks * BS, 0x5EED0710 + cl, r900_rows(cl, starts[~weak], STRONG, cl),
              r900_rows(cl, starts[weak], WEAK, cl + 1))
    iq[0], iq[1] = 100, 150              # stream sample 0: a magnitude whose addition rounds
    for s in starts[:2]:
        rounding_probe(iq, g, int(s), cl)
    want = oracle_r900_digits(mt, cl, iq)
    early = [k for k in want if (k[0] + 1) * BS < g["BUF"]]      # chains that start before the stream
    assert len(early) >= 20 or g["BUF"] % BS == 0   # (b + 1) * BS - BUF < 0 with idx < BS needs BUF % BS != 0

    h1 = handle(mt, cl)
    whole = h1.decode(iq, cap=1 << 16)
    kernels(h1)
    n, fails = compare_r900_digits(whole, mt, want)
    h2 = handle(mt, cl, max_blocks=4)
    parts, off = [], 0
    for m in sizes:
        part = h2.decode(iq[off * g["bs2"]:(off + m) * g["bs2"]], cap=1 << 16)
        if off > 0 and ((part["block"] == off) & (part["preamble_id"] == r900_preamble_id(mt))).any():
            SEEN.add("carried_history")
        parts.append(part)
        off += m
    split = np.concatenate(parts)
    compare_r900_digits(split, mt, want)
    assert len(split) == len(whole)
    for f in ("block", "idx", "preamble_id", "check_mask", "flags", "bytes", "r900_digits"):
        assert np.array_equal(split[f], whole[f]), f
    COMPARED[("seams", mt, cl)] = (n, fails)
    assert n >= 200 and fails >= 40, (n, fails)

    # reset == a fresh handle
    first = 2 * g["BUF"] // BS
    h2.reset()
    again = h2.decode(iq[: first * g["bs2"]], cap=1 << 16)
    fresh = handle(mt, cl).decode(iq[: first * g["bs2"]], cap=1 << 16)
    for f in ("block", "idx", "preamble_id", "check_mask", "flags", "r900_digits"):
        assert np.array_equal(again[f], fresh[f]), f
    compare_r900_digits(again, mt, {k: v for k, v in want.items() if k[0] < first})
    h1.close()
    h2.close()


# ---------------------------------------------------------------- 3. scratch overflow
@gpu
@pytest.mark.parametrize("mt,cl", [("r900", 40), ("scm,scm+,idm,r900", 72)])
def test_scratch_overflow(built, monkeypatch, mt, cl):
    """ERTGPU_R900_SLOTS at 1, half the detecting blocks, all but one and exactly all of them: one call served mostly
    by replay, by chain and replay, by the chain with one replayed block, by the chain alone."""
    g = geometry(mt, cl)
    nblocks = 300
    iq = seam_sweep(mt, cl, nblocks, cl + 3)
    want = oracle_r900_digits(mt, cl, iq)
    D = detecting_blocks(want)
    assert D >= 30
    for slots, path in ((1, "mostly_replay"), (D // 2, "mixed"), (D - 1, "mixed"), (D, "chain_only")):
        h = handle(mt, cl, max_blocks=nblocks, max_cands=1 << 16, slots=slots, monkeypatch=monkeypatch)
        got = h.decode(iq, cap=1 << 16)
        assert "r900_chain2_kernel" in h.last_kernels().split(";")
        n, fails = compare_r900_digits(got, mt, want)
        assert n >= 300 and fails >= 50, (slots, n, fails)
        SEEN.add(path)
        h.close()


# ---------------------------------------------------------------- 4. more detecting blocks than one pass of the chain grid
@gpu
@pytest.mark.parametrize("cl", [32, 64])
def test_multi_pass_chain_schedule(built, monkeypatch, cl):
    """One device-resident call whose detecting blocks fill the chain grid (2 CTAs per SM x kChainsPerCta chains) three
    times and part of a fourth: the slot0 loop, the barrier phases carried from one group of chains to the next and
    the producer drain all run.  Packets back to back; every detecting block has a scratch slot."""
    import torch
    mt = "r900"
    g = geometry(mt, cl)
    per_sm, per_cta = chain_grid()
    cap = sm_count() * per_sm * per_cta
    npk = 3 * cap + cap // 3 + 200
    plen = 232 * cl
    pk, _ = synth.make_packets(mt, cl, npk * (plen // 2), seed=cl, spacing=plen // 2)
    assert len(pk) == npk
    nblocks = -(-(int(pk["start_sample"][-1]) + plen) // g["BS"]) + 2
    h = handle(mt, cl, max_blocks=nblocks, max_cands=1 << 22, slots=npk + 4096, monkeypatch=monkeypatch)
    d = torch.empty(nblocks * g["bs2"], dtype=torch.uint8, device="cuda")
    capi.synth_fill(0, d.data_ptr(), 0, nblocks * g["BS"], 0x5EED0720 + cl, pk)
    torch.cuda.synchronize()
    h.decode_device_async(d.data_ptr(), d.numel(), 0, torch.cuda.current_stream().cuda_stream)
    got = h.fetch(1 << 20)
    kernels(h)
    iq = d.cpu().numpy()
    del d
    want = oracle_r900_digits(mt, cl, iq)
    D = detecting_blocks(want)
    assert 3 * cap <= D < npk + 4096 and D % cap != 0, (D, cap)
    n, fails = compare_r900_digits(got, mt, want)
    COMPARED[("multi_pass", cl)] = (n, fails, D, cap)
    assert n >= 20 * D and fails >= D // 2, (n, fails)
    SEEN.add("multi_pass")
    h.close()


# ---------------------------------------------------------------- coverage
def test_chain_grid_restatement():
    per_sm, per_cta = chain_grid()
    assert per_sm == 2 and per_cta == 16


@gpu
def test_every_r900_path_was_seen(built):
    """Runs last: chain only, chain and replay in one call, mostly replay, several passes of the chain grid and
    call-first blocks whose chains read carried history were all compared with the oracle above."""
    if not SEEN:
        pytest.skip("collects what the other tests of this file ran: run the whole file")
    for k, v in sorted(COMPARED.items(), key=str):
        print("r900 digits compared", k, v)
    assert SEEN == {"chain_only", "mixed", "mostly_replay", "multi_pass", "carried_history"}, SEEN
