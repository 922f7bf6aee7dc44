"""Full-size checks at BASELINE.json's sizes, one GPU (SURVEY.md section 8d correctness gate):

  configs[1]  scm           ChipLength 72, 1 GiB   (131 072 blocks of 4096 samples)
  configs[2]  scm,scm+,idm  ChipLength 72, 8 GiB   (524 288 blocks of 8192; three preambles in one pass)
  configs[3]  r900          ChipLength 72, 4 GiB   (262 144 blocks of 8192; incl. the parser's filter+quantize)
  configs[4]  scm           ChipLength 72, 8 GiB   (the per-GPU share of the 64 GiB / 8 GPU run)

Size-independent properties (every injected packet decodes and nothing else passes a screen, sorted unique
output, one call == many calls, N shards with halo == one stream) plus bit-exact comparison with the CPU oracle
on windows of the stream: its start, places that hold a packet, every seam of an 8-way shard plan that is
checked, and the very end."""
import numpy as np
import pytest

import oracle
from helpers import assert_check_masks_exact, cand_key_gpu, cand_key_oracle, compare_r900_digits, oracle_r900_digits
from rtlamr_b200 import capi, shard, synth

pytestmark = pytest.mark.gpu

CL = 72
CONFIGS = {
    "scm1g": ("scm", 1 << 30, 0x5EED0002),
    "multi8g": ("scm,scm+,idm", 8 << 30, 0x5EED0003),
    "r9004g": ("r900", 4 << 30, 0x5EED0004),
    "scm8g": ("scm", 8 << 30, 0x5EED0005),
}
KEY_BYTES = {"scm": 12, "scm+": 16, "idm": 92}


class Big:
    def __init__(self, name):
        import torch
        self.name = name
        self.mt, self.nbytes, self.seed = CONFIGS[name]
        self.msgtypes = self.mt.split(",")
        probe = capi.new_decoder(self.mt, CL, max_blocks_per_call=1)
        self.bs, self.bs2, self.pkl, self.buf = (probe.cfg.block_size, probe.cfg.block_size2, probe.cfg.packet_length,
                                                 probe.cfg.buffer_length)
        self.pk_symbols = probe.cfg.packet_symbols
        probe.close()
        self.nblocks = self.nbytes // self.bs2
        self.nsamples = self.nbytes // 2
        self.h = capi.new_decoder(self.mt, CL, max_blocks_per_call=self.nblocks, max_candidates=1 << 20)
        self.pk, self.truth = synth.make_packets(self.mt, CL, self.nsamples, seed=1, spacing=1 << 20)
        self.d = torch.empty(self.nbytes, dtype=torch.uint8, device="cuda")
        capi.synth_fill(0, self.d.data_ptr(), 0, self.nsamples, self.seed, self.pk)
        self.stream = torch.cuda.Stream()
        self.h.decode_device_async(self.d.data_ptr(), self.nbytes, 0, self.stream.cuda_stream)
        self.got = self.h.fetch(1 << 20)

    def close(self):
        self.h.close()
        self.d = None


@pytest.fixture(scope="module", params=list(CONFIGS))
def big(built, request):
    import torch
    b = Big(request.param)
    yield b
    b.close()
    torch.cuda.empty_cache()


def truth_key(t):
    return (t.msgtype, t.data)


def valid_keys(got, msgtypes):
    keys = set()
    for i, mt in enumerate(msgtypes):
        sel = got[(got["check_mask"] >> i) & 1 == 1]
        if mt == "r900":
            d = sel["r900_digits"].astype(np.int32)
            sym = d[:, 0::2] * 6 + d[:, 1::2]
            keys |= {(mt, bytes(r.astype(np.uint8))) for r in np.unique(sym, axis=0)}
        else:
            keys |= {(mt, bytes(r)) for r in np.unique(sel["bytes"][:, :KEY_BYTES[mt]], axis=0)}
    return keys


def test_every_injected_packet_is_recovered_and_nothing_else(big):
    b = big
    usable = [t for t in b.truth if t.start_sample + b.buf < b.nsamples]
    assert len(usable) >= len(b.truth) - 1 >= 500
    keys = valid_keys(b.got, b.msgtypes)
    missing = [t for t in usable if truth_key(t) not in keys]
    assert not missing
    # nothing passes a screen that was not injected -- except what a 16-bit CRC lets through on noise: the 16-bit scm+
    # preamble matches ~2^-16 of all start positions of an 8 GiB stream (~65 000 noise candidates), each of which
    # passes the CCITT check with probability 2^-16 (the parser's ProtocolID test, scmplus.go:84, is not a GPU screen)
    extra = keys - {truth_key(t) for t in b.truth}
    assert all(k[0] == "scm+" for k in extra) and len(extra) <= 8, extra
    # candidates are sorted by (block, preamble, idx) and unique
    key = (b.got["block"].astype(np.int64) * 4 + b.got["preamble_id"]) * 8192 + b.got["idx"]
    assert np.all(np.diff(key) > 0)
    assert int(b.got["block"].max()) < b.nblocks and int(b.got["idx"].max()) < b.bs


def window_starts(b):
    """Block ranges compared with the oracle: stream start, two packets, seams of the 8-way shard plan, the end."""
    n = 512 if b.bs == 8192 else 1024
    plans = shard.plan(b.nblocks, 8, b.bs, b.pkl)
    ti = [len(b.truth) // 4, (3 * len(b.truth)) // 4]
    starts = [0] + [max(0, int(b.truth[i].start_sample // b.bs) - n // 3) for i in ti]
    starts += [plans[k].first_block - n // 2 for k in (1, 4, 7)]      # windows straddling shard seams
    starts += [b.nblocks - n]
    return n, starts


def test_windows_match_the_oracle_bit_for_bit(big):
    b = big
    halo = shard.halo_blocks(b.bs, b.pkl)
    n, starts = window_starts(b)
    nbytes_key = (b.pk_symbols + 7) >> 3
    total_cands = 0
    for w0 in starts:
        w1 = min(b.nblocks, w0 + n)
        f0 = max(0, w0 - halo)
        iq = b.d[f0 * b.bs2:w1 * b.bs2].cpu().numpy()
        # the device generator and the host generator agree on this window
        assert np.array_equal(iq[:1 << 16], synth.host_fill(f0 * b.bs, 1 << 15, b.seed, b.pk))
        o = oracle.Oracle(b.mt, CL, oracle.SEARCH_GO)
        cands, msgs = o.decode(iq, cand_cap=1 << 18)
        want = sorted(cand_key_oracle(c, nbytes_key, b.pk_symbols) for c in cands if c.block + f0 >= w0)
        want = [(k[0] + f0,) + k[1:] for k in want]
        sel = b.got[(b.got["block"] >= w0) & (b.got["block"] < w1)]
        have = sorted(cand_key_gpu(r, nbytes_key, b.pk_symbols) for r in sel)
        assert have == want, (b.name, w0, len(have), len(want))
        total_cands += len(want)
        assert_check_masks_exact(sel, b.mt)
        if "r900" in b.msgtypes:   # every r900 candidate's 42 digits against the r900 parser fed the window, halo included
            digits = {k: v for k, v in oracle_r900_digits(b.mt, CL, iq, first_block=f0).items() if k[0] >= w0}
            assert compare_r900_digits(sel, b.mt, digits)[0] > 0
        # the parsers' verdicts: every message the oracle's parsers emit sits on a candidate with that bit set
        protos = oracle.proto_ids(b.mt)
        masks = {(int(r["block"]), int(r["idx"])): int(r["check_mask"]) for r in sel}
        for m in msgs:
            if m.block + f0 >= w0:
                assert masks[(m.block + f0, m.idx)] & (1 << protos.index(m.proto)), m
        # Quantized (and the r900 parser's quantized) of the window's last block, bit for bit.  The tap works on the
        # last decode call of a handle: a second handle replays the window's blocks from the same device bytes.
        h2 = capi.new_decoder(b.mt, CL, max_blocks_per_call=w1 - f0)
        h2.decode_device_async(b.d.data_ptr() + f0 * b.bs2, (w1 - f0) * b.bs2, 0, b.stream.cuda_stream)
        h2.fetch(1 << 18)
        assert np.array_equal(h2.tap(capi.TAP_QUANTIZED, w1 - f0 - 1), o.quantized())
        assert np.array_equal(h2.tap(capi.TAP_PACKED, w1 - f0 - 1), o.packed())
        if "r900" in b.msgtypes:
            assert np.array_equal(h2.tap(capi.TAP_R900_QUANTIZED, w1 - f0 - 1), o.r900_quantized())
        h2.close()
    assert total_cands > 0


def test_quantized_of_the_whole_call_at_window_ends(big):
    """The big call itself (not a replay): Quantized after the LAST block of the call against an oracle fed the tail."""
    b = big
    halo = shard.halo_blocks(b.bs, b.pkl)
    f0 = b.nblocks - 256 - halo
    iq = b.d[f0 * b.bs2:].cpu().numpy()
    o = oracle.Oracle(b.mt, CL, oracle.SEARCH_EXACT)
    for k in range(iq.size // b.bs2):
        o.dsp_only(iq[k * b.bs2:(k + 1) * b.bs2])
    assert np.array_equal(b.h.tap(capi.TAP_QUANTIZED, b.nblocks - 1), o.quantized())


def test_one_call_equals_many_calls_at_full_size(big):
    b = big
    cap = 20000 if b.bs == 4096 else 90000
    h2 = capi.new_decoder(b.mt, CL, max_blocks_per_call=cap, max_candidates=1 << 20)
    parts, off = [], 0
    sizes = [1, cap - 1, 3] + [cap] * (b.nblocks // cap + 1)
    for n in sizes:
        n = min(n, b.nblocks - off)
        if n <= 0:
            break
        h2.decode_device_async(b.d.data_ptr() + off * b.bs2, n * b.bs2, 0, b.stream.cuda_stream)
        parts.append(h2.fetch(1 << 20))
        off += n
    assert off == b.nblocks
    split = np.concatenate(parts)
    assert len(split) == len(b.got)
    for f in ("block", "idx", "preamble_id", "check_mask", "bytes", "r900_digits"):
        assert np.array_equal(split[f], b.got[f]), f
    h2.close()


def test_shards_with_halo_equal_the_single_stream(big):
    """The multi-GPU decomposition on one GPU: every shard of the 8-way plan (halo + owned blocks, device
    resident, its own fresh handle) reports exactly the single-stream candidates of its owned blocks."""
    b = big
    plans = shard.plan(b.nblocks, 8, b.bs, b.pkl)
    assert [tuple(p) for p in capi.plan_shards(b.nblocks, 8, b.bs, b.pkl)] == \
        [(p.first_block, p.last_block, p.first_fed_block) for p in plans]
    fed_max = max(p.last_block - p.first_fed_block for p in plans)
    h2 = capi.new_decoder(b.mt, CL, max_blocks_per_call=fed_max, max_candidates=1 << 20)
    total = 0
    for p in plans:
        h2.reset()
        nfed = p.last_block - p.first_fed_block
        h2.decode_device_async(b.d.data_ptr() + p.first_fed_block * b.bs2, nfed * b.bs2, 0, b.stream.cuda_stream)
        part = h2.fetch(1 << 20)
        part = part[part["block"] >= p.halo_blocks].copy()
        part["block"] += p.first_fed_block
        ref = b.got[(b.got["block"] >= p.first_block) & (b.got["block"] < p.last_block)]
        assert len(part) == len(ref), (p, len(part), len(ref))
        for f in ("block", "idx", "preamble_id", "check_mask", "bytes", "r900_digits"):
            assert np.array_equal(part[f], ref[f]), (p.rank, f)
        total += len(part)
    assert total == len(b.got)
    h2.close()
