"""GPU parity tests (-m gpu): the CUDA path, called through the C ABI, against the CPU oracle on
the same bytes.  Bar: bit-exact at Quantize / Pack / Search / Slice / CRC; float taps
(Signal, csum) within 1 ulp (in practice identical)."""
import numpy as np
import pytest

import oracle
from helpers import assert_check_masks_exact, cand_key_gpu, cand_key_oracle, oracle_run, synth_stream, whole_blocks
from rtlamr_b200 import capi

pytestmark = pytest.mark.gpu


def ulp_diff(a, b):
    ai = a.view(np.int32).astype(np.int64)
    bi = b.view(np.int32).astype(np.int64)
    return np.abs(ai - bi).max() if a.size else 0


def compare_candidates(h, got, o, cands):
    nb, pk = o.cfg.packet_symbols + 7 >> 3, o.cfg.packet_symbols
    a = sorted(cand_key_gpu(r, nb, pk) for r in got)
    b = sorted(cand_key_oracle(c, nb, pk) for c in cands)
    assert len(a) == len(b), (len(a), len(b))
    assert a == b


def expected_masks(o, msgs):
    """(block, idx, proto) of every candidate whose parser accepted it (first occurrence per block)."""
    return {(m.block, m.idx, m.proto) for m in msgs}


@pytest.mark.parametrize("variant", [0, -1])
def test_sample_bin_cl78(built, sample_iq, variant):
    o, cands, msgs = oracle_run("scm", 78, sample_iq, oracle.SEARCH_EXACT)
    h = capi.new_decoder("scm", 78)
    h.set_demod_variant(variant)
    iq = whole_blocks(sample_iq, h.cfg.block_size2)
    got = h.decode(iq)
    assert len(got) == 853
    compare_candidates(h, got, o, cands)
    valid = {(int(r["block"]), int(r["idx"])) for r in got if r["check_mask"] & 1}
    for m in msgs:
        assert (m.block, m.idx) in valid
    # taps after the last block
    last = iq.size // h.cfg.block_size2 - 1
    assert np.array_equal(h.tap(capi.TAP_QUANTIZED, last), o.quantized())
    assert np.array_equal(h.tap(capi.TAP_PACKED, last), o.packed())
    assert ulp_diff(h.tap(capi.TAP_SIGNAL, last), o.signal()) <= 1
    assert ulp_diff(h.tap(capi.TAP_CSUM, last), o.csum()) <= 1
    assert np.array_equal(h.tap(capi.TAP_SIGNAL, last), o.signal())
    assert np.array_equal(h.tap(capi.TAP_CSUM, last), o.csum())
    h.close()


def test_sample_bin_cl72_is_empty(built, sample_iq):
    h = capi.new_decoder("scm", 72)
    got = h.decode(whole_blocks(sample_iq, h.cfg.block_size2))
    assert len(got) == 0
    h.close()


CASES = [("scm", 72), ("scm+", 72), ("idm", 72), ("netidm", 48), ("r900", 72), ("r900bcd", 32),
         ("scm,scm+,idm", 72), ("scm,scm+,idm,r900", 72), ("scm", 8), ("scm", 96), ("scm", 78), ("scm,idm", 40)]


@pytest.mark.parametrize("mt,cl", CASES)
@pytest.mark.parametrize("variant", [0, -1])
def test_synthetic_candidates_match_oracle(built, mt, cl, variant):
    n = 1 << 21
    iq, pk, truth = synth_stream(mt, cl, n, spacing=1 << 19)
    o, cands, msgs = oracle_run(mt, cl, iq)
    h = capi.new_decoder(mt, cl)
    h.set_demod_variant(variant)
    iq = whole_blocks(iq, h.cfg.block_size2)
    got = h.decode(iq)
    compare_candidates(h, got, o, cands)
    # the on-GPU screens agree with the parsers: every message's candidate carries its bit, and a
    # candidate with a bit set is one the parser accepts (or a same-block duplicate of one)
    protos = oracle.proto_ids(mt)
    bit_of = {p: i for i, p in enumerate(protos)}
    by_key = {(int(r["block"]), int(r["idx"]), int(r["preamble_id"])): int(r["check_mask"]) for r in got}
    accepted_bytes = {}
    for m in msgs:
        masks = [v for (b, i, _), v in by_key.items() if b == m.block and i == m.idx]
        assert any(v & (1 << bit_of[m.proto]) for v in masks), m
        accepted_bytes.setdefault(m.proto, set()).add(m.data)
    assert len(msgs) >= 1
    # ... and the converse, for EVERY candidate: a bit is set iff that parser's check passes on the returned bytes
    assert_check_masks_exact(got, mt)
    # every tap of the last block, for every geometry and both kernels (Signal/csum: identical, bar is 1 ulp)
    nblk = iq.size // h.cfg.block_size2
    assert np.array_equal(h.tap(capi.TAP_QUANTIZED, nblk - 1), o.quantized())
    assert np.array_equal(h.tap(capi.TAP_PACKED, nblk - 1), o.packed())
    assert ulp_diff(h.tap(capi.TAP_SIGNAL, nblk - 1), o.signal()) <= 1
    assert ulp_diff(h.tap(capi.TAP_CSUM, nblk - 1), o.csum()) <= 1
    assert np.array_equal(h.tap(capi.TAP_SIGNAL, nblk - 1), o.signal())
    assert np.array_equal(h.tap(capi.TAP_CSUM, nblk - 1), o.csum())
    # ... and of a block in the middle (DSP only: Search/Parse do not change the taps)
    o2 = oracle.Oracle(mt, cl, oracle.SEARCH_EXACT)
    mid = nblk // 2
    for b in range(mid + 1):
        o2.dsp_only(iq[b * h.cfg.block_size2:(b + 1) * h.cfg.block_size2])
    assert np.array_equal(h.tap(capi.TAP_QUANTIZED, mid), o2.quantized())
    assert np.array_equal(h.tap(capi.TAP_CSUM, mid), o2.csum())
    h.close()


@pytest.mark.parametrize("knob", ["7", "8"])
def test_demod_tuning_variants_are_bit_exact(built, sample_iq, knob):
    """The headline kernel gives the same bits with 7 and with 8 resident warps.  The call size picks the count
    (fast_round_cost): a call of a few work tiles runs 7 warps, one of exactly 8 x SMs tiles (one full round of
    8 warps, where 7 would need a second round) runs 8."""
    import torch
    ntiles = None if knob == "7" else 8 * torch.cuda.get_device_properties(0).multi_processor_count
    _variant_is_bit_exact(sample_iq, f"demod_fast_kernel<72,{knob}>", ntiles)


def test_register_ring_default_is_bit_exact(built, sample_iq):
    """The default kernel of the headline chip length (both rings in registers, 7 or 8 warps) is exact."""
    _variant_is_bit_exact(sample_iq)


def _variant_is_bit_exact(sample_iq, kernel=None, ntiles=None):
    """Synthetic, sample and uniform-random bytes against the oracle.  ntiles: tile each source to that many demod
    work tiles (32 blocks each) and decode it in one device-resident call; kernel: the demod instance that must run."""
    import torch
    mt, cl = "scm", 72
    for src in ("synthetic", "sample", "extremes"):
        if src == "synthetic":
            iq, _, _ = synth_stream(mt, cl, 1 << 21, spacing=1 << 18)
        elif src == "sample":
            iq = sample_iq
        else:
            iq = np.random.default_rng(3).integers(0, 256, 1 << 21, dtype=np.uint8)   # every byte value, uniformly
        if ntiles is None:
            h = capi.new_decoder(mt, cl)
            iqb = whole_blocks(iq, h.cfg.block_size2)
            got = h.decode(iqb)
        else:
            h = capi.new_decoder(mt, cl, max_blocks_per_call=32 * ntiles, max_candidates=1 << 20)
            src_b = whole_blocks(iq, h.cfg.block_size2)
            reps = -(-32 * ntiles * h.cfg.block_size2 // src_b.size)
            iqb = np.tile(src_b, reps)[: 32 * ntiles * h.cfg.block_size2]
            d = torch.from_numpy(iqb).cuda()
            h.decode_device_async(d.data_ptr(), d.numel(), 0, torch.cuda.current_stream().cuda_stream)
            got = h.fetch(1 << 20)
        o, cands, msgs = oracle_run(mt, cl, iqb, oracle.SEARCH_EXACT)
        compare_candidates(h, got, o, cands)
        last = iqb.size // h.cfg.block_size2 - 1
        assert np.array_equal(h.tap(capi.TAP_QUANTIZED, last), o.quantized())
        if kernel is not None:
            assert h.demod_kernel_name() == kernel, (src, h.last_kernels())
        h.close()


# Search instance each geometry reaches by default (the second entry of last_kernels()): the sliding-window kernel for
# the stock geometries, with the stock preamble sets' patterns as compile-time constants; search_generic_kernel for
# every geometry it does not fit (SL % 16 != 0, SL outside [64, 192], more than 4 preambles, preambles under 16 bits)
SEARCH_KERNEL = {("scm", 72): "search_slide_kernel<1,true,0xF953u>",    # SL 144: odd bits half a word in
                 ("scm,scm+,idm", 72): "search_slide_kernel<3,true,0xF953u, 0x16A3u, 0x5555u>",
                 ("scm,scm+,idm,r900", 72): "search_slide_kernel<4,true,0xF953u, 0x16A3u, 0x5555u, 0x0000u>",
                 ("scm,scm+", 72): "search_slide_kernel<2,true>",        # no stock set: patterns read at run time
                 ("r900", 72): "search_slide_kernel<1,true,0x0000u>",
                 ("scm", 64): "search_slide_kernel<1,false,0xF953u>",   # SL 128
                 ("scm", 78): "search_generic_kernel",      # SL 156: SL % 16 != 0, SL % 32 == 28
                 ("scm", 16): "search_generic_kernel",      # SL 32 < 64, SL % 32 == 0
                 ("scm", 24): "search_generic_kernel",      # SL 48 < 64, SL % 32 == 16
                 ("idm", 100): "search_generic_kernel"}     # SL 200 > 192
# symbol lengths below 64 or not a multiple of 16: each residue of SL mod 32 a chip length can give (0, 16, other)
SHORT_OR_ODD_SL = [("scm", 78), ("scm", 16), ("scm", 24)]


@pytest.mark.parametrize("mt,cl", [g for g in SEARCH_KERNEL if g not in SHORT_OR_ODD_SL])
def test_legacy_search_kernel_agrees(built, mt, cl):
    """Every Search kernel finds the oracle's candidates on a geometry that reaches it by default."""
    iq, _, _ = synth_stream(mt, cl, 1 << 21, spacing=1 << 18)
    o, cands, msgs = oracle_run(mt, cl, iq)
    assert len(cands) > 0
    h = capi.new_decoder(mt, cl)
    got = h.decode(whole_blocks(iq, h.cfg.block_size2))
    assert h.last_kernels().split(";")[1] == SEARCH_KERNEL[(mt, cl)], h.last_kernels()
    compare_candidates(h, got, o, cands)
    h.close()


@pytest.mark.parametrize("mt,cl", SHORT_OR_ODD_SL)
def test_short_or_odd_symbol_search_agrees(built, mt, cl):
    """search_generic_kernel finds the oracle's candidates where the sliding-window Search does not run."""
    test_legacy_search_kernel_agrees(built, mt, cl)


@pytest.mark.parametrize("mt,cl", [("r900", 72), ("scm,scm+,idm,r900", 72), ("r900bcd", 32)])
def test_r900_chain_shuffle_form_agrees(built, mt, cl):
    """The r900 running sums of the producer / consumer chain kernel give the oracle's candidate list with digits that
    pass the syndrome screen; its digits are compared with the oracle's quantized buffer in test_r900_digits_and_tap."""
    iq, _, _ = synth_stream(mt, cl, 1 << 21, spacing=1 << 18)
    o, cands, msgs = oracle_run(mt, cl, iq)
    h = capi.new_decoder(mt, cl)
    got = h.decode(whole_blocks(iq, h.cfg.block_size2))
    assert "r900_chain2_kernel" in h.last_kernels().split(";"), h.last_kernels()
    compare_candidates(h, got, o, cands)
    assert (got["flags"] & capi.CAND_HAS_R900).any()
    assert (got["check_mask"] != 0).any()
    h.close()


def test_r900_replay_when_packet_length_is_not_a_multiple_of_8(built):
    """r900 with 118 packet symbols at chip length 73 (PacketLength 17 228 samples): the chain starts are not 16-byte
    aligned, so every block takes the exact per-candidate replay.  Its digits are the r900 parser's quantized buffer."""
    mt, cl = "r900", 73
    p = capi.stock_protocol(mt, cl)
    p.packet_symbols = 118
    h = capi.Handle()
    h.register(p)
    h.allocate()
    assert h.cfg.packet_length % 8 != 0
    iq, _, _ = synth_stream(mt, cl, 1 << 21, spacing=1 << 18)
    got = h.decode(whole_blocks(iq, h.cfg.block_size2))
    kernels = h.last_kernels().split(";")
    assert "r900_replay_kernel" in kernels and "r900_chain2_kernel" not in kernels, kernels
    assert len(got) > 0
    taps = {}
    for r in got:
        assert r["flags"] & capi.CAND_HAS_R900
        b = int(r["block"])
        q = taps[b] if b in taps else taps.setdefault(b, h.tap(capi.TAP_R900_QUANTIZED, b))
        payload = int(r["idx"]) + h.cfg.preamble_length - h.cfg.symbol_length
        assert list(r["r900_digits"]) == [int(q[payload + k * 4 * cl]) for k in range(42)]
    h.close()


def test_r900_digits_and_tap(built):
    mt, cl = "r900", 72
    iq, pk, truth = synth_stream(mt, cl, 1 << 20, spacing=1 << 18)
    o = oracle.Oracle(mt, cl, oracle.SEARCH_GO)
    h = capi.new_decoder(mt, cl)
    iq = whole_blocks(iq, h.cfg.block_size2)
    nblk = iq.size // h.cfg.block_size2
    got = h.decode(iq)
    # feed the oracle block by block and compare the digits of every candidate of that block
    rows = {}
    for r in got:
        rows.setdefault(int(r["block"]), []).append(r)
    checked = 0
    for b in range(nblk):
        cands, _ = o.decode(iq[b * h.cfg.block_size2:(b + 1) * h.cfg.block_size2])
        q = o.r900_quantized()
        for r in rows.get(b, []):
            assert r["flags"] & capi.CAND_HAS_R900
            payload = int(r["idx"]) + o.cfg.preamble_length - o.cfg.symbol_length
            want = [int(q[payload + k * 4 * cl]) for k in range(42)]
            assert list(r["r900_digits"]) == want
            checked += 1
    assert checked == len(got) and checked > 0
    assert np.array_equal(h.tap(capi.TAP_R900_QUANTIZED, nblk - 1), o.r900_quantized())
    h.close()


@pytest.mark.parametrize("seed", range(6))
def test_random_geometries_and_call_patterns(built, seed):
    """Chip lengths the CLI would refuse (odd, tiny, large: generic kernel), random protocol sets, random call
    sizes: candidates must still equal the reference restatement (exact-search mode where SL % 8 != 0)."""
    rng = np.random.default_rng(100 + seed)
    cl = int(rng.choice([9, 16, 33, 50, 100, 120, 24, 61]))
    names = ["scm", "scm+", "idm", "netidm", "r900", "r900bcd"]
    k = int(rng.integers(1, 4))
    mt = ",".join(rng.choice(names, size=k, replace=False))
    n = 1 << 20
    iq, pk, truth = synth_stream(mt, cl, n, spacing=1 << 18, pkt_seed=seed)
    o, cands, msgs = oracle_run(mt, cl, iq)
    h = capi.new_decoder(mt, cl, max_blocks_per_call=64)
    bs2 = h.cfg.block_size2
    iq = whole_blocks(iq, bs2)
    parts, off, nblk = [], 0, iq.size // bs2
    while off < nblk:
        m = int(min(nblk - off, rng.integers(1, 100)))
        parts.append(h.decode(iq[off * bs2:(off + m) * bs2]))
        off += m
    got = np.concatenate(parts)
    compare_candidates(h, got, o, cands)
    want_valid = {(m.block, m.idx) for m in msgs}
    have_valid = {(int(r["block"]), int(r["idx"])) for r in got if r["check_mask"]}
    assert want_valid <= have_valid
    h.close()


def test_r900_scratch_overflow_falls_back_to_replay(built, monkeypatch):
    """With a single scratch slot most blocks must take the per-candidate replay path: same digits."""
    mt, cl = "r900", 72
    iq, pk, truth = synth_stream(mt, cl, 1 << 21, spacing=1 << 18)
    h = capi.new_decoder(mt, cl)
    iq = whole_blocks(iq, h.cfg.block_size2)
    ref = h.decode(iq)
    monkeypatch.setenv("ERTGPU_R900_SLOTS", "1")
    h1 = capi.new_decoder(mt, cl)
    got = h1.decode(iq)
    assert len(got) == len(ref) > 0
    for f in ("block", "idx", "check_mask", "r900_digits"):
        assert np.array_equal(got[f], ref[f]), f
    assert (ref["check_mask"] != 0).sum() >= 7
    h.close()
    h1.close()


def test_call_splitting_is_invisible(built):
    """N calls of any sizes == one long stream (history carried in the handle, decode.go:165-166)."""
    mt, cl = "scm,scm+,idm,r900", 72
    iq, _, _ = synth_stream(mt, cl, 1 << 21, spacing=1 << 18)
    h1 = capi.new_decoder(mt, cl)
    bs2 = h1.cfg.block_size2
    iq = whole_blocks(iq, bs2)
    whole = h1.decode(iq)
    h2 = capi.new_decoder(mt, cl, max_blocks_per_call=7)   # forces internal chunking too
    rng = np.random.default_rng(1)
    parts, off, nblk = [], 0, iq.size // bs2
    while off < nblk:
        n = int(min(nblk - off, rng.integers(1, 40)))
        parts.append(h2.decode(iq[off * bs2:(off + n) * bs2]))
        off += n
    split = np.concatenate(parts)
    assert len(whole) == len(split) and len(whole) > 0
    for f in ("block", "idx", "preamble_id", "check_mask", "bytes", "r900_digits"):
        assert np.array_equal(whole[f], split[f]), f
    # reset == fresh decoder
    h2.reset()
    again = h2.decode(iq[: 16 * bs2])
    first = whole[whole["block"] < 16]
    assert np.array_equal(again["idx"], first["idx"]) and np.array_equal(again["bytes"], first["bytes"])
    h1.close()
    h2.close()


def test_device_resident_path_and_flags(built):
    import torch
    mt, cl = "scm", 72
    iq, _, _ = synth_stream(mt, cl, 1 << 21, spacing=1 << 18)
    h = capi.new_decoder(mt, cl)
    iq = whole_blocks(iq, h.cfg.block_size2)
    host = h.decode(iq)
    h.reset()
    d = torch.from_numpy(iq).cuda()
    h.decode_device_async(d.data_ptr(), d.numel(), 0, torch.cuda.current_stream().cuda_stream)
    dev = h.fetch()
    assert np.array_equal(host["idx"], dev["idx"]) and np.array_equal(host["bytes"], dev["bytes"])
    ncand, nvalid = h.last_counts()
    assert ncand == len(host) and nvalid == int((host["check_mask"] != 0).sum()) and nvalid > 0
    assert h.last_launches() >= 3          # demod, Search, Slice (+ history carry in the same kernel)
    h.reset()
    only = h.decode(iq, flags=capi.DECODE_ONLY_VALID)
    assert len(only) == nvalid and (only["check_mask"] != 0).all()
    h.close()


def test_edge_cases(built):
    h = capi.new_decoder("scm", 72)
    bs2 = h.cfg.block_size2
    assert len(h.decode(np.zeros(0, dtype=np.uint8))) == 0            # empty input
    with pytest.raises(capi.ErtGpuError) as e:                        # ragged input: Go panics (decode.go:222)
        h.decode(np.zeros(bs2 + 2, dtype=np.uint8))
    assert e.value.code == capi.ESIZE
    # all-zero and all-255 IQ: magnitude saturates at 2.0, filter output is exactly +0 -> bit 1 everywhere
    for v in (0, 255, 127):
        h.reset()
        got = h.decode(np.full(4 * bs2, v, dtype=np.uint8))
        o = oracle.Oracle("scm", 72)
        cands, _ = o.decode(np.full(4 * bs2, v, dtype=np.uint8))
        assert len(got) == len(cands)
        assert np.array_equal(h.tap(capi.TAP_QUANTIZED, 3), o.quantized())
    h.close()   # the candidate capacity: tests/test_gpu_capacity.py


def test_synth_device_generator_matches_host(built):
    import torch
    from rtlamr_b200 import synth
    n = 1 << 20
    pk, _ = synth.make_packets("scm,idm,r900", 72, n, seed=11, spacing=1 << 18)
    host = synth.host_fill(12345, n - 12345, 0x5EED0003, pk)
    d = torch.empty(2 * (n - 12345), dtype=torch.uint8, device="cuda")
    capi.synth_fill(0, d.data_ptr(), 12345, n - 12345, 0x5EED0003, pk)
    assert np.array_equal(d.cpu().numpy(), host)
