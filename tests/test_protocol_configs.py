"""Custom protocol configurations on the CPU: the oracle built from ertgpu_protocol structs (Oracle.from_protocols)
equals the stock oracle on every stock set, it reports where the reference would index past a slice, and a Python
restatement of the rules ertgpu_allocate applies (include/ertgpu.h, R1-R4) gives the library's verdict on the boundary
of each rule and on seeded random configurations.  Nothing here decodes on a GPU."""
import numpy as np
import pytest

import oracle
from helpers import allocate_verdict, make_protocol, merged_geometry, rule_violated, synth_stream, whole_blocks
from rtlamr_b200 import capi

STOCK_SETS = ["scm", "scm+", "idm", "netidm", "r900", "r900bcd", "scm,scm+", "scm,scm+,idm", "scm,scm+,idm,r900",
              "r900,r900bcd,scm", "idm,netidm"]
SUITE_CLS = [8, 9, 16, 24, 32, 33, 40, 48, 50, 56, 61, 64, 72, 73, 78, 80, 88, 96, 100, 120]


def search_mode(cl):
    return oracle.SEARCH_GO if (2 * cl) % 8 == 0 else oracle.SEARCH_EXACT


def stock_structs(mt, cl):
    return [capi.stock_protocol(m, cl) for m in mt.split(",")]


# ---------------------------------------------------------------- the oracle on protocol structs
@pytest.mark.parametrize("cl", [8, 33, 72])
@pytest.mark.parametrize("mt", STOCK_SETS)
def test_oracle_from_protocols_equals_stock_oracle(built, mt, cl):
    """Every stock set through from_protocols: byte-identical candidates, messages and taps (SL = 66 at chip length
    33 takes the exact search)."""
    a = oracle.Oracle(mt, cl, search_mode(cl))
    b = oracle.Oracle.from_protocols(stock_structs(mt, cl), search_mode(cl))
    for f in ("block_size", "chip_length", "preamble_symbols", "packet_symbols", "buffer_length", "center_freq"):
        assert getattr(a.cfg, f) == getattr(b.cfg, f), f
    assert a.npreambles == b.npreambles
    bs = a.cfg.block_size
    nblocks = max(24, -(-3 * a.cfg.buffer_length // bs))
    iq, _, truth = synth_stream(mt, cl, nblocks * bs, spacing=max(bs * 4, a.cfg.buffer_length + bs))
    iq = whole_blocks(iq, a.cfg.block_size2)
    seen_msgs = 0
    for part in np.array_split(np.arange(iq.size // a.cfg.block_size2), 3):
        chunk = iq[part[0] * a.cfg.block_size2:(part[-1] + 1) * a.cfg.block_size2]
        ca, ma = a.decode(chunk)
        cb, mb = b.decode(chunk)
        assert ca == cb and ma == mb
        seen_msgs += len(ma)
        for tap in ("signal", "csum", "quantized", "packed", "r900_quantized"):
            ta, tb = getattr(a, tap)(), getattr(b, tap)()
            assert (ta is None) == (tb is None) and (ta is None or np.array_equal(ta, tb)), tap
    assert seen_msgs > 0 or cl == 33    # the synthetic packets decode (SL = 66: the stock sets still give candidates)
    a.close()
    b.close()


def test_oracle_rejects_bad_protocol_structs(built):
    ok = make_protocol("1" * 8, 32, 8, 16)
    oracle.Oracle.from_protocols([ok]).close()
    for bad in (make_protocol("", 32, 8, 16), make_protocol("10x", 32, 8, 16), make_protocol("1", 0, 8, 16),
                make_protocol("1", 32, 0, 16), make_protocol("1", 32, 8, 0), make_protocol("1", 32, 8, 8 * oracle.MAX_PKT + 1)):
        with pytest.raises(ValueError):
            oracle.Oracle.from_protocols([bad])
    with pytest.raises(ValueError):
        oracle.Oracle.from_protocols([ok] * 9)


# ---------------------------------------------------------------- the reference's panics
def constant_blocks(o, extra=1, v=0):
    """Constant IQ: once the zeros in front of the stream have left Quantized, every bit is 1 (the filter's output is
    exactly +0, tests/test_gpu_parity.py test_edge_cases).  Returns (iq, the first block with all-ones Quantized)."""
    warm = -(-o.cfg.buffer_length // o.cfg.block_size) + 1
    return np.full((warm + extra) * o.cfg.block_size2, v, np.uint8), warm


PANICS = {
    # PreambleSymbols > PacketSymbols: packing d.packed reads past Quantized on the first call (R1)
    "R1": ([make_protocol("1" * 8, 32, 20, 10)], oracle.SEARCH_GO),
    # 18 bits, PS = PK = 16: the byte pre-filter of bit 17 indexes past d.packed (R2)
    "R2": ([make_protocol("1" * 18, 32, 16, 16)], oracle.SEARCH_GO),
    # odd SL, 10 bits, PK = 8: the exact test of bit 9 indexes past Quantized (R2)
    "R2_exact": ([make_protocol("1" * 10, 33, 8, 8)], oracle.SEARCH_EXACT),
    # r900 digits with PK = PS + 80: the last digit of a late start indexes past the parser's quantized (R3)
    "R3": ([make_protocol("1" * 32, 32, 32, 112, check=capi.CHECK_R900)], oracle.SEARCH_GO),
}


@pytest.mark.parametrize("case", sorted(PANICS))
def test_oracle_reports_reference_panics(built, case):
    protos, search = PANICS[case]
    assert rule_violated(protos) == case[:2]
    o = oracle.Oracle.from_protocols(protos, search)
    with pytest.raises(oracle.ReferencePanic):
        o.decode(constant_blocks(o)[0])
    with pytest.raises(oracle.ReferencePanic):   # the reference has died: every later call too
        o.decode(np.zeros(o.cfg.block_size2, np.uint8))
    o.close()


@pytest.mark.parametrize("pk_over_ps", [81, 82, 83])
def test_r900_short_packets_that_do_not_panic(built, pk_over_ps):
    """PK = PS + 81 and + 82 read never-written zeros in the reference instead of panicking (R3 rejects them all
    the same); PK = PS + 83 is the shortest r900 packet whose digits are all computed.  Every start is a candidate on
    constant input, so the latest digit position is reached."""
    p = make_protocol("1" * 32, 32, 32, 32 + pk_over_ps, check=capi.CHECK_R900)
    assert rule_violated([p]) == (None if pk_over_ps == 83 else "R3")
    o = oracle.Oracle.from_protocols([p])
    iq, last_block = constant_blocks(o)
    cands, _ = o.decode(iq)
    assert {c.idx for c in cands if c.block == last_block} == set(range(o.cfg.block_size))
    q = o.r900_quantized()
    cfg = o.cfg
    last = cfg.block_size - 1 + cfg.preamble_length - cfg.symbol_length + 164 * cfg.chip_length
    written = cfg.buffer_length - 4 * cfg.chip_length
    assert (last < written) == (pk_over_ps == 83) and last < cfg.buffer_length
    assert not q[written:].any()
    o.close()


def test_partial_last_byte_carries_the_previous_candidate(built):
    """R4: with PK % 8 != 0 the reference's last packet byte keeps the previous candidate's high bits
    (decode.go:363-366), so it differs from a zero-filled slice of the same bits; masked to its PK % 8 low bits it
    does not."""
    pk = 12
    o = oracle.Oracle.from_protocols([make_protocol("1" * 8, 32, 8, pk)])
    iq, last_block = constant_blocks(o)
    cands, _ = o.decode(iq)
    last = [c for c in cands if c.block == last_block]
    assert len(last) == o.cfg.block_size
    zeroed = 0xFF >> (8 - pk % 8)                 # the candidate's own bits sliced into a zeroed buffer: 0xFF, 0x0F
    assert all(c.data == b"\xff\xff" for c in last)
    assert cands[0].data[-1] & ~zeroed == 0        # d.pkt starts zeroed
    o.close()


# ---------------------------------------------------------------- the rules of ertgpu_allocate
def assert_verdict(protos):
    want = rule_violated(protos)
    rc, msg = allocate_verdict(protos)
    if want is None:
        assert rc in (capi.OK, capi.ECUDA), (rc, msg)      # ECUDA: no device on this machine, every check passed
    else:
        assert rc == capi.EINVAL, (want, rc, msg)
        assert msg.startswith(want + ":") or (want == "BS" and "block size" in msg), (want, msg)
    return want


def r4(pk, crc_to, crc_from=0):
    return [make_protocol("1" * 8, 32, 8, pk, check=capi.CHECK_CRC16, crc_range=(crc_from, crc_to))]


BOUNDARIES = {
    # R1: PS = PK packs exactly BUF bits when PL % 8 == 0; at odd SL the rounding of ceil(PL/8) already rejects PS = PK
    "R1": [([make_protocol("1", 32, 20, 20)], None), ([make_protocol("1", 32, 21, 20)], "R1"),
           ([make_protocol("1", 33, 4, 5)], None), ([make_protocol("1", 33, 5, 5)], "R1")],
    # R2: the byte pre-filter (SL % 8 == 0: n <= PS + 1) and, where SL >> 3 == 0, n <= PK + 1
    "R2": [([make_protocol("1" * 17, 32, 16, 16)], None), ([make_protocol("1" * 18, 32, 16, 16)], "R2"),
           ([make_protocol("1" * 17, 32, 16, 40)], None), ([make_protocol("1" * 18, 32, 16, 40)], "R2"),
           ([make_protocol("1" * 8, 3, 6, 7)], None), ([make_protocol("1" * 9, 3, 6, 7)], "R2"),
           ([make_protocol("1" * 9, 3, 6, 8)], None)],
    # R3: PK = PS + 83 against PS + 82, stock preamble and a mixed set
    "R3": [([make_protocol("0" * 16 + "1110010101100100", 32, 32, 115, check=capi.CHECK_R900)], None),
           ([make_protocol("0" * 16 + "1110010101100100", 32, 32, 114, check=capi.CHECK_R900)], "R3"),
           ([make_protocol("1" * 21, 40, 21, 96), make_protocol("1" * 20, 40, 40, 123, check=capi.CHECK_R900)], None),
           ([make_protocol("1" * 21, 40, 21, 96), make_protocol("1" * 20, 40, 40, 122, check=capi.CHECK_R900)], "R3")],
    # R4: a CRC range ending at the last whole byte against one holding the partial byte (PK = 100: byte 12)
    "R4": [(r4(100, 12), None), (r4(100, 13), "R4"), (r4(100, 13, 12), "R4"), (r4(104, 13), None)],
}


@pytest.mark.parametrize("rule", sorted(BOUNDARIES))
def test_allocate_rules_at_their_boundaries(built, rule):
    for protos, want in BOUNDARIES[rule]:
        assert rule_violated(protos) == want, (rule, [(p.preamble, p.preamble_symbols, p.packet_symbols) for p in protos])
        assert_verdict(protos)


def test_every_stock_set_passes_the_rules(built):
    for mt in STOCK_SETS + ["scm,scm+,idm,r900,r900bcd,netidm"]:
        for cl in SUITE_CLS:
            assert assert_verdict(stock_structs(mt, cl)) is None, (mt, cl)


def test_hand_built_protocols_of_the_suite_pass_the_rules(built):
    """The custom protocols the GPU tests of the stock decode path build (a 21-bit custom or all-ones preamble on the
    scm geometry, scm with PacketSymbols >= 96, r900 with 118 symbols) are still accepted."""
    for cl in (56, 72, 80):
        for pre in ("110100111000101101001", "1" * 21):
            p = capi.stock_protocol("scm", cl)
            p.preamble = pre.encode()
            assert assert_verdict([p]) is None
    for cl in (32, 40, 64, 96):
        for pk in range(96, 140):
            p = capi.stock_protocol("scm", cl)
            p.packet_symbols = pk
            assert assert_verdict([p]) is None
    for cl in (32, 48, 72):
        p = capi.stock_protocol("r900", cl)
        p.packet_symbols = 118
        assert assert_verdict([p]) is None


def random_protocol(rng, cls):
    """A protocol ertgpu_register_protocol accepts, drawn so that every rule is met and broken now and then."""
    cl = int(rng.choice(cls))
    n = int(rng.integers(1, 33))
    pre = "".join(rng.choice(["0", "1"], n))
    ps = int(rng.integers(1, 40))
    pk = int(rng.choice([rng.integers(1, ps + 2), rng.integers(1, 130), rng.integers(ps, ps + 120), rng.integers(1, 737)]))
    kind = int(rng.choice([capi.CHECK_NONE, capi.CHECK_CRC16, capi.CHECK_CRC16, capi.CHECK_R900]))
    if kind == capi.CHECK_CRC16:
        nbytes = (pk + 7) // 8
        lo = int(rng.integers(0, nbytes))
        return make_protocol(pre, cl, ps, pk, kind, (int(rng.integers(0, 1 << 16)), int(rng.integers(1, 1 << 16)),
                                                      int(rng.integers(0, 1 << 16))), (lo, int(rng.integers(lo + 1, nbytes + 1))))
    return make_protocol(pre, cl, ps, pk, kind)


def random_config(rng, cls):
    return [random_protocol(rng, cls) for _ in range(int(rng.choice([1, 1, 1, 2, 3, 4, 5, 6, 7, 8])))]


def test_allocate_rules_on_random_configurations(built):
    rng = np.random.default_rng(0xC0F16)
    cls = [3, 8, 9, 16, 32, 33, 40, 56, 64, 72, 78, 96, 120, 200]
    seen = {}
    for _ in range(200):
        protos = random_config(rng, cls)
        want = assert_verdict(protos)
        seen[want] = seen.get(want, 0) + 1
    assert all(seen.get(r, 0) >= 3 for r in (None, "R1", "R2", "R3", "R4")), seen


def test_merged_geometry_matches_the_oracle(built):
    """merged_geometry is the configuration the oracle merges (decode.go:100-141)."""
    rng = np.random.default_rng(7)
    for _ in range(40):
        protos = random_config(rng, [8, 16, 33, 72, 100])
        g = merged_geometry(protos)
        o = oracle.Oracle.from_protocols(protos)
        assert (o.cfg.chip_length, o.cfg.preamble_symbols, o.cfg.packet_symbols, o.cfg.block_size, o.cfg.buffer_length) == \
            (g["CL"], g["PS"], g["PK"], g["BS"], g["BUF"])
        o.close()
