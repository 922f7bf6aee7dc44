"""Custom protocol configurations through the C ABI against the oracle built from the same ertgpu_protocol structs
(Oracle.from_protocols): the edges of the geometry the ABI accepts and a seeded sweep of random accepted configurations.

Each configuration decodes a seeded stream with packets behind its own preambles (CRC-valid bodies where a CRC16 screen
is registered, r900-coded payloads behind an r900 screen).  Checked: candidates (block, preamble, idx, bytes) exactly,
check_mask in both directions from each protocol's own screen, r900 digits against the oracle's r900 quantized, the
Quantized and Packed taps on both sides of tile seams, the two demod kernels where the fast one applies, and host-call
splits with max_blocks_per_call chunking against one call.  The first rejected configuration of every rule of
ertgpu_allocate is never decoded: allocate must refuse it."""
import time

import numpy as np
import pytest

import oracle
from helpers import (assert_check_masks_exact, cand_key_gpu, cand_key_oracle, make_protocol, merged_geometry,
                     preamble_of, rule_violated, whole_blocks)
from rtlamr_b200 import capi, synth

gpu = pytest.mark.gpu
SEEN = set()        # every kernel the decodes of this file launched
SEEN_GENERIC_NPRE = set()
TIMES = {}
NONE, CRC, R900 = capi.CHECK_NONE, capi.CHECK_CRC16, capi.CHECK_R900
R900_PRE = "00000000000000001110010101100100"


def bits(rng, n):
    return "".join(rng.choice(["0", "1"], n))


def crc_proto(pre, cl, ps, pk, rng, to=None):
    """A CRC16 screen with a custom init, polynomial and residue over [1, to) (the last whole byte by default)."""
    to = to or pk // 8
    return make_protocol(pre, cl, ps, pk, CRC, (int(rng.integers(0, 1 << 16)), int(rng.integers(1, 1 << 16)) | 1,
                                                 int(rng.integers(0, 1 << 16))), (1, to))


def r900_proto(cl, pk):
    return make_protocol(R900_PRE, cl, 32, pk, R900)


# ---------------------------------------------------------------- the edge configurations
def edge_configs():
    rng = np.random.default_rng(0xED6E)
    out = {
        # PreambleSymbols = 1: BlockSize shorter than two fast-kernel bodies (issue: demod_fast launch failed)
        "ps1_cl32": [make_protocol("0", 32, 1, 40)],
        "ps1_cl56": [make_protocol("01", 56, 1, 40)],
        "ps1_cl64": [make_protocol("10", 64, 1, 40)],
        # PacketSymbols = 1 at a specialised chip length: a packet shorter than the fast kernel's lead-in
        "pk1_cl72": [make_protocol("0", 72, 1, 1)],
    }
    for pk in (1, 7, 8, 9, 31, 32, 33, 127, 128, 129, 735, 736):   # extract_words_kernel<4> up to 128, <23> above
        ps = min(pk, 24)
        n = min(ps + 1, 20)
        pre = "0" + bits(rng, n - 1)   # not all ones: short preambles hit only inside the packets of a quiet stream
        out[f"pk{pk}"] = [crc_proto(pre, 40, ps, pk, rng) if pk >= 8 * (n // 8 + 4) else make_protocol(pre, 40, ps, pk)]
    out["pre15_generic"] = [crc_proto(bits(rng, 15), 48, 15, 100, rng)]
    out["pre16_slide1"] = [crc_proto("0110100111010010", 48, 16, 100, rng)]
    out["pre17_31_slide2"] = [crc_proto(bits(rng, 17), 40, 17, 100, rng), crc_proto(bits(rng, 31), 40, 31, 104, rng)]
    out["pre32_slide3"] = [crc_proto(bits(rng, 32), 56, 32, 96, rng), make_protocol(bits(rng, 16), 56, 16, 90),
                           crc_proto(bits(rng, 17), 56, 17, 120, rng)]
    out["pre_slide4"] = [crc_proto(bits(rng, n), 64, n, 100, rng) for n in (20, 32, 16, 25)]
    out["npre5_generic"] = [crc_proto(bits(rng, 16 + 3 * i), 48, 16 + 3 * i, 96 + 8 * i, rng) for i in range(5)]
    out["npre8_generic"] = [crc_proto(bits(rng, 18 + i), 72, 18 + i, 100 + i, rng) if i % 3 else
                            make_protocol(bits(rng, 18 + i), 72, 18 + i, 100 + i) for i in range(8)]
    shared = bits(rng, 21)
    out["shared_and_prefix"] = [crc_proto(shared, 40, 21, 96, rng), make_protocol(shared, 40, 21, 96),
                                make_protocol("0101", 40, 4, 64), crc_proto("01010", 40, 5, 80, rng),
                                make_protocol(bits(rng, 24), 40, 24, 100)]
    out["r900_pk115_chain"] = [r900_proto(32, 115)]
    out["r900_pk115_replay"] = [r900_proto(33, 115)]
    out["r900_mixed"] = [crc_proto(bits(rng, 21), 48, 21, 96, rng), r900_proto(48, 115),
                         make_protocol(R900_PRE, 48, 32, 100)]
    # PacketLength % 8 == 4 at a specialised chip length: the fast kernel's lead-in could not be bulk-copied from the
    # history of the previous call (16-byte alignment), the generic kernel runs
    out["pkl4mod8_cl78"] = [crc_proto(bits(rng, 21), 78, 21, 97, rng)]
    for name, protos in out.items():
        assert rule_violated(protos) is None, name
    return out


EDGES = edge_configs()


def random_configs(n=24, seed=0x5EE9):
    """Accepted configurations: 1-8 protocols, chip lengths specialised, odd, small and large, mixed screens."""
    rng = np.random.default_rng(seed)
    cls = [32, 40, 48, 56, 64, 72, 78, 80, 88, 96, 33, 61, 73, 8, 9, 16, 100, 120, 200]
    out = []
    while len(out) < n:
        cl = int(rng.choice(cls))
        protos = []
        for _ in range(int(rng.choice([1, 1, 2, 3, 4, 5, 6, 7, 8]))):
            nb = int(rng.integers(8, 33))
            ps = int(rng.integers(nb - 1, 40))
            pk = int(rng.integers(max(ps, nb + 40), 200))
            kind = int(rng.choice([NONE, CRC, CRC, R900]))
            if kind == R900:
                protos.append(r900_proto(cl, int(rng.integers(115, 160))))
            elif kind == CRC:
                protos.append(crc_proto(bits(rng, nb), cl, ps, pk, rng, int(rng.integers(nb // 8 + 4, pk // 8 + 1))))
            else:
                protos.append(make_protocol(bits(rng, nb), cl, ps, pk))
        if rule_violated(protos) is None:
            out.append(protos)
    return out


RANDOM = random_configs()


# ---------------------------------------------------------------- streams
def crc_fix(data: bytearray, p):
    """Set bytes crc_to-2, crc_to-1 so that the CRC over [crc_from, crc_to) equals the residue: the register is linear,
    so crc(M || b) = crc(M || 00) ^ crc_0(b) with crc_0 the CRC from a zero register."""
    table = oracle.crc_table(p.crc_poly).astype(np.uint32)
    lo, hi = p.crc_from, p.crc_to
    data[hi - 2:hi] = b"\0\0"
    base = oracle.crc_checksum(p.crc_init, bytes(data[lo:hi]), p.crc_poly)
    b = np.arange(1 << 16, dtype=np.uint32)
    c = table[b >> 8]                                   # crc_0 of byte b>>8, then of byte b & 0xFF
    c = ((c << 8) & 0xFFFF) ^ table[(c >> 8) ^ (b & 0xFF)]
    v = int(np.nonzero(c == (base ^ p.crc_residue))[0][0])
    data[hi - 2:hi] = v.to_bytes(2, "big")
    assert oracle.crc_checksum(p.crc_init, bytes(data[lo:hi]), p.crc_poly) == p.crc_residue


def packet_chips(rng, p, cl):
    pre = preamble_of(p)
    if p.check_kind == R900:
        chips, _ = synth.encode_r900(*(int(rng.integers(0, hi)) for hi in (1 << 32, 256, 64, 4, 1 << 24, 4, 16, 4)))
        return chips
    nbits = max(p.packet_symbols, 8 * p.crc_to if p.check_kind == CRC else 0)
    nbits = min(nbits, 8 * 96)
    body = [int(c) for c in pre] + list(rng.integers(0, 2, max(0, nbits - len(pre))))
    data = bytearray(np.packbits(np.array(body, np.uint8)).tobytes())
    if p.check_kind == CRC:
        crc_fix(data, p)
    return synth.manchester_chips(np.unpackbits(np.frombuffer(bytes(data), np.uint8))[:nbits].tolist())


def make_stream(protos, g, nsamples, seed, quiet):
    """Seeded noise with packets of every protocol in turn; quiet: constant bytes outside the packets (every Quantized
    bit 1), so that preambles of a few bits hit only inside packets."""
    rng = np.random.default_rng(seed)
    rows, s, i = [], int(rng.integers(0, 3 * g["SL"])), 0
    while True:
        p = protos[i % len(protos)]
        chips = packet_chips(rng, p, g["CL"])
        if s + len(chips) * g["CL"] + 2 * g["SL"] > nsamples:
            break
        row = np.zeros((), dtype=capi.SYNTH_DTYPE)
        row["start_sample"], row["n_chips"], row["chip_length"] = s, len(chips), g["CL"]
        row["amp_i"], row["amp_q"] = 40, 30
        pk = np.packbits(np.array(chips, np.uint8))
        row["chips"][:len(pk)] = pk
        rows.append(row)
        s += len(chips) * g["CL"] + int(rng.integers(g["SL"], max(g["SL"] + 1, nsamples // 24)))
        i += 1
    rows = np.array(rows, dtype=capi.SYNTH_DTYPE)
    iq = synth.host_fill(0, nsamples, seed, rows)
    if quiet:
        keep = np.zeros(nsamples, bool)
        for r in rows:
            keep[r["start_sample"]:r["start_sample"] + r["n_chips"] * r["chip_length"]] = True
        iq.reshape(-1, 2)[~keep] = 0     # magnitude 2.0: exact running sums, filter output +0
    return iq, len(rows)


# ---------------------------------------------------------------- the oracle
def oracle_run(protos, g, iq, stops, r900_pid):
    """Candidates of the oracle over the whole stream, fed in segments ending at each block of `stops`, with the
    Quantized / Packed / r900 quantized taps after those blocks."""
    search = oracle.SEARCH_GO if g["SL"] % 8 == 0 else oracle.SEARCH_EXACT
    o = oracle.Oracle.from_protocols(protos, search)
    bs2 = o.cfg.block_size2
    nblk = iq.size // bs2
    cands, taps, prev = [], {}, 0
    for b in sorted(set(stops)) + [nblk - 1]:
        if b < prev:
            continue
        n = b + 1 - prev
        c, _ = o.decode(iq[prev * bs2:(b + 1) * bs2], cand_cap=4096 + g["BS"] * n, msg_cap=1 << 12)
        cands += c
        prev = b + 1
        taps[b] = (o.quantized(), o.packed(), o.r900_quantized() if r900_pid is not None else None)
    o.close()
    return cands, taps


def handle(protos, max_blocks=0, max_cands=1 << 20, variant=-1):
    h = capi.Handle()
    for p in protos:
        h.register(p)
    h.allocate(0, max_blocks, max_cands)
    if variant == 0:
        h.set_demod_variant(0)
    return h


def same_records(a, b, what):
    assert len(a) == len(b), (what, len(a), len(b))
    for f in ("block", "idx", "preamble_id", "check_mask", "flags", "bytes", "r900_digits"):
        assert np.array_equal(a[f], b[f]), (what, f)


def record(h, npre):
    k = [x.strip() for x in h.last_kernels().split(";")]
    SEEN.update(k)
    if k[1] == "search_generic_kernel":
        SEEN_GENERIC_NPRE.add(npre)
    return k


def distinct(protos):
    out = []
    for p in protos:
        if preamble_of(p) not in out:
            out.append(preamble_of(p))
    return out


def check_config(name, protos, nsamples=1 << 20, seed=1, full=True, constant=False, max_cands=1 << 20):
    t0 = time.perf_counter()
    g = merged_geometry(protos)
    pres = distinct(protos)
    quiet = min(len(p) for p in pres) < 16
    if constant:
        iq, npk = np.zeros(2 * nsamples, np.uint8), 0
    else:
        iq, npk = make_stream(protos, g, nsamples, seed, quiet)
    h = handle(protos, max_cands=max_cands)
    c = h.cfg
    assert (c.block_size, c.buffer_length, c.packet_symbols) == (g["BS"], g["BUF"], g["PK"])
    iq = whole_blocks(iq, c.block_size2)
    nblk = iq.size // c.block_size2
    nbytes = (g["PK"] + 7) >> 3
    got = h.decode(iq, cap=1 << 16)
    k = record(h, len(pres))

    r900_pid = next((pres.index(preamble_of(p)) for p in protos if p.check_kind == R900), None)
    stops = {0, 31, 32, nblk // 2, nblk - 1} if full else set()
    if r900_pid is not None:
        stops |= {int(b) for b in got["block"][got["preamble_id"] == r900_pid]}
    cands, taps = oracle_run(protos, g, iq, stops, r900_pid)
    want = sorted(cand_key_oracle(x, nbytes, g["PK"]) for x in cands)
    have = sorted(cand_key_gpu(r, nbytes, g["PK"]) for r in got)
    assert have == want, (name, len(have), len(want), sorted(set(have) ^ set(want))[:4])
    assert len(want) > 0
    assert_check_masks_exact(got, protos)

    if r900_pid is not None:   # r900 digit k = the parser's quantized[idx + PL - SL + 4*k*CL] after the candidate's block
        pos = g["PL"] - g["SL"] + 4 * g["CL"] * np.arange(capi.R900_DIGITS)
        rec = got[got["preamble_id"] == r900_pid]
        assert len(rec) > 0 and (rec["flags"] & capi.CAND_HAS_R900).all()
        for r in rec:
            q = taps[int(r["block"])][2]
            assert np.array_equal(r["r900_digits"], q[int(r["idx"]) + pos]), (name, int(r["block"]), int(r["idx"]))
    if full:
        for b in sorted({0, 31, 32, nblk // 2, nblk - 1}):
            q, pk, _ = taps[b]
            assert np.array_equal(h.tap(capi.TAP_QUANTIZED, b), q), (name, b)
            assert np.array_equal(h.tap(capi.TAP_PACKED, b), pk), (name, b)
        if k[0] != "demod_generic_kernel":      # the same bytes on the other demod kernel
            hg = handle(protos, max_cands=max_cands, variant=0)
            same_records(hg.decode(iq, cap=1 << 16), got, f"{name}: fast vs generic")
            record(hg, len(pres))
            hg.close()

    # host-call splits with max_blocks_per_call chunking equal one call
    rng = np.random.default_rng(seed + 17)
    h2 = handle(protos, max_blocks=int(rng.integers(3, 40)), max_cands=max_cands)
    parts, off = [], 0
    while off < nblk:
        n = int(min(nblk - off, rng.integers(1, 3 * 40)))
        parts.append(h2.decode(iq[off * c.block_size2:(off + n) * c.block_size2], cap=1 << 16))
        off += n
    same_records(np.concatenate(parts), got, f"{name}: split calls")
    h.close()
    h2.close()
    TIMES[name] = time.perf_counter() - t0
    return k, got, npk


# ---------------------------------------------------------------- tests
@gpu
@pytest.mark.parametrize("name", sorted(EDGES))
def test_edge_configuration(built, name):
    protos = EDGES[name]
    k, got, npk = check_config(name, protos)
    g = merged_geometry(protos)
    if name.startswith(("ps1_", "pk1_", "pkl4mod8")):   # the fast kernel's geometry does not fit: the generic kernel runs
        assert g["CL"] in (32, 56, 64, 72, 78) and k[0] == "demod_generic_kernel", k
    assert k[-1] == f"extract_words_kernel<{4 if g['PK'] <= 128 else 23}>", k
    if name.startswith("r900_pk115"):
        assert ("r900_chain2_kernel" in k) == (g["PKL"] % 8 == 0), k
    if any(p.check_kind == CRC for p in protos) and npk:
        assert (got["check_mask"] != 0).any(), name   # the injected CRC-valid packets pass their screen


@gpu
def test_r2_boundary_on_constant_input(built):
    """A 17-bit all-ones preamble with PreambleSymbols = PacketSymbols = 16 (n = PK + 1, the last length R2 accepts) on
    constant input: every start of every block whose Quantized holds no stream-start zeros is a candidate, and the
    Search reads plane bits up to the last one of the call."""
    protos = [make_protocol("1" * 17, 32, 16, 16)]
    g = merged_geometry(protos)
    assert rule_violated(protos) is None
    nblk = 48
    k, got, _ = check_config("r2_boundary", protos, nsamples=nblk * g["BS"], constant=True, max_cands=nblk * g["BS"])
    warm = -(-g["BUF"] // g["BS"])
    assert len(got) >= (nblk - warm) * g["BS"]


@gpu
@pytest.mark.parametrize("i", range(len(RANDOM)))
def test_random_accepted_configuration(built, i):
    check_config(f"random{i}", RANDOM[i], nsamples=1 << 20, seed=100 + i, full=False)


REJECTED = {
    "R1": [make_protocol("1" * 8, 32, 21, 20)],
    "R2": [make_protocol("1" * 18, 32, 16, 16)],
    "R3": [r900_proto(32, 114), make_protocol("1" * 21, 32, 21, 96)],
    "R4": [make_protocol("1" * 16, 40, 16, 100, CRC, (0xFFFF, 0x1021, 0x1D0F), (2, 13))],
}


@gpu
@pytest.mark.parametrize("rule", sorted(REJECTED))
def test_first_rejected_configuration_is_refused(built, rule):
    """Never decoded: on a library without the rule some of these read past the caller's buffer."""
    protos = REJECTED[rule]
    assert rule_violated(protos) == rule
    h = capi.Handle()
    for p in protos:
        h.register(p)
    rc = h._L.ertgpu_allocate(h._h, 0, 0, 0)
    msg = (h._L.ertgpu_last_error(h._h) or b"").decode()
    h.close()
    assert rc == capi.EINVAL and msg.startswith(rule + ":"), (rc, msg)


@gpu
def test_every_custom_geometry_kernel_was_seen(built):
    """Runs last: both demod kernels, search_generic_kernel with 5 or more preambles, every run-time-pattern slide
    instance, both extract instances and both r900 paths were launched by the tests above."""
    if not SEEN:
        pytest.skip("collects what the other tests of this file launched: run the whole file")
    print("seconds per configuration:", {k: round(v, 2) for k, v in sorted(TIMES.items())})
    assert "demod_generic_kernel" in SEEN and any(s.startswith("demod_fast_kernel<") for s in SEEN), SEEN
    assert max(SEEN_GENERIC_NPRE, default=0) >= 5, SEEN_GENERIC_NPRE
    slides = {s for s in SEEN if s.startswith("search_slide_kernel<") and "0x" not in s}
    assert {s.split(",")[0] for s in slides} == {f"search_slide_kernel<{n}" for n in (1, 2, 3, 4)}, slides
    assert {"extract_words_kernel<4>", "extract_words_kernel<23>"} <= SEEN, SEEN
    assert {"r900_chain2_kernel", "r900_replay_kernel"} <= SEEN, SEEN
