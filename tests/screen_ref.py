"""The parsers' integrity screens restated from the reference, a corpus of packets with designed verdicts near the screens'
decision boundaries, and single wrong variants of the screens that the corpus must tell apart from the right ones.

The restatement shares no code with the kernel (table CRC, linearised syndrome table) nor with the oracle (C):
  * CRC: bit by bit, crc/crc.go:34-55 (a table entry is eight of these shifts);
  * IDM pair: the packet CRC over Bytes[4:92] and the serial CRC over Bytes[9:13] + Bytes[88:90], idm/idm.go:77-87 and
    netidm/netidm.go:88-98, with the protocol's own init, polynomial and residue;
  * r900: two base-6 digits per symbol, a symbol above 31 fails, and Syndrome(msg, 5, 29) of the 31-symbol word (16 data
    symbols, 10 zeros, 5 parity symbols) by Horner's rule, r900/r900.go:195-221 and r900/gf/gf.go:20-57,152-172.

A corpus group is a protocol set and its entries.  An entry is one transmitted packet (its bits from the first preamble
bit, or the 42 payload digits of an r900 packet) and one view per protocol that screens it: the candidate `offset`
symbols after the packet's first symbol and the verdict it was designed to get."""
from __future__ import annotations

import functools
from dataclasses import dataclass

import numpy as np

import oracle
from helpers import _feed, make_protocol, merged_geometry
from rtlamr_b200 import capi, synth

NONE, CRC16, IDM, R900 = capi.CHECK_NONE, capi.CHECK_CRC16, capi.CHECK_IDM, capi.CHECK_R900
R900_PRE = synth.PREAMBLE["r900"]


# ---------------------------------------------------------------- the screens, restated
def crc(init: int, poly: int, data: bytes) -> int:
    """crc.Checksum(init, data, NewTable(poly)) one bit at a time."""
    reg = init
    for v in data:
        for k in range(7, -1, -1):
            top = ((reg >> 15) ^ (v >> k)) & 1
            reg = (reg << 1) & 0xFFFF
            if top:
                reg ^= poly
    return reg


def _gf_mul_slow(x: int, y: int) -> int:   # gf.go:81-94, order 32, polynomial 37
    z = 0
    while x > 0:
        if x & 1:
            z ^= y
        x >>= 1
        y <<= 1
        if y & 32:
            y ^= 37
    return z


GF_EXP, GF_LOG = [0] * 62, [0] * 32   # gf.NewField(32, 37, 2), r900.go:68
_x = 1
for _i in range(31):
    GF_EXP[_i] = GF_EXP[_i + 31] = _x
    GF_LOG[_x] = _i
    _x = _gf_mul_slow(_x, 2)


def gf_mul(x: int, y: int) -> int:
    return 0 if x == 0 or y == 0 else GF_EXP[GF_LOG[x] + GF_LOG[y]]


def syndrome(message, nparity: int = 5, offset: int = 29) -> list[int]:
    """Field.Syndrome (gf.go:152-172): Horner's rule at Exp(offset + idx) for each idx."""
    out = []
    for idx in range(nparity):
        root = GF_EXP[(offset + idx) % 31]
        syn = message[0]
        for v in message[1:]:
            syn = gf_mul(syn, root) ^ v
        out.append(syn)
    return out


def r900_symbols(digits) -> list[int]:
    """strconv.ParseInt(digits[2k:2k+2], 6, 32) for the 21 symbols (r900.go:199-207), before the > 31 test."""
    return [int(digits[2 * k]) * 6 + int(digits[2 * k + 1]) for k in range(21)]


MUTANTS = ("no_serial_crc", "serial_89_91", "range_end_minus_1", "range_start_plus_1", "residue_ignored",
           "four_syndromes", "no_gt31_test", "position_map_15")


def screen(p, data: bytes = b"", digits=None, mutant: str | None = None) -> bool:
    """Bit of check_mask for a candidate filed under protocol struct `p` (its bytes `data`, its r900 digits), or the
    verdict of one wrong variant of that screen (`mutant`, one of MUTANTS)."""
    kind = p.check_kind
    if kind == NONE:
        return True
    if kind in (CRC16, IDM):
        lo, hi = (p.crc_from, p.crc_to) if kind == CRC16 else (4, 92)
        lo += mutant == "range_start_plus_1"
        hi -= mutant == "range_end_minus_1"
        res = 0 if mutant == "residue_ignored" else p.crc_residue
        ok = crc(p.crc_init, p.crc_poly, data[lo:hi]) == res
        if kind == IDM and mutant != "no_serial_crc":
            tail = data[89:91] if mutant == "serial_89_91" else data[88:90]
            ok = ok and crc(p.crc_init, p.crc_poly, data[9:13] + tail) == res
        return ok
    if kind == R900:
        sym = r900_symbols(digits)
        if mutant == "no_gt31_test":
            sym = [s & 31 for s in sym]
        elif max(sym) > 31:
            return False
        split = 15 if mutant == "position_map_15" else 16
        word = sym[:split] + [0] * 10 + sym[split:]      # r900.go:215-216
        return not any(syndrome(word, 4 if mutant == "four_syndromes" else 5, 29))
    raise ValueError(f"check kind {kind}")


def parser_emits(name: str, data: bytes = b"", digits=None) -> bool:
    """The stock parser's rules after its checksum (a message needs both): scm.go:83-85 ID != 0, scmplus.go:84-86
    EndpointID != 0 and ProtocolID == 0x1E, idm.go:90-92 / netidm.go:103-105 ERTSerialNumber != 0; r900 has none."""
    if name == "scm":
        bits = np.unpackbits(np.frombuffer(data[:12], np.uint8))
        return bool(bits[21:23].any() or bits[56:80].any())
    if name == "scm+":
        return data[2] == 0x1E and data[4:8] != bytes(4)
    if name in ("idm", "netidm"):
        return data[9:13] != bytes(4)
    return name in ("r900", "r900bcd")


# ---------------------------------------------------------------- building packets
_ZZ = {}


def solve_tail(prefix: bytes, init: int, poly: int, residue: int) -> bytes | None:
    """Two bytes b with crc(init, prefix + b) == residue, or None.  Feeding b from register R equals feeding two zero
    bytes from R ^ b, so b = R ^ u for any u that two zero bytes take to the residue."""
    if poly not in _ZZ:
        r = np.arange(1 << 16, dtype=np.uint32)
        for _ in range(16):
            r = np.where(r & 0x8000, ((r << 1) ^ poly) & 0xFFFF, (r << 1) & 0xFFFF)
        _ZZ[poly] = r
    u = np.nonzero(_ZZ[poly] == residue)[0]
    if u.size == 0:
        return None
    b = crc(init, poly, prefix) ^ int(u[0])
    out = b.to_bytes(2, "big")
    assert crc(init, poly, prefix + out) == residue
    return out


def to_bits(b: bytes) -> list[int]:
    return [int(x) for x in np.unpackbits(np.frombuffer(bytes(b), np.uint8))]


def to_bytes(bits) -> bytes:
    return np.packbits(np.array(list(bits), np.uint8)).tobytes()


def cand_bytes(bits, pk: int) -> bytes:
    """A candidate's bytes of PacketSymbols pk: MSB first, a trailing partial byte holds its pk%8 bits in the low bits."""
    b = bytearray(to_bytes(list(bits[:pk])))
    if pk % 8:
        b[-1] >>= 8 - pk % 8
    return bytes(b)


def digits_of(symbols) -> tuple:
    return tuple(d for s in symbols for d in (s // 6, s % 6))


def gf_poly(nroots: int) -> list[int]:
    """prod_j (x + a^(29+j)), j < nroots, highest degree first."""
    g = [1]
    for j in range(nroots):
        root = GF_EXP[(29 + j) % 31]
        ng = g + [0]
        for i, c in enumerate(g):
            ng[i + 1] ^= gf_mul(c, root)
        g = ng
    return g


def r900_valid(rng, fixed: dict | None = None) -> list[int]:
    """21 symbols of a valid codeword: 16 data symbols (some fixed) and their parity."""
    data = [int(v) for v in rng.integers(0, 32, 16)]
    for k, v in (fixed or {}).items():
        data[k] = v
    sym = data + synth.rs_parity(data)
    assert not any(syndrome(sym[:16] + [0] * 10 + sym[16:]))
    return sym


# ---------------------------------------------------------------- corpus
@dataclass(frozen=True)
class View:
    proto: int      # index of the protocol in the group's list
    offset: int     # symbols from the packet's first symbol to the candidate's symbol 0
    passes: bool    # the verdict the entry was designed to get


@dataclass(frozen=True)
class Entry:
    cls: str
    bits: tuple | None      # transmitted bits, preamble first (byte protocols)
    digits: tuple | None    # the 42 payload digits (r900)
    views: tuple


@dataclass
class Group:
    name: str
    msgtypes: str | None    # stock parsers (oracle messages, host.Parsers), None for custom protocols
    protos: object          # chip length -> list of capi.Protocol
    entries: list
    chip_lengths: tuple


def _views(protos_idx, passes, offset=0):
    return tuple(View(i, offset, passes) for i in protos_idx)


def _flip(bits, positions):
    b = list(bits)
    for q in positions:
        b[q] ^= 1
    return tuple(b)


def crc_entries(rng, p, pre: int, pk: int, packets, views=(0,), full_sweep=True):
    """Entries for a CRC16 screen over bits [8 crc_from, 8 crc_to) of packets `packets` (bit tuples of pk bits)."""
    lo, hi = 8 * p.crc_from, 8 * p.crc_to
    args = (p.crc_init, p.crc_poly, p.crc_residue)
    inside = lambda qs: all(lo <= q < hi for q in qs)                   # noqa: E731
    base = packets[0]
    out = [Entry("valid", b, None, _views(views, True)) for b in packets]
    sweep = range(pre, pk) if full_sweep else sorted(rng.choice(np.arange(pre, pk), 24, replace=False))
    for q in sweep:                                                     # a single flip fails inside the range only
        out.append(Entry("flip1", _flip(base, [q]), None, _views(views, not lo <= q < hi)))
    first = max(pre, lo)
    for n in range(2, 17):                                              # bursts: first and last bit flipped
        for _ in range(2):
            s = int(rng.integers(first, hi - n + 1))
            qs = [s, s + n - 1] + [s + 1 + int(i) for i in np.nonzero(rng.integers(0, 2, n - 2))[0]]
            out.append(Entry(f"burst{n}", _flip(base, qs), None, _views(views, False)))
    for _ in range(20):                                                 # two flips: the restatement decides
        qs = sorted(int(x) for x in rng.choice(np.arange(pre, pk), 2, replace=False))
        b = _flip(base, qs)
        out.append(Entry("flip2", b, None, _views(views, screen(p, cand_bytes(b, pk)))))
    for _ in range(3):                                                  # forged: bytes changed, CRC recomputed
        d = bytearray(to_bytes(base[:8 * (pk // 8)]) + bytes(1))
        for k in rng.choice(np.arange(max(p.crc_from, -(-pre // 8)), p.crc_to - 2), 3, replace=False):
            d[int(k)] = int(rng.integers(0, 256))
        d[p.crc_to - 2:p.crc_to] = solve_tail(bytes(d[p.crc_from:p.crc_to - 2]), *args)
        b = tuple(to_bits(d)[:8 * (pk // 8)]) + tuple(base[8 * (pk // 8):])
        out.append(Entry("forged", b, None, _views(views, True)))
    g = [1] + [(p.crc_poly >> (15 - j)) & 1 for j in range(16)]          # g(x) = x^16 + poly, highest degree first
    gq = [j for j in range(17) if g[j]]
    for s in range(first, hi - 16, 3):                                  # g(x) x^k wholly inside: passes
        out.append(Entry("gxk", _flip(base, [s + j for j in gq]), None, _views(views, True)))
    edges = [s for s in range(lo - 17, lo + 2)] + [s for s in range(hi - 18, hi + 1)]
    for s in sorted(set(edges)):                                        # slid across a range edge one bit at a time
        qs = [s + j for j in gq]
        if qs[0] < pre or qs[-1] >= pk:
            continue
        n_in = sum(lo <= q < hi for q in qs)
        out.append(Entry("gxk_edge", _flip(base, qs), None, _views(views, n_in in (0, len(qs)))))
    return out


def scm_packets(rng, n):
    out = []
    for _ in range(n):
        d = synth.encode_scm(int(rng.integers(1, 1 << 26)) | 1, int(rng.integers(0, 16)), int(rng.integers(0, 4)),
                             int(rng.integers(0, 4)), int(rng.integers(0, 1 << 24)))
        out.append(tuple(to_bits(d)))
    return out


def scmplus_packets(rng, n):
    return [tuple(to_bits(synth.encode_scmplus(int(rng.integers(0, 256)), int(rng.integers(1, 1 << 32)) | 1,
                                               int(rng.integers(0, 1 << 32)), int(rng.integers(0, 1 << 16)))))
            for _ in range(n)]


def custom_crc_packets(rng, p, pre: str, pk: int, n):
    out = []
    for _ in range(n):
        b = [int(c) for c in pre] + [int(x) for x in rng.integers(0, 2, pk - len(pre))]
        d = bytearray(to_bytes(b[:8 * (pk // 8)]))
        d[p.crc_to - 2:p.crc_to] = solve_tail(bytes(d[p.crc_from:p.crc_to - 2]), p.crc_init, p.crc_poly, p.crc_residue)
        out.append(tuple(to_bits(d)) + tuple(b[8 * (pk // 8):]))
    return out


def idm_bytes(rng, pre4: bytes, crcp, ptype=0x1C, serial=None) -> bytearray:
    """A valid IDM-layout packet (idm.go:121-156) under CRC parameters crcp = (init, poly, residue)."""
    b = bytearray(92)
    b[0:4] = pre4
    b[4], b[5], b[6], b[7] = ptype, 0x5C, 0xC6, 0x01
    b[8] = int(rng.integers(0, 16))
    b[9:13] = (serial or int(rng.integers(1 << 24, 1 << 32))).to_bytes(4, "big")
    b[13:88] = rng.integers(0, 256, 75, dtype=np.uint8).tobytes()
    idm_repair(b, crcp, serial_too=True)
    return b


def idm_repair(b: bytearray, crcp, serial_too=False):
    if serial_too:
        b[88:90] = solve_tail(bytes(b[9:13]), *crcp)
    b[90:92] = solve_tail(bytes(b[4:90]), *crcp)


def idm_entries(rng, pre4: bytes, crcp, views, flips="full"):
    """The four quadrants of the IDM pair and single flips of the bytes both CRCs read."""
    mk = lambda b, cls, ok: Entry(cls, tuple(to_bits(b)), None, _views(views, ok))   # noqa: E731
    out = []
    for _ in range(3):
        out.append(mk(idm_bytes(rng, pre4, crcp), "valid", True))
    for _ in range(3):                                      # the packet CRC fails only: a filler bit flipped
        b = idm_bytes(rng, pre4, crcp)
        b[int(rng.integers(14, 86))] ^= 1 << int(rng.integers(0, 8))
        out.append(mk(b, "packet_crc_fails", False))
    for k in range(3):                                      # the serial CRC fails only: tampered, packet CRC repaired
        b = idm_bytes(rng, pre4, crcp)
        b[9 + k if k < 2 else 88] ^= 0x10
        idm_repair(b, crcp)
        assert b[9:13] != bytes(4)
        out.append(mk(b, "serial_crc_fails", False))
    for k in range(3):                                      # both fail
        b = idm_bytes(rng, pre4, crcp)
        b[10 + k if k < 2 else 89] ^= 0x21
        out.append(mk(b, "both_fail", False))
    base = idm_bytes(rng, pre4, crcp)
    qs = [8 * k + j for k in list(range(4, 14)) + list(range(86, 92)) for j in range(8)]
    if flips != "full":
        qs = qs[::3]
    qs += sorted(int(x) for x in rng.choice(np.arange(8 * 14, 8 * 86), 24 if flips == "full" else 8, replace=False))
    for q in qs:
        b = bytearray(base)
        b[q >> 3] ^= 0x80 >> (q & 7)
        out.append(mk(b, "flip1", False))
    return out


def cross_entry(rng, idx_scmplus: int, idx_idm: int) -> Entry:
    """An idm packet whose scm+-aligned slice (the scm+ preamble is the idm preamble's last 16 bits) passes scm+'s CRC
    and carries ProtocolID 0x1E, so that both parsers emit it."""
    b = idm_bytes(rng, bytes.fromhex("555516A3"), (0xFFFF, 0x1021, 0x1D0F), ptype=0x1E)
    b[16:18] = solve_tail(bytes(b[4:16]), 0xFFFF, 0x1021, 0x1D0F)   # scm+ bytes [2,16) are idm bytes [4,18)
    idm_repair(b, (0xFFFF, 0x1021, 0x1D0F))
    return Entry("cross_preamble", tuple(to_bits(b)), None, (View(idx_scmplus, 16, True), View(idx_idm, 0, True)))


def r900_entries(rng, views, full=True):
    mk = lambda sym, cls, ok: Entry(cls, None, digits_of(sym), _views(views, ok))   # noqa: E731
    out = [mk(r900_valid(rng, {15: 17 + k}), "valid", True) for k in range(4)]
    base = r900_valid(rng, {15: 9})
    for pi in range(21):                                    # one symbol wrong: every position, every nonzero error
        for e in (range(1, 32) if full else [1 + (7 * pi) % 31]):
            s = list(base)
            s[pi] ^= e
            out.append(mk(s, "symbol_error", False))
    for n in (2, 3, 4, 5):                                  # 2..5 symbols wrong: below the minimum distance 6
        for _ in range(5 if full else 1):
            s = list(base)
            for pi in rng.choice(21, n, replace=False):
                s[int(pi)] ^= int(rng.integers(1, 32))
            out.append(mk(s, f"errors{n}", False))
    for nroots, ok in ((5, True), (4, False)):              # g(x) x^k wholly in the data symbols (degrees 15..30):
        g = gf_poly(nroots)                                 # a codeword of weight 6; the 4-root polynomial leaves
        for k in range(15, 31 - nroots, 1 if full or nroots == 5 else 4):   # only the 5th syndrome
            s = list(base)
            for j, c in enumerate(g):
                pi = 30 - (k + nroots - j)                  # degree d sits at word position 30 - d, data symbol pi
                assert 0 <= pi < 16
                s[pi] ^= c
            out.append(mk(s, f"codeword_x{k}" if ok else f"four_roots_x{k}", ok))
    for pi in range(21):                                    # symbol v <= 3 written as the digit pair of v + 32
        v = pi % 4
        while True:
            s = r900_valid(rng, {pi: v} if pi < 16 else None)
            if s[pi] == v:
                break
        d = list(digits_of(s))
        d[2 * pi], d[2 * pi + 1] = divmod(v + 32, 6)
        out.append(Entry("pair_over_31", None, tuple(d), _views(views, False)))
    return out


CUSTOM_CRC_A = ("010011101100011110100101", 24, 160, (0x3A5C, 0x8005, 0x4B37), (5, 17))   # bytes 3,4 and 17,18,19 outside
CUSTOM_CRC_B = ("01100101110100011011", 20, 150, (0xFFFF, 0x1020, None), (3, 18))         # even polynomial, PK % 8 = 6
CUSTOM_IDM_PRE = "10110010011101001100101011110001"
CUSTOM_IDM_CRC = (0x4C11, 0x8BB7, 0x2F0D)
CUSTOM_IDM_RANGES = ((0, 0), (4, 92), (2, 50), (10, 92))


def custom_crc_protocol(spec, cl):
    pre, ps, pk, (init, poly, res), rng_ = spec
    if res is None:     # a residue the even polynomial can reach: the CRC of some message
        res = crc(init, poly, bytes(range(40, 55)))
    return make_protocol(pre, cl, ps, pk, CRC16, (init, poly, res), rng_, name="crc_custom")


def custom_idm_protocols(cl):
    return [make_protocol(CUSTOM_IDM_PRE, cl, 32, 92 * 8, IDM, CUSTOM_IDM_CRC, r, name=f"idm_custom{i}")
            for i, r in enumerate(CUSTOM_IDM_RANGES)]


def custom_r900_protocol(cl):
    return make_protocol(R900_PRE, cl, 32, 115, R900, name="r900_custom")


def _stock(names):
    return lambda cl: [capi.stock_protocol(m, cl) for m in names.split(",")]


# (group name, stock message types or None, chip lengths): what the tests parametrize over, known without the library
GROUPS = (("scm", "scm", (72, 16)), ("scm+", "scm+", (72, 16)), ("idm,netidm", "idm,netidm", (72, 16)),
          ("scm+,idm", "scm+,idm", (72, 16)), ("r900,r900bcd", "r900,r900bcd", (72, 16)),
          ("crc_custom_a", None, (72, 16)), ("crc_custom_b", None, (72, 16)), ("idm_custom", None, (72, 16)),
          ("all", "scm,scm+,idm,r900", (72, 16)), ("r900_custom", None, (33,)))


@functools.lru_cache(maxsize=None)
def corpus() -> dict:
    """build_corpus(), once per process (it needs libertgpu.so for the stock protocol structs)."""
    G = build_corpus()
    assert [(g.name, g.msgtypes, g.chip_lengths) for g in G.values()] == list(GROUPS)
    return G


def build_corpus() -> dict:
    """{group name: Group}, the same on every call."""
    G = {}
    rng = np.random.default_rng(0x5C4EE7)
    scm = _stock("scm")(72)[0]
    G["scm"] = Group("scm", "scm", _stock("scm"), crc_entries(rng, scm, 21, 96, scm_packets(rng, 3)), (72, 16))
    sp = _stock("scm+")(72)[0]
    G["scm+"] = Group("scm+", "scm+", _stock("scm+"), crc_entries(rng, sp, 16, 128, scmplus_packets(rng, 3)), (72, 16))
    pre4 = bytes.fromhex("555516A3")
    G["idm,netidm"] = Group("idm,netidm", "idm,netidm", _stock("idm,netidm"),
                            idm_entries(rng, pre4, (0xFFFF, 0x1021, 0x1D0F), (0, 1)), (72, 16))
    cross = [cross_entry(rng, 0, 1) for _ in range(2)]
    plain = idm_bytes(rng, pre4, (0xFFFF, 0x1021, 0x1D0F))
    cross.append(Entry("cross_preamble", tuple(to_bits(plain)), None,
                       (View(0, 16, screen(sp, cand_bytes(to_bits(plain)[16:], 128))), View(1, 0, True))))
    cross += [Entry("valid", b, None, (View(0, 0, True),)) for b in scmplus_packets(rng, 2)]
    G["scm+,idm"] = Group("scm+,idm", "scm+,idm", _stock("scm+,idm"), cross, (72, 16))
    G["r900,r900bcd"] = Group("r900,r900bcd", "r900,r900bcd", _stock("r900,r900bcd"), r900_entries(rng, (0, 1)),
                              (72, 16))
    for name, spec in (("crc_custom_a", CUSTOM_CRC_A), ("crc_custom_b", CUSTOM_CRC_B)):
        p = custom_crc_protocol(spec, 72)
        pk = spec[2]
        G[name] = Group(name, None, lambda cl, s=spec: [custom_crc_protocol(s, cl)],
                        crc_entries(rng, p, spec[1], pk, custom_crc_packets(rng, p, spec[0], pk, 2)), (72, 16))
    G["idm_custom"] = Group("idm_custom", None, custom_idm_protocols,
                            idm_entries(rng, to_bytes(int(c) for c in CUSTOM_IDM_PRE), CUSTOM_IDM_CRC, (0, 1, 2, 3),
                                        flips="sample"), (72, 16))
    # -msgtype=all: a few entries of every kind, the cross-preamble packet among them; views re-filed under the index
    # of their protocol in "scm,scm+,idm,r900"
    def pick(group, counts, proto, offset=0):
        out = []
        for cls, n in counts:
            es = [e for e in G[group].entries if e.cls == cls]
            assert len(es) >= n, (group, cls)
            out += [Entry(e.cls, e.bits, e.digits, (View(proto, offset, e.views[0].passes),)) for e in es[:n]]
        return out
    allg = pick("scm", (("valid", 2), ("gxk", 2), ("flip1", 2)), 0)
    allg += pick("scm+", (("valid", 2), ("flip1", 1), ("burst9", 1)), 1)
    allg += pick("idm,netidm", (("valid", 2), ("packet_crc_fails", 1), ("serial_crc_fails", 2), ("both_fail", 1)), 2)
    allg += [Entry(e.cls, e.bits, None, (View(1, 16, True), View(2, 0, True)))
             for e in G["scm+,idm"].entries if e.cls == "cross_preamble" and all(v.passes for v in e.views)][:1]
    allg += pick("r900,r900bcd", (("valid", 2), ("symbol_error", 2), ("errors5", 2), ("codeword_x20", 1),
                                  ("four_roots_x15", 1), ("pair_over_31", 4)), 3)
    G["all"] = Group("all", "scm,scm+,idm,r900", _stock("scm,scm+,idm,r900"), allg, (72, 16))
    G["r900_custom"] = Group("r900_custom", None, lambda cl: [custom_r900_protocol(cl)],
                             r900_entries(np.random.default_rng(0x900C), (0,), full=False), (33,))
    return G


# ---------------------------------------------------------------- streams
@dataclass
class Stream:
    iq: np.ndarray
    starts: list            # first sample of each entry's packet
    geo: dict               # helpers.merged_geometry
    protos: list


def view_data(entry: Entry, view: View, protos) -> tuple[bytes, tuple | None]:
    """(candidate bytes of the view's protocol, r900 digits) the entry was designed to give."""
    if entry.digits is not None:
        return b"", entry.digits
    pk = protos[view.proto].packet_symbols
    return cand_bytes(entry.bits[view.offset:view.offset + pk], pk), None


def make_stream(group: Group, cl: int, seed: int = 0x51EA) -> Stream:
    """The group's packets in order behind seeded noise (synth.host_fill, carrier 40/30 as the protocol-config tests),
    whole blocks, with room after the last packet for its candidates."""
    protos = group.protos(cl)
    g = merged_geometry(protos)
    rng = np.random.default_rng(seed + cl)
    rows, starts = [], []
    s = g["BUF"] + int(rng.integers(0, g["BS"]))
    for e in group.entries:
        chips = synth.manchester_chips(list(e.bits)) if e.digits is None else synth.r900_chips(e.digits)
        row = np.zeros((), dtype=capi.SYNTH_DTYPE)
        row["start_sample"], row["n_chips"], row["chip_length"] = s, len(chips), cl
        row["amp_i"], row["amp_q"] = 40, 30
        pk = np.packbits(np.array(chips, np.uint8))
        row["chips"][:len(pk)] = pk
        rows.append(row)
        starts.append(s)
        s += len(chips) * cl + 4 * g["SL"] + int(rng.integers(0, g["BS"]))
    n = s + 2 * g["BUF"] + 2 * g["BS"]
    n = -(-n // g["BS"]) * g["BS"]
    iq = synth.host_fill(0, n, seed, np.array(rows, dtype=capi.SYNTH_DTYPE))
    return Stream(iq, starts, g, protos)


def first_sample(geo, block: int, idx: int) -> int:
    """Sample at which symbol 0 of candidate (block, idx) starts (decode.go:163-197, 229-245, 369)."""
    return (block + 1) * geo["BS"] - geo["BUF"] + idx - geo["SL"]


def preamble_ids(protos) -> list[int]:
    order, ids = [], []
    for p in protos:
        pre = bytes(p.preamble).split(b"\0")[0]
        if pre not in order:
            order.append(pre)
        ids.append(order.index(pre))
    return ids


def locate(stream: Stream, group: Group, cands, tol: int = 2):
    """{(entry index, view index): [candidates]}: the candidates (anything with .block, .idx, .preamble_id) of the
    view's preamble whose symbol 0 lies within `tol` samples of the view's first symbol."""
    ids = preamble_ids(stream.protos)
    geo = stream.geo
    by_pid = {}
    for c in cands:
        by_pid.setdefault(int(c.preamble_id), []).append((first_sample(geo, int(c.block), int(c.idx)), c))
    for v in by_pid.values():
        v.sort(key=lambda t: t[0])
    keys = {k: np.array([t[0] for t in v]) for k, v in by_pid.items()}
    out = {}
    for i, (e, s) in enumerate(zip(group.entries, stream.starts)):
        for j, v in enumerate(e.views):
            pid = ids[v.proto]
            want = s + v.offset * geo["SL"]
            if pid not in keys:
                out[(i, j)] = []
                continue
            a, b = np.searchsorted(keys[pid], [want - tol, want + tol + 1])
            out[(i, j)] = [t[1] for t in by_pid[pid][a:b]]
    return out


def entry_of_sample(stream: Stream, sample: int) -> int:
    """Index of the entry whose packet holds `sample`."""
    return int(np.searchsorted(np.array(stream.starts), sample, side="right")) - 1


def oracle_digits(protos, iq, pid):
    """{(block, idx): 42 digits} of every candidate of preamble `pid`, read from the oracle's r900 quantized after the
    candidate's own block (helpers.oracle_r900_digits for protocol structs)."""
    search = oracle.SEARCH_GO if (2 * protos[0].chip_length) % 8 == 0 else oracle.SEARCH_EXACT
    o = oracle.Oracle.from_protocols(protos, search)
    bs2, bs, cl = o.cfg.block_size2, o.cfg.block_size, o.cfg.chip_length
    pos = o.cfg.preamble_length - o.cfg.symbol_length + 4 * cl * np.arange(42)
    ends = sorted({x.block for x in _feed(o, iq) if x.preamble_id == pid})
    o.close()
    o = oracle.Oracle.from_protocols(protos, search)
    out, prev = {}, 0
    for b in ends:
        n = b + 1 - prev
        part, _ = o.decode(iq[prev * bs2:(b + 1) * bs2], cand_cap=4096 + bs * n, msg_cap=256 + 16 * n)
        prev = b + 1
        q = o.r900_quantized()
        for x in part:
            if x.preamble_id == pid and x.block == b:
                out[(x.block, x.idx)] = tuple(int(d) for d in q[x.idx + pos])
    o.close()
    return out
