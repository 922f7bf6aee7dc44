"""Shared helpers for the parity tests: run the oracle and the CUDA path on the same bytes."""
from __future__ import annotations

import numpy as np

import oracle
from rtlamr_b200 import capi, synth


def whole_blocks(iq: np.ndarray, bs2: int) -> np.ndarray:
    return iq[: (iq.size // bs2) * bs2]


def oracle_run(msgtypes, cl, iq, search=None):
    if search is None:
        search = oracle.SEARCH_GO if (2 * cl) % 8 == 0 else oracle.SEARCH_EXACT
    o = oracle.Oracle(msgtypes, cl, search)
    iq = whole_blocks(iq, o.cfg.block_size2)
    cands, msgs = o.decode(iq, cand_cap=1 << 18, msg_cap=1 << 16)
    return o, cands, msgs


def cand_key_oracle(c, nbytes, pk_symbols):
    data = bytearray(c.data[:nbytes])
    if pk_symbols % 8:  # stale bits of the reused d.pkt in the last byte (decode.go:363-366): not comparable
        data[-1] &= (0xFF >> (8 - pk_symbols % 8))
    return (c.block, c.preamble_id, c.idx, bytes(data))


def cand_key_gpu(row, nbytes, pk_symbols):
    data = bytearray(row["bytes"][:nbytes].tobytes())
    if pk_symbols % 8:
        data[-1] &= (0xFF >> (8 - pk_symbols % 8))
    return (int(row["block"]), int(row["preamble_id"]), int(row["idx"]), bytes(data))


def synth_stream(msgtypes, cl, nsamples, seed=0x5EED0001, spacing=1 << 19, pkt_seed=7):
    pk, truth = synth.make_packets(msgtypes, cl, nsamples, seed=pkt_seed, spacing=spacing)
    return synth.host_fill(0, nsamples, seed, pk), pk, truth


# ---- the integrity screens, restated with the oracle's own crc/gf functions (crc/crc.go, r900/gf/gf.go) ----
def screen_expected(proto, data: bytes, digits=None) -> bool:
    """What bit i of check_mask must be for a candidate filed under parser `proto` (a stock name or a capi.Protocol):
    scm/scm.go:76, scmplus/scmplus.go:77, idm/idm.go:77-87, netidm/netidm.go:88-98, r900/r900.go:199-221; a protocol
    struct's own CRC16 (init, polynomial, residue over bytes [crc_from, crc_to)), its own IDM pair (init, polynomial,
    residue over Bytes[4:92] and Bytes[9:13] + Bytes[88:90], whatever its range fields say) or ERTGPU_CHECK_NONE
    (always set)."""
    if not isinstance(proto, str):
        kind = proto.check_kind
        if kind == capi.CHECK_NONE:
            return True
        if kind == capi.CHECK_CRC16:
            return oracle.crc_checksum(proto.crc_init, data[proto.crc_from:proto.crc_to], proto.crc_poly) == proto.crc_residue
        if kind == capi.CHECK_IDM:
            init, poly, res = proto.crc_init, proto.crc_poly, proto.crc_residue
            return (oracle.crc_checksum(init, data[4:92], poly) == res
                    and oracle.crc_checksum(init, data[9:13] + data[88:90], poly) == res)
        proto = {capi.CHECK_R900: "r900"}[kind]
    if proto == "scm":
        return oracle.crc_checksum(0, data[2:12], 0x6F63) == 0
    if proto == "scm+":
        return oracle.crc_checksum(0xFFFF, data[2:16], 0x1021) == 0x1D0F
    if proto in ("idm", "netidm"):
        return (oracle.crc_checksum(0xFFFF, data[4:92], 0x1021) == 0x1D0F
                and oracle.crc_checksum(0xFFFF, data[9:13] + data[88:90], 0x1021) == 0x1D0F)
    if proto in ("r900", "r900bcd"):
        sym = [digits[2 * k] * 6 + digits[2 * k + 1] for k in range(21)]
        if max(sym) > 31:
            return False
        msg = bytes(sym[:16]) + bytes(10) + bytes(sym[16:])
        return oracle.gf32_syndrome(msg, 5, 29) == bytes(5)
    raise ValueError(proto)


PREAMBLES = {"scm": "111110010101001100000", "scm+": "0001011010100011", "idm": "01010101010101010001011010100011",
             "netidm": "01010101010101010001011010100011", "r900": "00000000000000001110010101100100",
             "r900bcd": "00000000000000001110010101100100"}


def _names(msgtypes):
    return [m.strip() for m in msgtypes.split(",") if m.strip()] if isinstance(msgtypes, str) else list(msgtypes)


def r900_preamble_id(msgtypes):
    """preamble_id of the r900 preamble among the distinct preambles in registration order (decode.go:121-124)."""
    order = []
    for m in _names(msgtypes):
        if PREAMBLES[m] not in order:
            order.append(PREAMBLES[m])
    return order.index(PREAMBLES["r900"])


def _feed(o, iq, chunk=128):
    """Decode whole blocks in chunks whose candidate arrays stay small (the oracle's state runs on across calls)."""
    bs2, out = o.cfg.block_size2, []
    for a in range(0, iq.size // bs2, chunk):
        part = iq[a * bs2:(a + chunk) * bs2]
        n = part.size // bs2
        out += o.decode(part, cand_cap=4096 + 512 * n, msg_cap=256 + 16 * n)[0]
    return out


def oracle_r900_digits(mt, cl, iq, first_block=0, cuts=()):
    """{(block, idx, preamble_id): 42 digits as bytes} for every r900-preamble candidate the oracle finds in `iq` (whole
    blocks, the stream's first bytes: nothing in front of them), blocks numbered from `first_block`.  Digit k is the r900
    parser's quantized[idx + PL - SL + 4*k*CL] (r900.go:187-193) after the candidate's own block: a first pass finds those
    blocks, a second one feeds the oracle in segments ending at each of them (and at the blocks in `cuts`)."""
    search = oracle.SEARCH_GO if (2 * cl) % 8 == 0 else oracle.SEARCH_EXACT
    pid = r900_preamble_id(mt)
    o = oracle.Oracle(mt, cl, search)
    bs2 = o.cfg.block_size2
    iq = whole_blocks(iq, bs2)
    ends = sorted({c.block for c in _feed(o, iq) if c.preamble_id == pid} | set(cuts))
    o.close()
    o = oracle.Oracle(mt, cl, search)
    c = o.cfg
    pos = c.preamble_length - c.symbol_length + 4 * cl * np.arange(42)
    out, prev = {}, 0
    for b in ends:
        cands = _feed(o, iq[prev * bs2:(b + 1) * bs2])
        prev = b + 1
        hits = [x for x in cands if x.preamble_id == pid and x.block == b]
        if hits:
            q = o.r900_quantized()
            for x in hits:
                out[(x.block + first_block, x.idx, pid)] = q[x.idx + pos].tobytes()
    o.close()
    return out


def r900_symbols(digits):
    """The 21 symbols of 42 base-6 digits (r900.go:188-197); None if one exceeds 31 (the parser drops the candidate)."""
    sym = [digits[2 * k] * 6 + digits[2 * k + 1] for k in range(21)]
    return None if max(sym) > 31 else sym


def compare_r900_digits(got, msgtypes, want):
    """Every GPU record against oracle_r900_digits: a record of the r900 preamble carries CAND_HAS_R900 and exactly the
    oracle's 42 digits, every other record neither; the r900 records are exactly the oracle's r900 candidates; and every
    r900 / r900bcd bit of check_mask is screen_expected of the ORACLE's digits.  Returns (records compared, of those
    failing the screen)."""
    names = _names(msgtypes)
    pid = r900_preamble_id(names)
    bits = [i for i, m in enumerate(names) if m in ("r900", "r900bcd")]
    rmask = sum(1 << i for i in bits)
    is_r = got["preamble_id"] == pid
    other = got[~is_r]
    assert not (other["flags"] & capi.CAND_HAS_R900).any() and not other["r900_digits"].any()
    assert not (other["check_mask"] & rmask).any()
    rec = got[is_r]
    keys = list(zip(rec["block"].tolist(), rec["idx"].tolist(), rec["preamble_id"].tolist()))
    assert len(set(keys)) == len(keys)
    assert set(keys) == set(want), (len(set(keys) - set(want)), len(set(want) - set(keys)),
                                    sorted(set(keys) ^ set(want))[:8])
    assert (rec["flags"] & capi.CAND_HAS_R900).all()
    fails = 0
    for r, k in zip(rec, keys):
        d = want[k]
        assert r["r900_digits"].tobytes() == d, (k, list(r["r900_digits"]), list(d))
        ok = screen_expected("r900", b"", d)
        fails += not ok
        assert int(r["check_mask"]) & rmask == (rmask if ok else 0), (k, int(r["check_mask"]), ok)
    return len(keys), fails


def preamble_of(proto) -> str:
    """The preamble of a stock name or a capi.Protocol."""
    return PREAMBLES[proto] if isinstance(proto, str) else bytes(proto.preamble).split(b"\0")[0].decode()


def _is_r900(proto) -> bool:
    return proto in ("r900", "r900bcd") if isinstance(proto, str) else proto.check_kind == capi.CHECK_R900


def assert_check_masks_exact(got, msgtypes):
    """BOTH directions: bit i of check_mask is set iff the candidate is filed under parser i's preamble and
    passes that parser's integrity check (recomputed here from the returned bytes / digits).  msgtypes: stock names
    or capi.Protocol structs, in registration order."""
    if isinstance(msgtypes, str):
        msgtypes = [m.strip() for m in msgtypes.split(",") if m.strip()]
    pre_ids, order = [], []
    for m in msgtypes:          # distinct preambles in registration order (decode.go:121-124)
        if preamble_of(m) not in order:
            order.append(preamble_of(m))
        pre_ids.append(order.index(preamble_of(m)))
    cache = {}
    for r in got:
        data, dig, pid = r["bytes"].tobytes(), r["r900_digits"].tobytes(), int(r["preamble_id"])
        want = 0
        for i, m in enumerate(msgtypes):
            if pre_ids[i] != pid:
                continue
            key = (i, data if not _is_r900(m) else dig)
            if key not in cache:
                cache[key] = screen_expected(m, data, list(dig))
            if cache[key]:
                want |= 1 << i
        assert int(r["check_mask"]) == want, (int(r["block"]), int(r["idx"]), pid, int(r["check_mask"]), want)


# ---- custom protocol configurations (ertgpu_protocol) and the rules ertgpu_allocate applies to them ----
def make_protocol(preamble, cl, ps, pk, check=capi.CHECK_NONE, crc=(0xFFFF, 0x1021, 0x1D0F), crc_range=(0, 0),
                  name="custom"):
    """A capi.Protocol: `preamble` a '0'/'1' string, ChipLength cl, PreambleSymbols ps, PacketSymbols pk, a check kind
    and, for CHECK_CRC16 / CHECK_IDM, (init, polynomial, residue) over bytes [crc_range)."""
    p = capi.Protocol()
    p.name, p.preamble = name.encode(), preamble.encode()
    p.data_rate, p.chip_length, p.preamble_symbols, p.packet_symbols = 32768, cl, ps, pk
    p.center_freq, p.check_kind = 912600155, check
    p.crc_init, p.crc_poly, p.crc_residue = crc
    p.crc_from, p.crc_to = crc_range
    return p


def merged_geometry(protos):
    """Decoder.Cfg after RegisterProtocol of every protocol and Allocate (decode.go:100-141)."""
    cl = max(p.chip_length for p in protos)
    ps = max(p.preamble_symbols for p in protos)
    pk = max(p.packet_symbols for p in protos)
    sl = 2 * cl
    pl, pkl = ps * sl, pk * sl
    bs = 1 << max(0, (pl - 1).bit_length())
    return {"CL": cl, "SL": sl, "PS": ps, "PK": pk, "PL": pl, "PKL": pkl, "BS": bs, "BUF": pkl + bs}


def rule_violated(protos):
    """The first rule of ertgpu_allocate (include/ertgpu.h) the merged configuration breaks, in the order the library
    checks them ("BS": block size below 32, then R1, R2 / R4 per protocol in registration order, R3), or None."""
    g = merged_geometry(protos)
    BS, PL, SL, CL, PS, PK, BUF = g["BS"], g["PL"], g["SL"], g["CL"], g["PS"], g["PK"], g["BUF"]
    if BS < 32:
        return "BS"
    npacked = -(-(BS + PL) // 8)
    if 8 * npacked > BUF:
        return "R1"
    for p in protos:
        n = len(preamble_of(p))
        if n - 1 > PK or (n - 1) * (SL >> 3) + BS // 8 > npacked:
            return "R2"
        if p.check_kind == capi.CHECK_CRC16 and PK % 8 and p.crc_from <= PK >> 3 < p.crc_to:
            return "R4"
    if any(p.check_kind == capi.CHECK_R900 for p in protos) and BS - 1 + PL - SL + 164 * CL >= BUF - 4 * CL:
        return "R3"
    return None


def allocate_verdict(protos, max_blocks=1, max_cands=1):
    """(return code of ertgpu_allocate, its message) for the protocols registered in order; never decodes."""
    h = capi.Handle()
    try:
        for p in protos:
            h.register(p)
        rc = h._L.ertgpu_allocate(h._h, 0, max_blocks, max_cands)
        return rc, (h._L.ertgpu_last_error(h._h) or b"").decode()
    finally:
        h.close()
