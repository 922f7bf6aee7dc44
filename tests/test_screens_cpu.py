"""The integrity screens at their decision boundary, without a GPU: the corpus of tests/screen_ref.py against the
restatement and helpers.screen_expected, every wrong variant of a screen against the corpus, the oracle's candidates
and messages on the corpus streams, the host parsers' re-check, and the check kinds ertgpu_register_protocol takes."""
import numpy as np
import pytest

import oracle
import screen_ref as S
from helpers import make_protocol, screen_expected
from rtlamr_b200 import capi, host

@pytest.fixture(scope="module")
def corpus(built):
    return S.corpus()


def _views(corpus):
    for name, g in corpus.items():
        protos = g.protos(g.chip_lengths[0])
        for e in g.entries:
            for v in e.views:
                data, dig = S.view_data(e, v, protos)
                yield name, g, protos, e, v, data, dig


def test_corpus_is_deterministic(corpus):
    again = S.build_corpus()
    assert list(again) == list(corpus) == [name for name, _, _ in S.GROUPS]
    for name in corpus:
        assert again[name].entries == corpus[name].entries, name
    for name, g in corpus.items():
        cls = {e.cls for e in g.entries}
        assert any(v.passes for e in g.entries for v in e.views) and any(not v.passes for e in g.entries for v in e.views), name
        assert "valid" in cls or "cross_preamble" in cls, name


def test_designed_verdicts_equal_the_restatement_and_screen_expected(corpus):
    n = 0
    for name, g, protos, e, v, data, dig in _views(corpus):
        p = protos[v.proto]
        assert S.screen(p, data, dig) == v.passes, (name, e.cls)
        assert screen_expected(p, data, list(dig or ())) == v.passes, (name, e.cls)
        if g.msgtypes:
            stock = g.msgtypes.split(",")[v.proto]
            assert screen_expected(stock, data, list(dig or ())) == v.passes, (name, e.cls)
        n += 1
    assert n > 1900


def test_designed_packets_keep_their_preamble(corpus):
    """Search must find every packet: no entry touches a preamble bit, and r900 digits stay in 0..5."""
    for name, g in corpus.items():
        protos = g.protos(g.chip_lengths[0])
        for e in g.entries:
            for v in e.views:
                pre = bytes(protos[v.proto].preamble).split(b"\0")[0].decode()
                if e.bits is not None:
                    assert "".join(map(str, e.bits[v.offset:v.offset + len(pre)])) == pre, (name, e.cls)
                else:
                    assert len(e.digits) == 42 and 0 <= min(e.digits) and max(e.digits) <= 5, (name, e.cls)


@pytest.mark.parametrize("mutant", S.MUTANTS)
def test_every_wrong_screen_disagrees_with_the_corpus(corpus, mutant):
    for name, g, protos, e, v, data, dig in _views(corpus):
        if S.screen(protos[v.proto], data, dig, mutant) != v.passes:
            return
    pytest.fail(f"no corpus entry tells {mutant} from the screen")


def test_restated_crc_and_syndrome_match_known_values(built):
    """crc/crc_test.go's CCITT check value and a codeword of the encoder; the restatement's field is gf.go's."""
    assert S.crc(0xFFFF, 0x1021, b"123456789") == 0x29B1
    assert S.crc(0, 0x6F63, b"") == 0
    assert all(S.GF_EXP[S.GF_LOG[x]] == x for x in range(1, 32))
    assert S.syndrome([0] * 30 + [1]) == [1] * 5
    assert S.gf_poly(5)[0] == 1 and all(S.gf_poly(5))


def parser_names(g, protos):
    """The parser the oracle runs on each protocol's candidates: the stock one, the r900 parser for a custom r900
    screen (Oracle.from_protocols), none otherwise."""
    if g.msgtypes:
        return g.msgtypes.split(",")
    return ["r900" if p.check_kind == S.R900 else None for p in protos]


def expected_messages(g, protos):
    """{(entry, parser name)} the parsers must emit: designed passes the parser's own rules keep."""
    names = parser_names(g, protos)
    out = set()
    for i, e in enumerate(g.entries):
        for v in e.views:
            data, dig = S.view_data(e, v, protos)
            if v.passes and names[v.proto] and S.parser_emits(names[v.proto], data, dig):
                out.add((i, names[v.proto]))
    return out


def _same_data(c_bytes, data, pk):
    if pk % 8:     # the oracle's partial last byte holds stale bits of the previous candidate (decode.go:363-366)
        return c_bytes[:pk // 8] == data[:pk // 8] and (c_bytes[pk // 8] & ((1 << pk % 8) - 1)) == data[pk // 8]
    return c_bytes[:len(data)] == data


CPU_CASES = [(n, 16 if 16 in cls else cls[0]) for n, _, cls in S.GROUPS]


@pytest.mark.parametrize("name,cl", CPU_CASES)
def test_oracle_finds_designed_packets_and_emits_designed_passes(corpus, name, cl):
    g = corpus[name]
    st = S.make_stream(g, cl)
    search = oracle.SEARCH_GO if (2 * cl) % 8 == 0 else oracle.SEARCH_EXACT
    o = oracle.Oracle.from_protocols(st.protos, search)
    nblk = st.iq.size // o.cfg.block_size2
    cands, msgs = o.decode(st.iq, cand_cap=4096 + o.cfg.block_size * nblk, msg_cap=1 << 14)
    o.close()
    ids = S.preamble_ids(st.protos)
    r900_pid = next((ids[i] for i, p in enumerate(st.protos) if p.check_kind == S.R900), None)
    digits = S.oracle_digits(st.protos, st.iq, r900_pid) if r900_pid is not None else {}
    found = S.locate(st, g, cands)
    for (i, j), cs in found.items():
        e = g.entries[i]
        v = e.views[j]
        data, dig = S.view_data(e, v, st.protos)
        assert cs, (name, i, e.cls, "no candidate")
        for c in cs:
            if dig is None:
                assert _same_data(c.data, data, st.protos[v.proto].packet_symbols), (name, i, e.cls)
            else:
                assert digits[(c.block, c.idx)] == dig, (name, i, e.cls)
    names = parser_names(g, st.protos)
    got = set()
    for m in msgs:
        s = S.first_sample(st.geo, m.block, m.idx)
        i = S.entry_of_sample(st, s + st.geo["SL"])
        pname = oracle.PROTO_NAMES[m.proto]
        v = next(v for v in g.entries[i].views if names[v.proto] == pname)
        # the parser keeps the first of the adjacent sample phases that decode to the same bytes
        assert abs(s - st.starts[i] - v.offset * st.geo["SL"]) <= cl, (name, i, pname)
        got.add((i, pname))
    assert got == expected_messages(g, st.protos)


@pytest.mark.parametrize("name", [n for n, mt, _ in S.GROUPS if mt])
def test_host_parsers_emit_designed_passes(corpus, name):
    """host.Parsers re-checks every candidate itself: records built straight from the corpus, check_mask 0."""
    g = corpus[name]
    cl = g.chip_lengths[0]
    protos = g.protos(cl)
    ids = S.preamble_ids(protos)
    pk = max(p.packet_symbols for p in protos)
    recs = []
    for i, e in enumerate(g.entries):
        for v in e.views:
            r = np.zeros((), dtype=capi.CAND_DTYPE)
            r["block"], r["idx"], r["preamble_id"] = i, 0, ids[v.proto]
            if e.digits is None:
                b = S.cand_bytes(e.bits[v.offset:v.offset + pk] + (0,) * pk, pk)
                r["bytes"][:len(b)] = np.frombuffer(b, np.uint8)
            else:
                r["r900_digits"][:] = e.digits
                r["flags"] = capi.CAND_HAS_R900
            recs.append(r)
    recs = np.sort(np.array(recs, dtype=capi.CAND_DTYPE), order=["block", "preamble_id", "idx"])
    P = host.Parsers(g.msgtypes, cl)
    msgs = P.parse(recs, cap=1 << 14)
    P.close()
    names = {"scm": "SCM", "scm+": "SCM+", "idm": "IDM", "netidm": "NetIDM", "r900": "R900", "r900bcd": "R900BCD"}
    got = {(m.block, m.msgtype) for m in msgs}
    want = {(i, names[n]) for i, n in expected_messages(g, protos)}
    assert got == want, (sorted(got - want)[:4], sorted(want - got)[:4])


def test_registration_rejects_unknown_check_kinds(built):
    for kind in (-1, 4, 5, 1 << 20):
        h = capi.Handle()
        try:
            p = make_protocol("0101", 32, 4, 96, kind)
            with pytest.raises(capi.ErtGpuError) as ex:
                h.register(p)
            assert ex.value.code == capi.EINVAL and f"check_kind {kind}" in str(ex.value), str(ex.value)
        finally:
            h.close()
    h = capi.Handle()
    try:
        for p in S.custom_idm_protocols(72):       # every range field registers: the IDM screen ignores them
            h.register(p)
        h.register(make_protocol("0110", 32, 4, 96, S.NONE, crc_range=(-5, 200)))
    finally:
        h.close()
