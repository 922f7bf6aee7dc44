"""extract_words_kernel's integrity screens at their decision boundary: every stream of the tests/screen_ref.py corpus
decoded on the GPU.  Per stream: check_mask in both directions on every candidate, every designed packet's candidate
with its designed bytes or digits and its designed bit, candidates and r900 digits equal to the oracle's, the
DECODE_ONLY_VALID records and n_valid, and no host-parser message from a record whose bit for that parser is clear.
The custom CHECK_IDM group registers range fields (0,0), (4,92), (2,50) and (10,92): every one must screen [4,92)."""
from collections import namedtuple

import numpy as np
import pytest

import oracle
import screen_ref as S
from helpers import _feed, assert_check_masks_exact, cand_key_gpu, cand_key_oracle
from rtlamr_b200 import capi, host

gpu = pytest.mark.gpu
CASES = [(n, cl) for n, _, cls in S.GROUPS for cl in cls]
Rec = namedtuple("Rec", "block idx preamble_id row")
HOST_NAMES = {"SCM": "scm", "SCM+": "scm+", "IDM": "idm", "NetIDM": "netidm", "R900": "r900", "R900BCD": "r900bcd"}


@pytest.fixture(scope="module")
def corpus(built):
    return S.corpus()


def _handle(protos):
    h = capi.Handle()
    for p in protos:
        h.register(p)
    h.allocate(0, 0, 1 << 20)
    return h


def _sorted(recs):
    return np.sort(recs, order=["block", "preamble_id", "idx"], kind="stable")


@gpu
@pytest.mark.parametrize("name,cl", CASES)
def test_screens_on_the_corpus(corpus, name, cl):
    g = corpus[name]
    st = S.make_stream(g, cl)
    protos, geo = st.protos, st.geo
    h = _handle(protos)
    got = _sorted(h.decode(st.iq, cap=1 << 16))
    kernels = h.last_kernels()
    n_cand, n_valid = h.last_counts()
    h.close()
    assert n_cand == len(got)
    assert_check_masks_exact(got, protos)

    # every designed packet: its candidate, its bytes or digits, its designed bit
    recs = [Rec(int(r["block"]), int(r["idx"]), int(r["preamble_id"]), r) for r in got]
    for (i, j), cs in S.locate(st, g, recs).items():
        e, v = g.entries[i], g.entries[i].views[j]
        data, dig = S.view_data(e, v, protos)
        assert cs, (name, cl, i, e.cls, "no candidate")
        for c in cs:
            r = c.row
            if dig is None:
                assert r["bytes"][:len(data)].tobytes() == data, (name, cl, i, e.cls)
            else:
                assert tuple(int(d) for d in r["r900_digits"]) == dig, (name, cl, i, e.cls)
            assert bool(int(r["check_mask"]) >> v.proto & 1) == v.passes, (name, cl, i, e.cls, int(r["check_mask"]))

    # the oracle's candidates and r900 digits (the masks follow from the bytes through assert_check_masks_exact)
    search = oracle.SEARCH_GO if (2 * cl) % 8 == 0 else oracle.SEARCH_EXACT
    o = oracle.Oracle.from_protocols(protos, search)
    want = sorted(cand_key_oracle(x, (geo["PK"] + 7) >> 3, geo["PK"]) for x in _feed(o, st.iq))
    o.close()
    have = sorted(cand_key_gpu(r, (geo["PK"] + 7) >> 3, geo["PK"]) for r in got)
    assert have == want, (name, cl, len(have), len(want), sorted(set(have) ^ set(want))[:4])
    ids = S.preamble_ids(protos)
    r900_pid = next((ids[i] for i, p in enumerate(protos) if p.check_kind == S.R900), None)
    if r900_pid is not None:
        digits = S.oracle_digits(protos, st.iq, r900_pid)
        rec = got[got["preamble_id"] == r900_pid]
        assert len(rec) == len(digits)
        for r in rec:
            assert tuple(int(d) for d in r["r900_digits"]) == digits[(int(r["block"]), int(r["idx"]))]
        if name == "r900_custom":       # PacketLength not a multiple of 8 samples: the replay kernel
            assert "r900_replay_kernel" in kernels, kernels
        elif name == "r900,r900bcd":
            assert "r900_chain2_kernel" in kernels, kernels

    # DECODE_ONLY_VALID: exactly the records whose mask is not 0, byte for byte, and n_valid counts them
    valid = got[got["check_mask"] != 0]
    assert n_valid == len(valid) > 0
    h = _handle(protos)
    only = _sorted(h.decode(st.iq, flags=capi.DECODE_ONLY_VALID, cap=1 << 16))
    assert h.last_counts() == (n_cand, n_valid)
    h.close()
    assert only.tobytes() == valid.tobytes(), (name, cl, len(only), len(valid))

    # the shim's safety property: a parser message only ever comes from a record whose bit for that parser is set
    if g.msgtypes:
        names = g.msgtypes.split(",")
        P = host.Parsers(g.msgtypes, cl)
        msgs = P.parse(got, cap=1 << 14)
        P.close()
        assert msgs
        at = {(int(r["block"]), int(r["idx"]), int(r["preamble_id"])): int(r["check_mask"]) for r in got}
        for m in msgs:
            i = names.index(HOST_NAMES[m.msgtype])
            assert at[(m.block, m.idx, ids[i])] >> i & 1, (name, cl, m.msgtype, m.block, m.idx)
