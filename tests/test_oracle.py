"""CPU tests: pin the oracle against the reference's golden vectors and known answers.

Sources of truth (SURVEY.md section 8c): crc/crc_test.go:22-41 (TestIdentity) and the standard
CRC check values; the MagLUT and geometry known answers; and the CRC-self-verifying SCM
messages recovered from the reference fixture assets/sample.bin (captured at chip length 78).
"""
import json
import os

import numpy as np
import pytest

import oracle
from conftest import GOLDEN
from helpers import synth_stream
from rtlamr_b200 import synth


def test_crc_known_answers():
    assert oracle.crc_checksum(0, b"123456789", 0x6F63) == 0xBDF4
    assert oracle.crc_checksum(0xFFFF, b"123456789", 0x1021) == 0x29B1
    assert oracle.crc_checksum(0, b"123456789", 0x8005) == 0xFEE8
    assert list(oracle.crc_table(0x6F63)[1:4]) == [0x6F63, 0xDEC6, 0xB1A5]
    assert list(oracle.crc_table(0x1021)[1:4]) == [0x1021, 0x2042, 0x3063]


@pytest.mark.parametrize("init,poly", [(0, 0x8005), (0, 0x6F63), (0xFFFF, 0x1021)])
def test_crc_identity(init, poly):
    # crc/crc_test.go:22-41 TestIdentity: crc(data || BE16(crc(data))) == 0 (for init 0: plain;
    # the reference runs the same loop for CCITT with its init, checking against 0 too)
    rng = np.random.default_rng(poly)
    for _ in range(512):
        data = bytes(rng.integers(0, 256, 10, dtype=np.uint8))
        crc = oracle.crc_checksum(init, data, poly)
        assert oracle.crc_checksum(init, data + crc.to_bytes(2, "big"), poly) == 0
        # the product-side Python CRC used by the packet encoders agrees with the oracle
        assert synth.crc16(init, poly, data) == crc


def test_maglut_known_answers():
    lut = oracle.maglut()
    bits = lut.view(np.uint32)
    assert bits[0] == bits[255] == 0x3F800000
    assert bits[127] == bits[128] == 0x37810183
    assert np.array_equal(lut, lut[::-1])
    ref = ((np.float32(127.5) - np.arange(256, dtype=np.float32)) / np.float32(127.5)).astype(np.float32)
    assert np.array_equal(lut, (ref * ref).astype(np.float32))


GEOMETRY = [  # SURVEY.md section 8d
    ("scm", 72, dict(symbol_length=144, preamble_length=3024, packet_length=13824, block_size=4096,
                     block_size2=8192, buffer_length=17920, sample_rate=2359296)),
    ("scm,scm+,idm", 72, dict(preamble_symbols=32, packet_symbols=736, preamble_length=4608,
                              packet_length=105984, block_size=8192, block_size2=16384, buffer_length=114176)),
    ("r900", 72, dict(preamble_symbols=32, packet_symbols=116, preamble_length=4608, packet_length=16704,
                      block_size=8192, buffer_length=24896, center_freq=912380000)),
    ("scm", 78, dict(preamble_length=3276, packet_length=14976, block_size=4096, buffer_length=19072)),
]


@pytest.mark.parametrize("msgtypes,cl,want", GEOMETRY)
def test_geometry(msgtypes, cl, want):
    o = oracle.Oracle(msgtypes, cl)
    for k, v in want.items():
        assert getattr(o.cfg, k) == v, k


def test_sample_bin_cl72_decodes_to_nothing(sample_iq):
    # BASELINE config 1: `scm -symbollength=72` on assets/sample.bin -> plumbing only, zero messages
    o = oracle.Oracle("scm", 72, oracle.SEARCH_GO)
    n = sample_iq.size // o.cfg.block_size2
    assert n == 69
    cands, msgs = o.decode(sample_iq[: n * o.cfg.block_size2])
    assert len(cands) == 0 and len(msgs) == 0


def test_sample_bin_cl78_golden(sample_iq):
    with open(os.path.join(GOLDEN, "sample_cl78_scm.json")) as f:
        gold = json.load(f)
    o = oracle.Oracle("scm", 78, oracle.SEARCH_EXACT)
    n = sample_iq.size // o.cfg.block_size2
    cands, msgs = o.decode(sample_iq[: n * o.cfg.block_size2])
    assert len(cands) == gold["exact"]["n_candidates"] == 853
    got = [[m.block, m.idx, m.data.hex(), m.meter_id, m.meter_type, m.consumption] for m in msgs]
    assert got == gold["exact"]["messages"]
    assert len(got) == 14
    # every golden message is self-verifying: BCH over bytes[2:12] is zero
    for _, _, hx, *_ in got:
        assert oracle.crc_checksum(0, bytes.fromhex(hx)[2:12], 0x6F63) == 0
    # the literal Go search (byte pre-filter with SL>>3 = 19 for SL = 156) keeps one message
    o2 = oracle.Oracle("scm", 78, oracle.SEARCH_GO)
    cands2, msgs2 = o2.decode(sample_iq[: n * o2.cfg.block_size2])
    assert len(cands2) == gold["go_faithful"]["n_candidates"] == 6
    assert [[m.block, m.idx, m.data.hex()] for m in msgs2] == gold["go_faithful"]["messages"]


def test_numpy_restatement_agrees_with_c(sample_iq):
    """Independent restatement of decode.go:219-245 with numpy (sequential float32 cumsum)."""
    o = oracle.Oracle("scm", 78, oracle.SEARCH_EXACT)
    c = o.cfg
    bs, sl, cl = c.block_size, c.symbol_length, c.chip_length
    lut = oracle.maglut()
    signal = np.zeros(bs + sl, dtype=np.float32)
    for b in range(6):
        blk = sample_iq[b * c.block_size2:(b + 1) * c.block_size2]
        o.decode(blk)
        signal[:sl] = signal[bs:]
        signal[sl:] = lut[blk[0::2]] + lut[blk[1::2]]
        csum = np.concatenate([[np.float32(0)], np.cumsum(signal, dtype=np.float32)])
        f = (csum[cl:cl + bs] - csum[:bs]) - (csum[sl:sl + bs] - csum[cl:cl + bs])
        q = (1 - (f.view(np.uint32) >> 31)).astype(np.uint8)
        assert np.array_equal(o.signal(), signal)
        assert np.array_equal(o.csum(), csum.astype(np.float32))
        assert np.array_equal(o.quantized()[c.packet_length:], q)


def test_go_search_equals_exact_search_when_sl_multiple_of_8():
    for mt, cl in (("scm", 72), ("scm,scm+,idm", 32), ("r900", 40)):
        iq, _, _ = synth_stream(mt, cl, 1 << 20, spacing=1 << 18)
        a = oracle.Oracle(mt, cl, oracle.SEARCH_GO)
        b = oracle.Oracle(mt, cl, oracle.SEARCH_EXACT)
        n = iq.size // a.cfg.block_size2 * a.cfg.block_size2
        ca, ma = a.decode(iq[:n])
        cb, mb = b.decode(iq[:n])
        assert ca == cb and ma == mb and len(ca) > 0


@pytest.mark.parametrize("mt,cl", [("scm", 72), ("scm+", 72), ("idm", 72), ("netidm", 48), ("r900", 72),
                                   ("r900bcd", 32), ("scm,scm+,idm,r900", 72)])
def test_injected_packets_are_recovered(mt, cl):
    n = 1 << 21
    iq, pk, truth = synth_stream(mt, cl, n, spacing=1 << 19)
    o = oracle.Oracle(mt, cl, oracle.SEARCH_GO)
    nb = iq.size // o.cfg.block_size2
    cands, msgs = o.decode(iq[: nb * o.cfg.block_size2])
    got = {(oracle.PROTO_NAMES[m.proto], m.meter_id) for m in msgs}
    usable = [t for t in truth if t.start_sample + o.cfg.packet_length + o.cfg.block_size < nb * o.cfg.block_size]
    assert usable
    for t in usable:
        assert (t.msgtype, t.meter_id) in got, t
    # no false messages: everything decoded was injected
    want = {(t.msgtype, t.meter_id) for t in truth}
    assert got <= want


def test_gf32_syndrome_of_encoded_r900_is_zero():
    chips, sym = synth.encode_r900(0xDEADBEEF, 3, 5, 1, 777777, 2, 9, 1)
    assert len(chips) == 232
    msg = bytes(sym[:16]) + bytes(10) + bytes(sym[16:])
    assert oracle.gf32_syndrome(msg) == bytes(5)
    bad = bytearray(msg)
    bad[3] ^= 1
    assert oracle.gf32_syndrome(bytes(bad)) != bytes(5)


def test_two_constant_reciprocal_reproduces_the_lut_division_exactly():
    """r900_chain2_kernel computes x = fl((127.5 - v) / 127.5) as fma(n, rhi, fl(n * rlo)).
    Exhaustive proof over the 256 byte values with exact rational arithmetic (a true single-rounding fma)."""
    from fractions import Fraction

    def rn32(fr):
        x = np.float32(float(fr))
        best = None
        for d in (-1, 0, 1):
            c = np.uint32(int(x.view(np.uint32)) + d).view(np.float32)
            err = abs(Fraction(float(c)) - fr)
            if best is None or err < best[0] or (err == best[0] and (int(c.view(np.uint32)) & 1) == 0):
                best = (err, c)
        return best[1]

    rhi = np.uint32(1006665857).view(np.float32)
    rlo = np.uint32(2952724223).view(np.float32)
    lut = oracle.maglut()
    for v in range(256):
        m = np.uint32(0x47000000 | (v << 8)).view(np.float32)        # the byte-permuted float 32768 + v
        assert float(m) == 32768.0 + v
        n = np.float32(32895.5) - m
        assert float(n) == 127.5 - v                                   # exact
        t = rn32(Fraction(float(n)) * Fraction(float(rlo)))
        x = rn32(Fraction(float(n)) * Fraction(float(rhi)) + Fraction(float(t)))
        assert x == np.float32(np.float32(127.5 - v) / np.float32(127.5)), v
        assert np.float32(x * x) == lut[v], v
