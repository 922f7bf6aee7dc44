"""Synthetic ERT traffic: packet encoders and the packet table of the synthetic IQ stream.

Bench/test tooling (the reference has no transmitter side).  Field layouts are the inverse of
the reference parsers: scm/scm.go:103-119, scmplus/scmplus.go:94-109, idm/idm.go:101-156,
netidm/netidm.go:112-160, r900/r900.go:187-242; CRC per crc/crc.go:34-55; RS(31,26)-style
parity per r900/gf/gf.go:152-172 (syndromes at alpha^29..alpha^33 of GF(32), poly 37).

The IQ bytes themselves come from include/ertgpu_synth.h (one definition shared by the CUDA
generator `ertgpu_synth_fill` and the gcc-built host generator used on CPU-only machines).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass, field

import numpy as np

from .capi import SYNTH_DTYPE

_HERE = os.path.dirname(os.path.abspath(__file__))
_HOST_LIB = os.path.join(_HERE, "libertsynth_host.so")

PREAMBLE = {
    "scm": "111110010101001100000",
    "scm+": "0001011010100011",
    "idm": "01010101010101010001011010100011",
    "netidm": "01010101010101010001011010100011",
    "r900": "00000000000000001110010101100100",
}


# ---------------------------------------------------------------- CRC / GF(32)
def crc16(init: int, poly: int, data: bytes) -> int:
    crc = init
    for v in data:
        crc ^= v << 8
        for _ in range(8):
            crc = ((crc << 1) ^ poly) & 0xFFFF if crc & 0x8000 else (crc << 1) & 0xFFFF
    return crc


def _gf32():
    exp, log = [0] * 62, [0] * 32
    x = 1
    for i in range(31):
        exp[i] = exp[i + 31] = x
        log[x] = i
        x <<= 1
        if x & 32:
            x ^= 37
    return exp, log


_EXP, _LOG = _gf32()


def _gmul(a: int, b: int) -> int:
    return 0 if a == 0 or b == 0 else _EXP[_LOG[a] + _LOG[b]]


def _rs_generator():
    g = [1]
    for j in range(5):
        root = _EXP[(29 + j) % 31]
        ng = [0] * (len(g) + 1)
        for i, c in enumerate(g):  # g * (x + root), highest degree first
            ng[i] ^= c
            ng[i + 1] ^= _gmul(c, root)
        g = ng
    return g  # degree 5, monic


_RS_G = _rs_generator()


def rs_parity(data16: list[int]) -> list[int]:
    """5 parity symbols so that [data(16), 0*10, parity(5)] has zero syndromes at alpha^29..33."""
    msg = list(data16) + [0] * 15  # degrees 30..0, data in 30..15
    rem = list(msg)
    for i in range(len(msg) - 5):
        c = rem[i]
        if c:
            for j, g in enumerate(_RS_G):
                rem[i + j] ^= _gmul(c, g)
    return rem[-5:]


# ---------------------------------------------------------------- bit helpers
def _bits_from_bytes(b: bytes) -> list[int]:
    return [(v >> (7 - k)) & 1 for v in b for k in range(8)]


def _bytes_from_bits(bits: list[int]) -> bytes:
    assert len(bits) % 8 == 0
    out = bytearray()
    for i in range(0, len(bits), 8):
        v = 0
        for k in range(8):
            v = (v << 1) | bits[i + k]
        out.append(v)
    return bytes(out)


def _field(v: int, n: int) -> list[int]:
    return [(v >> (n - 1 - k)) & 1 for k in range(n)]


def manchester_chips(bits: list[int]) -> list[int]:
    """bit 1 -> chips high,low ; bit 0 -> low,high (sign of first-minus-second chip, decode.go:242-243)."""
    out = []
    for b in bits:
        out += [1, 0] if b else [0, 1]
    return out


# ---------------------------------------------------------------- encoders
def encode_scm(ert_id: int, ert_type: int, tamper_phy: int, tamper_enc: int, consumption: int) -> bytes:
    bits = [int(c) for c in PREAMBLE["scm"]]
    bits += _field((ert_id >> 24) & 3, 2) + [0] + _field(tamper_phy, 2) + _field(ert_type, 4)
    bits += _field(tamper_enc, 2) + _field(consumption, 24) + _field(ert_id & 0xFFFFFF, 24)
    body = _bytes_from_bits(bits)  # 10 bytes
    crc = crc16(0, 0x6F63, body[2:10])
    return body + crc.to_bytes(2, "big")


def encode_scmplus(endpoint_type: int, endpoint_id: int, consumption: int, tamper: int) -> bytes:
    body = bytes([0x16, 0xA3, 0x1E, endpoint_type & 0xFF]) + endpoint_id.to_bytes(4, "big") \
        + consumption.to_bytes(4, "big") + tamper.to_bytes(2, "big")
    crc = crc16(0xFFFF, 0x1021, body[2:14]) ^ 0xFFFF
    return body + crc.to_bytes(2, "big")


def _encode_idm_like(packet_type: int, ert_type: int, serial: int, filler: bytes) -> bytes:
    assert len(filler) == 75  # bytes 13..87
    b = bytearray(92)
    b[0:4] = bytes([0x55, 0x55, 0x16, 0xA3])
    b[4], b[5], b[6], b[7] = packet_type, 0x5C, 0xC6, 0x01
    b[8] = ert_type & 0x0F
    b[9:13] = serial.to_bytes(4, "big")
    b[13:88] = filler
    b[88:90] = (crc16(0xFFFF, 0x1021, bytes(b[9:13])) ^ 0xFFFF).to_bytes(2, "big")
    b[90:92] = (crc16(0xFFFF, 0x1021, bytes(b[4:90])) ^ 0xFFFF).to_bytes(2, "big")
    return bytes(b)


def encode_idm(ert_type: int, serial: int, filler: bytes) -> bytes:
    return _encode_idm_like(0x1C, ert_type, serial, filler)


def encode_netidm(ert_type: int, serial: int, filler: bytes) -> bytes:
    return _encode_idm_like(0x1C, ert_type, serial, filler)


_R900_CHIPS = {3: [1, 1, 0, 0], 0: [0, 0, 1, 1], 4: [1, 0, 1, 0], 1: [0, 1, 0, 1], 5: [1, 0, 0, 1], 2: [0, 1, 1, 0]}


def encode_r900(meter_id: int, unkn1: int, nouse: int, backflow: int, consumption: int, unkn3: int,
                leak: int, leaknow: int):
    """Returns (chips, symbols21): 32 Manchester preamble bits (64 chips) followed by 42 base-6
    digits of 4 chips each = 232 chips = 116 symbols (PacketSymbols, r900.go:62).  The parser
    reads the payload at Idx + PL - SL in ITS buffer (r900.go:187), whose index i is sample i,
    while Decoder.Quantized[Idx] is the filter window starting SL samples earlier
    (decode.go:169,239-244): so the payload starts right after the 32-symbol preamble."""
    bits = _field(meter_id, 32) + _field(unkn1, 8) + _field(nouse, 6) + _field(backflow, 2) \
        + _field(consumption, 24) + _field(unkn3, 2) + _field(leak, 4) + _field(leaknow, 2)
    data = [int("".join(map(str, bits[i:i + 5])), 2) for i in range(0, 80, 5)]
    symbols = data + rs_parity(data)
    digits = []
    for s in symbols:
        digits += [s // 6, s % 6]
    return r900_chips(digits), symbols


def r900_chips(digits) -> list[int]:
    """The r900 preamble's Manchester chips followed by 4 chips per base-6 digit: any 42 digits, valid or not."""
    chips = manchester_chips([int(c) for c in PREAMBLE["r900"]])
    for d in digits:
        chips += _R900_CHIPS[int(d)]
    return chips


# ---------------------------------------------------------------- packet table
@dataclass
class Truth:
    msgtype: str
    start_sample: int
    data: bytes           # packet bytes (r900: the 21 symbols)
    meter_id: int
    fields: dict = field(default_factory=dict)


def _amp(rng, amplitude: int):
    ph = rng.integers(0, 16)
    return int(round(amplitude * np.cos(2 * np.pi * ph / 16))), int(round(amplitude * np.sin(2 * np.pi * ph / 16)))


def make_packets(msgtypes, chip_length: int, nsamples: int, seed: int, spacing: int = 1 << 20,
                 first_sample: int = 0, amplitude=(24, 60)):
    """One packet per `spacing` samples at a pseudo-random offset (never overlapping the next
    window's packet), message types cycling through `msgtypes`.  Returns (table, truth)."""
    if isinstance(msgtypes, str):
        msgtypes = [m.strip() for m in msgtypes.split(",") if m.strip()]
    rng = np.random.default_rng(seed)
    rows, truth = [], []
    nwin = max(1, (nsamples + spacing - 1) // spacing)
    prev_end = first_sample
    for w in range(nwin):
        mt = msgtypes[w % len(msgtypes)]
        if mt == "scm":
            mid = int(rng.integers(1, 1 << 26))
            data = encode_scm(mid, int(rng.integers(0, 16)), int(rng.integers(0, 4)), int(rng.integers(0, 4)),
                              int(rng.integers(0, 1 << 24)))
            chips = manchester_chips(_bits_from_bytes(data))
        elif mt == "scm+":
            mid = int(rng.integers(1, 1 << 32))
            data = encode_scmplus(int(rng.integers(0, 256)), mid, int(rng.integers(0, 1 << 32)), int(rng.integers(0, 1 << 16)))
            chips = manchester_chips(_bits_from_bytes(data))
        elif mt in ("idm", "netidm"):
            mid = int(rng.integers(1, 1 << 32))
            filler = bytes(rng.integers(0, 256, 75, dtype=np.uint8))
            data = (encode_idm if mt == "idm" else encode_netidm)(int(rng.integers(0, 16)), mid, filler)
            chips = manchester_chips(_bits_from_bytes(data))
        elif mt in ("r900", "r900bcd"):
            mid = int(rng.integers(1, 1 << 32))
            chips, symbols = encode_r900(mid, int(rng.integers(0, 256)), int(rng.integers(0, 64)), int(rng.integers(0, 4)),
                                         int(rng.integers(0, 1 << 24)), int(rng.integers(0, 4)), int(rng.integers(0, 16)),
                                         int(rng.integers(0, 4)))
            data = bytes(symbols)
        else:
            raise ValueError(mt)
        length = len(chips) * chip_length
        lo = max(first_sample + w * spacing, prev_end + 4 * chip_length)
        hi = first_sample + (w + 1) * spacing
        start = int(rng.integers(lo, max(lo + 1, hi)))
        prev_end = start + length
        row = np.zeros((), dtype=SYNTH_DTYPE)
        row["start_sample"] = start
        row["n_chips"] = len(chips)
        row["chip_length"] = chip_length
        a = int(rng.integers(amplitude[0], amplitude[1] + 1))
        row["amp_i"], row["amp_q"] = _amp(rng, a)
        packed = np.packbits(np.array(chips, dtype=np.uint8))
        row["chips"][:len(packed)] = packed
        rows.append(row)
        truth.append(Truth(mt, start, data, mid))
    return np.array(rows, dtype=SYNTH_DTYPE), truth


# ---------------------------------------------------------------- host generator
_host = None


def _host_lib():
    global _host
    if _host is None:
        src = os.path.join(_HERE, "csrc", "synth_host.c")
        if not os.path.exists(_HOST_LIB) or os.path.getmtime(_HOST_LIB) < os.path.getmtime(src):
            subprocess.run(["gcc", "-O2", "-fPIC", "-pthread", "-shared", "-o", _HOST_LIB, src], check=True)
        L = C.CDLL(_HOST_LIB)
        L.ertsynth_host_fill.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_uint64, C.c_void_p, C.c_int64]
        L.ertsynth_host_fill.restype = None
        L.ertsynth_host_fill_mt.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_uint64, C.c_void_p, C.c_int64, C.c_int32]
        L.ertsynth_host_fill_mt.restype = None
        _host = L
    return _host


def host_fill(first_sample: int, nsamples: int, seed: int, packets: np.ndarray | None,
              nthreads: int = 1, out: np.ndarray | None = None) -> np.ndarray:
    """The synthetic stream on the CPU (bit-identical to ertgpu_synth_fill); `nthreads` > 1 fills
    disjoint ranges in parallel (same bytes: the generator is counter based)."""
    if out is None:
        out = np.empty(2 * nsamples, dtype=np.uint8)
    assert out.dtype == np.uint8 and out.size >= 2 * nsamples and out.flags.c_contiguous
    if packets is None or len(packets) == 0:
        ptr, n = None, 0
    else:
        packets = np.ascontiguousarray(packets)
        ptr, n = packets.ctypes.data, len(packets)
    if nthreads > 1:
        _host_lib().ertsynth_host_fill_mt(out.ctypes.data, first_sample, nsamples, seed, ptr, n, nthreads)
    else:
        _host_lib().ertsynth_host_fill(out.ctypes.data, first_sample, nsamples, seed, ptr, n)
    return out[:2 * nsamples]
