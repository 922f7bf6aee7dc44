"""NumPy restatement of the per-packet signal record (include/ertgpu_signal.h), and a ctypes binding of the header's
own summary (tests/cpu_harness/signal_ref.c), compiled with gcc into a temporary directory on first use.

record() takes the decoder's byte stream from the stream's first sample, one candidate and the registered protocols,
and returns the record packet_signal_kernel must produce for it, field for field."""
from __future__ import annotations

import ctypes as C
import hashlib
import math
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(ROOT, "tests", "cpu_harness", "signal_ref.c")
_HDRS = [os.path.join(ROOT, "include", n) for n in ("ertgpu_signal.h", "ertgpu.h")]
CHECK_R900 = 3
FIELDS = ("n_on", "e_on", "n_off", "e_off", "r_re", "r_im", "n_pairs", "protocol", "symbols")
FULL_SCALE = 65025.0
SNR_MIN = -99.99


def _get(p, name):
    v = p[name] if isinstance(p, dict) else getattr(p, name)
    return v.decode() if isinstance(v, bytes) else v


def geometry(protos) -> dict:
    """The merged geometry of decode.go:100-141 and each protocol's preamble id and span."""
    cl = max(_get(p, "chip_length") for p in protos)
    ps = max(_get(p, "preamble_symbols") for p in protos)
    pk = max(_get(p, "packet_symbols") for p in protos)
    sl = 2 * cl
    bs = 1
    while bs < ps * sl:
        bs <<= 1
    pres, ids, spans = [], [], []
    for p in protos:
        pre = _get(p, "preamble")
        if pre not in pres:
            pres.append(pre)
        ids.append(pres.index(pre))
        spans.append(_get(p, "preamble_symbols") if _get(p, "check_kind") == CHECK_R900 else _get(p, "packet_symbols"))
    return {"CL": cl, "SL": sl, "BS": bs, "PK": pk, "BUF": pk * sl + bs, "preamble_id": ids, "span": spans}


def protocol_of(geo, preamble_id: int, check_mask: int) -> int:
    first = -1
    for i, pid in enumerate(geo["preamble_id"]):
        if pid != preamble_id:
            continue
        if (check_mask >> i) & 1:
            return i
        if first < 0:
            first = i
    return first


def first_sample(geo, block: int, idx: int) -> int:
    """Decoder sample at which symbol 0 of the candidate (block, idx) starts (decode.go:163-197, 229-245, 369)."""
    return (block + 1) * geo["BS"] - geo["BUF"] + idx - geo["SL"]


def bits(data, n: int, pk: int) -> np.ndarray:
    """Bits 0 .. n-1 of a candidate's bytes (MSB first; a trailing partial byte holds its pk%8 bits in the low bits)."""
    b = np.frombuffer(bytes(data), dtype=np.uint8)
    k = np.arange(n)
    shift = 7 - (k & 7)
    if pk & 7:
        last = (k >> 3) == (pk >> 3)
        shift = np.where(last, (pk & 7) - 1 - (k & 7), shift)
    return (b[k >> 3] >> shift) & 1


def record(u8, block: int, idx: int, preamble_id: int, check_mask: int, data, protos) -> dict:
    """The record of one candidate of the byte stream u8 (uint8 I,Q from the stream's first sample)."""
    geo = geometry(protos)
    s = 2 * np.asarray(u8, dtype=np.int64).reshape(-1, 2) - 255
    cl, sl = geo["CL"], geo["SL"]
    g = cl >> 2
    m = cl - 2 * g
    proto = protocol_of(geo, preamble_id, check_mask)
    span = geo["span"][proto]
    k = np.arange(1, span)
    bit = bits(data, span, geo["PK"])[1:]
    c0 = first_sample(geo, block, idx) + k * sl
    hi0 = np.where(bit == 1, c0, c0 + cl)
    lo0 = np.where(bit == 1, c0 + cl, c0)
    off = g + np.arange(m)
    hi, lo = hi0[:, None] + off, lo0[:, None] + off
    assert hi.max(initial=-1) < len(s) and lo.max(initial=-1) < len(s), "the span runs past the bytes given"

    def energy(pos):
        v = pos[pos >= 0]
        return int(v.size), int((s[v] ** 2).sum())

    n_on, e_on = energy(hi)
    n_off, e_off = energy(lo)
    cur, prev = hi[:, 1:].ravel(), hi[:, :-1].ravel()
    ok = prev >= 0
    a, b = s[cur[ok]], s[prev[ok]]
    r_re = int((a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]).sum())
    r_im = int((a[:, 1] * b[:, 0] - a[:, 0] * b[:, 1]).sum())
    return {"n_on": n_on, "e_on": e_on, "n_off": n_off, "e_off": e_off, "r_re": r_re, "r_im": r_im,
            "n_pairs": int(ok.sum()), "protocol": proto, "symbols": span - 1}


def summary(rec, channel_hz: int, rate_out: int):
    """Level, Noise, SNR (dB), Offset and Freq (Hz) of a record, or None when it has none."""
    if rec["n_on"] <= 0 or rec["n_off"] <= 0:
        return None
    p_on, p_off = rec["e_on"] / rec["n_on"], rec["e_off"] / rec["n_off"]
    x = (p_on - p_off) / p_off
    off = math.atan2(rec["r_im"], rec["r_re"]) * rate_out / (2 * math.pi)
    return {"level": 10 * math.log10(p_on / FULL_SCALE), "noise": 10 * math.log10(p_off / FULL_SCALE),
            "snr": max(10 * math.log10(x), SNR_MIN) if x > 0 else SNR_MIN, "offset": off,
            "freq": int(round(channel_hz + off))}


_lib = None


class _Summary(C.Structure):
    _fields_ = [("level_db", C.c_double), ("noise_db", C.c_double), ("snr_db", C.c_double), ("offset_hz", C.c_double),
                ("freq_hz", C.c_int64)]


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for p in [_SRC] + _HDRS:
            h.update(open(p, "rb").read())
        so = os.path.join(tempfile.gettempdir(), f"ertgpu_signal_ref_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-I", os.path.join(ROOT, "include"),
                            "-o", tmp, _SRC, "-lm"], check=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.sigref_summary.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.POINTER(_Summary)]
        L.sigref_protocol.argtypes = [C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_uint32]
        _lib = L
    return _lib


def header_summary(rec, channel_hz: int, rate_out: int):
    """ertsig_summary of include/ertgpu_signal.h on a record (dict or SIGNAL_DTYPE row)."""
    arr = (C.c_int64 * 8)(*[int(rec[f]) for f in FIELDS[:7]], (int(rec["protocol"]) & 0xFFFFFFFF) | (int(rec["symbols"]) << 32))
    out = _Summary()
    if not lib().sigref_summary(C.addressof(arr), channel_hz, rate_out, C.byref(out)):
        return None
    return {"level": out.level_db, "noise": out.noise_db, "snr": out.snr_db, "offset": out.offset_hz, "freq": out.freq_hz}


def header_protocol(geo, preamble_id: int, check_mask: int) -> int:
    """ertsig_protocol of include/ertgpu_signal.h."""
    n = len(geo["preamble_id"])
    ids = (C.c_int32 * n)(*geo["preamble_id"])
    return int(lib().sigref_protocol(n, ids, preamble_id, check_mask))
