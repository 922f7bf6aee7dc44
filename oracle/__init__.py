"""CPU oracle for the protocol.Decoder hot path -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this package; the product (rtlamr_b200/) never does.

`Oracle` wraps oracle/libert_oracle.so (ert_oracle.c, a plain-C restatement of
protocol/decode.go, crc/crc.go, r900/r900.go and the parsers' validity checks).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libert_oracle.so")

SCM, SCMPLUS, IDM, NETIDM, R900, R900BCD = range(6)
PROTO_NAMES = ["scm", "scm+", "idm", "netidm", "r900", "r900bcd"]
SEARCH_GO, SEARCH_EXACT = 0, 1
MAX_PKT = 96
PARSER_NONE = -1
CHECK_R900 = 3    # ERTGPU_CHECK_R900 of include/ertgpu.h
PANIC = -2        # ert_oracle_decode: the reference indexes a slice past its length here


def build(force: bool = False) -> str:
    """Compile libert_oracle.so with the committed Makefile (gcc only)."""
    srcs = [os.path.join(_HERE, f) for f in ("ert_oracle.c", "ert_oracle_bench.c", "ert_oracle.h", "Makefile")]
    if (force or not os.path.exists(_LIB_PATH)
            or os.path.getmtime(_LIB_PATH) < max(os.path.getmtime(f) for f in srcs)):
        subprocess.run(["make", "-C", _HERE, "-B", "libert_oracle.so"], check=True,
                       stdout=subprocess.DEVNULL)
    return _LIB_PATH


class Cfg(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "data_rate", "block_size", "block_size2", "chip_length", "symbol_length", "sample_rate",
        "preamble_symbols", "packet_symbols", "preamble_length", "packet_length",
        "buffer_length")] + [("center_freq", C.c_uint32)]


class Proto(C.Structure):
    """ert_oracle_proto: one parser's PacketConfig and the parser run on its candidates."""
    _fields_ = [("preamble", C.c_char * 33), ("data_rate", C.c_int32), ("chip_length", C.c_int32),
                ("preamble_symbols", C.c_int32), ("packet_symbols", C.c_int32), ("center_freq", C.c_uint32),
                ("parser", C.c_int32)]


class ReferencePanic(RuntimeError):
    """The reference decoder would index a slice past its length on this input (it panics there)."""


class Cand(C.Structure):
    _fields_ = [("block", C.c_int64), ("idx", C.c_int32), ("preamble_id", C.c_int32),
                ("nbytes", C.c_int32), ("bytes", C.c_uint8 * MAX_PKT)]


class Msg(C.Structure):
    _fields_ = [("block", C.c_int64), ("idx", C.c_int32), ("proto", C.c_int32),
                ("meter_id", C.c_uint32), ("meter_type", C.c_uint32),
                ("consumption", C.c_uint32), ("nchecksum", C.c_int32),
                ("checksum", C.c_uint8 * 8), ("nbytes", C.c_int32),
                ("bytes", C.c_uint8 * MAX_PKT)]


@dataclass(frozen=True)
class Candidate:
    block: int
    idx: int
    preamble_id: int
    data: bytes


@dataclass(frozen=True)
class Message:
    block: int
    idx: int
    proto: int
    meter_id: int
    meter_type: int
    consumption: int
    checksum: bytes
    data: bytes


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        L.ert_oracle_new.restype = C.c_void_p
        L.ert_oracle_new.argtypes = [C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_int32]
        L.ert_oracle_new_protocols.restype = C.c_void_p
        L.ert_oracle_new_protocols.argtypes = [C.POINTER(Proto), C.c_int32, C.c_int32]
        L.ert_oracle_free.argtypes = [C.c_void_p]
        L.ert_oracle_config.restype = C.POINTER(Cfg)
        L.ert_oracle_config.argtypes = [C.c_void_p]
        L.ert_oracle_npreambles.restype = C.c_int32
        L.ert_oracle_npreambles.argtypes = [C.c_void_p]
        L.ert_oracle_decode_stream.restype = C.c_int32
        L.ert_oracle_decode_stream.argtypes = [
            C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(Cand), C.c_int32, C.POINTER(C.c_int32),
            C.POINTER(Msg), C.c_int32, C.POINTER(C.c_int32)]
        L.ert_oracle_dsp_only.argtypes = [C.c_void_p, C.c_void_p]
        for name, ty in (("signal", C.c_float), ("csum", C.c_float), ("quantized", C.c_uint8),
                         ("packed", C.c_uint8), ("r900_quantized", C.c_uint8)):
            f = getattr(L, "ert_oracle_" + name)
            f.restype = C.POINTER(ty)
            f.argtypes = [C.c_void_p, C.POINTER(C.c_int32)]
        L.ert_oracle_maglut.restype = C.POINTER(C.c_float)
        L.ert_crc_table.argtypes = [C.c_uint16, C.POINTER(C.c_uint16)]
        L.ert_crc_checksum.restype = C.c_uint16
        L.ert_crc_checksum.argtypes = [C.c_uint16, C.c_char_p, C.c_size_t, C.POINTER(C.c_uint16)]
        L.ert_gf32_syndrome.argtypes = [C.c_char_p, C.c_int32, C.c_int32, C.c_int32, C.c_char_p]
        L.ert_oracle_bench_threads.restype = C.c_double
        L.ert_oracle_bench_threads.argtypes = [C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                               C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                               C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.ert_oracle_host_cpus.restype = C.c_int32
        _lib = L
    return _lib


def proto_ids(msgtypes) -> list[int]:
    if isinstance(msgtypes, str):
        msgtypes = [m.strip() for m in msgtypes.split(",") if m.strip()]
    return [m if isinstance(m, int) else PROTO_NAMES.index(m) for m in msgtypes]


def crc_table(poly: int) -> np.ndarray:
    t = (C.c_uint16 * 256)()
    lib().ert_crc_table(poly, t)
    return np.frombuffer(t, dtype=np.uint16).copy()


def crc_checksum(init: int, data: bytes, poly: int) -> int:
    t = (C.c_uint16 * 256)()
    lib().ert_crc_table(poly, t)
    return int(lib().ert_crc_checksum(init, bytes(data), len(data), t))


def gf32_syndrome(message: bytes, nparity: int = 5, offset: int = 29) -> bytes:
    out = C.create_string_buffer(nparity)
    lib().ert_gf32_syndrome(bytes(message), len(message), nparity, offset, out)
    return out.raw


def maglut() -> np.ndarray:
    p = lib().ert_oracle_maglut()
    return np.ctypeslib.as_array(p, shape=(256,)).copy()


def host_cpus() -> int:
    """CPUs this process may run on."""
    return int(lib().ert_oracle_host_cpus())


def bench_threads(msgtypes, chip_length: int, iq, nthreads: int, repeats: int = 1, search: int = SEARCH_GO,
                  pin: bool = True):
    """Timed CPU baseline (ert_oracle_bench.c): `nthreads` independent decoders over contiguous
    block-aligned shards of `iq` (numpy uint8 or (address, nbytes)), everything inside C (no GIL,
    no allocation in the timed region).  Returns (seconds, n_candidates, n_messages, nblocks)."""
    ids = proto_ids(msgtypes)
    arr = (C.c_int32 * len(ids))(*ids)
    probe = Oracle(msgtypes, chip_length, search)
    bs2 = probe.cfg.block_size2
    probe.close()
    if isinstance(iq, tuple):
        addr, nbytes = iq
    else:
        iq = np.ascontiguousarray(iq, dtype=np.uint8)
        addr, nbytes = iq.ctypes.data, iq.size
    nblocks = nbytes // bs2
    nc, nm = C.c_int64(0), C.c_int64(0)
    dt = lib().ert_oracle_bench_threads(arr, len(ids), chip_length, search, addr, nblocks, nthreads, repeats,
                                        1 if pin else 0, C.byref(nc), C.byref(nm))
    if dt < 0:
        raise RuntimeError("ert_oracle_bench_threads failed")
    return dt, nc.value, nm.value, nblocks


class Oracle:
    """One protocol.Decoder with its registered parsers (decode.go:65-160)."""

    def __init__(self, msgtypes="scm", chip_length: int = 72, search: int = SEARCH_GO, _protocols=None):
        self._L = lib()
        if _protocols is None:
            ids = proto_ids(msgtypes)
            arr = (C.c_int32 * len(ids))(*ids)
            self._h = self._L.ert_oracle_new(arr, len(ids), chip_length, search)
        else:
            ids = [p.parser for p in _protocols]
            arr = (Proto * len(ids))(*_protocols)
            self._h = self._L.ert_oracle_new_protocols(arr, len(ids), search)
        if not self._h:
            raise ValueError("ert_oracle_new failed")
        self.protos = ids
        self.cfg = self._L.ert_oracle_config(self._h).contents
        self.npreambles = self._L.ert_oracle_npreambles(self._h)

    @classmethod
    def from_protocols(cls, protocols, search: int = SEARCH_GO, parsers=None):
        """A decoder with the libertgpu protocol structs `protocols` (rtlamr_b200.capi.Protocol) registered in order.
        parsers[i] is the parser run on protocol i's candidates (an ERT_* id or PARSER_NONE); by default the stock
        parser of the protocol's name, else the r900 DSP parser for an r900 check, else none."""
        out = []
        for i, p in enumerate(protocols):
            if parsers is not None:
                parser = parsers[i]
            else:
                name = bytes(p.name).split(b"\0")[0].decode()
                parser = PROTO_NAMES.index(name) if name in PROTO_NAMES else R900 if p.check_kind == CHECK_R900 else PARSER_NONE
            out.append(Proto(bytes(p.preamble).split(b"\0")[0], p.data_rate, p.chip_length, p.preamble_symbols,
                             p.packet_symbols, p.center_freq, parser))
        return cls(search=search, _protocols=out)

    def close(self):
        if self._h:
            self._L.ert_oracle_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def decode(self, iq, cand_cap: int = 1 << 16, msg_cap: int = 1 << 16):
        """Feed whole blocks (len(iq) multiple of BlockSize2). Returns (candidates, messages)."""
        iq = np.ascontiguousarray(iq, dtype=np.uint8)
        bs2 = self.cfg.block_size2
        if iq.size % bs2:
            raise ValueError(f"input must be a multiple of BlockSize2={bs2} bytes")
        nblocks = iq.size // bs2
        cands = (Cand * cand_cap)()
        msgs = (Msg * msg_cap)()
        nc, nm = C.c_int32(0), C.c_int32(0)
        rc = self._L.ert_oracle_decode_stream(self._h, iq.ctypes.data, nblocks, cands, cand_cap,
                                              C.byref(nc), msgs, msg_cap, C.byref(nm))
        if rc == PANIC:
            raise ReferencePanic("the reference indexes a slice past its length on this input")
        if rc != 0:
            raise OverflowError(f"oracle caps too small: {nc.value} candidates, {nm.value} messages")
        co = [Candidate(c.block, c.idx, c.preamble_id, bytes(c.bytes[:c.nbytes]))
              for c in cands[:nc.value]]
        mo = [Message(m.block, m.idx, m.proto, m.meter_id, m.meter_type, m.consumption,
                      bytes(m.checksum[:m.nchecksum]), bytes(m.bytes[:m.nbytes]))
              for m in msgs[:nm.value]]
        return co, mo

    def dsp_only(self, iq):
        """Timed-baseline helper: shift + magnitude + Filter for each whole block."""
        iq = np.ascontiguousarray(iq, dtype=np.uint8)
        bs2 = self.cfg.block_size2
        base = iq.ctypes.data
        for b in range(iq.size // bs2):
            self._L.ert_oracle_dsp_only(self._h, base + b * bs2)

    def _tap(self, name, dtype):
        n = C.c_int32(0)
        p = getattr(self._L, "ert_oracle_" + name)(self._h, C.byref(n))
        if not p:
            return None
        return np.ctypeslib.as_array(p, shape=(n.value,)).astype(dtype, copy=True)

    def signal(self):
        return self._tap("signal", np.float32)

    def csum(self):
        return self._tap("csum", np.float32)

    def quantized(self):
        return self._tap("quantized", np.uint8)

    def packed(self):
        return self._tap("packed", np.uint8)

    def r900_quantized(self):
        return self._tap("r900_quantized", np.uint8)
