"""ctypes binding of the CPU restatement of the wide channel path (tests/cpu_harness/wide_ref.c), the numpy restatement
of the wide component s_w of every input format, and of the channel level and its gain rule, written from
include/ertgpu_resample.h.

The library is compiled with gcc into a temporary directory on first use (the tree stays untouched)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from rtlamr_b200 import capi

import format_ref
from decimate_ref import DecInfo
from resample_ref import Info
from test_sigmf import SIGMF, components

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(ROOT, "tests", "cpu_harness", "wide_ref.c")
_HDRS = [os.path.join(ROOT, "include", n) for n in ("ertgpu_resample.h", "ertgpu.h")]
_lib = None
K_MAX = 14
S = 14
WIDE_MAX = 16383
# components float32 holds exactly take the float32 product; the others the float64 one (convert.cuh)
F32_EXACT = {capi.FORMAT_CS8, capi.FORMAT_CS16, capi.FORMAT_CF32, capi.FORMAT_CS16BE, capi.FORMAT_CU16,
             capi.FORMAT_CU16BE, capi.FORMAT_CF32BE}


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for p in [_SRC] + _HDRS:
            h.update(open(p, "rb").read())
        so = os.path.join(tempfile.gettempdir(), f"ertgpu_wide_ref_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-std=gnu11", "-Wall", "-I", os.path.join(ROOT, "include"),
                            "-o", tmp, _SRC], check=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.wideref_state_size.restype = C.c_size_t
        L.wideref_init.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int32]
        L.wideref_info.restype = C.POINTER(Info)
        L.wideref_info.argtypes = [C.c_void_p]
        L.wideref_dec.restype = C.POINTER(DecInfo)
        L.wideref_dec.argtypes = [C.c_void_p]
        L.wideref_table.restype = C.POINTER(C.c_int16)
        L.wideref_table.argtypes = [C.c_void_p]
        L.wideref_taps.restype = C.POINTER(C.c_int16)
        L.wideref_taps.argtypes = [C.c_void_p]
        L.wideref_max_acc.restype = C.c_int64
        L.wideref_max_acc.argtypes = [C.c_void_p]
        L.wideref_set_gain.argtypes = [C.c_void_p, C.c_int32]
        L.wideref_feed.restype = C.c_int64
        L.wideref_feed.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64]
        L.wideref_channel_gain.restype = C.c_int32
        L.wideref_channel_gain.argtypes = [C.c_void_p, C.c_int64]
        _lib = L
    return _lib


def _d(s):
    return {k: getattr(s, k) for k, _ in s._fields_}


def wide_components(raw, fmt: int, scale: float = 0.0) -> np.ndarray:
    """s_w of every component of the raw capture bytes (int32, I and Q interleaved): isnan(p) ? 0 :
    clamp(rint(p * 2^7), +-16383) with p = fl32(x * g) or fl64(x * g); cu8 gives 64 * (2u - 255)."""
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    if fmt == capi.FORMAT_CU8:
        return 64 * (2 * raw.astype(np.int32) - 255)
    if fmt in SIGMF:
        x, g = components(raw, fmt), scale or SIGMF[fmt][3]
    else:
        x, g = raw.view(format_ref.DTYPE[fmt]), scale or format_ref.DEFAULT_SCALE[fmt]
    with np.errstate(invalid="ignore", over="ignore"):
        if fmt in F32_EXACT:
            p = (np.asarray(x).astype(np.float32) * np.float32(g)) * np.float32(128)
        else:
            p = (np.asarray(x).astype(np.float64) * np.float64(np.float32(g))) * 128.0
        v = np.where(np.isnan(p), 0, np.clip(np.rint(p), -WIDE_MAX, WIDE_MAX))
    return v.astype(np.int32)


class Wide:
    """One stream through the wide path: feed() takes s_w pairs (int32, interleaved) at rate_in and returns the uint8
    IQ bytes at rate_out whose windows are complete, and their accumulators."""

    def __init__(self, rate_in: int, rate_out: int, offset_hz: int, k: int = 0):
        L = lib()
        self._buf = C.create_string_buffer(L.wideref_state_size())
        if L.wideref_init(self._buf, rate_in, rate_out, offset_hz, k) != 0:
            raise ValueError(f"rate {rate_in} -> {rate_out} at offset {offset_hz} rejected")
        self.info = _d(L.wideref_info(self._buf).contents)
        self.dec = _d(L.wideref_dec(self._buf).contents)

    def table(self) -> np.ndarray:
        n = (self.info["P"] + 1) * self.info["T"]
        return np.ctypeslib.as_array(lib().wideref_table(self._buf), shape=(n,)).copy()

    def taps(self) -> np.ndarray:
        return np.ctypeslib.as_array(lib().wideref_taps(self._buf), shape=(self.dec["T1"],)).copy()

    def max_acc(self) -> int:
        return int(lib().wideref_max_acc(self._buf))

    def set_gain(self, k: int):
        lib().wideref_set_gain(self._buf, k)

    def feed(self, sw):
        sw = np.ascontiguousarray(sw, dtype=np.int32)
        assert sw.size % 2 == 0
        n = sw.size // 2
        cap = n * 4 + 4 * self.info["T"] + 64
        out = np.empty(2 * cap, dtype=np.uint8)
        acc = np.empty(2 * cap, dtype=np.int32)
        got = lib().wideref_feed(self._buf, sw.ctypes.data if n else None, n, out.ctypes.data, acc.ctypes.data, cap)
        assert got >= 0
        return out[:2 * got], acc[:2 * got]


def wide(raw, fmt, rate_in, rate_out, offset_hz, k, scale=0.0):
    """The wide path's bytes and accumulators of a whole capture."""
    return Wide(rate_in, rate_out, offset_hz, k).feed(wide_components(raw, fmt, scale))


def level(acc) -> dict:
    """The channel level of accumulators: bins[e] counts 2^e <= |acc| < 2^(e+1), e in [0, 31]."""
    a = np.abs(np.asarray(acc, dtype=np.int64))
    nz = a[a > 0]
    e = np.floor(np.log2(nz.astype(np.float64))).astype(np.int64)
    # log2 of an int32 in float64 can round up at 2^e - 1: correct from the integers
    e -= (np.left_shift(np.int64(1), e) > nz)
    bins = np.bincount(e, minlength=32).astype(np.int64)
    return {"components": int(a.size), "zeros": int(a.size - nz.size), "bins": bins, "k": channel_gain(bins, a.size)}


def channel_gain(bins, components) -> int:
    """The auto rule: the largest k in [0, 14] at which at most components // 65536 components have
    e >= S + 14 - k; 0 when none is non-zero."""
    bins = np.asarray(bins, dtype=np.int64)
    if bins.sum() == 0:
        return 0
    for k in range(K_MAX, 0, -1):
        if bins[S + 14 - k:].sum() <= components // 65536:
            return k
    return 0
