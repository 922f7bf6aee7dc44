"""ctypes binding of the CPU restatement of the input-rate resampler (tests/cpu_harness/resample_ref.c).

The library is compiled with gcc into a temporary directory on first use (the tree stays untouched)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(ROOT, "tests", "cpu_harness", "resample_ref.c")
_HDRS = [os.path.join(ROOT, "include", n) for n in ("ertgpu_resample.h", "ertgpu.h")]
_lib = None


class Info(C.Structure):
    _fields_ = [("rate_in", C.c_int64), ("rate_out", C.c_int64), ("L", C.c_int64), ("M", C.c_int64),
                ("T", C.c_int32), ("P", C.c_int32), ("S", C.c_int32), ("F", C.c_int32)]


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for p in [_SRC] + _HDRS:
            h.update(open(p, "rb").read())
        so = os.path.join(tempfile.gettempdir(), f"ertgpu_resample_ref_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-std=gnu11", "-Wall", "-I", os.path.join(ROOT, "include"),
                            "-o", tmp, _SRC, "-lm"], check=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.rsref_state_size.restype = C.c_size_t
        L.rsref_init.argtypes = [C.c_void_p, C.c_int64, C.c_int64]
        L.rsref_table.restype = C.POINTER(C.c_int16)
        L.rsref_table.argtypes = [C.c_void_p]
        L.rsref_info.restype = C.POINTER(Info)
        L.rsref_info.argtypes = [C.c_void_p]
        L.rsref_feed.restype = C.c_int64
        L.rsref_feed.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
        _lib = L
    return _lib


class Resampler:
    """One stream: feed() takes uint8 IQ bytes (even length) at rate_in and returns the uint8 IQ bytes at
    rate_out whose filter window is complete."""

    def __init__(self, rate_in: int, rate_out: int):
        L = lib()
        self._buf = C.create_string_buffer(L.rsref_state_size())
        rc = L.rsref_init(self._buf, rate_in, rate_out)
        if rc != 0:
            raise ValueError(f"rate {rate_in} -> {rate_out} rejected")
        inf = L.rsref_info(self._buf).contents
        self.info = {k: getattr(inf, k) for k, _ in Info._fields_}

    def table(self) -> np.ndarray:
        n = (self.info["P"] + 1) * self.info["T"]
        return np.ctypeslib.as_array(lib().rsref_table(self._buf), shape=(n,)).copy()

    def feed(self, iq) -> np.ndarray:
        iq = np.ascontiguousarray(iq, dtype=np.uint8)
        assert iq.size % 2 == 0
        n = iq.size // 2
        cap = (n * 4 + 4 * self.info["T"] + 16) if n else 4 * self.info["T"] + 16
        out = np.empty(2 * cap, dtype=np.uint8)
        got = lib().rsref_feed(self._buf, iq.ctypes.data if n else None, n, out.ctypes.data, cap)
        assert got >= 0
        return out[:2 * got]


def resample(iq, rate_in: int, rate_out: int) -> np.ndarray:
    return Resampler(rate_in, rate_out).feed(iq)
