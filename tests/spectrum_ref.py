"""NumPy float64 restatement of the input spectrum (include/ertgpu_spectrum.h) from raw capture bytes, and a ctypes
binding of the header's own helpers (tests/cpu_harness/spectrum_ref.c), compiled with gcc into a temporary directory
on first use."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from wide_ref import wide_components

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(ROOT, "tests", "cpu_harness", "spectrum_ref.c")
_HDRS = [os.path.join(ROOT, "include", n) for n in ("ertgpu_spectrum.h", "ertgpu.h")]
FULL_SCALE = 16320.0
DB_FLOOR = -200.0
ROW_MIN = 1 << 18
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for p in [_SRC] + _HDRS:
            h.update(open(p, "rb").read())
        so = os.path.join(tempfile.gettempdir(), f"ertgpu_spectrum_ref_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-std=gnu11", "-Wall", "-I", os.path.join(ROOT, "include"),
                            "-o", tmp, _SRC, "-lm"], check=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.specref_window.argtypes = [C.c_int32, C.c_void_p]
        L.specref_power_scale.restype = C.c_float
        L.specref_power_scale.argtypes = [C.c_int32]
        L.specref_db.restype = C.c_double
        L.specref_db.argtypes = [C.c_double]
        L.specref_log2_for_bin.restype = C.c_int32
        L.specref_log2_for_bin.argtypes = [C.c_int64, C.c_double]
        L.specref_frames_per_row.restype = C.c_int64
        L.specref_frames_per_row.argtypes = [C.c_int32, C.c_int64, C.c_int64]
        L.specref_bin_hz.restype = C.c_double
        L.specref_bin_hz.argtypes = [C.c_int64, C.c_int64, C.c_int32, C.c_int32]
        L.specref_csv_line.restype = C.c_int
        L.specref_csv_line.argtypes = [C.c_char_p, C.c_size_t, C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_int64,
                                       C.c_void_p]
        _lib = L
    return _lib


def window(log2_n: int) -> np.ndarray:
    """The periodic Hann window in double, rounded to float (as the library builds it)."""
    n = 1 << log2_n
    return (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(n) / n)).astype(np.float32)


def frame_powers(raw, fmt: int, log2_n: int, scale: float = 0.0) -> np.ndarray:
    """P_f[k] of every whole frame of the capture bytes, float64, bins in ascending frequency order."""
    sw = wide_components(raw, fmt, scale).astype(np.float64).reshape(-1, 2)
    n = 1 << log2_n
    nf = sw.shape[0] // n
    v = (sw[:nf * n, 0] + 1j * sw[:nf * n, 1]) / FULL_SCALE
    w = window(log2_n).astype(np.float64)
    x = np.fft.fft(v.reshape(nf, n) * w, axis=1)
    p = (x.real ** 2 + x.imag ** 2) / (n / 2.0) ** 2
    return np.fft.fftshift(p, axes=1)


def rows(raw, fmt: int, log2_n: int, frames_per_row: int, scale: float = 0.0, partial: bool = False):
    """(rows, mean, peak) as ertgpu_fetch_spectrum returns them for the whole capture in one stream: rows a list of
    (first_sample, frames)."""
    p = frame_powers(raw, fmt, log2_n, scale)
    n, F = 1 << log2_n, frames_per_row
    nr = p.shape[0] // F
    out, mean, peak = [], [], []
    ends = [(r * F, (r + 1) * F) for r in range(nr)]
    if partial and p.shape[0] % F:
        ends.append((nr * F, p.shape[0]))
    for a, b in ends:
        out.append((a * n, b - a))
        mean.append(p[a:b].mean(axis=0))
        peak.append(p[a:b].max(axis=0))
    z = np.zeros((0, n))
    return out, np.array(mean) if mean else z, np.array(peak) if peak else z


def db(p) -> np.ndarray:
    p = np.asarray(p, dtype=np.float64)
    with np.errstate(divide="ignore"):
        d = 10 * np.log10(np.where(p > 0, p, 1.0))
    return np.where(p > 0, np.maximum(d, DB_FLOOR), DB_FLOOR)


def assert_close(got, want, what=""):
    """mean or peak within 0.01 dB for every bin within 60 dB of the row's strongest bin; below that an absolute error
    of at most 1e-8 of the strongest bin's power."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    for r in range(want.shape[0]):
        top = want[r].max()
        strong = want[r] >= top * 1e-6
        if top > 0:
            err_db = np.abs(db(got[r][strong]) - db(want[r][strong]))
            assert err_db.max() <= 0.01, (what, r, float(err_db.max()), int(np.argmax(err_db)))
        weak = ~strong
        if weak.any():
            assert np.abs(got[r][weak] - want[r][weak]).max() <= 1e-8 * max(top, 0.0), (what, r)
