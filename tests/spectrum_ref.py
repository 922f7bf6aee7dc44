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

from rtlamr_b200 import capi
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
    return rows_of_powers(p, frames_per_row, partial=partial)


def rows_of_powers(p, frames_per_row: int, frames: int | None = None, first_row: int = 0, partial: bool = False):
    """rows() from frame powers p: the rows of the stream's first `frames` frames (all of p by default), from row
    first_row on, as a fetch after the rows before first_row were fetched returns them."""
    F, n = frames_per_row, p.shape[1]
    frames = p.shape[0] if frames is None else frames
    nr = frames // F
    out, mean, peak = [], [], []
    ends = [(r * F, (r + 1) * F) for r in range(first_row, nr)]
    if partial and frames % F:
        ends.append((nr * F, frames))
    for a, b in ends:
        out.append((a * n, b - a))
        mean.append(p[a:b].mean(axis=0))
        peak.append(p[a:b].max(axis=0))
    z = np.zeros((0, n))
    return out, np.array(mean) if mean else z, np.array(peak) if peak else z


def group_frames(log2_n: int) -> int:
    """G, the frames of one of spectrum_kernel's groups (rtlamr_b200/csrc/spectrum.cuh): max(4, 2^14 / N)."""
    return max(4, 1 << max(0, 14 - log2_n))


def least_frames(log2_n: int) -> int:
    """The fewest frames per row ertgpu_enable_spectrum takes: ceil(2^18 / N)."""
    return -(-ROW_MIN >> log2_n)


def row_shapes() -> list:
    """(log2 N, F) for every N: the least F, one more, the least F above them whose last group is one frame short of
    G, and 3 least F + 5.  Their last groups are whole, one frame, G - 1 frames and five or one frames long."""
    out = []
    for log2_n in range(6, 15):
        lf, g = least_frames(log2_n), group_frames(log2_n)
        out += [(log2_n, lf), (log2_n, lf + 1), (log2_n, lf + 2 + (g - 1 - (lf + 2) % g) % g), (log2_n, 3 * lf + 5)]
    return out


def cut_plan(log2_n: int, frames_per_row: int) -> list:
    """Ends, in input samples, of the calls that feed one stream of four rows, the last one open: (a) inside a frame,
    then inside the same frame again (a call of no whole frame); (b) on a frame boundary inside a group; (c) on a group
    boundary inside a row; (d) at the first row's end; (e) inside the second row's last group, on a frame boundary
    when it has two frames or more, then inside a frame; then a call over the rest of that row and all of the third to
    a frame boundary inside the fourth; and the stream's end, inside a frame of the fourth row's last group."""
    n, g, F = 1 << log2_n, group_frames(log2_n), frames_per_row
    last = F - (-(-F // g) - 1) * g          # frames of a row's last group
    lg = F - last                            # its first frame, from the row's start
    cuts = [(g + 1) * n + n // 2 + 1, (g + 1) * n + n // 2 + 4, (2 * g + 3) * n, 3 * g * n, F * n]
    if last > 1:
        cuts.append((F + lg + 1) * n)
    return cuts + [(F + lg + last // 2) * n + n // 3, (3 * F + 2) * n, (3 * F + lg + last // 2) * n + n // 3]


# The frame-tagged capture.  Frame f holds one tone at the centre of FFT bin (c + a f) mod N, a odd, so that neighbouring
# frames land far apart, at a level from a cycle of three: odd, so that frames f and f + F differ in level even where N
# divides F and their bins agree.  White noise lies 45 dB below the tone in its bin, which keeps every bin of a row
# within the 60 dB that assert_close checks to 0.01 dB.  Each frame is then visible in its row's mean, and where a row
# has fewer frames than N, also in its peak.
TAG_LEVELS_DB = (0.0, -1.5, -3.0)
TAG_SNR_DB = 45.0


def tag_bins(log2_n: int, seed: int) -> tuple:
    """(c, a) of the tagged capture of this seed: frame f's tone is at FFT bin (c + a f) mod N."""
    n = 1 << log2_n
    rng = np.random.default_rng(seed)
    return int(rng.integers(0, n)), 2 * int(rng.integers(n // 8, n // 4)) + 1


def tag_amplitude(log2_n: int) -> tuple:
    """(tone amplitude at level 0, noise per component), in 8-bit units: A^2 N / (3 sigma^2) is TAG_SNR_DB, and the
    tone and three sigma of noise stay inside the cu8 range."""
    rel = np.sqrt((1 << log2_n) / (3.0 * 10 ** (TAG_SNR_DB / 10)))
    amp = 125.0 / (1.0 + 3.0 * rel)
    return amp, amp * rel


def tagged_components(log2_n: int, samples: int, seed: int) -> np.ndarray:
    """s_w (int32, I and Q interleaved) of the first `samples` samples of the tagged capture: odd multiples of 64
    (64 (2u - 255) of a cu8 byte u), which every format of tagged_bytes stores exactly."""
    n = 1 << log2_n
    c, a = tag_bins(log2_n, seed)
    amp, sigma = tag_amplitude(log2_n)
    rng = np.random.default_rng([seed, 1])
    out = np.empty(2 * samples, np.int32)
    j = np.arange(n)
    step = max(1, (1 << 20) // n)
    nf = -(-samples // n)
    for f0 in range(0, nf, step):
        f = np.arange(f0, min(f0 + step, nf))
        lv = amp * 10 ** (np.asarray(TAG_LEVELS_DB)[f % len(TAG_LEVELS_DB)] / 20)
        ph = rng.uniform(0, 2 * np.pi, f.size)
        z = lv[:, None] * np.exp(1j * (2 * np.pi * np.outer((c + a * f) % n, j) / n + ph[:, None]))
        z = z.reshape(-1) + sigma * (rng.standard_normal(z.size) + 1j * rng.standard_normal(z.size))
        s0, s1 = f0 * n, min((f0 + f.size) * n, samples)
        for part, o in ((z.real, 0), (z.imag, 1)):
            u = np.clip(np.round(part[:s1 - s0] + 127.5), 0, 255).astype(np.int32)
            out[2 * s0 + o:2 * s1:2] = 64 * (2 * u - 255)
    return out


# the formats tagged_bytes writes, one per read path (byte, int16, float, double); at their default gains they give s_w
# back exactly
TAG_FORMATS = (capi.FORMAT_CU8, capi.FORMAT_CS16, capi.FORMAT_CF32, capi.FORMAT_CF64BE)


def tagged_bytes(sw, fmt: int) -> np.ndarray:
    """Raw bytes of format fmt (cu8, cs16, cf32 or cf64_be) whose s_w at the default gain are sw."""
    sw = np.asarray(sw, np.int64)
    if fmt == capi.FORMAT_CU8:
        return ((sw // 64 + 255) // 2).astype(np.uint8)
    if fmt == capi.FORMAT_CS16:       # x 2^-8 2^7 = s_w
        return (2 * sw).astype("<i2").view(np.uint8)
    dt = {capi.FORMAT_CF32: "<f4", capi.FORMAT_CF64BE: ">f8"}[fmt]   # x 2^7 2^7 = s_w
    return (sw / 16384.0).astype(dt).view(np.uint8)


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


def assert_rows(got, want, what=""):
    """A fetch (rows, mean, peak) against the restatement's: the same rows (first_sample, frames), mean and peak within
    assert_close, and each row's mean summed over its bins within 1 / (4 frames) of the restatement's.  A divisor or a
    frame count off by one scales a whole row by 1 / F, under assert_close's 0.01 dB once F > 434; it moves the sum by
    four times that bound, and float32 rounding by far less."""
    rows = [tuple(int(x) for x in r) for r in got[0]]
    assert rows == list(want[0]), (what, rows, want[0])
    assert_close(got[1], want[1], f"{what} mean")
    assert_close(got[2], want[2], f"{what} peak")
    for i, (_, frames) in enumerate(want[0]):
        s, t = float(np.sum(got[1][i], dtype=np.float64)), float(np.sum(want[1][i]))
        assert abs(s - t) <= t / (4 * frames), (what, "sum", i, s / t - 1)
