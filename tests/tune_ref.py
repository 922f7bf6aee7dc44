"""ctypes binding of the CPU restatement of the tuned input resampler (tests/cpu_harness/tune_ref.c), and the
numpy rendering of wideband test captures: packets drawn like test_gpu_resample.stream, rotated to an offset.

The library is compiled with gcc into a temporary directory on first use (the tree stays untouched)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from resample_ref import Info

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(ROOT, "tests", "cpu_harness", "tune_ref.c")
_HDRS = [os.path.join(ROOT, "include", n) for n in ("ertgpu_resample.h", "ertgpu.h")]
_lib = None
NCO_N = 4096
DATA_RATE = 32768


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for p in [_SRC] + _HDRS:
            h.update(open(p, "rb").read())
        so = os.path.join(tempfile.gettempdir(), f"ertgpu_tune_ref_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-std=gnu11", "-Wall", "-I", os.path.join(ROOT, "include"),
                            "-o", tmp, _SRC], check=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.tuneref_state_size.restype = C.c_size_t
        L.tuneref_init.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int64]
        L.tuneref_table.restype = C.POINTER(C.c_int16)
        L.tuneref_table.argtypes = [C.c_void_p]
        L.tuneref_info.restype = C.POINTER(Info)
        L.tuneref_info.argtypes = [C.c_void_p]
        L.tuneref_feed.restype = C.c_int64
        L.tuneref_feed.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
        L.tuneref_nco_step.restype = C.c_uint32
        L.tuneref_nco_step.argtypes = [C.c_int64, C.c_int64]
        L.tuneref_nco_table.argtypes = [C.c_void_p]
        L.tuneref_plan.argtypes = [C.c_int64, C.c_int64, C.c_int64, C.POINTER(Info)]
        _lib = L
    return _lib


def nco_step(offset_hz: int, rate_in: int) -> int:
    return int(lib().tuneref_nco_step(offset_hz, rate_in))


def nco_table() -> np.ndarray:
    """E as an (4096, 2) int32 array of (C, S)."""
    e = np.zeros(NCO_N, dtype=np.uint32)
    lib().tuneref_nco_table(e.ctypes.data)
    return np.stack([(e & 0xFFFF).astype(np.uint16).view(np.int16), (e >> 16).astype(np.uint16).view(np.int16)],
                    axis=1).astype(np.int32)


def plan(rate_in: int, rate_out: int, offset_hz: int):
    """ertrs_plan_tuned as a dict, or None when rejected."""
    inf = Info()
    if lib().tuneref_plan(rate_in, rate_out, offset_hz, C.byref(inf)) != 0:
        return None
    return {k: getattr(inf, k) for k, _ in Info._fields_}


class Tuner:
    """One stream: feed() takes uint8 IQ bytes (even length) at rate_in and returns the uint8 IQ bytes of the channel
    at offset_hz, at rate_out, whose filter window is complete."""

    def __init__(self, rate_in: int, rate_out: int, offset_hz: int):
        L = lib()
        self._buf = C.create_string_buffer(L.tuneref_state_size())
        if L.tuneref_init(self._buf, rate_in, rate_out, offset_hz) != 0:
            raise ValueError(f"rate {rate_in} -> {rate_out} at offset {offset_hz} rejected")
        inf = L.tuneref_info(self._buf).contents
        self.info = {k: getattr(inf, k) for k, _ in Info._fields_}

    def table(self) -> np.ndarray:
        n = (self.info["P"] + 1) * self.info["T"]
        return np.ctypeslib.as_array(lib().tuneref_table(self._buf), shape=(n,)).copy()

    def feed(self, iq) -> np.ndarray:
        iq = np.ascontiguousarray(iq, dtype=np.uint8)
        assert iq.size % 2 == 0
        n = iq.size // 2
        cap = (n * 4 + 4 * self.info["T"] + 16) if n else 4 * self.info["T"] + 16
        out = np.empty(2 * cap, dtype=np.uint8)
        got = lib().tuneref_feed(self._buf, iq.ctypes.data if n else None, n, out.ctypes.data, cap)
        assert got >= 0
        return out[:2 * got]


def tune(iq, rate_in: int, rate_out: int, offset_hz: int) -> np.ndarray:
    return Tuner(rate_in, rate_out, offset_hz).feed(iq)


def wideband(channels, rate_in: int, nsamples: int, seed: int, noise: float = 6.0, full_scale: float = 1.0):
    """Complex baseband at rate_in: Gaussian noise of sigma `noise` plus, for each (msgtypes, offset_hz, pk_seed) in
    channels, packets drawn as test_gpu_resample.stream draws them (carrier amp_i + j amp_q on high chips) and
    rotated by e^(j 2 pi offset n / rate_in).  Returns (complex128 signal in 8-bit units, truth per channel)."""
    from rtlamr_b200 import synth
    rng = np.random.default_rng(seed)
    z = noise * (rng.standard_normal(nsamples) + 1j * rng.standard_normal(nsamples))
    truths = []
    spacing = 1 << 17 if rate_in < 4_000_000 else 1 << 19   # an idm packet at 8 MS/s is 360 000 samples long
    cl_guess = -(-rate_in // DATA_RATE)
    n_all = np.arange(nsamples)
    for msgtypes, off, pk_seed, shift in channels:
        pk, truth = synth.make_packets(msgtypes, cl_guess, nsamples - 2 * spacing - shift, seed=pk_seed, spacing=spacing)
        sig = np.zeros(nsamples, dtype=np.complex128)
        for row in pk:
            n_chips = int(row["n_chips"])
            chips = np.unpackbits(row["chips"])[:n_chips]
            start = int(row["start_sample"]) + shift
            n = -(-n_chips * rate_in // DATA_RATE)
            s = np.arange(n)
            c = s * DATA_RATE // rate_in
            hi = chips[np.minimum(c, n_chips - 1)].astype(bool) & (c < n_chips)
            idx = start + s[hi]
            idx = idx[idx < nsamples]
            sig[idx] += complex(int(row["amp_i"]), int(row["amp_q"])) * full_scale
        z += sig * np.exp(2j * np.pi * (off * (n_all % rate_in) / rate_in))
        truths.append(truth)
    return z, truths


def quantize(z, fmt: int) -> np.ndarray:
    """Raw capture bytes of z (8-bit units) as cs8 or cs16 (cs16 = 256 * the 8-bit value, so its default scale maps it
    back)."""
    from rtlamr_b200.capi import FORMAT_CS8, FORMAT_CS16
    iq = np.empty(2 * z.size, dtype=np.float64)
    iq[0::2], iq[1::2] = z.real, z.imag
    if fmt == FORMAT_CS8:
        return np.clip(np.round(iq), -128, 127).astype(np.int8).view(np.uint8)
    assert fmt == FORMAT_CS16
    return np.clip(np.round(iq * 256), -32768, 32767).astype("<i2").view(np.uint8)
