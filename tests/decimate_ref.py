"""ctypes binding of the CPU restatement of the decimating tuned input: its first stage (tests/cpu_harness/decimate_ref.c)
into the untuned resampler's restatement (resample_ref), or the tuned restatement (tune_ref) alone when D = 1, and the
rendering of wideband test captures with packets far enough apart for 30-61 MS/s.

The library is compiled with gcc into a temporary directory on first use (the tree stays untouched)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import resample_ref
import tune_ref
from resample_ref import Info

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(ROOT, "tests", "cpu_harness", "decimate_ref.c")
_HDRS = [os.path.join(ROOT, "include", n) for n in ("ertgpu_resample.h", "ertgpu.h")]
_lib = None


class DecInfo(C.Structure):
    _fields_ = [("rate_in", C.c_int64), ("rate_out", C.c_int64), ("D", C.c_int32), ("T1", C.c_int32), ("S", C.c_int32),
                ("reserved", C.c_int32)]


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for p in [_SRC] + _HDRS:
            h.update(open(p, "rb").read())
        so = os.path.join(tempfile.gettempdir(), f"ertgpu_decimate_ref_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-std=gnu11", "-Wall", "-I", os.path.join(ROOT, "include"),
                            "-o", tmp, _SRC], check=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.dcref_state_size.restype = C.c_size_t
        L.dcref_plan.argtypes = [C.c_int64, C.c_int64, C.c_int64, C.POINTER(DecInfo), C.POINTER(Info)]
        L.dcref_init.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int64]
        L.dcref_dec.restype = C.POINTER(DecInfo)
        L.dcref_dec.argtypes = [C.c_void_p]
        L.dcref_info.restype = C.POINTER(Info)
        L.dcref_info.argtypes = [C.c_void_p]
        L.dcref_taps.restype = C.POINTER(C.c_int16)
        L.dcref_taps.argtypes = [C.c_void_p]
        L.dcref_feed.restype = C.c_int64
        L.dcref_feed.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
        _lib = L
    return _lib


def _d(s):
    return {k: getattr(s, k) for k, _ in s._fields_}


def plan(rate_in: int, rate_out: int, offset_hz: int):
    """ertrs_plan_decimated as (decimator dict, resampler dict), or None when rejected."""
    dec, inf = DecInfo(), Info()
    if lib().dcref_plan(rate_in, rate_out, offset_hz, C.byref(dec), C.byref(inf)) != 0:
        return None
    return _d(dec), _d(inf)


class Stage1:
    """The first stage of one stream (D >= 2): feed() takes uint8 IQ bytes at rate_in and returns the uint8 IQ bytes at
    R_mid = rate_in / D whose window is complete."""

    def __init__(self, rate_in: int, rate_out: int, offset_hz: int):
        L = lib()
        self._buf = C.create_string_buffer(L.dcref_state_size())
        if L.dcref_init(self._buf, rate_in, rate_out, offset_hz) != 0:
            raise ValueError(f"rate {rate_in} -> {rate_out} at offset {offset_hz}: no first stage")
        self.dec = _d(L.dcref_dec(self._buf).contents)
        self.info = _d(L.dcref_info(self._buf).contents)

    def taps(self) -> np.ndarray:
        return np.ctypeslib.as_array(lib().dcref_taps(self._buf), shape=(self.dec["T1"],)).copy()

    def feed(self, iq) -> np.ndarray:
        iq = np.ascontiguousarray(iq, dtype=np.uint8)
        assert iq.size % 2 == 0
        n = iq.size // 2
        cap = n // self.dec["D"] + 16
        out = np.empty(2 * cap, dtype=np.uint8)
        got = lib().dcref_feed(self._buf, iq.ctypes.data if n else None, n, out.ctypes.data, cap)
        assert got >= 0
        return out[:2 * got]


class Cascade:
    """One stream through the whole decimating input: feed() takes uint8 IQ bytes at rate_in and returns the uint8 IQ
    bytes at rate_out whose windows are complete.  D = 1 is the tuned restatement alone."""

    def __init__(self, rate_in: int, rate_out: int, offset_hz: int):
        p = plan(rate_in, rate_out, offset_hz)
        if p is None:
            raise ValueError(f"rate {rate_in} -> {rate_out} at offset {offset_hz} rejected")
        self.dec, self.info = p
        if self.dec["D"] == 1:
            self._tuner = tune_ref.Tuner(rate_in, rate_out, offset_hz)
            self.stage1 = None
        else:
            self.stage1 = Stage1(rate_in, rate_out, offset_hz)
            self._stage2 = resample_ref.Resampler(rate_in, self.dec["D"] * rate_out)
            assert self._stage2.info == self.info

    def feed(self, iq) -> np.ndarray:
        if self.stage1 is None:
            return self._tuner.feed(iq)
        return self._stage2.feed(self.stage1.feed(iq))


def decimate(iq, rate_in: int, rate_out: int, offset_hz: int) -> np.ndarray:
    return Cascade(rate_in, rate_out, offset_hz).feed(iq)


def wideband(channels, rate_in: int, nsamples: int, seed: int, spacing: int, noise: float = 6.0):
    """tune_ref.wideband with `spacing` samples between packet starts: at 30-61 MS/s one idm packet is 1.4-2.8 million
    samples long, longer than tune_ref's fixed 2^19.  Complex baseband at rate_in (8-bit units): Gaussian noise of sigma
    `noise` plus, for each (msgtypes, offset_hz, pk_seed, shift) in channels, packets whose high chips carry
    amp_i + j amp_q, rotated by e^(j 2 pi offset n / rate_in).  Returns (signal, truth per channel)."""
    from rtlamr_b200 import synth
    rng = np.random.default_rng(seed)
    z = noise * (rng.standard_normal(nsamples) + 1j * rng.standard_normal(nsamples))
    truths = []
    cl_guess = -(-rate_in // tune_ref.DATA_RATE)
    n_all = np.arange(nsamples)
    for msgtypes, off, pk_seed, shift in channels:
        pk, truth = synth.make_packets(msgtypes, cl_guess, nsamples - 2 * spacing - shift, seed=pk_seed, spacing=spacing)
        sig = np.zeros(nsamples, dtype=np.complex128)
        for row in pk:
            n_chips = int(row["n_chips"])
            chips = np.unpackbits(row["chips"])[:n_chips]
            start = int(row["start_sample"]) + shift
            s = np.arange(-(-n_chips * rate_in // tune_ref.DATA_RATE))
            c = s * tune_ref.DATA_RATE // rate_in
            hi = chips[np.minimum(c, n_chips - 1)].astype(bool) & (c < n_chips)
            idx = start + s[hi]
            sig[idx[idx < nsamples]] += complex(int(row["amp_i"]), int(row["amp_q"]))
        z += sig * np.exp(2j * np.pi * (off * (n_all % rate_in) / rate_in))
        truths.append(truth)
    return z, truths
