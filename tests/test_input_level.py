"""CPU tests of the automatic gain: the rule of include/ertgpu_level.h (compiled through a small C harness) against a
NumPy restatement, and the CLI's handling of -samplescale=auto."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import ROOT
from format_ref import wav_bytes
from test_sigmf import write_recording

CLI = os.path.join(ROOT, "rtlamr_b200", "ertgpu_decode_file")
_SRC = os.path.join(ROOT, "tests", "cpu_harness", "level_ref.c")
_HDR = os.path.join(ROOT, "include", "ertgpu_level.h")
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for p in (_SRC, _HDR):
            h.update(open(p, "rb").read())
        so = os.path.join(tempfile.gettempdir(), f"ertgpu_level_ref_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-std=gnu11", "-Wall", "-I", os.path.join(ROOT, "include"),
                            "-o", tmp, _SRC], check=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.lvref_exponent.restype = C.c_int32
        L.lvref_exponent.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int32]
        _lib = L
    return _lib


def rule(bins, components, zeros, nans, default_k):
    bins = np.ascontiguousarray(bins, dtype=np.int64)
    assert bins.size == 256
    return lib().lvref_exponent(bins.ctypes.data, components, zeros, nans, default_k)


def rule_ref(bins, components, zeros, nans, default_k):
    """The rule from its definition: the largest k in [-120, 120] at which at most floor(N / 65536) components have
    |x| * 2^k >= 128, i.e. e >= 7 - k; -120 when none; the default when nothing is non-zero and non-NaN."""
    if components - zeros - nans <= 0:
        return default_k
    allow = components // 65536
    for k in range(120, -121, -1):
        if int(np.sum(bins[7 - k + 128:])) <= allow:
            return k
    return -120


def test_window_is_two_to_the_22():
    assert lib().lvref_window() == 1 << 22


def test_rule_on_random_histograms():
    rng = np.random.default_rng(1)
    for trial in range(400):
        bins = np.zeros(256, dtype=np.int64)
        lo, hi = sorted(rng.integers(0, 256, 2))
        bins[lo:hi + 1] = rng.integers(0, 1 << rng.integers(1, 30), hi - lo + 1)
        if trial % 3 == 0:   # a few outliers far above the bulk
            bins[rng.integers(lo, 256, 3)] += rng.integers(0, 40, 3)
        zeros, nans = int(rng.integers(0, 1000)), int(rng.integers(0, 50))
        n = int(bins.sum()) + zeros + nans
        dk = int(rng.integers(-24, 8))
        assert rule(bins, n, zeros, nans, dk) == rule_ref(bins, n, zeros, nans, dk), trial


def test_rule_edge_cases():
    z = np.zeros(256, dtype=np.int64)
    assert rule(z, 1000, 1000, 0, -8) == -8                 # all zero
    assert rule(z, 1000, 0, 1000, 7) == 7                   # all NaN
    assert rule(z, 1000, 600, 400, -24) == -24              # zeros and NaNs only
    assert rule(z, 0, 0, 0, 0) == 0                         # nothing measured
    inf = z.copy()
    inf[255] = 10                                           # infinities (top bin) and nothing else
    assert rule(inf, 10, 0, 0, -8) == -120
    # e = 3 only (|x| in [8, 16)): 7 - k <= 3 clips, so k = 3 is the largest that does not
    b = z.copy()
    b[3 + 128] = 1 << 20
    assert rule(b, 1 << 20, 0, 0, 0) == 3
    # exactly A and A + 1 components over the threshold
    n = 1 << 22
    A = n // 65536
    for over, want in ((A, 8), (A + 1, 1)):
        b = z.copy()
        b[-2 + 128] = n - over                              # the bulk at e = -2: k <= 8 keeps it unclipped
        b[5 + 128] = over                                   # the loud ones at e = 5: k <= 1 keeps them unclipped
        assert rule(b, n, 0, 0, 0) == want == rule_ref(b, n, 0, 0, 0), over
    # infinities count against the allowance at every k
    b = z.copy()
    b[0 + 128] = n - A - 1
    b[255] = A + 1
    assert rule(b, n, 0, 0, 0) == -120
    b[255] = A
    assert rule(b, n, 0, 0, 0) == 6
    # the k bounds: tiny and huge components
    b = z.copy()
    b[0] = 100                                              # e <= -128: even 2^120 leaves them below 128
    assert rule(b, 100, 0, 0, 0) == 120
    b = z.copy()
    b[-113 + 128] = 100                                     # e = -113: 2^120 clips, 2^119 does not
    assert rule(b, 100, 0, 0, 0) == 119
    b = z.copy()
    b[127 + 128] = 100                                      # e >= 127 (a float64 of 2^200, say): clips even at 2^-120
    assert rule(b, 100, 0, 0, 0) == -120
    b = z.copy()
    b[126 + 128] = 100                                      # e = 126: 2^-119 clips, 2^-120 does not
    assert rule(b, 100, 0, 0, 0) == -120
    b = z.copy()
    b[125 + 128] = 100
    assert rule(b, 100, 0, 0, 0) == -119


def _cli(*args, stdin=None):
    r = subprocess.run([CLI, *args], capture_output=True, timeout=60, input=stdin)
    r.stderr = r.stderr.decode(errors="replace")
    return r


def test_cli_takes_auto_for_every_converted_format(built, tmp_path):
    """-samplescale=auto passes the argument checks for cs16, cf32, a 16-bit WAV and a SigMF recording (without a GPU
    the run then fails at the device, with exit status 1), and is a usage error for cu8 and an 8-bit WAV."""
    raw = tmp_path / "in.bin"
    np.zeros(1 << 14, dtype=np.uint8).tofile(raw)
    w8 = tmp_path / "a8.wav"
    w8.write_bytes(wav_bytes(bytes(1 << 14), bits=8, rate=2_359_296))
    w16 = tmp_path / "a16.wav"
    w16.write_bytes(wav_bytes(bytes(1 << 14), bits=16, rate=2_400_000))
    rec = write_recording(tmp_path / "r", bytes(1 << 14), "cf32_le", 2_400_000)
    u8rec = write_recording(tmp_path / "u", bytes(1 << 14), "cu8", 2_400_000)
    try:
        import torch
        gpu = torch.cuda.is_available()
    except Exception:
        gpu = False
    for args in (["-sampleformat=cs16", str(raw)], ["-sampleformat=cf32", str(raw)], ["-sampleformat=ci16_be", str(raw)],
                 ["-sampleformat=wav", str(w16)], ["-sampleformat=sigmf", rec]):
        r = _cli("-samplescale=auto", *args)
        assert "invalid value" not in r.stderr and "does not apply" not in r.stderr, (args, r.stderr)
        assert r.returncode == (0 if gpu else 1), (args, r.returncode, r.stderr)
    for args in (["-sampleformat=cu8", str(raw)], [str(raw)], ["-sampleformat=wav", str(w8)], ["-sampleformat=sigmf", u8rec]):
        r = _cli("-samplescale=auto", *args)
        assert r.returncode == 2 and "-samplescale" in r.stderr and "CenterFreq" not in r.stderr, (args, r.stderr)
    for word in ("AUTO", "Auto", "auto ", " auto", "autox", "auto=1", ""):
        r = _cli(f"-samplescale={word}", "-sampleformat=cs16", str(raw))
        assert r.returncode == 2 and "invalid value" in r.stderr and "CenterFreq" not in r.stderr, (word, r.stderr)


def test_host_receiver_input_scale_argument(built):
    """host.Receiver takes a gain or the word "auto": another string is refused before a device is touched, and auto
    on cu8 input is refused as the CLI refuses it."""
    from rtlamr_b200 import capi, host
    with pytest.raises(ValueError):
        host.Receiver("scm", 72, input_format=capi.FORMAT_CS16, input_scale="Auto")
    with pytest.raises(RuntimeError, match="cu8"):
        host.Receiver("scm", 72, input_scale="auto")
