"""CPU test of the input-format table of include/ertgpu_format.h (compiled through a small C harness) against the
Python copies the bindings and tests use: capi.FORMAT_BYTES, the short names, the SigMF datatypes and the default
gains."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import pytest

from conftest import ROOT
from rtlamr_b200 import capi

import format_ref
from test_sigmf import DATATYPES, NAME, SIGMF

_SRC = os.path.join(ROOT, "tests", "cpu_harness", "format_ref.c")
_HDRS = [os.path.join(ROOT, "include", h) for h in ("ertgpu_format.h", "ertgpu.h")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for p in [_SRC] + _HDRS:
            h.update(open(p, "rb").read())
        so = os.path.join(tempfile.gettempdir(), f"ertgpu_format_ref_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-std=gnu11", "-Wall", "-Wextra", "-Werror", "-I",
                            os.path.join(ROOT, "include"), "-o", tmp, _SRC], check=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.fmtref_sigmf.restype = L.fmtref_name.restype = C.c_char_p
        L.fmtref_default_scale.restype = C.c_float
        L.fmtref_from_sigmf.argtypes = L.fmtref_from_name.argtypes = [C.c_char_p]
        _lib = L
    return _lib


DEFAULT_SCALE = {capi.FORMAT_CU8: 0.0, **format_ref.DEFAULT_SCALE, **{f: v[3] for f, v in SIGMF.items()}}


@pytest.mark.parametrize("fmt", sorted(capi.FORMAT_BYTES))
def test_format_row(fmt):
    L = lib()
    sigmf = next(n for n, f in DATATYPES.items() if f == fmt)
    assert L.fmtref_bytes(fmt) == capi.FORMAT_BYTES[fmt]
    assert L.fmtref_name(fmt).decode() == NAME[fmt]
    assert L.fmtref_sigmf(fmt).decode() == sigmf
    assert L.fmtref_default_scale(fmt) == DEFAULT_SCALE[fmt]
    assert L.fmtref_from_sigmf(sigmf.encode()) == fmt
    assert L.fmtref_from_name(sigmf.encode()) == fmt
    assert L.fmtref_from_name(NAME[fmt].encode()) == fmt


def test_every_format_is_in_the_table():
    L = lib()
    assert sorted(DATATYPES.values()) == sorted(capi.FORMAT_BYTES) == sorted(NAME)
    known = [f for f in range(-4, 64) if L.fmtref_bytes(f)]
    assert known == sorted(capi.FORMAT_BYTES)
    assert all(L.fmtref_name(f) is None and L.fmtref_sigmf(f) is None for f in range(-4, 64) if f not in known)


@pytest.mark.parametrize("name", ["", "cs8 ", "CS16", "ci16", "cs16_le", "rf32_le", "wav", "sigmf", "cu8,cs8"])
def test_unknown_names(name):
    L = lib()
    assert L.fmtref_from_sigmf(name.encode()) == -1
    assert L.fmtref_from_name(name.encode()) == -1


def test_short_names_are_not_sigmf_datatypes():
    L = lib()
    for short in ("cs8", "cs16", "cf32"):
        assert L.fmtref_from_sigmf(short.encode()) == -1
