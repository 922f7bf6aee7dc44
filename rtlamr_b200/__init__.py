"""rtlamr_b200 -- Hopper-native (H100, sm_90a) ERT demodulator behind rtlamr's protocol.Decoder.

The product is `libertgpu.so` (C ABI in include/ertgpu.h, kernels in rtlamr_b200/csrc/).
This Python package only holds the ctypes binding and tooling used by tests/ and bench.py.
"""
from . import capi  # noqa: F401
