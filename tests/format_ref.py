"""numpy restatement of the input-format conversion (ertgpu_set_input_format), written from its definition and not
from the CUDA code, and writers of the test captures: raw cs8 / cs16 / cf32 and baseband WAV files."""
from __future__ import annotations

import struct

import numpy as np

from rtlamr_b200.capi import FORMAT_CF32, FORMAT_CS8, FORMAT_CS16, FORMAT_CU8

DEFAULT_SCALE = {FORMAT_CS8: 1.0, FORMAT_CS16: 2.0 ** -8, FORMAT_CF32: 2.0 ** 7}
DTYPE = {FORMAT_CS8: np.dtype("i1"), FORMAT_CS16: np.dtype("<i2"), FORMAT_CF32: np.dtype("<f4")}
NAME = {FORMAT_CU8: "cu8", FORMAT_CS8: "cs8", FORMAT_CS16: "cs16", FORMAT_CF32: "cf32"}


def to_u8(x, scale: float) -> np.ndarray:
    """u = (isnan(p) ? 0 : clamp(rint(p), -128, 127)) + 128 with p = fl32(x * scale) (float32 multiply, round half to
    even in both places)."""
    with np.errstate(invalid="ignore", over="ignore"):
        p = np.asarray(x).astype(np.float32) * np.float32(scale)
        v = np.where(np.isnan(p), np.float32(0), np.clip(np.rint(p), -128, 127))
    return (v + 128).astype(np.uint8)


def convert(raw: bytes | np.ndarray, fmt: int, scale: float = 0.0) -> np.ndarray:
    """The uint8 IQ bytes the decoder reads for the raw bytes of a capture in format fmt."""
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    if fmt == FORMAT_CU8:
        return raw.copy()
    return to_u8(raw.view(DTYPE[fmt]), scale or DEFAULT_SCALE[fmt])


def encode(u8: np.ndarray, fmt: int) -> np.ndarray:
    """uint8 IQ as raw bytes of format fmt that convert() at the default scale maps back exactly."""
    v = np.asarray(u8, dtype=np.int32) - 128
    if fmt == FORMAT_CU8:
        return np.asarray(u8, dtype=np.uint8).copy()
    if fmt == FORMAT_CS8:
        return v.astype(np.int8).view(np.uint8)
    if fmt == FORMAT_CS16:
        return (v * 256).astype("<i2").view(np.uint8)
    return (v.astype(np.float32) / np.float32(128)).astype("<f4").view(np.uint8)


def wav_bytes(payload: bytes, bits: int, rate: int, *, tag: int = 1, channels: int = 2, extensible: bool = False,
              rf64: bool = False, data_size: int | None = None, before_data: bytes = b"") -> bytes:
    """A WAV file around payload: RIFF or RF64 (ds64 chunk), plain or WAVE_FORMAT_EXTENSIBLE fmt, extra chunks in
    before_data, and the data chunk's size field (default: the payload's length)."""
    align = channels * bits // 8
    body = struct.pack("<HHIIHH", 0xFFFE if extensible else tag, channels, rate, rate * align, align, bits)
    if extensible:
        guid = struct.pack("<H", tag) + bytes([0, 0, 0, 0, 0x10, 0, 0x80, 0, 0, 0xAA, 0, 0x38, 0x9B, 0x71])
        body += struct.pack("<HHI", 22, bits, 3) + guid
    fmt = b"fmt " + struct.pack("<I", len(body)) + body
    n = len(payload) if data_size is None else data_size
    if rf64:
        ds64 = b"ds64" + struct.pack("<IQQQI", 28, 0, n, len(payload) // align, 0)
        head = b"RF64" + struct.pack("<I", 0xFFFFFFFF) + b"WAVE" + ds64 + fmt + before_data
        return head + b"data" + struct.pack("<I", 0xFFFFFFFF) + payload
    head = fmt + before_data + b"data" + struct.pack("<I", n & 0xFFFFFFFF)
    return b"RIFF" + struct.pack("<I", (4 + len(head) + len(payload)) & 0xFFFFFFFF) + b"WAVE" + head + payload
