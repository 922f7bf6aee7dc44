"""ctypes binding of the libertgpu C ABI (include/ertgpu.h).

This is plumbing for tests/ and bench.py: the product is libertgpu.so itself, bound from Go by
the cgo shim in go/ (INTEGRATION.md).  There is no fallback of any kind: if the shared library
is missing or CUDA is unusable every call raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libertgpu.so")

OK, EINVAL, ECUDA, ENOMEM, ECAPACITY, ESIZE = 0, -1, -2, -3, -4, -5
MAX_PROTOCOLS, MAX_PREAMBLE, MAX_PACKET_BYTES, R900_DIGITS = 8, 32, 92, 42
CHECK_NONE, CHECK_CRC16, CHECK_IDM, CHECK_R900 = 0, 1, 2, 3
DECODE_ONLY_VALID = 1
CAND_HAS_R900 = 1
TAP_SIGNAL, TAP_CSUM, TAP_QUANTIZED, TAP_PACKED, TAP_R900_QUANTIZED, TAP_RESAMPLED = range(6)
FORMAT_CU8, FORMAT_CS8, FORMAT_CS16, FORMAT_CF32 = range(4)
# the other complex SigMF datatypes: ci16_be, cf32_be, cu16_le, cu16_be, ci32_le, ci32_be, cu32_le, cu32_be, cf64_le, cf64_be
(FORMAT_CS16BE, FORMAT_CF32BE, FORMAT_CU16, FORMAT_CU16BE, FORMAT_CS32, FORMAT_CS32BE, FORMAT_CU32, FORMAT_CU32BE, FORMAT_CF64,
 FORMAT_CF64BE) = range(16, 26)
FORMAT_BYTES = {FORMAT_CU8: 2, FORMAT_CS8: 2, FORMAT_CS16: 4, FORMAT_CF32: 8,   # bytes per IQ sample
                FORMAT_CS16BE: 4, FORMAT_CF32BE: 8, FORMAT_CU16: 4, FORMAT_CU16BE: 4, FORMAT_CS32: 8, FORMAT_CS32BE: 8,
                FORMAT_CU32: 8, FORMAT_CU32BE: 8, FORMAT_CF64: 16, FORMAT_CF64BE: 16}


class Protocol(C.Structure):
    _fields_ = [("name", C.c_char * 16), ("preamble", C.c_char * (MAX_PREAMBLE + 1)),
                ("data_rate", C.c_int32), ("chip_length", C.c_int32),
                ("preamble_symbols", C.c_int32), ("packet_symbols", C.c_int32),
                ("center_freq", C.c_uint32), ("check_kind", C.c_int32),
                ("crc_init", C.c_uint16), ("crc_poly", C.c_uint16), ("crc_residue", C.c_uint16),
                ("reserved", C.c_uint16), ("crc_from", C.c_int32), ("crc_to", C.c_int32)]


class DecoderConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "data_rate", "block_size", "block_size2", "chip_length", "symbol_length", "sample_rate",
        "preamble_symbols", "packet_symbols", "preamble_length", "packet_length",
        "buffer_length")] + [("center_freq", C.c_uint32), ("n_protocols", C.c_int32),
                             ("n_preambles", C.c_int32), ("packet_bytes", C.c_int32)]


class Candidate(C.Structure):
    _fields_ = [("block", C.c_int64), ("idx", C.c_int32), ("preamble_id", C.c_int32),
                ("check_mask", C.c_uint32), ("flags", C.c_uint32),
                ("bytes", C.c_uint8 * MAX_PACKET_BYTES), ("r900_digits", C.c_uint8 * R900_DIGITS),
                ("pad", C.c_uint8 * 2)]


class ResamplerInfo(C.Structure):
    _fields_ = [("rate_in", C.c_int64), ("rate_out", C.c_int64), ("L", C.c_int64), ("M", C.c_int64),
                ("T", C.c_int32), ("P", C.c_int32), ("S", C.c_int32), ("F", C.c_int32)]


class DecimatorInfo(C.Structure):
    _fields_ = [("rate_in", C.c_int64), ("rate_out", C.c_int64), ("D", C.c_int32), ("T1", C.c_int32), ("S", C.c_int32),
                ("reserved", C.c_int32)]


class TuningInfo(C.Structure):
    _fields_ = [("capture_center_hz", C.c_int64), ("center_hz", C.c_int64), ("offset_hz", C.c_int64),
                ("nco_step", C.c_uint32), ("nco_bits", C.c_int32)]


class ChannelLevel(C.Structure):
    _fields_ = [("components", C.c_int64), ("zeros", C.c_int64), ("bins", C.c_int64 * 32), ("k", C.c_int32),
                ("reserved", C.c_int32)]


CHANNEL_GAIN_K_MAX = 14


class InputLevel(C.Structure):
    _fields_ = [("components", C.c_int64), ("zeros", C.c_int64), ("nans", C.c_int64), ("bins", C.c_int64 * 256),
                ("exponent", C.c_int32), ("scale", C.c_float)]


class Shard(C.Structure):
    _fields_ = [("first_block", C.c_int64), ("last_block", C.c_int64), ("first_fed_block", C.c_int64)]


class SynthPacket(C.Structure):
    _fields_ = [("start_sample", C.c_int64), ("n_chips", C.c_int32), ("chip_length", C.c_int32),
                ("amp_i", C.c_int16), ("amp_q", C.c_int16), ("chips", C.c_uint8 * 192),
                ("pad", C.c_int32)]


class Signal(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("n_on", "e_on", "n_off", "e_off", "r_re", "r_im", "n_pairs")] + \
        [("protocol", C.c_int32), ("symbols", C.c_int32)]


SIGNAL_DTYPE = np.dtype([(n, "<i8") for n in ("n_on", "e_on", "n_off", "e_off", "r_re", "r_im", "n_pairs")] +
                        [("protocol", "<i4"), ("symbols", "<i4")])
assert SIGNAL_DTYPE.itemsize == C.sizeof(Signal) == 64

CAND_DTYPE = np.dtype([("block", "<i8"), ("idx", "<i4"), ("preamble_id", "<i4"),
                       ("check_mask", "<u4"), ("flags", "<u4"),
                       ("bytes", "u1", (MAX_PACKET_BYTES,)), ("r900_digits", "u1", (R900_DIGITS,)),
                       ("pad", "u1", (2,))])
assert CAND_DTYPE.itemsize == C.sizeof(Candidate) == 160

# every symbol include/ertgpu.h declares
EXPORTS = [
    "ertgpu_abi_version", "ertgpu_last_error", "ertgpu_create", "ertgpu_destroy",
    "ertgpu_register_protocol", "ertgpu_stock_protocol", "ertgpu_allocate", "ertgpu_get_config",
    "ertgpu_reset", "ertgpu_decode", "ertgpu_decode_device_async", "ertgpu_fetch",
    "ertgpu_last_counts", "ertgpu_last_launches", "ertgpu_set_stage_timing",
    "ertgpu_last_stage_ms", "ertgpu_stage_ms_mean", "ertgpu_tap", "ertgpu_set_demod_variant",
    "ertgpu_host_alloc", "ertgpu_host_free", "ertgpu_synth_fill",
    "ertgpu_bind_host_thread", "ertgpu_last_kernels", "ertgpu_plan_shards", "ertgpu_decode_sharded",
    "ertgpu_set_input_rate", "ertgpu_get_resampler", "ertgpu_set_input_format", "ertgpu_get_input_format",
    "ertgpu_set_input_tuning", "ertgpu_get_tuning", "ertgpu_measure_input", "ertgpu_set_input_scale",
    "ertgpu_allow_input_decimation", "ertgpu_get_decimator",
    "ertgpu_decode_channels", "ertgpu_decode_channels_device_async",
    "ertgpu_set_channel_gain", "ertgpu_get_channel_gain", "ertgpu_measure_channel",
    "ertgpu_enable_signal", "ertgpu_fetch_signal",
]

_lib = None


class ErtGpuError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libertgpu error {code}: {msg}")
        self.code = code


def lib() -> C.CDLL:
    """Load libertgpu.so (built in-tree by __graft_entry__.build()).  Fails loudly if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FileNotFoundError(
            f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp, i32, i64, u32, u64, sz = C.c_void_p, C.c_int32, C.c_int64, C.c_uint32, C.c_uint64, C.c_size_t
    L.ertgpu_abi_version.restype = C.c_int
    L.ertgpu_last_error.restype = C.c_char_p
    L.ertgpu_last_error.argtypes = [vp]
    L.ertgpu_create.argtypes = [C.POINTER(vp)]
    L.ertgpu_destroy.restype = None
    L.ertgpu_destroy.argtypes = [vp]
    L.ertgpu_register_protocol.argtypes = [vp, C.POINTER(Protocol)]
    L.ertgpu_stock_protocol.argtypes = [C.c_char_p, i32, C.POINTER(Protocol)]
    L.ertgpu_allocate.argtypes = [vp, i32, i64, i64]
    L.ertgpu_get_config.argtypes = [vp, C.POINTER(DecoderConfig)]
    L.ertgpu_reset.argtypes = [vp]
    L.ertgpu_decode.argtypes = [vp, vp, sz, u32, vp, sz, C.POINTER(sz)]
    L.ertgpu_decode_device_async.argtypes = [vp, vp, sz, u32, vp]
    L.ertgpu_fetch.argtypes = [vp, vp, sz, C.POINTER(sz)]
    L.ertgpu_last_counts.argtypes = [vp, C.POINTER(i64), C.POINTER(i64)]
    L.ertgpu_last_launches.restype = i64
    L.ertgpu_last_launches.argtypes = [vp]
    L.ertgpu_tap.argtypes = [vp, i32, i64, vp, sz, C.POINTER(sz)]
    L.ertgpu_set_stage_timing.argtypes = [vp, i32]
    L.ertgpu_last_stage_ms.argtypes = [vp, C.POINTER(C.c_float)]
    L.ertgpu_stage_ms_mean.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(i64)]
    L.ertgpu_set_demod_variant.argtypes = [vp, i32]
    L.ertgpu_host_alloc.argtypes = [C.POINTER(vp), sz]
    L.ertgpu_host_free.argtypes = [vp]
    L.ertgpu_synth_fill.argtypes = [i32, vp, i64, i64, u64, vp, i64, vp]
    L.ertgpu_bind_host_thread.argtypes = [i32, C.POINTER(i32), C.POINTER(i32)]
    L.ertgpu_last_kernels.restype = C.c_char_p
    L.ertgpu_last_kernels.argtypes = [vp]
    L.ertgpu_plan_shards.argtypes = [i64, i32, i32, i32, C.POINTER(Shard)]
    L.ertgpu_decode_sharded.argtypes = [C.POINTER(vp), i32, vp, sz, u32, vp, sz, C.POINTER(sz)]
    L.ertgpu_decode_channels.argtypes = [C.POINTER(vp), i32, vp, sz, u32]
    L.ertgpu_decode_channels_device_async.argtypes = [C.POINTER(vp), i32, vp, sz, u32, vp]
    L.ertgpu_set_input_rate.argtypes = [vp, i64]
    L.ertgpu_get_resampler.argtypes = [vp, C.POINTER(ResamplerInfo), vp, sz, C.POINTER(sz)]
    L.ertgpu_set_input_format.argtypes = [vp, i32, C.c_float]
    L.ertgpu_get_input_format.argtypes = [vp, C.POINTER(i32), C.POINTER(C.c_float)]
    L.ertgpu_set_input_tuning.argtypes = [vp, i64, i64]
    L.ertgpu_get_tuning.argtypes = [vp, C.POINTER(TuningInfo)]
    L.ertgpu_measure_input.argtypes = [vp, vp, sz, C.POINTER(InputLevel)]
    L.ertgpu_set_input_scale.argtypes = [vp, C.c_float]
    L.ertgpu_allow_input_decimation.argtypes = [vp]
    L.ertgpu_get_decimator.argtypes = [vp, C.POINTER(DecimatorInfo), vp, sz, C.POINTER(sz)]
    L.ertgpu_set_channel_gain.argtypes = [vp, i32]
    L.ertgpu_get_channel_gain.argtypes = [vp, C.POINTER(i32)]
    L.ertgpu_measure_channel.argtypes = [vp, vp, sz, C.POINTER(ChannelLevel)]
    L.ertgpu_enable_signal.argtypes = [vp]
    L.ertgpu_fetch_signal.argtypes = [vp, vp, sz, C.POINTER(sz)]
    for name in EXPORTS:
        getattr(L, name)  # AttributeError if the library does not export it
    _lib = L
    return L


def stock_protocol(msgtype: str, chip_length: int) -> Protocol:
    p = Protocol()
    rc = lib().ertgpu_stock_protocol(msgtype.encode(), chip_length, C.byref(p))
    if rc != OK:
        raise ErtGpuError(rc, f"invalid message type: {msgtype!r}")
    return p


class Handle:
    """One ertgpu_handle == one protocol.Decoder (reference protocol/decode.go:45-63)."""

    def __init__(self):
        self._L = lib()
        self._h = C.c_void_p()
        self._check(self._L.ertgpu_create(C.byref(self._h)))
        self.cfg = None

    def _check(self, rc: int):
        if rc != OK:
            raise ErtGpuError(rc, (self._L.ertgpu_last_error(self._h) or b"").decode())

    def close(self):
        if self._h:
            self._L.ertgpu_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def register(self, proto: Protocol):
        self._check(self._L.ertgpu_register_protocol(self._h, C.byref(proto)))

    def set_input_rate(self, hz: int):
        """ertgpu_set_input_rate: the IQ fed to this handle is sampled at `hz` (between register and allocate)."""
        self._check(self._L.ertgpu_set_input_rate(self._h, int(hz)))

    def set_input_tuning(self, capture_hz: int, center_hz: int = 0):
        """ertgpu_set_input_tuning: the IQ was recorded centred at capture_hz; decode the channel at center_hz (0: the
        decoder's CenterFreq).  After the protocols, before the rate and allocate."""
        self._check(self._L.ertgpu_set_input_tuning(self._h, int(capture_hz), int(center_hz)))

    def allow_input_decimation(self):
        """ertgpu_allow_input_decimation: a tuned handle may take captures at up to 256 times the decoder's rate (after
        the tuning, before the rate and allocate)."""
        self._check(self._L.ertgpu_allow_input_decimation(self._h))

    def decimator(self):
        """ertgpu_get_decimator: (info dict, int16 taps of the first stage, T1 entries)."""
        info, n = DecimatorInfo(), C.c_size_t(0)
        self._check(self._L.ertgpu_get_decimator(self._h, C.byref(info), None, 0, C.byref(n)))
        taps = np.zeros(n.value, dtype=np.int16)
        self._check(self._L.ertgpu_get_decimator(self._h, C.byref(info), taps.ctypes.data, taps.size, C.byref(n)))
        return {k: getattr(info, k) for k, _ in DecimatorInfo._fields_}, taps

    def tuning(self):
        """ertgpu_get_tuning as a dict."""
        info = TuningInfo()
        self._check(self._L.ertgpu_get_tuning(self._h, C.byref(info)))
        return {k: getattr(info, k) for k, _ in TuningInfo._fields_}

    def set_input_format(self, fmt: int, scale: float = 0.0):
        """ertgpu_set_input_format: the IQ fed to this handle is in format FORMAT_* with gain `scale` (0: the format's
        default), before allocate."""
        self._check(self._L.ertgpu_set_input_format(self._h, int(fmt), float(scale)))

    def input_format(self):
        """ertgpu_get_input_format: (format, scale in effect)."""
        f, g = C.c_int32(0), C.c_float(0)
        self._check(self._L.ertgpu_get_input_format(self._h, C.byref(f), C.byref(g)))
        return f.value, g.value

    def measure_input(self, buf) -> dict:
        """ertgpu_measure_input on a HOST buffer (numpy array of any dtype, or an address/size pair) of whole samples in
        the handle's format: {"components", "zeros", "nans", "bins" (int64[256], bins[e + 128]), "exponent", "scale"}."""
        if isinstance(buf, tuple):
            addr, nbytes = buf
        else:
            buf = np.ascontiguousarray(buf)
            addr, nbytes = buf.ctypes.data, buf.nbytes
        lv = InputLevel()
        self._check(self._L.ertgpu_measure_input(self._h, addr, nbytes, C.byref(lv)))
        return {"components": lv.components, "zeros": lv.zeros, "nans": lv.nans,
                "bins": np.array(lv.bins[:], dtype=np.int64), "exponent": lv.exponent, "scale": lv.scale}

    def set_input_scale(self, scale: float):
        """ertgpu_set_input_scale: the gain of the stream that starts now (after allocate or reset, before decode)."""
        self._check(self._L.ertgpu_set_input_scale(self._h, float(scale)))

    def set_channel_gain(self, k: int):
        """ertgpu_set_channel_gain: before allocate, the wide channel path of a tuned handle with gain 2^k; after it, k
        of the stream that starts now."""
        self._check(self._L.ertgpu_set_channel_gain(self._h, int(k)))

    def channel_gain(self) -> int:
        """ertgpu_get_channel_gain: k of a wide handle."""
        k = C.c_int32(0)
        self._check(self._L.ertgpu_get_channel_gain(self._h, C.byref(k)))
        return k.value

    def measure_channel(self, buf) -> dict:
        """ertgpu_measure_channel on a HOST buffer (numpy array, or an address/size pair) of whole samples in the
        handle's format: {"components", "zeros", "bins" (int64[32], bins[e] for 2^e <= |acc| < 2^(e+1)), "k"}."""
        if isinstance(buf, tuple):
            addr, nbytes = buf
        else:
            buf = np.ascontiguousarray(buf)
            addr, nbytes = buf.ctypes.data, buf.nbytes
        lv = ChannelLevel()
        self._check(self._L.ertgpu_measure_channel(self._h, addr, nbytes, C.byref(lv)))
        return {"components": lv.components, "zeros": lv.zeros, "bins": np.array(lv.bins[:], dtype=np.int64), "k": lv.k}

    def enable_signal(self):
        """ertgpu_enable_signal: measure every candidate's signal (before allocate)."""
        self._check(self._L.ertgpu_enable_signal(self._h))

    def fetch_signal(self, cap: int = 4096) -> np.ndarray:
        """ertgpu_fetch_signal: one SIGNAL_DTYPE record per candidate the last decode or fetch returned, same order."""
        while True:
            out = np.empty(cap, dtype=SIGNAL_DTYPE)
            n = C.c_size_t(0)
            rc = self._L.ertgpu_fetch_signal(self._h, out.ctypes.data, cap, C.byref(n))
            if rc == ECAPACITY and n.value > cap and "internal" not in (self._L.ertgpu_last_error(self._h) or b"").decode():
                cap = n.value
                continue
            self._check(rc)
            return out[:n.value].copy()

    def resampler(self):
        """ertgpu_get_resampler: (info dict, int16 table of (P+1)*T entries)."""
        info, n = ResamplerInfo(), C.c_size_t(0)
        self._check(self._L.ertgpu_get_resampler(self._h, C.byref(info), None, 0, C.byref(n)))
        table = np.zeros(n.value, dtype=np.int16)
        self._check(self._L.ertgpu_get_resampler(self._h, C.byref(info), table.ctypes.data, table.size, C.byref(n)))
        return {k: getattr(info, k) for k, _ in ResamplerInfo._fields_}, table

    def allocate(self, device: int = 0, max_blocks_per_call: int = 0, max_candidates: int = 0):
        self._check(self._L.ertgpu_allocate(self._h, device, max_blocks_per_call, max_candidates))
        cfg = DecoderConfig()
        self._check(self._L.ertgpu_get_config(self._h, C.byref(cfg)))
        self.cfg = cfg
        return cfg

    def reset(self):
        self._check(self._L.ertgpu_reset(self._h))

    def set_demod_variant(self, variant: int):
        self._check(self._L.ertgpu_set_demod_variant(self._h, variant))

    def _buffer(self, cap):
        # reused between calls: allocating and zeroing tens of MB per call would dominate small decodes
        buf = getattr(self, "_outbuf", None)
        if buf is None or len(buf) < cap:
            buf = np.empty(cap, dtype=CAND_DTYPE)
            self._outbuf = buf
        return buf[:cap]

    def _deliver(self, call, cap):
        while True:
            out = self._buffer(cap)
            n = C.c_size_t(0)
            rc = call(out.ctypes.data, cap, C.byref(n))
            if rc == ECAPACITY and n.value > cap and "internal" not in (
                    self._L.ertgpu_last_error(self._h) or b"").decode():
                cap = n.value
                call = lambda p, c, nn: self._L.ertgpu_fetch(self._h, p, c, nn)  # noqa: E731
                continue
            self._check(rc)
            return out[:n.value].copy()

    def decode(self, iq, flags: int = 0, cap: int = 4096) -> np.ndarray:
        """ertgpu_decode on a HOST buffer (numpy uint8 or an address/size pair)."""
        if isinstance(iq, tuple):
            addr, nbytes = iq
        else:
            iq = np.ascontiguousarray(iq, dtype=np.uint8)
            addr, nbytes = iq.ctypes.data, iq.size
        return self._deliver(
            lambda p, c, nn: self._L.ertgpu_decode(self._h, addr, nbytes, flags, p, c, nn), cap)

    def decode_device_async(self, d_ptr: int, nbytes: int, flags: int = 0, stream: int = 0):
        self._check(self._L.ertgpu_decode_device_async(self._h, d_ptr, nbytes, flags, stream))

    def fetch(self, cap: int = 4096) -> np.ndarray:
        return self._deliver(lambda p, c, nn: self._L.ertgpu_fetch(self._h, p, c, nn), cap)

    def last_counts(self):
        a, b = C.c_int64(0), C.c_int64(0)
        self._check(self._L.ertgpu_last_counts(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def last_launches(self) -> int:
        return int(self._L.ertgpu_last_launches(self._h))

    def set_stage_timing(self, enable: bool):
        self._check(self._L.ertgpu_set_stage_timing(self._h, 1 if enable else 0))

    def last_stage_ms(self):
        ms = (C.c_float * 4)()
        self._check(self._L.ertgpu_last_stage_ms(self._h, ms))
        return dict(zip(("demod", "search", "extract", "carry"), [float(x) for x in ms]))

    def stage_ms_mean(self):
        ms, n = (C.c_float * 4)(), C.c_int64(0)
        self._check(self._L.ertgpu_stage_ms_mean(self._h, ms, C.byref(n)))
        return dict(zip(("demod", "search", "extract", "carry"), [float(x) for x in ms])), n.value

    def demod_kernel_name(self) -> str:
        """The demod instantiation the last decode launched (first entry of ertgpu_last_kernels)."""
        return (self._L.ertgpu_last_kernels(self._h) or b"").decode().split(";")[0].strip()

    def last_kernels(self) -> str:
        return (self._L.ertgpu_last_kernels(self._h) or b"").decode()

    def tap(self, which: int, block: int) -> np.ndarray:
        n = C.c_size_t(0)
        self._check(self._L.ertgpu_tap(self._h, which, block, None, 0, C.byref(n)))
        buf = np.zeros(n.value, dtype=np.uint8)
        self._check(self._L.ertgpu_tap(self._h, which, block, buf.ctypes.data, buf.size, C.byref(n)))
        if which in (TAP_SIGNAL, TAP_CSUM):
            return buf.view(np.float32)
        return buf


def new_decoder(msgtypes, chip_length: int = 72, device: int = 0, max_blocks_per_call: int = 0,
                max_candidates: int = 0, input_rate: int = 0, input_format: int = FORMAT_CU8,
                input_scale: float = 0.0, capture_freq: int = 0, center_freq: int = 0,
                channel_gain: int | None = None, signal: bool = False) -> Handle:
    """NewDecoder + RegisterProtocol(NewParser(name, chip_length)) for each name + Allocate
    (reference main.go:64-86).  input_rate > 0: the IQ is sampled at that rate (ertgpu_set_input_rate);
    input_format / input_scale: its sample format and gain (ertgpu_set_input_format, not called for plain cu8);
    capture_freq > 0: the IQ was recorded centred there, and the channel at center_freq (0: the protocols'
    CenterFreq) is decoded (ertgpu_set_input_tuning, before the rate), at up to 256 times the decoder's rate
    (ertgpu_allow_input_decimation).  channel_gain k: the wide channel path with gain 2^k (ertgpu_set_channel_gain;
    tuned handles only).  signal: per-packet signal reports (ertgpu_enable_signal)."""
    if isinstance(msgtypes, str):
        msgtypes = [m.strip() for m in msgtypes.split(",") if m.strip()]
    h = Handle()
    for m in msgtypes:
        h.register(stock_protocol(m, chip_length))
    if capture_freq or center_freq:
        h.set_input_tuning(capture_freq, center_freq)
        h.allow_input_decimation()
    if input_rate:
        h.set_input_rate(input_rate)
    if input_format != FORMAT_CU8 or input_scale:
        h.set_input_format(input_format, input_scale)
    if channel_gain is not None:
        h.set_channel_gain(channel_gain)
    if signal:
        h.enable_signal()
    h.allocate(device, max_blocks_per_call, max_candidates)
    return h


def bind_host_thread(device: int):
    """ertgpu_bind_host_thread: pin the calling thread to the CPUs next to `device`.  Returns a
    small dict for the bench line (None fields when the topology is unknown: nothing changed)."""
    n, node = C.c_int32(0), C.c_int32(-1)
    rc = lib().ertgpu_bind_host_thread(device, C.byref(n), C.byref(node))
    return {"bound": rc == OK, "cpus": n.value if rc == OK else None, "numa_node": node.value if node.value >= 0 else None}


def plan_shards(total_blocks: int, nshards: int, block_size: int, packet_length: int):
    arr = (Shard * nshards)()
    rc = lib().ertgpu_plan_shards(total_blocks, nshards, block_size, packet_length, arr)
    if rc != OK:
        raise ErtGpuError(rc, "ertgpu_plan_shards: bad request")
    return [(s.first_block, s.last_block, s.first_fed_block) for s in arr]


def decode_sharded(handles, iq, flags: int = 0, cap: int = 1 << 16) -> np.ndarray:
    """ertgpu_decode_sharded: one host buffer over several handles (one host thread per handle)."""
    if isinstance(iq, tuple):
        addr, nbytes = iq
    else:
        iq = np.ascontiguousarray(iq, dtype=np.uint8)
        addr, nbytes = iq.ctypes.data, iq.size
    hs = (C.c_void_p * len(handles))(*[h._h for h in handles])
    while True:
        out = np.empty(cap, dtype=CAND_DTYPE)
        n = C.c_size_t(0)
        rc = lib().ertgpu_decode_sharded(hs, len(handles), addr, nbytes, flags, out.ctypes.data, cap, C.byref(n))
        if rc == ECAPACITY and n.value > cap:
            cap = n.value
            continue
        if rc != OK:
            msgs = [(lib().ertgpu_last_error(h._h) or b"").decode() for h in handles]
            raise ErtGpuError(rc, "; ".join(m for m in msgs if m) or "ertgpu_decode_sharded failed")
        return out[:n.value].copy()


def synth_fill(device: int, d_ptr: int, first_sample: int, nsamples: int, seed: int,
               packets: np.ndarray | None, stream: int = 0):
    """ertgpu_synth_fill: packets is a numpy array of SYNTH_DTYPE sorted by start_sample."""
    if packets is None or len(packets) == 0:
        ptr, n = None, 0
    else:
        packets = np.ascontiguousarray(packets)
        ptr, n = packets.ctypes.data, len(packets)
    rc = lib().ertgpu_synth_fill(device, d_ptr, first_sample, nsamples, seed, ptr, n, stream)
    if rc != OK:
        raise ErtGpuError(rc, "ertgpu_synth_fill failed")


SYNTH_DTYPE = np.dtype([("start_sample", "<i8"), ("n_chips", "<i4"), ("chip_length", "<i4"),
                        ("amp_i", "<i2"), ("amp_q", "<i2"), ("chips", "u1", (192,)),
                        ("pad", "<i4")])
assert SYNTH_DTYPE.itemsize == C.sizeof(SynthPacket) == 216


def _channel_call(handles, call):
    hs = (C.c_void_p * len(handles))(*[h._h if h is not None else None for h in handles])
    rc = call(hs, len(handles))
    if rc != OK:
        h0 = handles[0] if handles and handles[0] is not None else None
        msg = (lib().ertgpu_last_error(h0._h) or b"").decode() if h0 is not None and h0._h else ""
        raise ErtGpuError(rc, msg or "ertgpu_decode_channels failed")


def decode_channels(handles, iq, flags: int = 0, cap: int = 4096) -> list:
    """ertgpu_decode_channels: one HOST buffer (numpy uint8 or an address/size pair) through every handle, each tuned to
    another channel of the same capture, in one pass.  Returns each handle's candidates (ertgpu_fetch)."""
    if isinstance(iq, tuple):
        addr, nbytes = iq
    else:
        iq = np.ascontiguousarray(iq, dtype=np.uint8)
        addr, nbytes = iq.ctypes.data, iq.size
    _channel_call(handles, lambda hs, n: lib().ertgpu_decode_channels(hs, n, addr, nbytes, flags))
    return [h.fetch(cap) for h in handles]


def decode_channels_device_async(handles, d_ptr: int, nbytes: int, flags: int = 0, stream: int = 0):
    """ertgpu_decode_channels_device_async: the same for input in device memory; read each handle with fetch()."""
    _channel_call(handles, lambda hs, n: lib().ertgpu_decode_channels_device_async(hs, n, d_ptr, nbytes, flags, stream))
