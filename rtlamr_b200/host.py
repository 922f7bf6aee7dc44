"""ctypes binding of libertgpu_host.so: the C++ mirror of rtlamr's protocol.Decoder + parsers
(rtlamr_b200/host/protocol.hpp) sitting above the C ABI.  Test/bench plumbing only."""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libertgpu_host.so")


class _Msg(C.Structure):
    _fields_ = [("block", C.c_int64), ("idx", C.c_int32), ("meter_id", C.c_uint32), ("meter_type", C.c_uint32),
                ("nchecksum", C.c_int32), ("checksum", C.c_uint8 * 8), ("msgtype", C.c_char * 12),
                ("text", C.c_char * 1400), ("record", C.c_char * 1400), ("signal", C.c_int32), ("reserved", C.c_int32),
                ("channel", C.c_int64), ("freq", C.c_int64), ("level", C.c_double), ("noise", C.c_double),
                ("snr", C.c_double)]


@dataclass(frozen=True)
class HostMessage:
    block: int
    idx: int
    msgtype: str
    meter_id: int
    meter_type: int
    checksum: bytes
    text: str
    record: tuple
    # Receiver(signal=True): {"channel", "freq", "level", "noise", "snr"} (freq and the dB values None for a packet that
    # starts before the stream); None without reports
    signal: dict | None = None


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FileNotFoundError(f"{LIB_PATH} missing: run __graft_entry__.build()")
        L = C.CDLL(LIB_PATH)
        L.erthost_new.restype = C.c_void_p
        L.erthost_new.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_longlong, C.c_longlong, C.c_longlong, C.c_int, C.c_float,
                                  C.c_longlong, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_int, C.c_longlong, C.c_char_p,
                                  C.c_int]
        L.erthost_gpu_handle.restype = C.c_void_p
        L.erthost_gpu_handle.argtypes = [C.c_void_p]
        L.erthost_channel_gain.argtypes = [C.c_void_p]
        L.erthost_level.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_float), C.POINTER(C.c_longlong),
                                    C.POINTER(C.c_longlong)]
        L.erthost_wav_probe.argtypes = [C.c_char_p, C.POINTER(C.c_int), C.POINTER(C.c_longlong), C.POINTER(C.c_longlong),
                                        C.POINTER(C.c_longlong), C.c_char_p, C.c_int]
        ll, pll = C.c_longlong, C.POINTER(C.c_longlong)
        L.erthost_sigmf_probe.argtypes = [C.c_char_p, C.POINTER(C.c_int), pll, pll, C.c_char_p, C.c_int, pll, pll, pll, pll,
                                          C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int), C.c_char_p, C.c_int]
        L.erthost_sigmf_block_time.argtypes = [C.c_char_p, ll, ll, ll, pll, C.c_char_p, C.c_int]
        L.erthost_free.argtypes = [C.c_void_p]
        L.erthost_error.restype = C.c_char_p
        L.erthost_error.argtypes = [C.c_void_p]
        L.erthost_config.argtypes = [C.c_void_p, C.POINTER(C.c_int32)]
        L.erthost_reset.argtypes = [C.c_void_p]
        L.erthost_decode.restype = C.c_longlong
        L.erthost_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(_Msg), C.c_longlong]
        L.erthost_log.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
        L.erthost_new_parse_only.restype = C.c_void_p
        L.erthost_new_parse_only.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int]
        L.erthost_parse.restype = C.c_longlong
        L.erthost_parse.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.POINTER(_Msg), C.c_longlong]
        L.erthost_parse_dedup_channels.restype = C.c_longlong
        L.erthost_parse_dedup_channels.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_longlong), C.c_int, C.c_int,
                                                   C.POINTER(_Msg), C.POINTER(C.c_int), C.c_longlong, C.POINTER(C.c_longlong)]
        L.erthost_parse_filtered.restype = C.c_longlong
        L.erthost_parse_filtered.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.c_char_p, C.c_char_p, C.c_int, C.c_int,
                                             C.POINTER(_Msg), C.c_longlong, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]
        L.erthost_encode.restype = C.c_longlong
        L.erthost_encode.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_longlong, C.c_int, C.c_longlong, C.c_int,
                                     C.c_int, C.c_char_p, C.c_longlong]
        L.erthost_encode_signal.restype = C.c_longlong
        L.erthost_encode_signal.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_longlong, C.c_longlong,
                                            C.c_int, C.c_longlong, C.c_int, C.c_char_p, C.c_longlong]
        _lib = L
    return _lib


def _signal(m):
    if not m.signal:
        return None
    full = m.signal == 2
    return {"channel": m.channel, "freq": m.freq if full else None, "level": m.level if full else None,
            "noise": m.noise if full else None, "snr": m.snr if full else None}


def _messages(out, n):
    return [HostMessage(m.block, m.idx, m.msgtype.decode(), m.meter_id, m.meter_type, bytes(m.checksum[:m.nchecksum]),
                        m.text.decode(), tuple(m.record.decode().split(",")), _signal(m)) for m in out[:n]]


FORMATS = {"plain": 0, "csv": 1, "json": 2, "xml": 3}


class Parsers:
    """NewDecoder + RegisterProtocol(NewParser(..)) WITHOUT Allocate: no device is touched.  parse() is the second
    half of Decode (decode.go:177-187 and every parser's Parse) on candidate records from any source."""

    def __init__(self, msgtypes: str, chip_length: int = 72):
        self._L = lib()
        err = C.create_string_buffer(512)
        self._h = self._L.erthost_new_parse_only(msgtypes.encode(), chip_length, err, 512)
        if not self._h:
            raise RuntimeError(err.value.decode())

    def close(self):
        if self._h:
            self._L.erthost_free(self._h)
            self._h = None

    def _check(self, n):
        """n, the count an erthost_* call returned; a negative one raises with the handle's message."""
        if n < 0:
            raise RuntimeError(self._L.erthost_error(self._h).decode())
        return n

    def parse(self, cands: np.ndarray, cap: int = 4096) -> list[HostMessage]:
        """cands: structured array with capi.CAND_DTYPE, sorted by (block, preamble_id, idx)."""
        cands = np.ascontiguousarray(cands)
        assert cands.dtype.itemsize == 160
        out = (_Msg * cap)()
        n = self._check(self._L.erthost_parse(self._h, cands.ctypes.data, len(cands), out, cap))
        if n > cap:
            raise OverflowError(f"{n} messages, cap {cap}")
        return _messages(out, n)

    def parse_dedup(self, cands: np.ndarray, block_dedup: bool = True, cap: int = 4096):
        """parse() followed by the receive loop's cross-block dedup (main.go:244-260,292): (messages, duplicates
        dropped)."""
        msgs, dup, _ = self.parse_filtered(cands, block_dedup=block_dedup, cap=cap)
        return msgs, dup

    def parse_dedup_channels(self, per_channel, block_dedup: bool = True, cap: int = 4096):
        """parse() of each channel's candidates (a list of arrays, one per channel of one capture), then the receiver's
        cross-channel dedup in its print order (ascending block, then channel): ([(channel, message)], duplicates
        dropped)."""
        cands = np.ascontiguousarray(np.concatenate(per_channel)) if per_channel else np.zeros(0, np.uint8)
        counts = (C.c_longlong * len(per_channel))(*[len(c) for c in per_channel])
        out, chan = (_Msg * cap)(), (C.c_int * cap)()
        dup = C.c_longlong(0)
        n = self._check(self._L.erthost_parse_dedup_channels(self._h, cands.ctypes.data, counts, len(per_channel),
                                                             1 if block_dedup else 0, out, chan, cap, C.byref(dup)))
        n = min(n, cap)
        return list(zip(chan[:n], _messages(out, n))), int(dup.value)

    def parse_filtered(self, cands, filterid: str = "", filtertype: str = "", unique: bool = False,
                       block_dedup: bool = True, cap: int = 1 << 16):
        """erthost_parse_filtered: parsers, then the receive loop's filter chain (-filterid, -filtertype, -unique in the
        order flag.Visit adds them, main.go:97-113) and the cross-block dedup (main.go:236-260).  Returns (messages,
        dropped by the dedup, rejected by the filters)."""
        cands = np.ascontiguousarray(cands)
        out = (_Msg * cap)()
        dup, flt = C.c_longlong(0), C.c_longlong(0)
        n = self._check(self._L.erthost_parse_filtered(self._h, cands.ctypes.data, len(cands), filterid.encode(),
                                                       filtertype.encode(), 1 if unique else 0, 1 if block_dedup else 0,
                                                       out, cap, C.byref(dup), C.byref(flt)))
        return _messages(out, min(n, cap)), int(dup.value), int(flt.value)

    def encode(self, cands, fmt: str = "plain", unix_seconds: int = 0, nanos: int = 0, offset: int = 0, length: int = 0,
               sample_file_is_devnull: bool = True) -> str:
        """erthost_encode: every parsed message through the plain, csv, json or xml encoder (flags.go:140-170) as one
        string of lines."""
        cands = np.ascontiguousarray(cands)
        cap = 1 << 22
        buf = C.create_string_buffer(cap)
        n = self._L.erthost_encode(self._h, cands.ctypes.data, len(cands), FORMATS[fmt], unix_seconds, nanos, offset,
                                   length, 1 if sample_file_is_devnull else 0, buf, cap)
        if n < 0 or n >= cap:
            raise RuntimeError("erthost_encode failed" if n < 0 else "encode buffer too small")
        return buf.value.decode()

    def encode_signal(self, cands, sigs, channel_hz: int, rate_out: int, fmt: str = "plain", unix_seconds: int = 0,
                      nanos: int = 0) -> str:
        """erthost_encode_signal: every parsed message with the signal report of its candidate (sigs:
        capi.SIGNAL_DTYPE, one per candidate) through the encoders; "plain" is ertgpu_decode_file's plain line."""
        cands, sigs = np.ascontiguousarray(cands), np.ascontiguousarray(sigs)
        assert len(sigs) == len(cands)
        cap = 1 << 22
        buf = C.create_string_buffer(cap)
        n = self._check(self._L.erthost_encode_signal(self._h, cands.ctypes.data, sigs.ctypes.data, len(cands), channel_hz,
                                                      rate_out, FORMATS[fmt], unix_seconds, nanos, buf, cap))
        if n >= cap:
            raise RuntimeError("encode buffer too small")
        return buf.value.decode()


def wav_probe(path) -> dict:
    """erthost_wav_probe: the header of a baseband WAV file (format = capi.FORMAT_*, rate in Hz, data offset and size
    in bytes, size -1 = to the end of the file).  Raises ValueError naming the field that cannot be decoded."""
    L = lib()
    fmt, rate, off, size = C.c_int(0), C.c_longlong(0), C.c_longlong(0), C.c_longlong(0)
    err = C.create_string_buffer(512)
    if L.erthost_wav_probe(os.fsencode(path), C.byref(fmt), C.byref(rate), C.byref(off), C.byref(size), err, 512) != 0:
        raise ValueError(err.value.decode())
    return {"format": fmt.value, "rate": rate.value, "data_offset": off.value, "data_size": size.value}


def sigmf_probe(path) -> dict:
    """erthost_sigmf_probe: the metadata of a SigMF recording (NAME.sigmf-meta, NAME.sigmf-data or NAME): format =
    capi.FORMAT_*, rate in Hz, frequency in Hz or None, the data file's path and its number of samples, and the capture
    segments, each {"start", "header_bytes", "datetime_ns" (None: not dated)}.  Raises ValueError naming the field."""
    L = lib()
    fmt, rate, freq, samples, nseg = C.c_int(0), C.c_longlong(0), C.c_longlong(0), C.c_longlong(0), C.c_int(0)
    data, err = C.create_string_buffer(4096), C.create_string_buffer(512)
    cap = 1024
    starts, hdr, dt = (C.c_longlong * cap)(), (C.c_longlong * cap)(), (C.c_longlong * cap)()
    dated = (C.c_int * cap)()
    if L.erthost_sigmf_probe(os.fsencode(path), C.byref(fmt), C.byref(rate), C.byref(freq), data, 4096, C.byref(samples),
                             starts, hdr, dt, dated, cap, C.byref(nseg), err, 512) != 0:
        raise ValueError(err.value.decode())
    segs = [{"start": starts[k], "header_bytes": hdr[k], "datetime_ns": dt[k] if dated[k] else None}
            for k in range(min(nseg.value, cap))]
    return {"format": fmt.value, "rate": rate.value, "frequency": freq.value or None, "data_path": os.fsdecode(data.value),
            "samples": samples.value, "segments": segs}


def sigmf_block_time(path, block: int, block_size: int, rate_out: int) -> int:
    """erthost_sigmf_block_time: the time in ns since the Unix epoch at which a live receiver would have finished decoder
    block `block` of the recording (block_size samples at rate_out Hz).  Raises ValueError when no segment is dated."""
    L = lib()
    ns, err = C.c_longlong(0), C.create_string_buffer(512)
    if L.erthost_sigmf_block_time(os.fsencode(path), block, block_size, rate_out, C.byref(ns), err, 512) != 0:
        raise ValueError(err.value.decode())
    return ns.value


class Receiver:
    """NewDecoder + RegisterProtocol(NewParser(..)) + Allocate, then Decode (main.go:59-86,235)."""

    CFG = ("DataRate", "BlockSize", "BlockSize2", "ChipLength", "SymbolLength", "SampleRate", "PreambleSymbols",
           "PacketSymbols", "PreambleLength", "PacketLength", "BufferLength", "CenterFreq")

    def __init__(self, msgtypes: str, chip_length: int = 72, device: int = 0, max_blocks: int = 0, max_cands: int = 0,
                 input_rate: int = 0, input_format: int = 0, input_scale: float | str = 0.0, capture_freq: int = 0,
                 center_freq: int = 0, channel_gain: int | str | None = None, signal: bool = False,
                 spectrum: tuple | None = None):
        """The input arguments are protocol::Decoder::SetInput's.  input_rate > 0: the IQ given to decode() is sampled at
        that rate; any rate other than DataRate * ChipLength is resampled on the GPU and decode() then takes any whole
        number of IQ samples.  input_format / input_scale: the IQ's sample format (capi.FORMAT_*) and gain.
        capture_freq > 0: the IQ was recorded centred there; the channel at center_freq (0: the protocols' CenterFreq) is
        decoded.  input_scale="auto": the gain of each stream (until reset()) is measured from the first
        min(len, 2^22) samples of its first decode() call (ertgpu_measure_input) and stays fixed for the stream;
        input_level() tells which.  channel_gain=k: the wide channel path of a tuned input with gain 2^k
        (ertgpu_set_channel_gain); "auto": k of each stream is measured from the same samples after the input gain
        (ertgpu_measure_channel), and channel_gain() tells which.  signal: every message carries its signal report
        (HostMessage.signal; protocol::Decoder::EnableSignal).  spectrum=(log2_n, frames_per_row): the input's spectrum
        (protocol::Decoder::EnableSpectrum), whose rows each decode() collects and spectrum() returns."""
        self._L = lib()
        err = C.create_string_buffer(512)
        auto = isinstance(input_scale, str)
        if auto and input_scale != "auto":
            raise ValueError(f"input_scale {input_scale!r}: a gain or 'auto'")
        if isinstance(channel_gain, str) and channel_gain != "auto":
            raise ValueError(f"channel_gain {channel_gain!r}: k or 'auto'")
        cg = -1 if channel_gain is None else -2 if channel_gain == "auto" else int(channel_gain)
        self._h = self._L.erthost_new(msgtypes.encode(), chip_length, device, max_blocks, max_cands, input_rate, input_format,
                                      0.0 if auto else input_scale, capture_freq, center_freq, 1 if auto else 0, cg,
                                      1 if signal else 0, spectrum[0] if spectrum else 0, spectrum[1] if spectrum else 0,
                                      err, 512)
        if not self._h:
            raise RuntimeError(err.value.decode())
        v = (C.c_int32 * 12)()
        self._L.erthost_config(self._h, v)
        self.cfg = dict(zip(self.CFG, [int(x) for x in v]))
        self.cfg["CenterFreq"] &= 0xFFFFFFFF
        self._spectrum = spectrum
        self._rows = []

    def close(self):
        if self._h:
            self._L.erthost_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        self._rows = []
        if self._L.erthost_reset(self._h) != 0:
            raise RuntimeError(self._L.erthost_error(self._h).decode())

    def input_level(self) -> dict | None:
        """input_scale="auto": the level measured at the start of the current stream ({"exponent": k, "scale": 2^k,
        "components", "bins"}), or None before its first decode()."""
        k, g, n = C.c_int(0), C.c_float(0), C.c_longlong(0)
        bins = (C.c_longlong * 256)()
        if self._L.erthost_level(self._h, C.byref(k), C.byref(g), C.byref(n), bins) != 0:
            return None
        return {"exponent": k.value, "scale": g.value, "components": n.value, "bins": np.array(bins[:], dtype=np.int64)}

    def channel_gain(self) -> int | None:
        """k of the wide channel path (for "auto": once the first decode() measured it), or None without it."""
        k = self._L.erthost_channel_gain(self._h)
        return None if k < 0 else k

    def log(self) -> str:
        b = C.create_string_buffer(2048)
        self._L.erthost_log(self._h, b, 2048)
        return b.value.decode()

    def decode(self, iq, cap: int = 4096) -> list[HostMessage]:
        iq = np.ascontiguousarray(iq, dtype=np.uint8)
        out = (_Msg * cap)()
        n = self._L.erthost_decode(self._h, iq.ctypes.data, iq.size, out, cap)
        if n == -2:
            raise ValueError(self._L.erthost_error(self._h).decode())
        if n < 0:
            raise RuntimeError(self._L.erthost_error(self._h).decode())
        if n > cap:
            raise OverflowError(f"{n} messages, cap {cap}")
        if self._spectrum:
            self._rows.append(self._fetch_spectrum(False))
        return _messages(out, n)

    def _fetch_spectrum(self, partial: bool):
        from rtlamr_b200 import capi
        return capi.fetch_spectrum(C.c_void_p(self._L.erthost_gpu_handle(self._h)), 1 << self._spectrum[0], partial)

    def spectrum(self, partial: bool = False):
        """(rows, mean, peak) of the spectrum rows the decode() calls of the current stream completed (capi.Handle's
        fetch_spectrum layout), and with partial the open row last."""
        from rtlamr_b200 import capi
        parts = self._rows + ([self._fetch_spectrum(True)] if partial else [])
        n = 1 << self._spectrum[0]
        empty = (np.zeros(0, capi.SPECTRUM_ROW_DTYPE), np.zeros((0, n), np.float32), np.zeros((0, n), np.float32))
        return tuple(np.concatenate([e] + [p[k] for p in parts]) for k, e in enumerate(empty))
