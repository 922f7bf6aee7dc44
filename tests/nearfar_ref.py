"""The near-far capture of the wide channel path's tests, generated from a seed: cs16 at 10 MS/s centred at 915 MHz, a
strong carrier 3.5 MHz below the meter channel near full scale, scm packets in the channel PACKET_DB below it, over
Gaussian noise at a 12-bit radio's floor (one 12-bit LSB, 16 cs16 units, rms per component).

It also restates both input paths on the CPU as the file receiver runs them with automatic gains: the narrow tuned path
at -samplescale=auto, and the wide path at -samplescale=auto and -channelgain=auto, both measured on the stream's first
min(stream, 2^22) samples."""
from __future__ import annotations

import numpy as np

from rtlamr_b200 import capi

import format_ref
import tune_ref
import wide_ref

RATE = 10_000_000
CAPTURE = 915_000_000
OFFSET = 1_500_000          # the meter channel, from the capture's centre
STRONG_OFFSET = -2_000_000  # the strong carrier, 3.5 MHz below the channel
STRONG = 90.0               # its amplitude in 8-bit units (23 040 in cs16)
PACKET_DB = -46.0           # the packets' amplitude relative to the carrier
FLOOR = 1 / 16              # noise sigma in 8-bit units: 16 cs16 units
NSAMPLES = 4_200_000
R72 = 32768 * 72
WINDOW = 1 << 22


def capture(seed: int = 3, packet_db: float = PACKET_DB):
    """(raw cs16 bytes, the scm truth of the channel)."""
    amp = STRONG * 10 ** (packet_db / 20) / 56.0   # synth's packets have |amp| of about 56
    z, truths = tune_ref.wideband([("scm", OFFSET, seed, 0)], RATE, NSAMPLES, seed, noise=FLOOR, full_scale=amp)
    z = z + STRONG * np.exp(2j * np.pi * STRONG_OFFSET * (np.arange(NSAMPLES) % RATE) / RATE)
    return tune_ref.quantize(z, capi.FORMAT_CS16), truths[0]


def auto_scale(raw) -> float:
    """-samplescale=auto on cs16: 2^k for the largest k at which at most N >> 16 components have |x| 2^k >= 128."""
    x = np.abs(raw[: 4 * WINDOW].view("<i2").astype(np.int64))
    allow = x.size >> 16
    for k in range(120, -121, -1):
        if np.count_nonzero(x * 2.0 ** k >= 128) <= allow:
            return 2.0 ** k
    return 2.0 ** -120


def narrow(raw) -> np.ndarray:
    """The narrow tuned path's bytes at -samplescale=auto."""
    return tune_ref.tune(format_ref.convert(raw, capi.FORMAT_CS16, auto_scale(raw)), RATE, R72, OFFSET)


def wide(raw):
    """The wide path's bytes at -samplescale=auto and -channelgain=auto, and the k it picked."""
    g = auto_scale(raw)
    _, acc = wide_ref.wide(raw[: 4 * WINDOW], capi.FORMAT_CS16, RATE, R72, OFFSET, 0, g)
    k = wide_ref.level(acc)["k"]
    out, _ = wide_ref.wide(raw, capi.FORMAT_CS16, RATE, R72, OFFSET, k, g)
    return out, k


def found(meter_ids, truth) -> int:
    """How many of the truth's packets were decoded, by meter ID (each packet of the capture has its own)."""
    got = set(int(m) for m in meter_ids)
    return sum(1 for t in truth if int(t.meter_id) in got)
