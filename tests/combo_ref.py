"""Seeded handle configurations that join the decoder's features (input format, rate, tuning, decimation, the wide
channel path, protocols, chip length, signal reports, the spectrum, channel groups, max_blocks_per_call and the host,
pinned and device input paths), their captures, and the expected outputs of every call composed from the restatements
the suite already trusts: test_sigmf.convert, resample_ref, tune_ref, decimate_ref and wide_ref for the decoder's
bytes, the oracle for the candidates and r900 digits, signal_ref for the signal records and spectrum_ref for the rows.

A configuration is a plain dict, printable and JSON-serialisable, so that a failure names it and it can be rerun
alone: test_gpu_combos.run_config(config)."""
from __future__ import annotations

import functools

import numpy as np

import decimate_ref
import oracle
import resample_ref
import signal_ref
import spectrum_ref
import tune_ref
import wide_ref
from helpers import _feed, oracle_r900_digits, rule_violated, screen_expected
from rtlamr_b200 import capi, synth
from test_sigmf import NAME, SIGMF, convert, encode

DATA_RATE = 32768
CAPTURE = 915_000_000
STOCK = ("scm", "scm+", "idm", "netidm", "r900", "r900bcd")
FORMATS = [capi.FORMAT_CU8, capi.FORMAT_CS8, capi.FORMAT_CS16, capi.FORMAT_CF32] + list(SIGMF)
MODES = ("pass", "convert", "resample", "tuned", "decimate", "wide", "wide_dec")
TUNED = ("tuned", "decimate", "wide", "wide_dec")
RESAMPLING = ("resample", "tuned", "decimate")
WIDE = ("wide", "wide_dec")
SPECIALISED_CL = (32, 40, 48, 56, 64, 72, 78, 80, 88, 96)   # demod_fast_kernel instances
GENERIC_CL = (8, 16, 100)
PATHS = ("pageable", "pinned", "device")
MAX_IN = 4_000_000          # input samples of a capture at most
SMALL_MAX_BLOCKS = 8        # max_blocks_per_call at or below this is "small"
# the component of each format: numpy dtype of a stored value and the offset subtracted from it
LAYOUT = {capi.FORMAT_CU8: ("u1", 128), capi.FORMAT_CS8: ("i1", 0), capi.FORMAT_CS16: ("<i2", 0),
          capi.FORMAT_CF32: ("<f4", 0), **{f: (v[1], v[2]) for f, v in SIGMF.items()}}


# ---------------------------------------------------------------- plans
def rate_out(cfg) -> int:
    return DATA_RATE * cfg["cl"]


def protos(cfg):
    return [capi.stock_protocol(m, cfg["cl"]) for m in cfg["protocols"]]


def geometry(cfg) -> dict:
    return signal_ref.geometry(protos(cfg))


def plan(cfg, member: int = 0):
    """(decimator dict or None, resampler dict or None) of the member's handle, from the restatements' planners."""
    return _plan(cfg["mode"], cfg["rate_in"], rate_out(cfg), cfg["offsets"][member], cfg["allow_decimation"])


@functools.lru_cache(maxsize=None)
def _plan(mode, rate_in, ro, off, allow):
    if mode in ("pass", "convert"):
        return None, None
    if mode == "resample":
        return None, resample_ref.Resampler(rate_in, ro).info
    p = decimate_ref.plan(rate_in, ro, off) if allow else (None, tune_ref.plan(rate_in, ro, off))
    assert p is not None and p[1] is not None, (mode, rate_in, ro, off)
    return p


def out_end(info, x: int) -> int:
    """ertrs_out_end: outputs whose window lies inside the first x input samples."""
    a = x - info["T"] // 2
    return 0 if a <= 0 else -(-a * info["L"] // info["M"])


def outputs_after(cfg, x: int) -> int:
    """Decoder samples a handle of cfg has produced once x input samples are in."""
    dec, info = plan(cfg)
    if info is None:
        return x
    if dec is not None and dec["D"] > 1:
        a = x - dec["T1"] // 2
        x = -(-a // dec["D"]) if a > 0 else 0
    return out_end(info, x)


def blocks_after(cfg, x: int) -> int:
    return outputs_after(cfg, x) // geometry(cfg)["BS"]


def sample_bytes(cfg) -> int:
    return capi.FORMAT_BYTES[cfg["fmt"]]


def group_size(cfg) -> int:
    return len(cfg["offsets"])


def configure(cfg, member: int = 0) -> capi.Handle:
    """The member's handle, configured through the C ABI in the order capi.new_decoder uses, not allocated.  A wide
    handle with k "auto" starts at k = 0 (the caller measures the channel and sets k at the stream start)."""
    mode = cfg["mode"]
    h = capi.Handle()
    for p in protos(cfg):
        h.register(p)
    if mode in TUNED:
        h.set_input_tuning(CAPTURE, CAPTURE + cfg["offsets"][member])
        if cfg["allow_decimation"]:
            h.allow_input_decimation()
    if mode not in ("pass", "convert"):
        h.set_input_rate(cfg["rate_in"])
    if cfg["fmt"] != capi.FORMAT_CU8 or cfg["scale"]:
        h.set_input_format(cfg["fmt"], cfg["scale"])
    if mode in WIDE:
        k = cfg["ks"][member]
        h.set_channel_gain(0 if k == "auto" else k)
    if cfg["signal"]:
        h.enable_signal()
    if cfg["spectrum"] and member == cfg["spectrum_member"]:
        h.enable_spectrum(*cfg["spectrum"])
    return h


# ---------------------------------------------------------------- configurations
def _f32(x: float) -> float:
    return float(np.float32(x))


def _default_scale(fmt) -> float:
    if fmt in SIGMF:
        return SIGMF[fmt][3]
    return {capi.FORMAT_CS8: 1.0, capi.FORMAT_CS16: 2.0 ** -8, capi.FORMAT_CF32: 2.0 ** 7}[fmt]


def _offset_limit(rate_in: int, ro: int) -> int:
    """The largest |offset| the tuned or decimating plan takes: 10 |D| + 4 min(R_in, R_out) <= 5 R_in."""
    return (5 * rate_in - 4 * min(rate_in, ro)) // 10


def _draw_protocols(rng, want_r900: bool) -> list:
    n = int(rng.integers(1, 5))
    names = [STOCK[i] for i in rng.permutation(len(STOCK))[:n]]
    if want_r900 and not ({"r900", "r900bcd"} & set(names)):
        names[int(rng.integers(0, n))] = ("r900", "r900bcd")[int(rng.integers(0, 2))]
    return names


def _valid_protocols(names, cl) -> bool:
    return rule_violated([capi.stock_protocol(m, cl) for m in names]) is None


def _draw_rate(rng, mode, ro):
    if mode in ("pass", "convert"):
        return ro
    if mode == "resample":
        lo, hi = 0.25, 4.0
    elif mode in ("tuned", "wide"):
        lo, hi = 0.25, 10.0
    else:
        lo, hi = 10.0 + 1e-6, 256.0
    while True:
        r = int(round(ro * float(np.exp(rng.uniform(np.log(lo), np.log(hi))))))
        r = max(r, -(-ro // 4))
        if mode in ("decimate", "wide_dec"):
            # at most 128 MS/s: longer packets than that rendered at the input rate outgrow the capture's memory
            r = min(max(r, 10 * ro + 1), 256 * ro, max(128_000_000, 10 * ro + 1))
        elif mode == "resample":
            r = min(r, 4 * ro)
        else:
            r = min(r, 10 * ro)
        if r != ro:
            return r


def _capture_samples(cfg, rng) -> int:
    """Input samples of the capture: about 16 to 48 decoder blocks (and room for two spectrum rows), at most MAX_IN."""
    bs = geometry(cfg)["BS"]
    if cfg["mode"] in ("pass", "convert"):
        nb = int(rng.integers(16, 48))
        if cfg["spectrum"]:
            nb = max(nb, -(-2 * cfg["spectrum"][1] * (1 << cfg["spectrum"][0]) // bs) + 1)
        return min(nb, MAX_IN // bs) * bs
    ratio = cfg["rate_in"] / rate_out(cfg)
    n = int(int(rng.integers(16, 48)) * bs * ratio)
    if cfg["spectrum"]:
        n = max(n, 2 * cfg["spectrum"][1] * (1 << cfg["spectrum"][0]) + 4096)
    return int(min(max(n, 200_000), MAX_IN))


def _draw_spectrum(rng):
    log2_n = int(rng.integers(6, 15))
    least = spectrum_ref.least_frames(log2_n)
    return [log2_n, int(least + rng.integers(0, max(2, least // 2)))]


def _cuts(cfg, rng, max_calls=9) -> list:
    """[(end sample, path)] of the calls that feed the capture: one-sample calls, calls that complete no block, calls of
    exactly max_blocks blocks, random ones and the rest; device calls only where they complete at most max_blocks."""
    n, mb_eff = cfg["nsamples"], max_blocks_effective(cfg)
    native = cfg["mode"] in ("pass", "convert")
    unit = geometry(cfg)["BS"] if native else 1
    exact = cfg["max_blocks"] or int(rng.integers(1, 4))
    out, x = [], 0
    kinds = ["one", "noblock", "exact", "random", "random"] if not native else ["exact", "random", "random"]
    while x < n and len(out) < max_calls - 1:
        kind = kinds[int(rng.integers(0, len(kinds)))]
        b0 = blocks_after(cfg, x)
        if kind == "one":
            y = x + 1
        elif kind == "noblock":   # the last input sample at which no further block is complete
            hi = _first_at(cfg, x, b0 + 1, n) - 1
            if hi <= x:
                continue
            y = int(rng.integers(x + 1, hi + 1))
        elif kind == "exact":
            y = x + exact * unit if native else _first_at(cfg, x, b0 + exact, n)
        else:
            y = x + unit * int(rng.integers(1, max(2, n // (4 * unit))))
        y = min(y, n, _spectrum_end(cfg, x))
        out.append([y, _path(rng, cfg, x, y, mb_eff)])
        x = y
    while x < n:
        y = min(n, _spectrum_end(cfg, x))
        out.append([y, _path(rng, cfg, x, y, mb_eff)])
        x = y
    return out


def spectrum_row_cap(cfg) -> int:
    """The fewest spectrum rows the handle holds (include/ertgpu.h): those of a call of max_blocks_per_call decoder blocks
    times the input rate over the decoder's rate (rounded up) input samples, plus two."""
    log2_n, F = cfg["spectrum"]
    in_max = max_blocks_effective(cfg) * geometry(cfg)["BS"] * -(-cfg["rate_in"] // rate_out(cfg))
    return ((in_max >> log2_n) + 1) // F + 2


def _spectrum_end(cfg, x) -> int:
    """The last end of a call from x whose spectrum rows fit the handle (the rows before x are fetched)."""
    if not cfg["spectrum"]:
        return cfg["nsamples"]
    log2_n, F = cfg["spectrum"]
    return ((x >> log2_n) // F + spectrum_row_cap(cfg) + 1) * F * (1 << log2_n) - 1


def _first_at(cfg, x, target, n) -> int:
    """The least y in (x, n] with blocks_after(y) >= target, else n."""
    lo, hi = x + 1, n
    if blocks_after(cfg, hi) < target:
        return n
    while lo < hi:
        mid = (lo + hi) // 2
        if blocks_after(cfg, mid) >= target:
            hi = mid
        else:
            lo = mid + 1
    return lo


def _path(rng, cfg, x, y, mb_eff) -> str:
    p = PATHS[int(rng.integers(0, 3))]
    if p == "device" and blocks_after(cfg, y) - blocks_after(cfg, x) > mb_eff:
        p = PATHS[int(rng.integers(0, 2))]
    return p


def max_blocks_effective(cfg) -> int:
    """max_blocks_per_call as ertgpu_allocate takes it (0: 64 MiB of decoder bytes)."""
    return cfg["max_blocks"] or max(1, (64 << 20) // (2 * geometry(cfg)["BS"]))


def make_config(name, seed, *, mode, protocols, cl, fmt=None, scale=0.0, rate_in=None, offsets=None, ks=None,
                allow_decimation=True, signal=False, spectrum=None, spectrum_member=0, max_blocks=0, flags=0,
                before_start=False, cuts=None, nsamples=None) -> dict:
    """One configuration; what is not given is drawn from seed."""
    rng = np.random.default_rng(seed)
    ro = DATA_RATE * cl
    if fmt is None:
        fmt = capi.FORMAT_CU8 if mode == "pass" else FORMATS[int(rng.integers(1 if mode == "convert" else 0, 14))]
    rate_in = rate_in or _draw_rate(rng, mode, ro)
    if offsets is None:
        offsets = [0]
        if mode in TUNED:
            lim = _offset_limit(rate_in, ro)
            offsets = [int(rng.integers(-lim, lim + 1)) or 1]
    if mode in WIDE and ks is None:
        ks = [int(rng.integers(0, 15)) if rng.random() < 0.7 else "auto" for _ in offsets]
    cfg = {"name": name, "seed": int(seed), "mode": mode, "protocols": list(protocols), "cl": int(cl), "fmt": int(fmt),
           "scale": float(scale), "rate_in": int(rate_in), "offsets": [int(o) for o in offsets],
           "ks": ks if mode in WIDE else None, "allow_decimation": bool(allow_decimation or mode in ("decimate", "wide_dec")),
           "signal": bool(signal), "spectrum": spectrum, "spectrum_member": int(spectrum_member),
           "max_blocks": int(max_blocks), "flags": int(flags), "before_start": bool(before_start)}
    cfg["nsamples"] = int(nsamples) if nsamples else _capture_samples(cfg, rng)
    cfg["cuts"] = cuts if cuts is not None else _cuts(cfg, rng)
    return cfg


def _draw(i: int) -> dict:
    seed = 0xC0_0000 + i
    rng = np.random.default_rng(seed)
    mode = MODES[i % len(MODES)] if i < 2 * len(MODES) else MODES[int(rng.integers(0, len(MODES)))]
    while True:
        names = _draw_protocols(rng, want_r900=(i % 3 == 0) or rng.random() < 0.2)
        cl = int(rng.choice(SPECIALISED_CL)) if rng.random() < 0.7 else int(rng.choice(GENERIC_CL))
        if _valid_protocols(names, cl):
            break
    ro = DATA_RATE * cl
    fmt = capi.FORMAT_CU8 if mode == "pass" else FORMATS[int(rng.integers(1 if mode == "convert" else 0, 14))]
    scale = 0.0 if fmt == capi.FORMAT_CU8 or rng.random() < 0.5 else _f32(_default_scale(fmt) * 2.0 ** rng.uniform(-1.5, 1.5))
    rate_in = _draw_rate(rng, mode, ro)
    offsets = [0]
    if mode in TUNED:
        lim = _offset_limit(rate_in, ro)
        nch = int(rng.integers(1, 5))
        offsets = sorted({int(rng.integers(-lim, lim + 1)) or 1 for _ in range(nch)})
    signal = bool(i < len(MODES) or rng.random() < 0.6)
    spectrum = _draw_spectrum(rng) if len(MODES) <= i < 2 * len(MODES) or rng.random() < 0.5 else None
    return make_config(f"random{i}", seed, mode=mode, protocols=names, cl=cl, fmt=fmt, scale=scale, rate_in=rate_in,
                       offsets=offsets, allow_decimation=bool(rng.random() < 0.5), signal=signal, spectrum=spectrum,
                       spectrum_member=int(rng.integers(0, len(offsets))),
                       max_blocks=int(rng.choice([0, 0, 0, 1, 2, 3, 5, 8, 33])), flags=int(rng.random() < 0.3),
                       before_start=bool(rng.random() < 0.4))


def _tuned_rate_for_t(ro: int, t: int) -> int:
    """The least input rate above 4 R_out whose tuned plan has T taps."""
    lo = 4 * ro
    r = lo
    while tune_ref.plan(r, ro, 0)["T"] < t:
        r += ro // 200
    while tune_ref.plan(r - 1, ro, 0)["T"] >= t:
        r -= 1
    assert tune_ref.plan(r, ro, 0)["T"] == t, (ro, t)
    return r


def fixed_configs() -> list:
    """The edges that always run."""
    r72 = DATA_RATE * 72
    out = [
        make_config("untuned_4_to_1_up", 11, mode="resample", protocols=["scm", "r900"], cl=72, rate_in=r72 // 4,
                    signal=True),
        make_config("untuned_1_to_4_down", 12, mode="resample", protocols=["scm+", "idm"], cl=72, rate_in=4 * r72,
                    fmt=capi.FORMAT_CS16, spectrum=[10, 300]),
        make_config("untuned_coprime_2_4M", 13, mode="resample", protocols=["scm"], cl=72, rate_in=2_400_001,
                    signal=True, max_blocks=3),
        make_config("tuned_10_to_1_T218", 14, mode="tuned", protocols=["scm", "netidm"], cl=72, rate_in=10 * r72,
                    offsets=[-2_000_000, 1_500_000], signal=True, allow_decimation=False),
        make_config("tuned_interpolating_1_to_4", 19, mode="tuned", protocols=["scm", "r900bcd"], cl=72,
                    rate_in=r72 // 4, offsets=[-40_000, 50_000], signal=True, fmt=capi.FORMAT_CF32),
        make_config("decimating_D64", 20, mode="decimate", protocols=["scm"], cl=8, rate_in=256 * DATA_RATE * 8,
                    offsets=[-3_000_000, 20_000_000], signal=True, fmt=capi.FORMAT_CS8),
        make_config("decimating_D4", 21, mode="decimate", protocols=["scm", "scm+"], cl=72, rate_in=30_720_000,
                    offsets=[-2_400_000], signal=True, fmt=capi.FORMAT_CS16, max_blocks=2, spectrum=[12, 64]),
        make_config("decimating_D5", 22, mode="decimate", protocols=["scm", "r900"], cl=72, rate_in=40_000_000,
                    offsets=[-2_400_000, 6_000_000], signal=True, fmt=capi.FORMAT_CU16),
        make_config("decimating_cl8", 23, mode="decimate", protocols=["scm", "idm", "r900"], cl=8, rate_in=20_000_000,
                    offsets=[-2_400_000], signal=True, fmt=capi.FORMAT_CS8),
        make_config("wide_r900_cl32", 24, mode="wide", protocols=["r900"], cl=32, rate_in=8_000_000,
                    offsets=[1_200_000], ks=[4], signal=True, fmt=capi.FORMAT_CS16),
    ]
    for t, seed in ((96, 15), (98, 16), (160, 17), (162, 18)):
        out.append(make_config(f"tuned_T{t}", seed, mode="tuned", protocols=["scm"], cl=72,
                               rate_in=_tuned_rate_for_t(r72, t), offsets=[700_000], signal=True,
                               fmt=capi.FORMAT_CS16))
    return out


N_FIXED = 14     # len(fixed_configs()), known without the library (the GPU test's parameters)
N_RANDOM = 40


def configs() -> list:
    """The fixed list: the edges, then N_RANDOM seeded draws."""
    return fixed_configs() + [_draw(i) for i in range(N_RANDOM)]


# ---------------------------------------------------------------- captures
def _quantize(z, fmt) -> np.ndarray:
    """Raw capture bytes of the complex signal z (8-bit units) in format fmt."""
    if fmt in (capi.FORMAT_CS8, capi.FORMAT_CS16):
        return tune_ref.quantize(z, fmt)
    u8 = np.empty(2 * z.size, dtype=np.uint8)
    u8[0::2] = np.clip(np.round(z.real + 127.5), 0, 255)
    u8[1::2] = np.clip(np.round(z.imag + 127.5), 0, 255)
    return encode(u8, fmt)


def special_values(fmt) -> np.ndarray:
    """Stored component values of fmt that the conversions must get right: for floats NaN, +-Inf, +-0, subnormals,
    the rint ties of both paths (p = x g at k + 1/2, and p 2^7 at k + 1/2) and values past both clamps; for integers the
    extremes, zero and the values next to them."""
    dtype, off = LAYOUT[fmt]
    dt = np.dtype(dtype)
    if dt.kind == "f":
        fi = np.finfo(dt)
        g = _default_scale(fmt)
        ties = [(k + 0.5) / g for k in (-129, -128, -1, 0, 1, 126, 127)] + \
            [(k + 0.5) / (g * 128) for k in (-16384, -1, 0, 1, 16383)]
        vals = [0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, fi.max, -fi.max, fi.tiny, -fi.tiny,
                fi.smallest_subnormal, -fi.smallest_subnormal, 1e30, -1e30, 200.0 / g, -200.0 / g] + ties
        with np.errstate(over="ignore"):
            return np.array(vals, dtype=np.float64).astype(dt)
    lo, hi = -(1 << (8 * dt.itemsize - 1)), (1 << (8 * dt.itemsize - 1)) - 1
    return np.array([x + off for x in (0, 1, -1, 2, -2, lo, hi, lo + 1, hi - 1)]).astype(dt)


def special_raw(fmt, nsamples, seed, density=0.5) -> np.ndarray:
    """Raw bytes of nsamples samples of fmt: random stored values (every bit pattern of the integers; for the floats
    ordinary levels and every bit pattern) with a fraction `density` of the components replaced by special_values."""
    dtype, _ = LAYOUT[fmt]
    dt = np.dtype(dtype)
    rng = np.random.default_rng(seed)
    raw = rng.integers(0, 256, 2 * nsamples * dt.itemsize, dtype=np.uint8)
    v = raw.view(dt)
    if dt.kind == "f":
        half = v.size // 2
        v[:half] = (rng.standard_normal(half) * 0.5).astype(dt)
        v[:] = v[rng.permutation(v.size)]
    sp = special_values(fmt)
    at = rng.choice(v.size, int(v.size * density), replace=False)
    v[at] = sp[rng.integers(0, sp.size, at.size)]
    return raw


def _spacing(cfg, n) -> int:
    return max(1 << 14, n // 5)


def capture(cfg, seed=None) -> np.ndarray:
    """The capture of cfg: packets of its protocols at each member's channel, an scm interferer and noise, quantised to
    its format, then, in the last fifth (no packet starts there), a stretch of special and extreme components.  With
    before_start the stream begins a third of the way into the first packet."""
    seed = cfg["seed"] if seed is None else seed
    rate_in, n = cfg["rate_in"], cfg["nsamples"]
    rng = np.random.default_rng([seed, 2])
    lim = _offset_limit(rate_in, rate_out(cfg)) if cfg["mode"] in TUNED else min(rate_in, rate_out(cfg)) // 3
    lead = 0
    spacing = _spacing(cfg, n)
    names = ",".join(cfg["protocols"])
    if cfg["before_start"]:
        cl_guess = -(-rate_in // DATA_RATE)
        total = n + spacing // 2
        pk, _ = synth.make_packets(names, cl_guess, total - 2 * spacing, seed=seed + 1, spacing=spacing)
        row = pk[0]
        lead = int(row["start_sample"]) + int(row["n_chips"]) * rate_in // DATA_RATE // 3
    total = n + lead
    chans = [(names, off, seed + 1 + i, 0) for i, off in enumerate(cfg["offsets"])]
    chans.append(("scm", int(rng.integers(-lim, lim + 1)), seed + 99, spacing // 3))
    z, _ = decimate_ref.wideband(chans, rate_in, total, seed, spacing=spacing)
    raw = _quantize(z[lead:], cfg["fmt"])
    s = sample_bytes(cfg)
    m = min(n // 8, 1 << 16)
    raw[(n - m) * s:] = special_raw(cfg["fmt"], m, seed + 7, density=0.25)
    return raw


# ---------------------------------------------------------------- the composed restatement
def decoder_bytes(cfg, raw, member=0, k=None) -> np.ndarray:
    """The uint8 IQ the member's decoder reads for the whole capture (outputs whose windows are complete)."""
    fmt, scale, mode, ro = cfg["fmt"], cfg["scale"], cfg["mode"], rate_out(cfg)
    if mode in WIDE:
        return wide_ref.Wide(cfg["rate_in"], ro, cfg["offsets"][member], k).feed(
            wide_ref.wide_components(raw, fmt, scale))[0]
    u8 = convert(raw, fmt, scale)
    if mode in ("pass", "convert"):
        return u8
    if mode == "resample":
        return resample_ref.resample(u8, cfg["rate_in"], ro)
    if cfg["allow_decimation"]:
        return decimate_ref.decimate(u8, cfg["rate_in"], ro, cfg["offsets"][member])
    return tune_ref.tune(u8, cfg["rate_in"], ro, cfg["offsets"][member])


def auto_gain(cfg, raw, member=0) -> int:
    """k of ertgpu_measure_channel over the whole capture: the auto rule on the accumulators at k = 0."""
    _, acc = wide_ref.Wide(cfg["rate_in"], rate_out(cfg), cfg["offsets"][member], 0).feed(
        wide_ref.wide_components(raw, cfg["fmt"], cfg["scale"]))
    return wide_ref.level(acc)["k"]


def gain_of(cfg, raw, member=0):
    if cfg["mode"] not in WIDE:
        return None
    k = cfg["ks"][member]
    return auto_gain(cfg, raw, member) if k == "auto" else k


def _mask_last(data: bytes, pk: int) -> bytes:
    data = bytearray(data)
    if pk % 8:
        data[-1] &= 0xFF >> (8 - pk % 8)
    return bytes(data)


def candidate_key(block, pid, idx, data, check_mask, has_r900, digits) -> tuple:
    return (int(block), int(pid), int(idx), bytes(data), int(check_mask), bool(has_r900),
            bytes(digits) if has_r900 else b"")


def gpu_keys(rows, cfg) -> list:
    """candidate_key of every GPU record, in the records' order."""
    geo = geometry(cfg)
    nbytes = (geo["PK"] + 7) >> 3
    return [candidate_key(r["block"], r["preamble_id"], r["idx"], _mask_last(r["bytes"][:nbytes].tobytes(), geo["PK"]),
                          r["check_mask"], int(r["flags"]) & capi.CAND_HAS_R900, r["r900_digits"].tobytes())
            for r in rows]


def oracle_candidates(cfg, u8) -> list:
    """[(candidate_key, data)] of the oracle over the whole blocks of u8, check masks from the protocols' own screens
    of the oracle's bytes and r900 digits, filtered by DECODE_ONLY_VALID when set."""
    names, cl = cfg["protocols"], cfg["cl"]
    geo = geometry(cfg)
    search = oracle.SEARCH_GO if (2 * cl) % 8 == 0 else oracle.SEARCH_EXACT
    o = oracle.Oracle(names, cl, search)
    bs2 = o.cfg.block_size2
    whole = u8[: u8.size // bs2 * bs2]
    cands = _feed(o, whole)
    o.close()
    r900 = any(m in ("r900", "r900bcd") for m in names)
    digits = oracle_r900_digits(names, cl, whole) if r900 and cands else {}
    pre_ids = geo["preamble_id"]
    r900_pid = next((pre_ids[i] for i, m in enumerate(names) if m in ("r900", "r900bcd")), None)
    nbytes = (geo["PK"] + 7) >> 3
    out = []
    for c in cands:
        data = _mask_last(c.data[:nbytes], geo["PK"])
        has = c.preamble_id == r900_pid
        dig = digits[(c.block, c.idx, c.preamble_id)] if has else b""
        mask = 0
        for i, m in enumerate(names):
            if pre_ids[i] == c.preamble_id and screen_expected(m, c.data[:nbytes], list(dig) if has else None):
                mask |= 1 << i
        if cfg["flags"] & capi.DECODE_ONLY_VALID and not mask:
            continue
        out.append((candidate_key(c.block, c.preamble_id, c.idx, data, mask, has, dig), c.data[:nbytes]))
    return out


def signal_of(u8, key, data, ps) -> tuple:
    """signal_ref.record of the candidate, given the bytes of whole blocks from the first one its span reaches (the
    record depends on positions only relative to the candidate's block, and excludes those before the stream start)."""
    geo = signal_ref.geometry(ps)
    block, bs = key[0], geo["BS"]
    w0 = max(0, signal_ref.first_sample(geo, block, key[2])) // bs
    rec = signal_ref.record(u8[2 * w0 * bs:2 * (block + 1) * bs], block - w0, key[2], key[1], key[4], data, ps)
    return tuple(rec[f] for f in signal_ref.FIELDS)


def expected(cfg, raw) -> dict:
    """The whole-stream expectations of every member: {"bytes", "k", "cands" [(key, signal record or None)],
    "blocks" (completed after each call), "spectrum" (frame powers or None)}."""
    ps = protos(cfg)
    bs = geometry(cfg)["BS"]
    ends = [c[0] for c in cfg["cuts"]]
    blocks = [blocks_after(cfg, x) for x in ends]
    members = []
    for i in range(group_size(cfg)):
        k = gain_of(cfg, raw, i)
        u8 = decoder_bytes(cfg, raw, i, k)
        nb = u8.size // (2 * bs)
        assert nb == blocks[-1], (cfg["name"], i, nb, blocks[-1])
        cands = [(key, signal_of(u8, key, data, ps) if cfg["signal"] else None)
                 for key, data in oracle_candidates(cfg, u8[:2 * nb * bs])]
        members.append({"bytes": u8[:2 * nb * bs], "k": k, "cands": cands, "blocks": blocks})
    if cfg["spectrum"]:
        p = spectrum_ref.frame_powers(raw, cfg["fmt"], cfg["spectrum"][0], cfg["scale"])
        members[cfg["spectrum_member"]]["spectrum"] = p
    return {"members": members, "ends": ends}


def call_expectation(cfg, exp, member, c) -> dict:
    """What call c (0-based) of the cut plan returns for the member: a prefix of the whole-stream expectations."""
    m = exp["members"][member]
    bs = geometry(cfg)["BS"]
    b0 = m["blocks"][c - 1] if c else 0
    b1 = m["blocks"][c]
    cands = sorted(x for x in m["cands"] if b0 <= x[0][0] < b1)
    out = {"b0": b0, "b1": b1, "bytes": m["bytes"][2 * b0 * bs:2 * b1 * bs], "cands": cands}
    if "spectrum" in m:
        log2_n, F = cfg["spectrum"]
        x0 = exp["ends"][c - 1] if c else 0
        out["rows"] = spectrum_ref.rows_of_powers(m["spectrum"], F, frames=exp["ends"][c] >> log2_n,
                                                  first_row=(x0 >> log2_n) // F, partial=True)
    return out


# ---------------------------------------------------------------- comparisons
def assert_bytes(got, want, what=""):
    assert got.size == want.size, (what, got.size, want.size)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, (what, "first differing byte", int(bad[0]) if bad.size else None, bad.size)


def assert_candidates(got_keys, got_signal, want, what=""):
    """got_keys: candidate_key of each GPU record; got_signal: their signal records (tuples) or None; want: the sorted
    [(key, record)] of the restatement."""
    have = sorted(zip(got_keys, got_signal if got_signal is not None else [None] * len(got_keys)))
    hk, wk = [h[0] for h in have], [w[0] for w in want]
    assert hk == wk, (what, len(hk), len(wk), sorted(set(hk) ^ set(wk))[:4])
    for h, w in zip(have, want):
        assert h[1] == w[1], (what, h[0][:3], h[1], w[1])


# ---------------------------------------------------------------- coverage cells
FEATURES = ("signal", "spectrum", "r900", "group", "device", "small_max_blocks")


def all_cells() -> set:
    """Every cell test_every_combination_cell_was_seen needs."""
    cells = set()
    for mode in MODES:
        for f in FEATURES:
            if f == "group" and mode not in TUNED:
                continue
            cells.add(("mode", mode, f))
    for fmt in FORMATS:
        cells.add(("format", NAME[fmt], "resampling"))
        cells.add(("format", NAME[fmt], "wide"))
    return cells | {("label", lb) for lb in all_labels()}


def all_labels() -> set:
    """Every name of an input-stage kernel ertgpu_last_kernels can give."""
    out = {"resample_kernel", "resample_kernel<cu8>", "resample_kernel<mid16,tuned,wide>"}
    for fmt in FORMATS:
        f = NAME[fmt]
        if fmt != capi.FORMAT_CU8:
            out |= {f"convert_kernel<{f}>", f"resample_kernel<{f}>"}
        out |= {f"resample_kernel<{f},tuned>", f"decimate_kernel<{f}>", f"decimate_channels_kernel<{f}>",
                f"resample_kernel<{f},tuned,wide>", f"decimate_kernel<{f},wide>"}
    return out


def input_labels(last_kernels: str) -> set:
    return {k.strip() for k in last_kernels.split(";")
            if k.strip().startswith(("convert_kernel", "resample_kernel", "decimate_kernel", "decimate_channels_kernel"))}


def labels_of(cfg) -> set:
    """The input-stage kernels a handle (group) of cfg launches."""
    f, mode = NAME[cfg["fmt"]], cfg["mode"]
    if mode == "pass":
        return set()
    if mode == "convert":
        return {f"convert_kernel<{f}>"}
    if mode == "resample":
        return {"resample_kernel" if cfg["fmt"] == capi.FORMAT_CU8 else f"resample_kernel<{f}>"}
    dec, info = plan(cfg)
    d = dec["D"] if dec else 1
    if mode in WIDE:
        return {f"decimate_kernel<{f},wide>", "resample_kernel<mid16,tuned,wide>"} if d > 1 else \
            {f"resample_kernel<{f},tuned,wide>"}
    if d > 1:
        first = "decimate_channels_kernel" if group_size(cfg) > 1 else "decimate_kernel"
        return {f"{first}<{f}>", "resample_kernel<cu8>"}
    return {f"resample_kernel<{f},tuned>"}


def cells_of(cfg, used_paths=None) -> set:
    mode = cfg["mode"]
    paths = used_paths if used_paths is not None else {c[1] for c in cfg["cuts"]}
    have = {"signal": cfg["signal"], "spectrum": bool(cfg["spectrum"]),
            "r900": bool({"r900", "r900bcd"} & set(cfg["protocols"])), "group": group_size(cfg) > 1,
            "device": "device" in paths, "small_max_blocks": 0 < cfg["max_blocks"] <= SMALL_MAX_BLOCKS}
    cells = {("mode", mode, f) for f, on in have.items() if on}
    if mode in RESAMPLING:
        cells.add(("format", NAME[cfg["fmt"]], "resampling"))
    if mode in WIDE:
        cells.add(("format", NAME[cfg["fmt"]], "wide"))
    return cells | {("label", lb) for lb in labels_of(cfg)}


# ---------------------------------------------------------------- the every-format sweep on special values
SWEEP_RATES = {"convert": None, "resample": (2_400_000, 0), "tuned": (10_000_000, -2_400_000),
               "decimate": (30_720_000, -2_400_000), "wide": (10_000_000, 1_500_000), "wide_dec": (30_720_000, -2_400_000)}


def sweep_configs(fmt) -> list:
    """The handles the special-value sweep runs for one format: every input mode, one call each on a capture dense in
    special values; the decimating one as a group of two (decimate_channels_kernel) and alone; the spectrum on the
    untuned resampler.  Each is a configuration whose cut plan is one pageable call."""
    out = []
    for mode, rates in SWEEP_RATES.items():
        if mode == "convert" and fmt == capi.FORMAT_CU8:
            mode, rates = "pass", None
        rate_in, off = rates if rates else (DATA_RATE * 72, 0)
        groups = [[off, off + 5_400_000], [off]] if mode == "decimate" else [[off]]
        for offs in groups:
            n = {"wide_dec": 1_200_000, "decimate": 1_200_000}.get(mode, 600_000)
            if mode in ("pass", "convert"):
                n = 40 * 4096
            cfg = make_config(f"sweep_{NAME[fmt]}_{mode}_{len(offs)}", 500 + fmt, mode=mode, protocols=["scm"], cl=72,
                              fmt=fmt, rate_in=rate_in, offsets=offs, ks=[3 if mode == "wide" else 5] * len(offs),
                              spectrum=[10, 256] if mode == "resample" else None, nsamples=n, cuts=[[n, "pageable"]])
            out.append(cfg)
    return out


def planned_cells() -> set:
    """The cells configs() and the sweep reach, as the CPU sees them."""
    cells = set()
    for cfg in configs():
        cells |= cells_of(cfg)
    for fmt in FORMATS:
        for cfg in sweep_configs(fmt):
            cells |= {c for c in cells_of(cfg) if c[0] != "mode"}
    return cells
