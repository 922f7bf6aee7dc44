"""GPU tests (-m gpu) of the decoder's features together: seeded handle configurations (tests/combo_ref.py) fed call by
call through pageable, pinned and device input, every call against the composed CPU restatement (the candidates and r900
digits against the oracle, ERTGPU_TAP_RESAMPLED of every block the call completed, the signal records and the spectrum
rows); then the calls' concatenation against one call on a fresh handle, each group member against a lone handle, and a
reset handle on a second capture.  Also every wide path and the spectrum of all 14 formats on captures dense in special
values, groups of ERTGPU_MAX_CHANNELS handles, and, last, the coverage of every combination cell."""
import ctypes as C
import functools
import json
import time

import numpy as np
import pytest

import combo_ref as cr
import signal_ref
import spectrum_ref
from rtlamr_b200 import capi

pytestmark = pytest.mark.gpu

SEEN = set()
TIMES = {}
N_CONFIGS = cr.N_FIXED + cr.N_RANDOM


@functools.lru_cache(maxsize=None)
def _configs():
    return cr.configs()


class Pinned:
    """One page-locked host buffer (ertgpu_host_alloc) that calls on the pinned path are copied into."""

    def __init__(self, nbytes):
        self.ptr = C.c_void_p()
        self.size = max(16, nbytes)
        assert capi.lib().ertgpu_host_alloc(C.byref(self.ptr), self.size) == capi.OK

    def load(self, part):
        assert part.size <= self.size
        C.memmove(self.ptr.value, part.ctypes.data, part.size)
        return self.ptr.value, part.size

    def close(self):
        if self.ptr.value:
            capi.lib().ertgpu_host_free(self.ptr)
            self.ptr = C.c_void_p()


def feed(hs, part, path, flags, pinned=None):
    """One decode call of every handle of hs (a group when there are several) on part; each handle's candidates."""
    part = np.ascontiguousarray(part, dtype=np.uint8)
    if path == "device":
        import torch
        d = torch.from_numpy(part.copy()).cuda()
        st = torch.cuda.current_stream().cuda_stream
        if len(hs) > 1:
            capi.decode_channels_device_async(hs, d.data_ptr(), d.numel(), flags, st)
        else:
            hs[0].decode_device_async(d.data_ptr(), d.numel(), flags, st)
        out = [h.fetch(cap=1 << 16) for h in hs]
        del d
        return out
    buf = pinned.load(part) if path == "pinned" else part
    if len(hs) > 1:
        return capi.decode_channels(hs, buf, flags, cap=1 << 16)
    return [hs[0].decode(buf, flags, cap=1 << 16)]


def signal_tuples(h, cfg):
    if not cfg["signal"]:
        return None
    return [tuple(int(r[f]) for f in signal_ref.FIELDS) for r in h.fetch_signal()]


def tapped(h, b0, b1):
    """ERTGPU_TAP_RESAMPLED of blocks [first, b1) of the last call, walking down from b1 - 1 to b0 while the tap
    reaches (the last chunk of a call that took several): (first, bytes).  Block b1 itself must be out of reach."""
    with pytest.raises(capi.ErtGpuError):
        h.tap(capi.TAP_RESAMPLED, b1)
    got = []
    for b in range(b1 - 1, b0 - 1, -1):
        try:
            got.append(h.tap(capi.TAP_RESAMPLED, b))
        except capi.ErtGpuError:
            break
    return b1 - len(got), np.concatenate(got[::-1]) if got else np.zeros(0, np.uint8)


def check_plan(h, cfg, i, what):
    dec, info = cr.plan(cfg, i)
    if info is None:
        with pytest.raises(capi.ErtGpuError):
            h.resampler()
    else:
        assert h.resampler()[0] == info, what
    if dec is not None:
        assert h.decimator()[0] == dec, what


def allocate(cfg, i, raw, max_blocks, what):
    """The member's handle, allocated, with the measured k of an "auto" wide handle set."""
    h = cr.configure(cfg, i)
    h.allocate(0, max_blocks, 0)
    check_plan(h, cfg, i, what)
    if cfg["mode"] in cr.WIDE and cfg["ks"][i] == "auto":
        k = h.measure_channel(raw)["k"]
        assert k == cr.auto_gain(cfg, raw, i), what
        h.set_channel_gain(k)
    return h


def record_bytes(rows, sig):
    """The records of a decode as sortable bytes (candidate, signal record)."""
    return sorted((r.tobytes(), s) for r, s in zip(rows, sig if sig is not None else [None] * len(rows)))


def run_config(cfg):
    """Every check of one configuration; failures name the configuration (rerun it alone with run_config)."""
    t0 = time.perf_counter()
    where = f"config {json.dumps(cfg)}"
    raw = cr.capture(cfg)
    exp = cr.expected(cfg, raw)
    n, s, bs = cr.group_size(cfg), cr.sample_bytes(cfg), cr.geometry(cfg)["BS"]
    native = cfg["mode"] == "pass"
    hs = [allocate(cfg, i, raw, cfg["max_blocks"], where) for i in range(n)]
    pinned = Pinned(max(y - x for x, y in zip([0] + exp["ends"], exp["ends"])) * s)
    labels, paths = set(), set()
    calls = [[] for _ in range(n)]
    x = 0
    try:
        for c, (y, path) in enumerate(cfg["cuts"]):
            outs = feed(hs, raw[x * s:y * s], path, cfg["flags"], pinned)
            paths.add(path)
            for i, (h, rows) in enumerate(zip(hs, outs)):
                what = f"{cfg['name']}: call {c} [{x}, {y}) on the {path} path, member {i}; {where}"
                e = cr.call_expectation(cfg, exp, i, c)
                sig = signal_tuples(h, cfg)
                cr.assert_candidates(cr.gpu_keys(rows, cfg), sig, e["cands"], what)
                if not native:
                    first, got = tapped(h, e["b0"], e["b1"])
                    assert e["b1"] == e["b0"] or first < e["b1"], what
                    cr.assert_bytes(got, e["bytes"][2 * (first - e["b0"]) * bs:], what)
                if "rows" in e:
                    spectrum_ref.assert_rows(h.fetch_spectrum(partial=True), e["rows"], what)
                labels |= cr.input_labels(h.last_kernels())
                calls[i].append((rows, sig))
            x = y
    finally:
        pinned.close()

    # the calls' concatenation equals one call on a fresh lone handle, bytes of every block included
    nb = exp["members"][0]["blocks"][-1]
    for i in range(n):
        what = f"{cfg['name']}: member {i} against one call on a lone handle; {where}"
        f = allocate(cfg, i, raw, 0, what)
        rows = f.decode(raw, cfg["flags"], cap=1 << 16)
        sig = signal_tuples(f, cfg)
        got = record_bytes(np.concatenate([r for r, _ in calls[i]]) if calls[i] else rows[:0],
                           sum((sg for _, sg in calls[i]), []) if cfg["signal"] else None)
        assert got == record_bytes(rows, sig), what
        if not native:
            first, b = tapped(f, 0, nb)
            assert first == 0, what
            cr.assert_bytes(b, exp["members"][i]["bytes"], what)
        if cfg["spectrum"] and i == cfg["spectrum_member"]:
            log2_n, F = cfg["spectrum"]
            p = exp["members"][i]["spectrum"]
            spectrum_ref.assert_rows(f.fetch_spectrum(partial=True),
                                     spectrum_ref.rows_of_powers(p, F, frames=cfg["nsamples"] >> log2_n, partial=True), what)
        f.close()

    # after reset a second capture, fed through the same cut plan, decodes as on fresh handles
    raw2 = cr.capture(cfg, seed=cfg["seed"] + 1000)
    for i, h in enumerate(hs):
        h.reset()
        if cfg["mode"] in cr.WIDE and cfg["ks"][i] == "auto":
            h.set_channel_gain(h.measure_channel(raw2)["k"])
    again = [[] for _ in range(n)]
    rows2 = [[] for _ in range(n)]
    pinned = Pinned(max(y - x for x, y in zip([0] + exp["ends"], exp["ends"])) * s)
    try:
        x = 0
        for y, path in cfg["cuts"]:
            for i, (h, rows) in enumerate(zip(hs, feed(hs, raw2[x * s:y * s], path, cfg["flags"], pinned))):
                again[i].append((rows, signal_tuples(h, cfg)))
                if cfg["spectrum"] and i == cfg["spectrum_member"]:
                    rows2[i].append(h.fetch_spectrum())
            x = y
    finally:
        pinned.close()
    for i in range(n):
        what = f"{cfg['name']}: member {i} after reset on a second capture; {where}"
        f = allocate(cfg, i, raw2, 0, what)
        want = f.decode(raw2, cfg["flags"], cap=1 << 16)
        got = record_bytes(np.concatenate([r for r, _ in again[i]]),
                           sum((sg for _, sg in again[i]), []) if cfg["signal"] else None)
        assert got == record_bytes(want, signal_tuples(f, cfg)), what
        if rows2[i]:
            log2_n, F = cfg["spectrum"]
            r = [np.concatenate([x[k] for x in rows2[i]]) for k in range(3)]
            spectrum_ref.assert_rows(r, spectrum_ref.rows(raw2, cfg["fmt"], log2_n, F, cfg["scale"]), what)
        f.close()
    for h in hs:
        h.close()

    assert labels == cr.labels_of(cfg), (labels, where)
    SEEN.update(cr.cells_of(cfg, paths))
    TIMES[cfg["name"]] = round(time.perf_counter() - t0, 2)
    return exp


@pytest.mark.parametrize("i", range(N_CONFIGS))
def test_configuration(built, i):
    run_config(_configs()[i])


@pytest.mark.parametrize("fmt", cr.FORMATS, ids=lambda f: cr.NAME[f])
def test_every_format_on_special_values(built, fmt):
    """Every input mode of the format, the wide ones and the spectrum included, on a capture dense in NaN, infinities,
    signed zeros, subnormals, rint ties and values past the clamps: every block's bytes against the restatement, the
    candidates against the oracle, the spectrum rows against the float64 restatement."""
    for cfg in cr.sweep_configs(fmt):
        where = f"config {json.dumps(cfg)}"
        raw = cr.special_raw(fmt, cfg["nsamples"], 900 + fmt)
        hs = [allocate(cfg, i, raw, 0, where) for i in range(cr.group_size(cfg))]
        outs = feed(hs, raw, "pageable", 0)
        labels = set()
        for i, (h, rows) in enumerate(zip(hs, outs)):
            what = f"{cfg['name']} member {i}; {where}"
            u8 = cr.decoder_bytes(cfg, raw, i, cr.gain_of(cfg, raw, i))
            nb = u8.size // (2 * h.cfg.block_size)
            assert nb > 4, what
            u8 = u8[:2 * nb * h.cfg.block_size]
            if cfg["mode"] != "pass":
                first, got = tapped(h, 0, nb)
                assert first == 0, what
                cr.assert_bytes(got, u8, what)
            want = sorted(k for k, _ in cr.oracle_candidates(cfg, u8))
            assert sorted(cr.gpu_keys(rows, cfg)) == want, what
            if cfg["spectrum"]:
                log2_n, F = cfg["spectrum"]
                spectrum_ref.assert_rows(h.fetch_spectrum(partial=True),
                                         spectrum_ref.rows(raw, fmt, log2_n, F, 0.0, partial=True), what)
            labels |= cr.input_labels(h.last_kernels())
            h.close()
        assert labels == cr.labels_of(cfg), (labels, where)
        SEEN.update({("label", lb) for lb in labels})
        SEEN.update({c for c in cr.cells_of(cfg) if c[0] == "format"})


@pytest.mark.parametrize("mode,rate_in", [("decimate", 30_720_000), ("tuned", 10_000_000)])
def test_largest_group(built, mode, rate_in):
    """ERTGPU_MAX_CHANNELS handles in one group across the capture: each equals its lone handle and the restatement,
    call by call, and after reset."""
    ro = cr.DATA_RATE * 72
    lim = cr._offset_limit(rate_in, ro)
    offs = [int(o) for o in np.linspace(-0.95 * lim, 0.95 * lim, 64)]
    n = 600_000
    cfg = cr.make_config(f"group64_{mode}", 64, mode=mode, protocols=["scm", "scm+"], cl=72, fmt=capi.FORMAT_CS16,
                         rate_in=rate_in, offsets=offs, signal=True, max_blocks=64, nsamples=n,
                         cuts=[[n // 3, "pinned"], [n // 3 + 1, "pageable"], [n, "device"]])
    assert cr.plan(cfg)[0] is None or (cr.plan(cfg)[0]["D"] > 1) == (mode == "decimate")
    run_config(cfg)


def test_every_combination_cell_was_seen(built):
    """Runs last: each input mode with each feature it allows (signal reports, the spectrum, r900, a group of several
    channels, the device path, a small max_blocks_per_call), every format in a resampling and a wide mode, and every
    input-stage kernel ertgpu_last_kernels names were reached by the tests above."""
    if not SEEN:
        pytest.skip("collects what the other tests of this file ran: run the whole file")
    print("seconds per configuration:", TIMES)
    print("cells:", sorted(SEEN))
    missing = cr.all_cells() - SEEN
    assert not missing, sorted(missing)
