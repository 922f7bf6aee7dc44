"""GPU tests (-m gpu) of what spectrum_kernel<F> and Spectrum (rtlamr_b200/csrc/spectrum.cuh) keep between calls,
against the NumPy restatement of a frame-tagged capture (tests/spectrum_ref.py), whose every frame shows in its row:
all nine frame lengths at four row lengths each, the complete rows and the open row after calls cut inside a frame, on
a frame, group or row boundary and inside a short last group, on the host and the device path; launch cuts of a long
device call; the row ring and the row capacity; reset; and channel groups.  tests/test_spectrum_rows_cpu.py shows that
rows built wrong at these shapes fail spectrum_ref.assert_rows."""
import functools

import pytest

import spectrum_ref as sr
from rtlamr_b200 import capi

pytestmark = pytest.mark.gpu

RATE_IN = 2_400_000     # a resampling handle takes calls of any whole number of samples
CAPTURE = 915_000_000
LAUNCH = 1 << 24        # input samples of one spectrum_kernel launch (kSpecLaunchSamples)


def _handle(fmt, log2n, F, **kw):
    return capi.new_decoder("scm", 72, input_rate=RATE_IN, input_format=fmt, spectrum=(log2n, F), **kw)


def _stream(log2n, F, samples, fmt, seed):
    """The tagged capture's raw bytes and its frame powers."""
    raw = sr.tagged_bytes(sr.tagged_components(log2n, samples, seed), fmt)
    return raw, sr.frame_powers(raw, fmt, log2n)


class Feed:
    """One handle's stream: feed() sends input samples [at, end) of raw as one host or device call, and check() fetches
    the rows completed since the last fetch and the open row, and compares them with the restatement of the prefix."""

    def __init__(self, h, raw, p, F, fmt):
        self.h, self.raw, self.p, self.F, self.S = h, raw, p, F, capi.FORMAT_BYTES[fmt]
        self.n = p.shape[1]
        self.at = self.fetched = 0
        self.d = None

    def feed(self, end, device=False):
        a, b = self.at * self.S, end * self.S
        if device:
            if self.d is None:
                import torch
                self.d = torch.from_numpy(self.raw).cuda()
                torch.cuda.synchronize()
            self.h.decode_device_async(self.d.data_ptr() + a, b - a)
            self.h.fetch(cap=1 << 16)
        else:
            self.h.decode(self.raw[a:b], cap=1 << 16)
        self.at = end

    def want(self, partial=True):
        return sr.rows_of_powers(self.p, self.F, frames=self.at // self.n, first_row=self.fetched, partial=partial)

    def check(self, what="", partial=True):
        got = self.h.fetch_spectrum(partial=partial)
        sr.assert_rows(got, self.want(partial), f"{what} at sample {self.at}")
        self.fetched = self.at // self.n // self.F
        return got

    def reset(self):
        self.h.reset()
        self.at = self.fetched = 0


CASES = [(n, F, sr.TAG_FORMATS[(i + i // 4) % 4]) for i, (n, F) in enumerate(sr.row_shapes())]


@pytest.mark.parametrize("log2n,F,fmt", CASES)
def test_rows_and_the_open_row_after_every_cut(built, log2n, F, fmt):
    """The stream of spectrum_ref.cut_plan as one call, then cut by the plan on the host path and on the device path:
    after every call the rows completed so far and the open row equal the restatement of the prefix."""
    cuts = sr.cut_plan(log2n, F)
    raw, p = _stream(log2n, F, cuts[-1], fmt, log2n * 100_000 + F)
    h = _handle(fmt, log2n, F)
    f = Feed(h, raw, p, F, fmt)
    f.feed(cuts[-1])
    got = f.check("one call")
    assert len(got[0]) == 4 and got[0][-1]["frames"] < F
    for device in (False, True):
        f.reset()
        for end in cuts:
            f.feed(end, device)
            f.check("device" if device else "host")
    h.close()


LAUNCH_SHAPE = (10, 271, capi.FORMAT_CU8)
LAUNCH_LONG = LAUNCH + (271 + 135) * 1024 + 7          # a device call of two launches, the second ending mid-row


@functools.lru_cache(maxsize=1)
def _launch_stream():
    log2n, F, fmt = LAUNCH_SHAPE
    return _stream(log2n, F, LAUNCH + (F + 2 * F) * (1 << log2n) + LAUNCH_LONG, fmt, 77)


@pytest.mark.parametrize("where", ["frame", "group", "row", "row end"])
def test_launch_cut_inside_a_frame_group_and_row(built, where):
    """A device call of more than 2^24 input samples is cut into two launches; a host call before it leaves the stream
    where that cut falls inside a frame (so inside a group and a row too), on a frame boundary inside a group, on a
    group boundary inside a row, or at a row's end."""
    log2n, F, fmt = LAUNCH_SHAPE
    n, g = 1 << log2n, sr.group_frames(log2n)
    r = LAUNCH // (F * n) + 1
    cut = {"frame": (r * F + 2 * g + 5) * n + n // 2 + 3, "group": (r * F + 2 * g + 5) * n,
           "row": (r * F + 2 * g) * n, "row end": r * F * n}[where]
    lead, long_call = cut - LAUNCH, LAUNCH_LONG
    raw, p = _launch_stream()
    assert 0 < lead and lead + long_call <= raw.size // capi.FORMAT_BYTES[fmt]
    h = _handle(fmt, log2n, F)
    f = Feed(h, raw, p, F, fmt)
    f.feed(lead)
    f.check("host lead")
    f.feed(lead + long_call, device=True)
    plain = capi.new_decoder("scm", 72, input_rate=RATE_IN, input_format=fmt)   # the same calls without a spectrum
    plain.decode(raw[:lead * f.S], cap=1 << 16)
    plain.decode_device_async(f.d.data_ptr() + lead * f.S, long_call * f.S)
    plain.fetch(cap=1 << 16)
    assert h.last_launches() == plain.last_launches() + 2
    got = f.check("long device call")
    assert len(got[0]) >= LAUNCH // (F * n)
    h.close()
    plain.close()


def _row_cap(f, one_row):
    """Send calls of one row each, leaving every row unfetched, until one is refused: the rows the handle holds."""
    k = 0
    while True:
        try:
            f.feed(f.at + one_row)
        except capi.ErtGpuError as e:
            assert e.code == capi.ECAPACITY, e
            return k
        k += 1
        assert k <= 64


def test_row_ring_and_capacity(built):
    """A handle of 64 blocks per call holds a few rows.  Rows left unfetched up to that capacity are kept; a call that
    needs one row more is refused before it enqueues anything, and goes through after a fetch.  Then more than three
    times the capacity of rows, fetched in batches across the ring's wrap, each equal to the restatement."""
    log2n, F, fmt = 10, 257, capi.FORMAT_CS16
    n = 1 << log2n
    one_row = F * n
    raw, p = _stream(log2n, F, 64 * one_row, fmt, 91)
    h = _handle(fmt, log2n, F, max_blocks_per_call=64)
    f = Feed(h, raw, p, F, fmt)
    f.feed(5 * n + 77)   # rows end inside the calls below, not at their ends
    cap = _row_cap(f, one_row)
    assert 2 <= cap <= 8, cap
    at = f.at
    f.check("after the refused call")    # all cap rows, and the open row without the refused bytes
    assert f.fetched == cap
    f.feed(at + one_row)                 # the refused bytes again
    f.check("the refused bytes again")
    # one call of exactly cap rows is taken, one of cap + 1 refused, with no row waiting
    f.feed(f.at + cap * one_row + n // 2)
    f.check("a call of cap rows")
    at = f.at
    with pytest.raises(capi.ErtGpuError) as e:
        f.feed(at + (cap + 1) * one_row)
    assert e.value.code == capi.ECAPACITY
    f.check("after a refused call of cap + 1 rows")
    # the ring: batches of 1 ... cap rows, calls ending inside frames, on frames and on groups
    start, straddles, k = f.fetched, 0, 0
    while f.fetched - start <= 3 * cap:
        rows = 1 + (3 * k + 1) % cap
        phase = [n // 3, 7 * n, 2 * sr.group_frames(log2n) * n, 0][k % 4]
        end = (f.fetched + rows) * one_row + phase
        first = f.fetched
        f.feed(end)
        got = f.check(f"ring batch {k}", partial=k % 2 == 0)
        assert len(got[0]) >= rows
        straddles += first % cap + rows > cap
        k += 1
    assert straddles >= 2
    h.close()


def test_reset_inside_a_group_and_inside_a_row(built):
    """A stream stopped inside a group (a partial group and an open row on the device) or on a group boundary inside a
    row (an open row only), reset, and another stream cut by the plan: its rows are its restatement alone."""
    log2n, F, fmt = 11, 135, capi.FORMAT_CF32
    n, g = 1 << log2n, sr.group_frames(log2n)
    cuts = sr.cut_plan(log2n, F)
    raw_a, p_a = _stream(log2n, F, 2 * F * n, fmt, 5)
    raw_b, p_b = _stream(log2n, F, cuts[-1], fmt, 6)
    h = _handle(fmt, log2n, F)
    for stop in ((F + 2 * g + 3) * n + n // 2, (F + 3 * g) * n):
        a = Feed(h, raw_a, p_a, F, fmt)
        a.reset()
        a.feed(stop)
        a.check("the first stream")
        b = Feed(h, raw_b, p_b, F, fmt)
        b.reset()
        for end in cuts:
            b.feed(end)
            b.check("the stream after reset")
    h.close()


@pytest.mark.parametrize("who", ["first", "last"])
def test_channel_group(built, who):
    """Three decimating channels of one cs16 capture, the spectrum on the first handle or on the last, fed by the cut
    plan: after every call its rows equal the restatement of the group's input."""
    log2n, F, fmt, rate_in = 13, 35, capi.FORMAT_CS16, 30_720_000
    cuts = sr.cut_plan(log2n, F)
    raw, p = _stream(log2n, F, cuts[-1], fmt, 13)
    offs = [-2_000_000, 500_000, 3_000_000]
    spec = 0 if who == "first" else len(offs) - 1
    group = [capi.new_decoder("scm", 72, input_rate=rate_in, input_format=fmt, capture_freq=CAPTURE,
                              center_freq=CAPTURE + o, spectrum=(log2n, F) if k == spec else None)
             for k, o in enumerate(offs)]
    f = Feed(group[spec], raw, p, F, fmt)
    for end in cuts:
        capi.decode_channels(group, raw[f.at * f.S:end * f.S], cap=1 << 16)
        f.at = end
        f.check(f"spectrum on the {who} channel")
    ks = group[spec].last_kernels()
    assert "decimate_channels_kernel<" in ks and ks.endswith(";spectrum_kernel<cs16>"), ks
    for h in group:
        h.close()
