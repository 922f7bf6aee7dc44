"""CPU tests of the frame-tagged capture (tests/spectrum_ref.py) that tests/test_gpu_spectrum_rows.py compares
spectrum_kernel's rows with: every format stores it exactly, each frame carries its tone, and, at every (log2 N, F) of
that file, rows built wrong from the restatement's own frame powers fail spectrum_ref.assert_rows."""
import numpy as np
import pytest

import spectrum_ref as sr
from wide_ref import wide_components

SHAPES = sr.row_shapes()


@pytest.mark.parametrize("fmt", sr.TAG_FORMATS)
def test_every_format_stores_the_tagged_components(fmt):
    sw = sr.tagged_components(10, 40 * 1024 + 77, seed=5)
    assert sw.size == 2 * (40 * 1024 + 77)
    assert (np.abs(sw) <= 16320).all() and (sw % 128 == 64).all()
    assert np.array_equal(wide_components(sr.tagged_bytes(sw, fmt), fmt), sw)


@pytest.mark.parametrize("log2n", [6, 10, 14])
def test_each_frame_carries_its_tone(log2n):
    """Frame f's strongest bin is its tone's, at the level of its place in the cycle; the noise floor lies 40 to 50 dB
    below the loudest level."""
    n, seed = 1 << log2n, 11
    nf = max(48, (1 << 20) // n)
    p = sr.frame_powers(sr.tagged_bytes(sr.tagged_components(log2n, nf * n, seed), 0), 0, log2n)
    c, a = sr.tag_bins(log2n, seed)
    k = (c + a * np.arange(nf) + n // 2) % n      # the tone's bin in ascending frequency order
    assert np.array_equal(np.argmax(p, axis=1), k)
    tone = sr.db(p[np.arange(nf), k])
    top = sr.db(sr.tag_amplitude(log2n)[0] ** 2 / 127.5 ** 2)
    for i, lv in enumerate(sr.TAG_LEVELS_DB):
        assert np.abs(tone[i::3] - (top + lv)).max() < 0.3
    others = np.ones_like(p, bool)
    for d in (-1, 0, 1):
        others[np.arange(nf), (k + d) % n] = False
    floor = top - sr.db(np.median(p[others]) / np.log(2))   # the median of an exponential is its mean times ln 2
    assert 40 <= floor <= 50, floor


def _rejects(got_mean, got_peak, want, i):
    """assert_rows rejects row i of want with got_mean and got_peak in its place."""
    rows, mean, peak = want
    m, pk = mean.copy(), peak.copy()
    m[i], pk[i] = got_mean, got_peak
    with pytest.raises(AssertionError):
        sr.assert_rows((np.array(rows), m, pk), want)


@pytest.mark.parametrize("log2n,F", SHAPES)
def test_wrong_rows_are_rejected(log2n, F):
    """Each row of the stream that test_gpu_spectrum_rows.py cuts, built wrong in the ways a bookkeeping error would
    build it, fails assert_rows: in its mean always, and in its peak too where the row and the frame after it fall in
    distinct bins (F < N).  A peak is a maximum, so neither a divisor nor a group added twice can move it; where more
    than one frame of a row share a bin, only the loudest of them shows in the peak."""
    n, g = 1 << log2n, sr.group_frames(log2n)
    cuts = sr.cut_plan(log2n, F)
    p = sr.frame_powers(sr.tagged_bytes(sr.tagged_components(log2n, cuts[-1], log2n * 100_000 + F), 0), 0, log2n)
    want = sr.rows_of_powers(p, F)
    sr.assert_rows((np.array(want[0]), want[1], want[2]), want)   # the restatement passes its own check
    assert len(want[0]) == 3
    peak_too = F < n
    lg = (-(-F // g) - 1) * g   # a row's last group starts here
    for r in range(3):
        a, b = r * F, (r + 1) * F
        s = p[a:b].sum(axis=0)
        frame_sets = {"shifted by one frame": p[a + 1:b + 1], "first frame dropped": p[a + 1:b],
                      "last frame dropped": p[a:b - 1], "next row's first frame added": p[a:b + 1]}
        if r < 2:
            frame_sets["the next row"] = p[b:b + F]
        for what, fs in frame_sets.items():
            _rejects(fs.sum(axis=0) / F, want[2][r], want, r)
            if peak_too or what == "the next row":
                _rejects(want[1][r], fs.max(axis=0), want, r)
        for wrong in (s / (F - 1), s / (F + 1), (s + p[a + lg:b].sum(axis=0)) / F):
            _rejects(wrong, want[2][r], want, r)
    # the open row after each call of the plan that ends inside a group: without the partial group's frames
    for cut in cuts:
        fr = cut // n - cut // n // F * F
        if fr % g == 0:
            continue
        a, done = cut // n - fr, (fr // g) * g
        open_row = sr.rows_of_powers(p, F, frames=cut // n, first_row=a // F, partial=True)
        assert open_row[0] == [(a * n, fr)]
        _rejects(p[a:a + done].sum(axis=0) / fr, open_row[2][0], open_row, 0)
        if peak_too:
            _rejects(open_row[1][0], p[a:a + done].max(axis=0) if done else np.zeros(n), open_row, 0)
