"""Index arithmetic of the sliding-window Search kernel (rtlamr_b200/csrc/search.cuh), checked on the CPU:
the launch constants make every start word of a tile belong to exactly one (thread, step), keep the 32 lanes of
a warp on 32 different shared-memory banks at every step, and keep every window read inside the staged words.
The kernel itself is compared with the oracle in the GPU tests; this pins the geometry for every symbol length
the reference CLI accepts (flags.go:127-132) without a GPU."""
import json
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpu_harness", "slide_params.cu")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def build(tmp_path_factory, name):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp(name) / name)
    src = os.path.join(ROOT, "tests", "cpu_harness", name + ".cu")
    subprocess.run([NVCC, "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe, src, "-lcuda"],
                   check=True, cwd=ROOT, capture_output=True)
    return exe


@pytest.fixture(scope="module")
def demod_geom_exe(tmp_path_factory):
    return build(tmp_path_factory, "demod_geom")


@pytest.fixture(scope="module")
def demod_geom(demod_geom_exe):
    return json.loads(subprocess.run([demod_geom_exe], check=True, capture_output=True, text=True).stdout)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("slide") / "slide_params")
    subprocess.run([NVCC, "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe, SRC],
                   check=True, cwd=ROOT, capture_output=True)
    return exe


def run(exe, cases):
    args = [str(x) for c in cases for x in c]
    return json.loads(subprocess.run([exe] + args, check=True, capture_output=True, text=True).stdout)


STOCK_SL = [64, 80, 96, 112, 128, 144, 160, 176, 192]   # 2 * ChipLength for ChipLength 32 .. 96


def test_slide_geometry_covers_each_start_word_once_without_bank_conflicts(harness):
    rows = run(harness, [(sl, nb, p0) for sl in STOCK_SL for nb, p0 in ((21, 0), (16, 0), (32, 0), (32, 64))])
    assert len(rows) == len(STOCK_SL) * 4
    for r in rows:
        assert r["ok"], r
        q, nseg, seg = r["q"], r["nseg"], r["seg"]
        assert q == r["SL"] // 16 and r["odd_off"] == r["SL"] >> 5 and r["half"] == r["SL"] % 32
        assert q * nseg <= r["threads"]
        assert r["tile_words"] == q * seg * nseg and r["tile_words"] % 4 == 0      # 16-byte aligned tile starts
        assert r["load_words"] % 4 == 0 and r["load_words"] <= r["max_load"]
        assert r["w0"] == r["p0"] // 32
        # every start word of the tile is visited by exactly one (thread, step)
        seen = [0] * r["tile_words"]
        for t in range(q * nseg):
            j0 = t % q + q * seg * (t // q)
            for i in range(seg):
                seen[j0 + q * i] += 1
        assert all(v == 1 for v in seen)
        # at every step the lanes of a warp read 32 different banks (word address mod 32)
        for w0 in range(0, q * nseg, 32):
            lanes = range(w0, min(w0 + 32, q * nseg))
            banks = {(t % q + q * seg * (t // q)) % 32 for t in lanes}
            assert len(banks) == len(lanes), (r["SL"], w0)
        # the furthest word any start of the tile reads: bit 31's window (even bits: 15 strides; odd bits: + odd_off,
        # two words when half a word in), and the one-window-ahead loads of the register rings (8 strides)
        last = r["tile_words"] - 1 + r["w0"]
        assert last + 15 * q + r["odd_off"] + 1 < r["load_words"]
        assert last + 8 * q + r["odd_off"] + 1 < r["load_words"]


def test_slide_rejects_what_it_does_not_cover(harness):
    rows = run(harness, [(156, 21, 0),    # ChipLength 78: SL % 16 != 0
                         (144, 12, 0),    # preamble shorter than the 16-bit probe
                         (144, 21, 5),    # first start not word aligned
                         (208, 21, 0)])   # beyond the CLI's largest symbol length
    assert [r["ok"] for r in rows] == [False, False, False, False]


def test_stock_probe_patterns(harness):
    # the first 16 preamble bits as the template constant of the specialised kernels (scm: 0x1F2A60 >> 5)
    (r,) = run(harness, [(144, 21, 0)])
    assert r["pattern"] == 0xF953


def test_demod_fast_geometry(demod_geom):
    """FastGeom of every specialised chip length: ring longer than the chip, 16-byte rows with an odd pitch
    (conflict-free LDS.128), an even alignment pad shorter than a body, and a shared-memory map that fits."""
    assert [r["CL"] for r in demod_geom] == [32, 40, 48, 56, 64, 72, 78, 80, 88, 96]
    for r in demod_geom:
        cl, L = r["CL"], r["L"]
        assert r["variant"] == cl
        assert L > cl and L % 8 == 0 and (L // 8) % 2 == 1 and L < cl + 17
        assert r["pad"] == 2 * L - 2 * cl and 0 <= r["pad"] < L and r["pad"] % 2 == 0
        assert r["row_bytes"] == 2 * L and (r["row_bytes"] // 16) % 2 == 1
        assert r["tail_bits"] == L % 32
        assert r["warps"] in (8, 12, 16) and r["stages"] == 2
        # registers are handed out per scheduler: 2 x L ring values + working set must fit the warp count
        assert 2 * L + 40 <= {8: 255, 12: 168, 16: 128}[r["warps"]]
        for key in ("smem", "smem7"):
            assert r[key] <= 227 * 1024, (cl, key, r[key])
        assert r["smem7"] <= r["smem"]
    by = {r["CL"]: r for r in demod_geom}
    assert by[72]["L"] == 88 and by[72]["pad"] == 32 and by[72]["smem"] == 65536 + 65536 + 3 * 2 * 32 * 176 - 1024


def test_demod_tile_plan_covers_every_tile_once(demod_geom_exe):
    """The last round of work tiles: when it would fill at most one warp per scheduler it is pre-assigned (tile
    dyn + SM + SMs * w to warp w < 4), otherwise everything stays dynamic.  Every tile is owned exactly once."""
    exe = demod_geom_exe
    for ntiles, sms, W in ((4096, 132, 8), (4096, 132, 7), (32768, 132, 8), (1056 * 3 + 528, 132, 8), (1056 * 3 + 529, 132, 8),
                           (1056 * 5, 132, 8), (100, 132, 8), (1, 132, 8), (1056 + 1, 132, 8), (4096, 148, 8), (16384, 148, 8)):
        r = json.loads(subprocess.run([exe, "plan", str(ntiles), str(sms), str(W)], check=True, capture_output=True, text=True).stdout)
        assert not r["dup"] and r["dyn"] + r["static_covered"] == ntiles, r
        cap = r["grid"] * W
        rest = ntiles % cap if ntiles >= cap else 0
        if ntiles >= cap and 0 < rest <= 4 * r["grid"]:
            assert r["dyn"] == ntiles - rest and r["per_sched_max"] == 1
        else:
            assert r["dyn"] == ntiles
    r = json.loads(subprocess.run([exe, "plan", "4096", "132", "8"], check=True, capture_output=True, text=True).stdout)
    assert r["dyn"] == 4096 and r["cost8"] < r["cost7"]      # 1 GiB scm on 132 SMs: the 4th round of 8 warps is too full to pre-assign
    r = json.loads(subprocess.run([exe, "plan", "3600", "132", "8"], check=True, capture_output=True, text=True).stdout)
    assert r["dyn"] == 3168 and r["per_sched_max"] == 1      # 3 dynamic rounds of 8 warps + 432 pre-assigned tiles
