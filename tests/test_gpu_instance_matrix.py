"""Every instance of the two template families on the hot path -- demod_fast_kernel<CL, W> and search_slide_kernel<NPRE,
HALF, PAT...> -- against the CPU oracle (or a numpy restatement over the oracle's Quantized bits), at the shapes where
their less travelled code paths run:

  * instance matrix: every specialised chip length, every slide instance (stock pattern sets and the run-time probe),
    candidates and the Quantized / Packed / r900 taps on both sides of every 32-block work tile seam;
  * work-tile schedules: call sizes derived from the device's SM count that end in a partial tile, one full round,
    several rounds with a dynamic or a pre-assigned last round, for 16, 12, 8 and 7 resident warps, compared with the
    independent demod_generic_kernel and with the oracle at the round seams;
  * plane alignment: every demod instance with the bit-plane at 0 and at 16 mod 32 bytes (sector-paired stores);
  * call seams: host-path splits and max_blocks_per_call chunking, packets placed across block, tile and call seams;
  * adversarial Search inputs: near-miss preambles, constant and uniform bytes, a custom preamble, an all-ones one.

The last test checks that every instance allocate can choose was seen."""
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import oracle
from helpers import PREAMBLES, assert_check_masks_exact, cand_key_gpu, cand_key_oracle, screen_expected, whole_blocks
from rtlamr_b200 import capi, shard, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
gpu = pytest.mark.gpu

FAST_CLS = [32, 40, 48, 56, 64, 72, 78, 80, 88, 96]
STOCK = {"scm": (21, 96), "scm+": (16, 128), "idm": (32, 736), "netidm": (32, 736), "r900": (32, 116),
         "r900bcd": (32, 116)}   # (PreambleSymbols, PacketSymbols)
STOCK_PATTERNS = {1: None, 3: [0xF953, 0x16A3, 0x5555], 4: [0xF953, 0x16A3, 0x5555, 0x0000]}
SEEN_DEMOD = set()    # (demod instance, plane alignment ph)
SEEN_SEARCH = set()   # Search instances


# ---------------------------------------------------------------- restated host arithmetic
def fast_body_len(cl):
    L = (cl + 1 + 7) // 8 * 8
    return L + 8 if (L // 8) % 2 == 0 else L


def fast_warps(cl):
    L2 = 2 * fast_body_len(cl) + 40
    return 16 if L2 <= 128 else 12 if L2 <= 168 else 8


def fast_dynamic_tiles(ntiles, grid, W):
    cap = grid * W
    if W < 4 or cap <= 0:
        return ntiles
    full, rest = divmod(ntiles, cap)
    if full < 1 or rest == 0 or rest > 4 * grid:
        return ntiles
    return full * cap


def fast_round_cost(ntiles, sms, W):
    cap = sms * W
    full, rest = divmod(ntiles, cap)
    unit = 1.0 if W == 8 else 0.94
    last = 0.0
    if rest > 0:
        last = 0.62 if (full >= 1 and rest <= 4 * sms) else unit
    return full * unit + last


def demod_plan(nblocks, sms, cl):
    """What launch_demod_fast does with a call of nblocks blocks: warps, grid, dynamic tiles."""
    T = -(-nblocks // 32)
    W = fast_warps(cl)
    if W == 8 and fast_round_cost(T, sms, 7) < fast_round_cost(T, sms, 8):
        W = 7
    grid = max(1, min(sms, -(-T // W)))
    return {"T": T, "W": W, "grid": grid, "cap": grid * W, "dyn": fast_dynamic_tiles(T, grid, W)}


def regime_of(nblocks, p, sms):
    T, cap, grid = p["T"], p["cap"], p["grid"]
    if nblocks % 32:
        return "one_partial_tile" if T == 1 else ("partial_last_tile" if T < cap else None)
    full, rest = divmod(T, cap)
    if grid != sms or full < 1:
        return None
    if rest == 0:
        return {1: "one_round", 2: "two_rounds"}.get(full)
    return "dynamic_tail" if rest > 4 * grid else "preassigned_tail"


def size_for(cl, W, regime, sms):
    """The smallest call (in blocks) whose work-tile plan has W warps and ends in `regime`."""
    if regime == "one_partial_tile":
        sizes = [17]
    elif regime == "partial_last_tile":
        sizes = (32 * t - 5 for t in range(2, 40 * sms))
    else:
        sizes = (32 * t for t in range(1, 40 * sms))
    for nb in sizes:
        p = demod_plan(nb, sms, cl)
        if p["W"] == W and regime_of(nb, p, sms) == regime:
            return nb, p
    raise AssertionError((cl, W, regime, sms))


class Geom:
    """Decoder geometry of a handle (ertgpu_allocate): the plane history in front of the call's first word is
    hist_words, so the call's plane rows start at 16 mod 32 bytes (ph = 4) exactly when hist_words % 8 == 4."""

    def __init__(self, h):
        c = h.cfg
        self.CL, self.SL, self.BS, self.bs2 = c.chip_length, c.symbol_length, c.block_size, c.block_size2
        self.PL, self.PKL, self.BUF, self.PK = c.preamble_length, c.packet_length, c.buffer_length, c.packet_symbols
        self.hist_words = ((self.PKL + 31) // 32 + 3) & ~3
        self.ph = 4 if self.hist_words % 8 == 4 else 0
        self.p0 = self.hist_words * 32 - self.PKL
        self.nbytes = (self.PK + 7) >> 3


def search_label(preambles, SL, p0):
    """The Search instance enqueue_pipeline picks for the distinct preambles (registration order)."""
    npre, nbits = len(preambles), [len(p) for p in preambles]
    if npre <= 4 and p0 % 32 == 0 and 0 <= p0 < 128 and SL % 16 == 0 and 64 <= SL <= 192 and \
            all(16 <= n <= 32 for n in nbits):
        pats = [int(p[:16], 2) for p in preambles]
        stock = (npre == 1 and pats[0] in (0xF953, 0x16A3, 0x5555, 0x0000)) or pats == STOCK_PATTERNS.get(npre)
        return f"search_slide_kernel<{npre},{'true' if SL % 32 == 16 else 'false'}" + \
            ("," + ", ".join("0x%04Xu" % v for v in pats) if stock else "") + ">"
    return "search_generic_kernel"


def distinct_preambles(names):
    out = []
    for m in names:
        if PREAMBLES[m] not in out:
            out.append(PREAMBLES[m])
    return out


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def record(h, g):
    k = h.last_kernels().split(";")
    SEEN_DEMOD.add((k[0], g.ph))
    SEEN_SEARCH.add(k[1])
    return k


# ---------------------------------------------------------------- references
def stream_bits(mt, cl, iq, bs2):
    """Row b = the BlockSize Quantized bits block b appends (the oracle's Filter fed block by block)."""
    o = oracle.Oracle(mt, cl, oracle.SEARCH_EXACT)
    n, bs, pkl = iq.size // bs2, bs2 // 2, o.cfg.packet_length
    out = np.empty((n, bs), np.uint8)
    for b in range(n):
        o.dsp_only(iq[b * bs2:(b + 1) * bs2])
        out[b] = o.quantized()[pkl:]
    o.close()
    return out


def q_window(bits, b, buf):
    """Quantized after block b (decode.go:166-172): the last BUF stream bits, zeros in front of the stream."""
    bs = bits.shape[1]
    lo = b + 1 - (-(-buf // bs))
    seg = bits[max(0, lo):b + 1].ravel()
    if lo < 0:
        seg = np.concatenate([np.zeros(-lo * bs, np.uint8), seg])
    return seg[-buf:]


def check_taps(h, g, bits, blocks, where, offset=0):
    """Quantized and Packed taps of the handle's last call at `blocks` (bits row b - offset = block b)."""
    npacked = (g.BS + g.PL + 7) >> 3
    for b in sorted(set(blocks)):
        want = q_window(bits, b - offset, g.BUF)
        got = h.tap(capi.TAP_QUANTIZED, b)
        if not np.array_equal(got, want):
            bad = np.nonzero(got != want)[0]
            raise AssertionError(f"{where}: Quantized of block {b} differs at {bad.size} bits, first at bit {bad[0]} "
                                 f"(stream bit {(b + 1) * g.BS - g.BUF + bad[0]})")
        assert np.array_equal(h.tap(capi.TAP_PACKED, b), np.packbits(want[:npacked * 8])), (where, b)


def seam_blocks(first, nblocks):
    """Both sides of every 32-block work tile seam of a call of nblocks blocks starting at block `first`, its first,
    middle and last block."""
    out = {first, first + nblocks // 2, first + nblocks - 1}
    for s in range(32, nblocks, 32):
        out |= {first + s - 1, first + s}
    return out


def oracle_keys(mt, cl, iq, g, from_block=0, offset=0, nbytes=None):
    search = oracle.SEARCH_GO if (2 * cl) % 8 == 0 else oracle.SEARCH_EXACT
    o = oracle.Oracle(mt, cl, search)
    cands, msgs = o.decode(iq, cand_cap=1 << 18, msg_cap=1 << 16)
    nb = nbytes or g.nbytes
    keys = sorted((c.block + offset,) + cand_key_oracle(c, nb, g.PK if nbytes is None else nb * 8)[1:]
                  for c in cands if c.block + offset >= from_block)
    o.close()
    return keys, msgs


def gpu_keys(got, g, nbytes=None):
    nb = nbytes or g.nbytes
    return sorted(cand_key_gpu(r, nb, g.PK if nbytes is None else nb * 8) for r in got)


def by_start(keys, BS, BUF, lo, hi):
    """(block, preamble, idx, bytes) -> (stream bit of the first preamble bit, preamble, bytes) for starts in [lo, hi):
    a start's block and idx depend on BufferLength (decode.go:166), the start itself does not."""
    return sorted(k for k in (((b + 1) * BS - BUF + i, p, d) for b, p, i, d in keys) if lo <= k[0] < hi)


def same_records(a, b, what):
    assert len(a) == len(b), (what, len(a), len(b))
    for f in ("block", "idx", "preamble_id", "check_mask", "flags", "bytes", "r900_digits"):
        assert np.array_equal(a[f], b[f]), (what, f)


def exact_search(q, bits, bs, sl, pk):
    """numpy exact Search over one block's Quantized q (decode.go:313-325 without the byte prefilter) and Slice."""
    ok = np.ones(bs, bool)
    for k, v in enumerate(bits):
        ok &= q[k * sl:k * sl + bs] == v
    idx = np.nonzero(ok)[0]
    data = np.packbits(q[idx[:, None] + sl * np.arange(pk)[None, :]], axis=1)
    return idx, data


def handle(protos, cl=None, variant=-1, max_blocks=0, max_cands=0):
    if isinstance(protos, str):
        protos = [capi.stock_protocol(m.strip(), cl) for m in protos.split(",")]
    h = capi.Handle()
    for p in protos:
        h.register(p)
    h.allocate(0, max_blocks, max_cands)
    if variant == 0:
        h.set_demod_variant(0)
    return h


def scm_with_packet_symbols(cl, ph):
    """The stock scm protocol with PacketSymbols (>= 96) changed so that the plane history puts the call's rows at
    ph = 0 or 4.  Quantized does not depend on PacketSymbols: the stock oracle gives the bits."""
    for pk in range(96, 1024):
        hw = ((pk * 2 * cl + 31) // 32 + 3) & ~3
        if (hw % 8 == 4) == (ph == 4):
            p = capi.stock_protocol("scm", cl)
            p.packet_symbols = pk
            return p
    raise AssertionError((cl, ph))


def synth_row(start, chips, cl, amp=(45, 30)):
    row = np.zeros((), dtype=capi.SYNTH_DTYPE)
    row["start_sample"], row["n_chips"], row["chip_length"] = start, len(chips), cl
    row["amp_i"], row["amp_q"] = amp
    packed = np.packbits(np.array(chips, dtype=np.uint8))
    row["chips"][:len(packed)] = packed
    return row


# ---------------------------------------------------------------- CPU: the tile plan restatement
@pytest.fixture(scope="module")
def demod_geom_exe(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("demod_geom") / "demod_geom")
    subprocess.run([NVCC, "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
                    os.path.join(ROOT, "tests", "cpu_harness", "demod_geom.cu"), "-lcuda"],
                   check=True, cwd=ROOT, capture_output=True)
    return exe


def test_tile_plan_restatement_matches_the_harness(demod_geom_exe):
    """fast_warps, fast_dynamic_tiles, fast_round_cost and the launch grid as restated here agree with the C++ (the
    `demod_geom plan` harness), at every call size the schedule tests below derive for 132 and 114 SMs."""
    geo = json.loads(subprocess.run([demod_geom_exe], check=True, capture_output=True, text=True).stdout)
    assert {r["CL"]: r["warps"] for r in geo} == {cl: fast_warps(cl) for cl in FAST_CLS}
    cases = set()
    for sms in (132, 114):
        for cl, _, W, regime in SCHEDULES:
            nb, p = size_for(cl, W, regime, sms)
            cases |= {(p["T"], sms, W), (p["T"], sms, 8), (p["T"], sms, 7)}
        for T in (1, 2, 7 * sms, 7 * sms + 1, 8 * sms, 11 * sms, 11 * sms + 1, 12 * sms + 1, 14 * sms, 14 * sms + 1,
                  16 * sms + 1, 20 * sms + 1, 16 * sms * 3 + 4 * sms, 16 * sms * 3 + 4 * sms + 1):
            cases |= {(T, sms, W) for W in (16, 12, 8, 7)}
    for T, sms, W in sorted(cases):
        r = json.loads(subprocess.run([demod_geom_exe, "plan", str(T), str(sms), str(W)], check=True,
                                      capture_output=True, text=True).stdout)
        grid = max(1, min(sms, -(-T // W)))
        assert r["grid"] == grid and r["dyn"] == fast_dynamic_tiles(T, grid, W), (T, sms, W, r)
        assert not r["dup"] and r["dyn"] + r["static_covered"] == T, r
        assert abs(r["cost7"] - fast_round_cost(T, sms, 7)) < 5e-4 and abs(r["cost8"] - fast_round_cost(T, sms, 8)) < 5e-4, r


def test_search_label_restatement():
    """The Search dispatch as restated here, on the labels tests/test_gpu_parity.py pins."""
    def lab(mt, cl):
        names = mt.split(",")
        pkl = max(STOCK[m][1] for m in names) * 2 * cl
        hw = ((pkl + 31) // 32 + 3) & ~3
        return search_label(distinct_preambles(names), 2 * cl, hw * 32 - pkl)
    assert lab("scm", 72) == "search_slide_kernel<1,true,0xF953u>"
    assert lab("scm,scm+,idm,r900", 72) == "search_slide_kernel<4,true,0xF953u, 0x16A3u, 0x5555u, 0x0000u>"
    assert lab("scm,scm+", 72) == "search_slide_kernel<2,true>"
    assert lab("scm", 64) == "search_slide_kernel<1,false,0xF953u>"
    assert lab("scm", 78) == "search_generic_kernel" and lab("scm", 16) == "search_generic_kernel"
    assert lab("scm", 24) == "search_generic_kernel" and lab("idm", 100) == "search_generic_kernel"


# ---------------------------------------------------------------- 1. instance matrix
# (message types, chip length): with the run-time probe test below, every search_slide_kernel instance; every chip length
MATRIX = [("scm", 40), ("scm+", 56), ("idm", 88), ("r900", 40), ("scm,idm", 88), ("scm,scm+,idm", 88),
          ("idm,scm,scm+", 40), ("scm,scm+,idm,r900", 56), ("r900,scm,scm+,idm", 72),
          ("scm", 48), ("scm+", 32), ("netidm", 64), ("r900bcd", 96), ("scm,r900", 80), ("scm,scm+,idm", 32),
          ("scm+,idm,r900", 48), ("scm,scm+,idm,r900", 80), ("idm,scm,scm+,r900", 96), ("scm,scm+", 64),
          ("idm", 100)]
# SL = 156, not a multiple of 16: the sliding-window Search does not take it and search_generic_kernel runs
ODD_SL_MATRIX = [("scm", 78), ("scm,scm+,idm,r900", 78)]


@gpu
@pytest.mark.parametrize("mt,cl", MATRIX)
def test_instance_matrix(built, mt, cl):
    names = mt.split(",")
    h = handle(mt, cl)
    g = Geom(h)
    nsamples = max(1 << 21, 16 * 32 * g.BS)   # at least 16 work tiles: seams inside the call
    iq, _, _ = synth_stream_any(mt, cl, nsamples)
    iq = whole_blocks(iq, g.bs2)
    nblk = iq.size // g.bs2
    got = h.decode(iq, cap=1 << 16)
    k = record(h, g)
    want_demod = "demod_generic_kernel" if cl not in FAST_CLS else \
        f"demod_fast_kernel<{cl},{demod_plan(nblk, sm_count(), cl)['W']}>"
    assert h.demod_kernel_name() == want_demod, k
    assert k[1] == search_label(distinct_preambles(names), g.SL, g.p0), k

    # the oracle, fed in segments ending at the tapped blocks (the r900 parser's quantized only exists after Decode)
    search = oracle.SEARCH_GO if (2 * cl) % 8 == 0 else oracle.SEARCH_EXACT
    o = oracle.Oracle(mt, cl, search)
    taps = sorted(seam_blocks(0, nblk))
    cands, r900q, prev = [], {}, 0
    for b in taps:
        c, _ = o.decode(iq[prev * g.bs2:(b + 1) * g.bs2], cand_cap=1 << 14, msg_cap=1 << 12)
        cands += c
        prev = b + 1
        if any(m.startswith("r900") for m in names):
            r900q[b] = o.r900_quantized()
    if prev < nblk:
        cands += o.decode(iq[prev * g.bs2:], cand_cap=1 << 14, msg_cap=1 << 12)[0]
    o.close()
    want = sorted(cand_key_oracle(c, g.nbytes, g.PK) for c in cands)
    assert gpu_keys(got, g) == want
    assert len(want) > 0
    assert_check_masks_exact(got, mt)
    check_taps(h, g, stream_bits(mt, cl, iq, g.bs2), taps, f"{mt}@{cl}")
    for b, q in r900q.items():
        assert np.array_equal(h.tap(capi.TAP_R900_QUANTIZED, b), q), b
    h.close()


@gpu
@pytest.mark.parametrize("mt,cl", ODD_SL_MATRIX)
def test_odd_symbol_length_matrix(built, mt, cl):
    """The instance-matrix checks on a symbol length that is not a multiple of 16 (search_generic_kernel)."""
    test_instance_matrix(built, mt, cl)


def synth_stream_any(mt, cl, nsamples):
    pk, truth = synth.make_packets(mt, cl, nsamples, seed=9, spacing=1 << 18)
    return synth.host_fill(0, nsamples, 0x5EED0011, pk), pk, truth


CUSTOM21 = "110100111000101101001"   # first 16 bits 0xD38B: no stock pattern, the single-preamble run-time probe


def custom_scm(cl, preamble):
    p = capi.stock_protocol("scm", cl)
    p.preamble = preamble.encode()
    return p


def custom_packet_bits(rng, preamble):
    """An scm-shaped packet behind a custom preamble: 80 bits, then the scm CRC over bytes 2..9 (scm.go:76)."""
    bits = [int(c) for c in preamble] + list(rng.integers(0, 2, 80 - len(preamble)))
    body = np.packbits(np.array(bits, np.uint8)).tobytes()
    crc = synth.crc16(0, 0x6F63, body[2:10])
    return np.unpackbits(np.frombuffer(body + crc.to_bytes(2, "big"), np.uint8)).tolist()


def numpy_candidates(bits_rows, g, preamble, pk, first_block=0):
    """(block, 0, idx, bytes) of the numpy exact search over every block's Quantized."""
    pre = [int(c) for c in preamble]
    out = []
    for b in range(first_block, bits_rows.shape[0]):
        q = q_window(bits_rows, b, g.BUF)
        idx, data = exact_search(q, pre, g.BS, g.SL, pk)
        out += [(b, 0, int(i), d.tobytes()) for i, d in zip(idx, data)]
    return sorted(out)


@gpu
@pytest.mark.parametrize("cl", [56, 80])
def test_runtime_single_preamble_probe(built, cl):
    """search_slide_kernel<1,HALF> with the pattern read at run time: a custom 21-bit preamble on the scm geometry,
    against a numpy exact search over the stock scm oracle's Quantized (the DSP does not depend on the preamble)."""
    h = handle([custom_scm(cl, CUSTOM21)], cl)
    g = Geom(h)
    rng = np.random.default_rng(cl)
    nsamples = 24 * 32 * g.BS
    plen = 96 * g.SL
    rows = [synth_row(s, synth.manchester_chips(custom_packet_bits(rng, CUSTOM21)), cl)
            for s in range(1000, nsamples - plen, nsamples // 16)]
    iq = synth.host_fill(0, nsamples, 0x5EED0012, np.array(rows, dtype=capi.SYNTH_DTYPE))
    got = h.decode(iq, cap=1 << 16)
    k = record(h, g)
    assert k[1] == f"search_slide_kernel<1,{'true' if g.SL % 32 == 16 else 'false'}>", k
    bits = stream_bits("scm", cl, iq, g.bs2)
    want = numpy_candidates(bits, g, CUSTOM21, g.PK)
    assert gpu_keys(got, g) == want
    valid = 0
    for r in got:
        ok = screen_expected("scm", r["bytes"].tobytes())
        assert int(r["check_mask"]) == int(ok)
        valid += ok
    assert valid >= 10
    check_taps(h, g, bits, seam_blocks(0, iq.size // g.bs2), f"custom@{cl}")
    h.close()


@gpu
def test_all_ones_preamble_on_constant_input_and_capacity(built):
    """Every start of every word a hit: the exact count, ERTGPU_ECAPACITY with the need reported when it does not fit,
    and all of them with enough capacity."""
    import ctypes as C
    cl, pre = 72, "1" * 21
    h = handle([custom_scm(cl, pre)], cl)
    g = Geom(h)
    iq = np.zeros(20 * g.bs2, np.uint8)
    bits = stream_bits("scm", cl, iq, g.bs2)
    want = numpy_candidates(bits, g, pre, g.PK)
    assert len(want) > 15 * g.BS
    small = handle([custom_scm(cl, pre)], cl, max_cands=1000)
    out = np.empty(1000, dtype=capi.CAND_DTYPE)
    n = C.c_size_t(0)
    rc = small._L.ertgpu_decode(small._h, iq.ctypes.data, iq.size, 0, out.ctypes.data, out.size, C.byref(n))
    assert rc == capi.ECAPACITY and n.value == len(want), (rc, n.value, len(want))
    small.close()
    big = handle([custom_scm(cl, pre)], cl, max_cands=len(want))
    got = big.decode(iq, cap=len(want))
    record(big, g)
    assert gpu_keys(got, g) == want
    for r in got[:: 97]:
        assert int(r["check_mask"]) == int(screen_expected("scm", r["bytes"].tobytes()))
    big.close()
    h.close()


# ---------------------------------------------------------------- 2. work-tile schedules
REGIMES = ["one_partial_tile", "partial_last_tile", "one_round", "dynamic_tail", "preassigned_tail"]
SCHEDULES = [(32, "scm", 16, r) for r in REGIMES] + [(40, "scm", 12, r) for r in REGIMES] + \
            [(56, "scm+", 7, r) for r in REGIMES + ["two_rounds"]] + \
            [(56, "scm+", 8, r) for r in ("one_round", "dynamic_tail", "preassigned_tail")]


def big_call(protos, ref_mt, cl, nblocks, fill, windows, compare_oracle_cands=True, extra_taps=lambda g: ()):
    """One device-resident call of nblocks blocks filled by fill(d, g) on the fast kernel and, on the same bytes, on
    demod_generic_kernel.  Full candidate lists and the Quantized taps at every tile seam (and extra_taps) must agree;
    the oracle (ref_mt: the stock set with the same DSP geometry) is checked on [w0, w1) windows with a halo lead-in.
    extra_taps(g): more blocks whose taps the two kernels must agree on."""
    import torch
    hf = handle(protos, cl, max_blocks=nblocks, max_cands=1 << 20)
    hg = handle(protos, cl, variant=0, max_blocks=nblocks, max_cands=1 << 20)
    g = Geom(hf)
    assert nblocks * g.bs2 < 1 << 30
    d = torch.empty(nblocks * g.bs2, dtype=torch.uint8, device="cuda")
    fill(d, g)
    torch.cuda.synchronize()
    st = torch.cuda.current_stream().cuda_stream
    res = []
    for h in (hf, hg):
        h.decode_device_async(d.data_ptr(), d.numel(), 0, st)
        res.append(h.fetch(1 << 20))
    k = record(hf, g)
    assert hg.demod_kernel_name() == "demod_generic_kernel" and hg.last_kernels().split(";")[1] == k[1]
    same_records(res[0], res[1], "fast vs generic")
    for b in sorted(seam_blocks(0, nblocks) | set(extra_taps(g))):
        assert np.array_equal(hf.tap(capi.TAP_QUANTIZED, b), hg.tap(capi.TAP_QUANTIZED, b)), b
    halo = shard.halo_blocks(g.BS, max(g.PKL, oracle.Oracle(ref_mt, cl).cfg.packet_length))
    ref_nbytes = (max(STOCK[m][1] for m in ref_mt.split(",")) + 7) >> 3
    ref_buf = oracle.Oracle(ref_mt, cl).cfg.buffer_length
    for w0, w1 in windows:
        w0, w1 = max(0, w0), min(nblocks, w1)
        f0 = max(0, w0 - halo)
        iq = d[f0 * g.bs2:w1 * g.bs2].cpu().numpy()
        check_taps(hf, g, stream_bits(ref_mt, cl, iq, g.bs2), range(w0, w1), f"window {w0}", offset=f0)
        if compare_oracle_cands:
            sel = res[0][(res[0]["block"] >= w0) & (res[0]["block"] < w1)]
            nbytes = min(ref_nbytes, g.nbytes)
            want, _ = oracle_keys(ref_mt, cl, iq, g, from_block=w0, offset=f0, nbytes=nbytes)
            lo, hi = (w0 + 1) * g.BS - min(g.BUF, ref_buf), (w1 + 1) * g.BS - max(g.BUF, ref_buf)
            have = by_start(gpu_keys(sel, g, nbytes=nbytes), g.BS, g.BUF, lo, hi)
            assert have == by_start(want, g.BS, ref_buf, lo, hi), (w0, w1)
    hf.close()
    hg.close()
    del d
    return res[0], k


@gpu
@pytest.mark.parametrize("cl,mt,W,regime", SCHEDULES)
def test_work_tile_schedule(built, cl, mt, W, regime):
    sms = sm_count()
    nb, p = size_for(cl, W, regime, sms)

    def fill(d, g):
        n = nb * g.BS
        pk, _ = synth.make_packets(mt, cl, n, seed=W, spacing=min(1 << 20, n // 2))
        capi.synth_fill(0, d.data_ptr(), 0, n, 0x5EED0020 + W, pk)

    T, cap, dyn = p["T"], p["cap"], p["dyn"]
    places = [0] + [32 * cap * r for r in range(1, T // cap + 1)] + ([32 * dyn] if dyn < T else []) + [nb]
    windows = [(x - 40, x + 40) for x in sorted(set(places))]

    def static_taps(g):   # the pre-assigned tiles: taps BUF // BS blocks apart cover every bit of them
        return list(range(32 * dyn, nb, g.BUF // g.BS)) + [nb - 1] if dyn < T else []
    got, k = big_call(mt, mt, cl, nb, fill, windows, extra_taps=static_taps)
    assert k[0] == f"demod_fast_kernel<{cl},{W}>", (k, p)
    if regime == "preassigned_tail":
        assert 0 < T - dyn <= 4 * sms
    assert len(got) > 0


# ---------------------------------------------------------------- 3. plane alignment
@gpu
@pytest.mark.parametrize("ph", [0, 4])
@pytest.mark.parametrize("cl", FAST_CLS)
def test_plane_alignment_short_calls(built, cl, ph):
    """Every demod instance a short call picks (16, 12 or 7 warps) with the plane rows at 0 and at 16 mod 32 bytes:
    every block's taps against the stock oracle's bits, candidate starts against the stock oracle's (first 12 bytes)
    and, on the same handle geometry, candidates against demod_generic_kernel."""
    p = scm_with_packet_symbols(cl, ph)
    hf, hg = handle([p], cl), handle([p], cl, variant=0)
    g = Geom(hf)
    assert g.ph == ph
    nb = 3 * 32 + 9
    iq, _, _ = synth_stream_any("scm", cl, nb * g.BS)
    a, b = hf.decode(iq, cap=1 << 14), hg.decode(iq, cap=1 << 14)
    k = record(hf, g)
    assert k[0] == f"demod_fast_kernel<{cl},{demod_plan(nb, sm_count(), cl)['W']}>", k
    same_records(a, b, "fast vs generic")
    want, _ = oracle_keys("scm", cl, iq, g, nbytes=12)
    ref_buf = oracle.Oracle("scm", cl).cfg.buffer_length
    hi = (nb + 1) * g.BS - max(g.BUF, ref_buf)
    want = by_start(want, g.BS, ref_buf, 0, hi)
    assert by_start(gpu_keys(a, g, nbytes=12), g.BS, g.BUF, 0, hi) == want and len(want) > 0
    check_taps(hf, g, stream_bits("scm", cl, iq, g.bs2), range(nb), f"ph{ph}@{cl}")
    hf.close()
    hg.close()


@gpu
@pytest.mark.parametrize("ph", [0, 4])
@pytest.mark.parametrize("cl", [c for c in FAST_CLS if fast_warps(c) == 8])
def test_eight_warp_instances_alignment_and_inputs(built, cl, ph):
    """demod_fast_kernel<CL,8> (a call of one full round of 8 warps) at both plane alignments, on one stream of
    synthetic packets, then constant 0, 127, 255 and uniform random bytes, each part checked against the oracle."""
    import torch
    sms = sm_count()
    nb, p = size_for(cl, 8, "one_round", sms)
    prot = scm_with_packet_symbols(cl, ph)
    cuts = [0, nb // 2 + 7, 5 * nb // 8 + 3, 6 * nb // 8 + 11, 7 * nb // 8 + 1, nb]

    def fill(d, g):
        s = [c * g.bs2 for c in cuts]
        pk, _ = synth.make_packets("scm", cl, cuts[1] * g.BS - 20 * g.BS, seed=cl, spacing=1 << 20)
        capi.synth_fill(0, d.data_ptr(), 0, cuts[1] * g.BS, 0x5EED0030 + cl, pk)
        for i, v in enumerate((0, 127, 255)):
            d[s[1 + i]:s[2 + i]].fill_(v)
        gen = torch.Generator(device="cuda").manual_seed(cl * 10 + ph)
        d[s[4]:] = torch.randint(0, 256, (s[5] - s[4],), dtype=torch.uint8, device="cuda", generator=gen)

    windows = [(0, 40)] + [(c - 20, c + 44) for c in cuts[1:-1]] + [(nb - 40, nb)]
    got, k = big_call([prot], "scm", cl, nb, fill, windows)
    assert k[0] == f"demod_fast_kernel<{cl},8>", k
    assert len(got) > 0


# ---------------------------------------------------------------- 4. call seams and placed packets
@gpu
@pytest.mark.parametrize("cl", FAST_CLS)
def test_call_seams_and_placed_packets(built, cl):
    """Host-path calls of 1, 31, 33, 32 and random block counts, chunked by max_blocks_per_call, equal one call and the
    oracle; packets straddle a block seam, a 32-block tile seam, call seams, and one starts in block 0.  The first
    block of every call's last chunk (its Quantized holds the bits carried over the seam) matches the oracle."""
    mt = "scm"
    h1 = handle(mt, cl)
    g = Geom(h1)
    nb = 200
    rng = np.random.default_rng(cl)
    sizes = [1, 31, 33, 32]
    while sum(sizes) < nb:
        sizes.append(int(min(nb - sum(sizes), rng.integers(1, 40))))
    seams = list(np.cumsum(sizes)[:-1])                       # 1, 32, 65, 97, ...
    plen = STOCK[mt][1] * g.SL
    pk, truth = synth.make_packets(mt, cl, 5 << 16, seed=cl, spacing=1 << 16)
    starts = [5, 8 * g.BS - plen // 2, 32 * g.BS - plen // 3, 65 * g.BS - plen // 2 + 3, 96 * g.BS - 2 * plen // 3]
    pk["start_sample"] = starts
    assert all(b - a > plen for a, b in zip(starts, starts[1:]))
    iq = synth.host_fill(0, nb * g.BS, 0x5EED0040, pk)
    whole = h1.decode(iq, cap=1 << 14)
    record(h1, g)
    bits = stream_bits(mt, cl, iq, g.bs2)
    check_taps(h1, g, bits, seam_blocks(0, nb), "one call")
    h2 = handle(mt, cl, max_blocks=16)
    parts, off = [], 0
    for n in sizes:
        parts.append(h2.decode(iq[off * g.bs2:(off + n) * g.bs2], cap=1 << 14))
        last0 = off + 16 * ((n - 1) // 16)
        check_taps(h2, g, bits, {last0, off + n - 1}, f"call at block {off}")
        off += n
    same_records(np.concatenate(parts), whole, "split vs one call")
    want, _ = oracle_keys(mt, cl, iq, g)
    assert gpu_keys(whole, g) == want
    assert_check_masks_exact(whole, mt)
    valid = {r["bytes"][:12].tobytes() for r in whole if r["check_mask"] & 1}
    assert all(t.data in valid for t in truth), [t.start_sample for t in truth if t.data not in valid]
    assert 32 in seams and 65 in seams
    h1.close()
    h2.close()


# ---------------------------------------------------------------- 5. adversarial Search inputs
@gpu
@pytest.mark.parametrize("cl", [40, 64, 72, 78, 96])
def test_near_miss_preambles(built, cl):
    """Every stock preamble with one bit flipped, for every bit, a few thousand samples apart (bits >= 16 reach the
    slide kernel's cold path): exactly the oracle's candidates."""
    mt = "scm,scm+,idm,r900"
    h = handle(mt, cl)
    g = Geom(h)
    rows, s = [], 3000
    for name in ("scm", "scm+", "idm", "r900"):
        pre = [int(c) for c in PREAMBLES[name]]
        for k in range(len(pre)):
            bits = list(pre)
            bits[k] ^= 1
            chips = synth.manchester_chips(bits + [1, 0, 1, 1, 0, 0, 1, 0])
            rows.append(synth_row(s, chips, cl))
            s += len(chips) * cl + 2500
    nb = -(-(s + 4 * g.BS) // g.BS)
    iq = synth.host_fill(0, nb * g.BS, 0x5EED0050, np.array(rows, dtype=capi.SYNTH_DTYPE))
    got = h.decode(iq, cap=1 << 16)
    record(h, g)
    want, _ = oracle_keys(mt, cl, iq, g)
    assert gpu_keys(got, g) == want
    assert_check_masks_exact(got, mt)
    h.close()


@gpu
@pytest.mark.parametrize("src", ["zeros", "c127", "c255", "uniform"])
@pytest.mark.parametrize("cl", FAST_CLS)
def test_constant_and_uniform_bytes(built, cl, src):
    """Constant and uniformly random bytes on the instance a short call picks: candidates and every block's taps."""
    mt = "scm,scm+"
    h = handle(mt, cl)
    g = Geom(h)
    nb = 2 * 32 + 21
    if src == "uniform":
        iq = np.random.default_rng(cl).integers(0, 256, nb * g.bs2, dtype=np.uint8)
    else:
        iq = np.full(nb * g.bs2, {"zeros": 0, "c127": 127, "c255": 255}[src], np.uint8)
    got = h.decode(iq, cap=1 << 16)
    record(h, g)
    want, _ = oracle_keys(mt, cl, iq, g)
    assert gpu_keys(got, g) == want
    assert_check_masks_exact(got, mt)
    check_taps(h, g, stream_bits(mt, cl, iq, g.bs2), range(nb), src)
    h.close()


# ---------------------------------------------------------------- coverage of the instance choices
def expected_instances():
    src = open(os.path.join(ROOT, "rtlamr_b200", "csrc", "demod_fast.cuh")).read()
    cls = sorted({int(x) for x in re.findall(r"fast_demod_of<(\d+)>\(", src)})
    demod = {f"demod_fast_kernel<{cl},{w}>" for cl in cls for w in ((8, 7) if fast_warps(cl) == 8 else (fast_warps(cl),))}
    src = open(os.path.join(ROOT, "rtlamr_b200", "csrc", "ertgpu.cu")).read()
    slide = set()
    for n, pats in re.findall(r"slide_instance<(\d+)((?:,\s*0x[0-9A-Fa-f]+u)*)>\(", src):
        pats = ", ".join("0x%04Xu" % int(p[2:-1], 16) for p in re.findall(r"0x[0-9A-Fa-f]+u", pats))
        for half in ("true", "false"):
            slide.add(f"search_slide_kernel<{n},{half}" + ("," + pats if pats else "") + ">")
    return cls, demod, slide


def test_instance_choices_have_the_expected_shape():
    cls, demod, slide = expected_instances()
    assert cls == FAST_CLS and len(demod) == 17 and len(slide) == 20


@gpu
def test_every_kernel_instance_was_seen(built):
    """Runs last: every demod_fast instance at both plane alignments, every slide instance, and search_generic_kernel
    were launched by the tests above."""
    if not SEEN_DEMOD:
        pytest.skip("collects what the other tests of this file launched: run the whole file")
    cls, demod, slide = expected_instances()
    missing = sorted((d, ph) for d in demod for ph in (0, 4) if (d, ph) not in SEEN_DEMOD)
    assert not missing, missing
    assert not sorted(slide - SEEN_SEARCH), sorted(slide - SEEN_SEARCH)
    assert "search_generic_kernel" in SEEN_SEARCH
