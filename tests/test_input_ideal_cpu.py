"""The input stage's CPU restatements (resample_ref, tune_ref, decimate_ref, wide_ref) against the float64 model of
tests/ideal_ref.py, sample by sample, over a seeded sweep of plans in every mode and at the edges of every rule: the
byte-exact GPU tests prove the kernels equal the header's integer design, these prove the design computes the
windowed-sinc resampler, the mixer and the decimator the header describes, within an error budget computed from the
plan.  Perturbed models (a late output, a wrong sub-phase, a conjugated or half-step mixer, an off-centre first stage,
a floor) must fail the same comparison."""
import functools

import numpy as np
import pytest

import decimate_ref
import ideal_ref as ir
import resample_ref
import tune_ref
import wide_ref
from rtlamr_b200 import capi

DATA_RATE = 32768
CAPTURE = 915_000_000
CHIP_LENGTHS = (8, 32, 72, 96, 100)     # 100: a chip length without a specialised demod
MODES = ("untuned", "tuned", "decimating", "wide", "wide_dec")
PER_MODE = 200
RANGES = {"untuned": (0.25, 4.0), "tuned": (0.25, 10.0), "decimating": (10.0, 256.0), "wide": (0.25, 10.0),
          "wide_dec": (10.0, 256.0)}
WIDE_K_MAX = 8     # above it an unclipped channel holds only a few s_w units


def offset_limit(rate_in: int, ro: int) -> int:
    """The largest |offset| a tuned or decimating plan takes: 10 |offset| + 4 min(R_in, R_out) <= 5 R_in."""
    return (5 * rate_in - 4 * min(rate_in, ro)) // 10


def prime_above(x: int) -> int:
    x += 1
    while any(x % d == 0 for d in range(2, int(x ** 0.5) + 1)):
        x += 1
    return x


def edge_rates(mode, ro):
    """The exact edges of the mode's rule, and a prime rate (coprime to every R_out: L/M unreduced)."""
    if mode == "untuned":
        return [ro // 4 + (ro % 4 > 0), 4 * ro, ro - 1, ro + 1, prime_above(3 * ro // 2)]
    if mode in ("tuned", "wide"):
        return [ro // 4 + (ro % 4 > 0), 4 * ro, 4 * ro + 1, 10 * ro, ro - 1, ro + 1, ro, prime_above(7 * ro)]
    return [10 * ro + 1, 256 * ro, 12 * ro, 12 * ro + 1, 64 * ro, 64 * ro + 1, 4 * 37 * ro, 4 * 37 * ro + 1,
            prime_above(100 * ro)]


def _plan_dict(mode, i, cl, rate_in, offset, k, rng):
    return {"mode": mode, "i": i, "cl": cl, "rate_in": int(rate_in), "offset": offset, "k": k,
            "seed": int(rng.integers(0, 2 ** 31))}


@functools.lru_cache(maxsize=None)
def sweep(mode) -> tuple:
    """PER_MODE seeded plans of the mode: every edge at every chip length (tuned modes cycling the offsets 0, +-1 and
    the largest |offset| either way), then rates drawn log-uniform over the mode's range with random offsets."""
    rng = np.random.default_rng(MODES.index(mode) + 0x1DEA)
    lo, hi = RANGES[mode]
    out = []
    for cl in CHIP_LENGTHS:
        ro = DATA_RATE * cl
        for rate_in in edge_rates(mode, ro):
            if mode == "untuned":
                out.append(_plan_dict(mode, len(out), cl, rate_in, None, None, rng))
                continue
            lim = offset_limit(rate_in, ro)
            offset = [0, 1, -1, lim, -lim][len(out) % 5]
            if rate_in == ro and offset == 0:
                offset = 1
            k = int(rng.integers(0, WIDE_K_MAX + 1)) if mode.startswith("wide") else None
            out.append(_plan_dict(mode, len(out), cl, rate_in, offset, k, rng))
    while len(out) < PER_MODE:
        cl = CHIP_LENGTHS[len(out) % len(CHIP_LENGTHS)]
        ro = DATA_RATE * cl
        r = int(round(ro * float(np.exp(rng.uniform(np.log(lo), np.log(hi))))))
        rate_in = min(max(r, -(-ro // 4), 10 * ro + 1 if mode in ("decimating", "wide_dec") else 0), int(hi * ro))
        if rate_in == ro:
            continue
        offset = k = None
        if mode != "untuned":
            lim = offset_limit(rate_in, ro)
            offset = int(rng.integers(-lim, lim + 1))
        if mode.startswith("wide"):
            k = int(rng.integers(0, WIDE_K_MAX + 1))
        out.append(_plan_dict(mode, len(out), cl, rate_in, offset, k, rng))
    return tuple(out)


def handle(plan, fmt=capi.FORMAT_CU8):
    """The plan's handle, configured through the C ABI and not allocated (no device needed)."""
    h = capi.Handle()
    h.register(capi.stock_protocol("scm", plan["cl"]))
    if plan["offset"] is not None:
        h.set_input_tuning(CAPTURE, CAPTURE + plan["offset"])
        if plan["mode"] in ("decimating", "wide_dec"):
            h.allow_input_decimation()
    h.set_input_rate(plan["rate_in"])
    if fmt != capi.FORMAT_CU8:
        h.set_input_format(fmt)
    if plan["k"] is not None:
        h.set_channel_gain(plan["k"])
    return h


def model_plan(plan) -> dict:
    h = handle(plan)
    try:
        return ir.plan_from_handle(h, plan["k"])
    finally:
        h.close()


def channel(plan, n, rng, amplitude, tones=((0.55, None), (0.45, None))):
    """n samples of complex baseband at rate_in, components within +-amplitude: uniform noise and in-band tones (at the
    channel's offset plus up to 0.35 min(R_in, R_out), random phases), relative amplitudes noise 1 - sum(tones)."""
    rate_in, ro = plan["rate_in"], DATA_RATE * plan["cl"]
    off = plan["offset"] or 0
    t = np.arange(n)
    a_noise = amplitude * (1.0 - sum(a for a, _ in tones)) / np.sqrt(2)
    z = rng.uniform(-a_noise, a_noise, n) + 1j * rng.uniform(-a_noise, a_noise, n)
    bw = 0.35 * min(rate_in, ro)
    for a, f in tones:
        f = off + (rng.uniform(-bw, bw) if f is None else f * min(rate_in, ro))
        z += a * amplitude / np.sqrt(2) * np.exp(2j * np.pi * (f * t % rate_in) / rate_in + 1j * rng.uniform(0, 2 * np.pi))
    return z


def narrow_bytes(z) -> np.ndarray:
    """uint8 IQ of z in s units (s = 2u - 255)."""
    u = np.empty(2 * z.size, dtype=np.uint8)
    u[0::2] = np.clip(np.round((z.real + 255) / 2), 0, 255)
    u[1::2] = np.clip(np.round((z.imag + 255) / 2), 0, 255)
    return u


def s_of_bytes(u) -> np.ndarray:
    u = np.asarray(u, dtype=np.float64)
    return (2 * u[0::2] - 255) + 1j * (2 * u[1::2] - 255)


def wide_pairs(z) -> np.ndarray:
    sw = np.empty(2 * z.size, dtype=np.int32)
    sw[0::2], sw[1::2] = np.clip(np.round(z.real), -16383, 16383), np.clip(np.round(z.imag), -16383, 16383)
    return sw


def amplitude_of(mp) -> float:
    """Largest component of the input such that no stage clips: 100 s units on the narrow path (|y| <= 2.5 * 141 <
    2 * 127.5 at the worst sum |c| / 2^S of 2.5); on the wide path an output within 100 LSB of 128."""
    if mp["k"] is None:
        return 100.0
    return min(12000.0, 100.0 * 2.0 ** ir.WIDE_BITS / 2.0 ** mp["k"] / 2.5)


def restated(plan, mp, data):
    """The restatement's decoder bytes for the whole input."""
    ro = DATA_RATE * plan["cl"]
    if mp["k"] is not None:
        return wide_ref.Wide(plan["rate_in"], ro, plan["offset"], mp["k"]).feed(data)[0]
    if plan["offset"] is None:
        return resample_ref.resample(data, plan["rate_in"], ro)
    if plan["mode"] == "decimating":
        return decimate_ref.decimate(data, plan["rate_in"], ro, plan["offset"])
    return tune_ref.tune(data, plan["rate_in"], ro, plan["offset"])


def run(plan, n_out, tones=((0.55, None), (0.45, None)), perturb=None, amplitude=None):
    """(errors, budget, plan of the model) of the restatement's first n_out or so outputs against the model."""
    mp = model_plan(plan)
    rng = np.random.default_rng(plan["seed"])
    x_in = int(n_out * plan["rate_in"] / (DATA_RATE * plan["cl"])) + mp["T"] + mp["D"] * mp["T1"] + 16
    z = channel(plan, x_in, rng, amplitude or amplitude_of(mp), tones)
    if mp["k"] is None:
        data = narrow_bytes(z)
        s = s_of_bytes(data)
    else:
        data = wide_pairs(z)
        s = data[0::2] + 1j * data[1::2].astype(np.float64)
    got = restated(plan, mp, data)
    want = ir.model(mp, s, x_in, perturb)
    assert got.size == want.size > 0, (plan, got.size, want.size)
    assert got.min() > 0 and got.max() < 255, plan     # nothing clipped
    return ir.errors(got, want, ir.centre(mp), ir.single_tap(mp, got.size // 2)), ir.budget(mp, s, x_in), mp


def _check(plan, n_out=1500):
    err, b, mp = run(plan, n_out)
    assert not ir.failures(err, b), (plan, mp, err, b, ir.failures(err, b))
    return err, b, mp


@pytest.mark.parametrize("mode", MODES)
def test_sweep_against_the_model(built, mode):
    """Every plan of the mode's sweep: max |err| within the budget, each component's mean within 0.02 LSB, no phase
    between the error and the signal; the budget below 1 LSB on the untuned path; the mixer step the nearest one."""
    worst = {}
    for plan in sweep(mode):
        err, b, mp = _check(plan)
        if mp["W"] or plan["offset"] is not None:
            assert ir.nco_offset_error(mp) <= mp["R_in"] / 2.0 ** 33, (plan, mp)
        if mode == "untuned":
            assert b["total"] < 1.0, (plan, b)
        for key, v in (("max", err["max"]), ("budget", b["total"]), ("mean", max(abs(err["mean_i"]), abs(err["mean_q"])))):
            worst[key] = max(worst.get(key, 0.0), v)
    print(mode, {k: round(v, 4) for k, v in worst.items()})


def test_sweep_covers_the_edges(built):
    """The sweep holds every edge of each rule, every chip length, offsets 0, +-1 and the largest, and both sides of
    the cascade's D steps."""
    for mode in MODES:
        plans = sweep(mode)
        mps = [model_plan(p) for p in plans]
        assert {p["cl"] for p in plans} == set(CHIP_LENGTHS), mode
        for cl in CHIP_LENGTHS:
            rates = {p["rate_in"] for p in plans if p["cl"] == cl}
            assert set(edge_rates(mode, DATA_RATE * cl)) <= rates, (mode, cl)
        if mode != "untuned":
            offs = {p["offset"] for p in plans}
            assert {0, 1, -1} <= offs, mode
            assert any(abs(p["offset"]) == offset_limit(p["rate_in"], DATA_RATE * p["cl"]) for p in plans), mode
        if mode in ("decimating", "wide_dec"):
            assert {m["D"] for m in mps} >= {3, 4, 16, 17, 37, 38, 64}, mode
            assert all(m["D"] > 1 for m in mps), mode
        else:
            assert all(m["D"] == 1 for m in mps), mode
        if mode in ("tuned", "wide"):
            assert {m["P"] for m in mps} >= {256, 128, 64}, mode


def test_model_tables_are_the_handles(built):
    """The model's own integer table and stage-1 taps (rebuilt from the header comment's definition for the budget) are
    the ones the handle reports, so the budget's coefficient term describes the coefficients the kernels apply."""
    for mode in MODES:
        for plan in sweep(mode)[::10]:
            h = handle(plan)
            mp = ir.plan_from_handle(h, plan["k"])
            _, tab = h.resampler()
            assert np.array_equal(tab.reshape(mp["P"] + 1, mp["T"]), ir.table(mp)), plan
            if mp["D"] > 1:
                assert np.array_equal(h.decimator()[1], ir.stage1_taps(mp)), plan
            h.close()


# ---------------------------------------------------------------- the comparison has teeth
def _fixed(mode, cl, rate_in, offset=None, k=None, seed=7):
    return {"mode": mode, "i": -1, "cl": cl, "rate_in": rate_in, "offset": offset, "k": k, "seed": seed}


R72 = DATA_RATE * 72
TEETH_PLANS = {
    "untuned": _fixed("untuned", 72, 2_400_000),
    "untuned_up": _fixed("untuned", 72, R72 // 4 + 1),
    "tuned": _fixed("tuned", 72, 8_000_001, 1_234_567),
    "tuned_near": _fixed("tuned", 72, 2_400_000, 200_000),
    "decimating": _fixed("decimating", 32, 30_720_000, -2_400_000),
    "wide": _fixed("wide", 72, 10_000_000, -2_400_000, k=2),
    "wide_dec": _fixed("wide_dec", 72, 61_440_000, 5_000_000, k=1),
}
PERTURBATIONS = [("shift_1_over_P", "untuned"), ("shift_1_over_P", "untuned_up"), ("shift_1_over_P", "tuned_near"),
                 ("shift_1_sample", "untuned"), ("shift_1_sample", "decimating"), ("shift_1_sample", "wide"),
                 ("row_wrong_way", "untuned"), ("row_wrong_way", "untuned_up"), ("row_wrong_way", "tuned_near"),
                 ("conjugate", "tuned"), ("conjugate", "decimating"), ("conjugate", "wide"),
                 ("nco_half", "tuned"), ("nco_half", "tuned_near"), ("nco_half", "decimating"), ("nco_half", "wide"),
                 ("stage1_centre", "decimating"), ("stage1_centre", "wide_dec"),
                 ("floor", "untuned"), ("floor", "tuned"), ("floor", "decimating"), ("floor", "wide_dec")]
TEETH_TONES = ((0.7, 0.38), (0.2, -0.3))    # strong tones near the band edge, a little noise
TEETH_OUTPUTS = 60_000


@functools.lru_cache(maxsize=None)
def _teeth_input(name):
    plan = TEETH_PLANS[name]
    mp = model_plan(plan)
    rng = np.random.default_rng(plan["seed"])
    x_in = int(TEETH_OUTPUTS * plan["rate_in"] / (DATA_RATE * plan["cl"])) + mp["T"] + mp["D"] * mp["T1"] + 16
    z = channel(plan, x_in, rng, amplitude_of(mp), TEETH_TONES)
    if mp["k"] is None:
        data = narrow_bytes(z)
        s = s_of_bytes(data)
    else:
        data = wide_pairs(z)
        s = data[0::2] + 1j * data[1::2].astype(np.float64)
    got = restated(plan, mp, data)
    return mp, s, x_in, got, ir.budget(mp, s, x_in)


@pytest.mark.parametrize("name", sorted(TEETH_PLANS))
def test_teeth_plans_pass_unperturbed(built, name):
    mp, s, x_in, got, b = _teeth_input(name)
    err = ir.errors(got, ir.model(mp, s, x_in), ir.centre(mp), ir.single_tap(mp, got.size // 2))
    assert not ir.failures(err, b), (name, err, b)


@pytest.mark.parametrize("perturb,name", PERTURBATIONS)
def test_perturbed_model_fails(built, perturb, name):
    """A model that is wrong in one of the ways a kernel or the header could be -- output time late by 1/P or by one
    input sample, interpolation towards the wrong neighbour row, the mixer conjugated or off by half an entry, the first
    stage centred at nD + 1, floor in place of round -- fails the comparison the sweep passes."""
    mp, s, x_in, got, b = _teeth_input(name)
    err = ir.errors(got, ir.model(mp, s, x_in, perturb), ir.centre(mp), ir.single_tap(mp, got.size // 2))
    assert ir.failures(err, b), (perturb, name, err, b)
