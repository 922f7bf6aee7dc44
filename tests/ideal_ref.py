"""A float64 model of the input stage: the tuned mixer, the decimating first stage, the resampler and the decoder's
byte, written from the definitions in the resampler header's comments and in DESIGN.md §3.7-3.12.  It
evaluates the Kaiser-windowed sinc with numpy and scipy and places every output at its exact rational input time; it
uses none of the header's code and none of the CPU restatements.  Next to it, the error budget of each mode: how far
the integer design may lie from the model, computed from the plan.

Units.  A stage's input is a complex array s in that path's integer units: s = 2u - 255 (u the converted byte, I and Q)
on the narrow path, the wide components s_w on the wide one; samples before the stream start are 0.  Every function
returns unrounded values.  A plan is a dict (plan_from_handle) of what the C ABI reports: the second (or only) stage's
rate_in, rate_out, L, M, T, P; D and T1 of the first stage (D = 1: none); the mixer step W and the offset; the channel
gain k of the wide path (None: narrow)."""
from __future__ import annotations

import numpy as np
from scipy.special import i0

S = 14                       # DC gain 2^S of the integer filters
F = 16                       # bits of the interpolation weight
NCO_N = 4096                 # entries of the mixer's phase table
WIDE_BITS = 7                # s_w = rint(x g 2^7)
BETA = 0.1102 * (70.0 - 8.7)  # Kaiser window of 70 dB
CHUNK = 4096                 # outputs per vectorised block


def kaiser_sinc(d, fc, half):
    """2 fc sinc(2 fc d) w(d / half) for |d| < half, else 0: the Kaiser-windowed sinc of unit DC gain cut off at fc
    cycles per sample, w(z) = I0(BETA sqrt(1 - z^2)) / I0(BETA)."""
    d = np.asarray(d, dtype=np.float64)
    z = np.clip(d / half, -1.0, 1.0)
    w = i0(BETA * np.sqrt(1.0 - z * z)) / i0(BETA)
    return np.where(np.abs(d) < half, 2.0 * fc * np.sinc(2.0 * fc * d) * w, 0.0)


def _round_half_away(v):
    return np.where(v >= 0, np.floor(v + 0.5), -np.floor(-v + 0.5)).astype(np.int64)


# ---------------------------------------------------------------- the plan
def plan_from_handle(h, k=None) -> dict:
    """The model's parameters from a configured handle (allocated or not): ertgpu_get_resampler, ertgpu_get_decimator
    (when the handle allows decimation) and ertgpu_get_tuning (when it is tuned).  k: the wide path's channel gain."""
    from rtlamr_b200 import capi
    info, _ = h.resampler()
    try:
        dec, _ = h.decimator()
    except capi.ErtGpuError:
        dec = {"D": 1, "T1": 0}
    try:
        t = h.tuning()
        W, offset = int(t["nco_step"]), int(t["offset_hz"])
    except capi.ErtGpuError:
        W, offset = 0, 0
    p = {key: int(info[key]) for key in ("rate_in", "rate_out", "L", "M", "T", "P")}
    p.update(D=int(dec["D"]), T1=int(dec["T1"]), W=W, offset=offset, k=k)
    p["R_in"] = p["rate_in"]   # the capture's rate (stage 2 of a cascade reports R_in -> D R_out)
    p["R_out"] = p["rate_out"] // p["D"]
    return p


def nco_offset_error(p) -> float:
    """|W R_in / 2^32 - offset| in Hz, W read as a signed step: at most R_in / 2^33 when W is the nearest step."""
    w = p["W"] - (1 << 32) if p["W"] >= 1 << 31 else p["W"]
    return abs(w * p["R_in"] / 2.0 ** 32 - p["offset"])


def stage1_fc(p) -> float:
    """Cut-off of the first stage, cycles per input sample: midway between the passband edge 0.4 R_out and the stopband
    edge R_mid - 0.6 R_out, R_mid = R_in / D."""
    mid = p["R_in"] / p["D"]
    return 0.5 * (0.4 * p["R_out"] + mid - 0.6 * p["R_out"]) / p["R_in"]


def stage2_nu(p) -> float:
    """min(R_in, R_out) of the resampler in cycles per input sample: its cut-off is half of it."""
    return min(1.0, p["L"] / p["M"])


# ---------------------------------------------------------------- the model
def mix(s, W, *, sign=-1.0, index_offset=0.0):
    """s_g e^(-2 pi i ((g W) mod 2^32) / 2^32), g the index since the stream start.  sign and index_offset (in entries
    of the 4096-entry table) exist to perturb the model."""
    g = np.arange(s.size, dtype=np.uint64)
    phase = ((g * np.uint64(W)) % np.uint64(1 << 32)).astype(np.float64) / 2.0 ** 32 + index_offset / NCO_N
    return s * np.exp(sign * 2j * np.pi * phase)


def stage1_outputs(p, x: int) -> int:
    """Outputs of the first stage whose window lies inside the first x input samples."""
    a = x - p["T1"] // 2
    return 0 if a <= 0 else -(-a // p["D"])


def out_end(p, x: int) -> int:
    """Outputs of the resampler whose window lies inside the first x of its input samples."""
    a = x - p["T"] // 2
    return 0 if a <= 0 else -(-a * p["L"] // p["M"])


def stage1(p, s, n_out, *, centre_shift=0):
    """y1(n) = sum_d h1(d) s_(nD + d), h1 the first stage's Kaiser sinc over |d| <= T1/2 - 1 (its taps are symmetric
    about the output, and tap T1 - 1 is 0).  centre_shift moves the output time (perturbation)."""
    D, half = p["D"], p["T1"] // 2
    fc = stage1_fc(p)
    y = np.zeros(n_out, dtype=np.complex128)
    base = np.arange(n_out, dtype=np.int64) * D + centre_shift
    for d in range(-(half - 1), half):
        j = base + d
        ok = (j >= 0) & (j < s.size)
        y += kaiser_sinc(d, fc, p["T1"] / 2) * np.where(ok, s[np.clip(j, 0, s.size - 1)], 0)
    return y


def _window(p, n):
    """For outputs n (int64): k_n, the input indices j of T + 2 taps around the output (the outer two have weight 0
    unperturbed), and the exact numerators j L - n M of the distances (j L - n M) / L."""
    L, M, T = p["L"], p["M"], p["T"]
    k = n * M // L
    j = k[:, None] - T // 2 + np.arange(T + 2, dtype=np.int64)[None, :]
    return k, j, j * L - (n * M)[:, None]


def resample(p, x, n_out, *, shift=None):
    """y(n) = sum_j h(j - n M / L) x_j, h the Kaiser sinc of T taps cut off at half of min(R_in, R_out), x_j = 0 for
    j < 0; the distance j - n M / L from an exact integer numerator.  shift(n) (input samples, added to every output
    time) exists to perturb the model."""
    nu = stage2_nu(p)
    y = np.zeros(n_out, dtype=np.complex128)
    for a in range(0, n_out, CHUNK):
        n = np.arange(a, min(a + CHUNK, n_out), dtype=np.int64)
        _, j, num = _window(p, n)
        d = num / p["L"]
        if shift is not None:
            d = d - shift(n)[:, None]
        xs = np.where((j >= 0) & (j < x.size), x[np.clip(j, 0, x.size - 1)], 0)
        y[a:a + n.size] = (kaiser_sinc(d, 0.5 * nu, p["T"] / 2) * xs).sum(axis=1)
    return y


def model(p, s, x_in: int, perturb=None):
    """The channel at the resampler's output, unrounded, in the decoder's byte units, for the outputs whose windows lie
    inside the first x_in input samples: (y + 255) / 2 on the narrow path, y 2^k / 2^7 + 128 on the wide one, I and Q
    interleaved (float64).  perturb: one of the perturbations the tests use to show that the comparison rejects wrong
    answers ("shift_1_over_P", "shift_1_sample", "row_wrong_way", "conjugate", "nco_half", "stage1_centre", "floor")."""
    s = np.asarray(s, dtype=np.complex128)[:x_in]
    if p["W"]:
        s = mix(s, p["W"], sign=1.0 if perturb == "conjugate" else -1.0,
                index_offset=0.5 if perturb == "nco_half" else 0.0)
    x = s
    if p["D"] > 1:
        x = stage1(p, s, stage1_outputs(p, x_in), centre_shift=1 if perturb == "stage1_centre" else 0)
    shift = None
    if perturb == "shift_1_over_P":
        shift = lambda n: np.full(n.size, 1.0 / p["P"])
    elif perturb == "shift_1_sample":
        shift = lambda n: np.ones(n.size)
    elif perturb == "row_wrong_way":
        def shift(n):   # towards row p - 1: (p - w / 2^F) / P in place of (p + w / 2^F) / P = q / (P 2^F)
            phi = n * p["M"] - (n * p["M"] // p["L"]) * p["L"]
            q = phi * (p["P"] << F) // p["L"]
            return (q - 2 * (q & ((1 << F) - 1))) / float(p["P"] << F) - phi / p["L"]
    y = resample(p, x, out_end(p, x.size), shift=shift)
    out = np.empty(2 * y.size, dtype=np.float64)
    out[0::2], out[1::2] = y.real, y.imag
    if p["k"] is None:
        out = (out + 255.0) / 2.0
    else:
        out = out * 2.0 ** p["k"] / 2.0 ** WIDE_BITS + 128.0
    return out - 0.5 if perturb == "floor" else out


# ---------------------------------------------------------------- the integer coefficients, rebuilt
def table(p) -> np.ndarray:
    """The (P+1) x T int16 table as the header's comment defines it: row p holds round(2^S h(t - T/2 + 1 - p/P)) (half
    away from zero), each row sums to 2^S (rows below P/2 take the residual on tap T/2 - 1, row P/2 splits it over its
    two centre taps), and row P - p mirrors row p."""
    T, P = p["T"], p["P"]
    nu = stage2_nu(p)
    t = np.arange(T)
    rows = np.arange(P // 2)[:, None]
    tab = np.zeros((P + 1, T), dtype=np.int64)
    tab[:P // 2] = _round_half_away((1 << S) * kaiser_sinc((t - T // 2 + 1)[None, :] - rows / P, 0.5 * nu, T / 2))
    tab[:P // 2, T // 2 - 1] += (1 << S) - tab[:P // 2].sum(axis=1)
    h = _round_half_away((1 << S) * kaiser_sinc(np.arange(T // 2) - T // 2 + 1 - 0.5, 0.5 * nu, T / 2))
    tab[P // 2] = np.concatenate([h, h[::-1]])
    r = ((1 << S) - tab[P // 2].sum()) // 2
    tab[P // 2, T // 2 - 1] += r
    tab[P // 2, T // 2] += r
    tab[P // 2 + 1:] = tab[P // 2 - 1::-1, ::-1]
    return tab


def stage1_taps(p) -> np.ndarray:
    """The T1 int16 taps of the first stage: round(2^S h1(t - T1/2 + 1)) for t <= T1/2 - 1, mirrored about that tap,
    tap T1 - 1 = 0, the residual to 2^S on the centre."""
    T1 = p["T1"]
    c = T1 // 2 - 1
    h = _round_half_away((1 << S) * kaiser_sinc(np.arange(c + 1) - c, stage1_fc(p), T1 / 2))
    taps = np.zeros(T1, dtype=np.int64)
    taps[:c + 1] = h
    taps[c:T1 - 1] = h[::-1]
    taps[c] += (1 << S) - taps.sum()
    return taps


def coefficients(p, tab, n):
    """The integer coefficients of outputs n (int64) over the T taps j = k_n - T/2 + 1 ..., as the header's comment
    defines them: q = floor(phi P 2^F / L), c = row_p + floor(((row_(p+1) - row_p) w + 2^(F-1)) / 2^F), and the tap
    nearest the output time, T/2 - 1 + (p >= P/2), takes the residual to 2^S."""
    phi = n * p["M"] - (n * p["M"] // p["L"]) * p["L"]
    q = phi * (p["P"] << F) // p["L"]
    r, w = q >> F, q & ((1 << F) - 1)
    h0, h1 = tab[r], tab[r + 1]
    c = h0 + (((h1 - h0) * w[:, None] + (1 << (F - 1))) >> F)
    near = p["T"] // 2 - 1 + (r >= p["P"] // 2)
    c[np.arange(n.size), near] += (1 << S) - c.sum(axis=1)
    return c


def coefficient_norms(p, n_out):
    """(max over the outputs of sum_t |c_t - 2^S h(d_t)|, max of sum_t |c_t|) of the resampler's first n_out outputs."""
    tab = table(p)
    nu = stage2_nu(p)
    dev = l1 = 0.0
    for a in range(0, n_out, CHUNK):
        n = np.arange(a, min(a + CHUNK, n_out), dtype=np.int64)
        _, _, num = _window(p, n)
        ideal = (1 << S) * kaiser_sinc(num[:, 1:-1] / p["L"], 0.5 * nu, p["T"] / 2)
        c = coefficients(p, tab, n)
        dev = max(dev, float(np.abs(c - ideal).sum(axis=1).max()))
        l1 = max(l1, float(np.abs(c).sum(axis=1).max()))
    return dev, l1


# ---------------------------------------------------------------- the error budget
def budget(p, s, x_in: int) -> dict:
    """The largest |output - model| the integer design may show, in output LSBs, for input s (complex, the path's units)
    over its first x_in samples.  Each term is a bound computed from the plan and the input's largest magnitude:
      final      the last rounding, 0.5;
      coef       sum |c_int - c_ideal| max|x| / 2^S of the resampler (c_int rebuilt by table() and coefficients());
      mix        the mixer's error per component, e = 0.5 (the rounding of s') + |s| pi / 4096 (the phase of the nearest
                 of 4096 entries) + (|s_I| + |s_Q|) / 2^15 (the entries' rounding), through the filter's sum |c| / 2^S;
      stage1     a cascade's first stage: its coefficient and mixer terms as above with its taps, plus its output rounding
                 (one byte = 2 s units on the narrow path, 0.5 s_w on the wide one), through stage 2's sum |c| / 2^S.
    The sum of the terms in s (or s_w) units is converted to output LSBs: / 2 on the narrow path, * 2^k / 2^7 on the wide
    one."""
    s = np.asarray(s, dtype=np.complex128)[:x_in]
    mag = float(np.abs(s).max()) if s.size else 0.0
    comp = float(max(np.abs(s.real).max(), np.abs(s.imag).max())) if s.size else 0.0
    e_mix = 0.0
    if p["W"]:
        e_mix = 0.5 + mag * np.pi / NCO_N + float((np.abs(s.real) + np.abs(s.imag)).max()) / 2.0 ** 15
        comp = mag
    wide = p["k"] is not None
    terms = {}
    if p["D"] > 1:
        taps = stage1_taps(p)
        half = p["T1"] // 2
        ideal1 = (1 << S) * kaiser_sinc(np.arange(p["T1"]) - half + 1, stage1_fc(p), p["T1"] / 2)
        e1 = (np.abs(taps - ideal1).sum() * comp + np.abs(taps).sum() * e_mix) / 2.0 ** S + (0.5 if wide else 1.0)
        n1 = stage1_outputs(p, x_in)
        y1 = stage1(p, s if not p["W"] else mix(s, p["W"]), n1)
        x2 = float(max(np.abs(y1.real).max(), np.abs(y1.imag).max())) + e1 if n1 else 0.0
        e_in = e1
    else:
        n1, x2, e_in = x_in, comp, e_mix
    dev, l1 = coefficient_norms(p, out_end(p, n1))
    unit = 2.0 ** p["k"] / 2.0 ** WIDE_BITS if wide else 0.5
    terms["final"] = 0.5
    terms["coef"] = dev * x2 / 2.0 ** S * unit
    terms["mix" if p["D"] == 1 else "stage1"] = l1 * e_in / 2.0 ** S * unit
    terms["total"] = sum(terms.values())
    w = p["W"] - (1 << 32) if p["W"] >= 1 << 31 else p["W"]
    terms["mixer_turns"] = abs(w) * x_in / 2.0 ** 32
    frac = (p["M"] % p["L"]) / p["L"]
    terms["phase_turns"] = float("inf") if p["L"] == 1 else out_end(p, n1) * min(frac, 1.0 - frac)
    return terms


# ---------------------------------------------------------------- the comparison
def centre(p) -> float:
    """The byte of a zero channel: 127.5 on the narrow path, 128 on the wide one."""
    return 127.5 if p["k"] is None else 128.0


def single_tap(p, n_out) -> np.ndarray:
    """Outputs (of n_out) whose filter is the single tap 2^S: they sit on an input sample (phi_n = 0) and the cut-off is
    the input's Nyquist frequency (L >= M), where the sinc vanishes at every other sample."""
    n = np.arange(n_out, dtype=np.int64)
    return (n * p["M"] % p["L"] == 0) & (p["L"] >= p["M"])


def errors(got, want, centre, single=None) -> dict:
    """Statistics of got - want (bytes against model values, I and Q interleaved): max |err|, the mean of each
    component over the outputs that are not `single` (single_tap()), and the phase of the error against the signal,
    Im(sum e conj(y)) / sum |y|^2 with y the model's output about its centre, with its statistical spread
    rms|e| / sqrt(sum |y|^2).
    A single-tap output is the input sample itself, an integer in s (or s_w) units, so its byte is a rounding tie as
    often as that integer has the parity (or, on the wide path at k <= 6, the low bits) of a half: the narrow path
    rounds ties up, the wide path down (so that a constant cu8 input keeps its byte).  With an integer mixer in front
    (s' of either parity) that is a bias of +0.25 LSB on those outputs on the narrow path: every output of a tuned plan
    at R_in = R_out, a quarter of them at R_in = R_out / 4.  The budget bounds them sample by sample; the mean leaves
    them out."""
    e = np.asarray(got, dtype=np.float64) - want
    keep = np.ones(e.size // 2, dtype=bool) if single is None else ~np.asarray(single, dtype=bool)
    ec = e[0::2] + 1j * e[1::2]
    y = (want[0::2] - centre) + 1j * (want[1::2] - centre)
    power = float((np.abs(y) ** 2).sum()) or 1.0
    ei, eq = e[0::2][keep], e[1::2][keep]
    return {"n": int(ec.size), "max": float(np.abs(e).max()) if e.size else 0.0, "n_mean": int(keep.sum()),
            "mean_i": float(ei.mean()) if ei.size else 0.0, "mean_q": float(eq.mean()) if eq.size else 0.0,
            "rms": float(np.sqrt((e * e).mean())),
            "phase": float((ec * np.conj(y)).sum().imag / power),
            "phase_spread": float(np.sqrt((np.abs(ec) ** 2).mean()) / np.sqrt(power))}


MEAN_TOL = 0.02                  # LSB: a biased rounding or a floor shows as 0.5
PHASE_TOL = np.pi / NCO_N / 4    # rad: a mixer off by half an entry turns the channel by pi / 4096
SPREADS = 6                      # statistical allowance of the mean and the phase, in standard deviations
MIN_TURNS = 8                    # whole turns of the mixer over the input before its phase is judged


def phase_judged(b) -> bool:
    """The phase of the error is judged only where the rounding cannot follow the signal: the mixer is off or turns
    through MIN_TURNS cycles or more, and the outputs' sub-phases turn through MIN_TURNS cycles of [0, 1) or more (or
    all sit on input samples, L = 1).  Otherwise neighbouring samples share nearly one rotation or one sub-phase, and an
    integer s' or output byte snaps them back towards the unrotated or uninterpolated sample: a 1 Hz channel leaves
    s' = s for thousands of samples, and at R_in = R_out - 7 a tone at 0.3 R_in keeps a phase of 6e-3 rad through the
    output rounding.  Both errors are within the budget's rounding terms sample by sample."""
    return (b["mixer_turns"] == 0 or b["mixer_turns"] >= MIN_TURNS) and b["phase_turns"] >= MIN_TURNS


def failures(err, b) -> list:
    """The criteria err (errors()) fails under budget b (budget()): max |err| above the budget; a component's mean
    beyond MEAN_TOL plus SPREADS standard deviations of a mean of err["n"] values of spread rms; the phase of the error
    against the signal beyond PHASE_TOL plus SPREADS times its spread (when phase_judged)."""
    out = []
    if err["max"] > b["total"]:
        out.append(f"max |err| {err['max']:.4f} > budget {b['total']:.4f}")
    for c in ("mean_i", "mean_q"):
        if abs(err[c]) > MEAN_TOL + SPREADS * err["rms"] / np.sqrt(max(err["n_mean"], 1)):
            out.append(f"{c} {err[c]:+.4f}")
    if phase_judged(b) and abs(err["phase"]) > PHASE_TOL + SPREADS * err["phase_spread"]:
        out.append(f"phase {err['phase']:+.2e} rad (spread {err['phase_spread']:.1e})")
    return out
