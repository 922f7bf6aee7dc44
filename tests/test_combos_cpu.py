"""CPU tests of tests/combo_ref.py: the configuration list is fixed and every entry is one the library accepts, the
coverage cells of test_gpu_combos are reachable from it, the composed restatement equals the per-stage restatements as
their own tests call them, call by call expectations are prefixes of the one-stream computation, and the comparisons
reject plausible wrong answers built from the restatement itself."""
import json

import numpy as np
import pytest

import combo_ref as cr
import decimate_ref
import resample_ref
import signal_ref
import spectrum_ref
import tune_ref
import wide_ref
from helpers import cand_key_oracle, oracle_run, rule_violated
from rtlamr_b200 import capi
from test_sigmf import convert

R72 = cr.DATA_RATE * 72


def _all():
    return cr.configs() + [c for f in cr.FORMATS for c in cr.sweep_configs(f)]


def test_generator_is_deterministic(built):
    a, b = cr.configs(), cr.configs()
    assert json.dumps(a) == json.dumps(b)
    assert len(cr.fixed_configs()) == cr.N_FIXED and len(a) == cr.N_FIXED + cr.N_RANDOM and len({c["name"] for c in a}) == len(a)
    rnd = [c for c in a if c["name"].startswith("random")]
    assert all(1 <= len(c["protocols"]) <= 4 and len(set(c["protocols"])) == len(c["protocols"]) for c in rnd)
    assert sum(bool({"r900", "r900bcd"} & set(c["protocols"])) for c in rnd) * 3 >= len(rnd)
    assert any(c["cl"] in cr.GENERIC_CL for c in rnd) and any(c["cl"] in cr.SPECIALISED_CL for c in rnd)
    assert any(c["scale"] for c in rnd) and any(c["flags"] for c in rnd) and any(c["before_start"] for c in rnd)
    assert any(isinstance(k, str) for c in rnd if c["ks"] for k in c["ks"])
    assert {c["mode"] for c in rnd} == set(cr.MODES)


def test_every_configuration_passes_the_plan_rules(built):
    for cfg in _all():
        what = json.dumps(cfg)
        ro = cr.rate_out(cfg)
        assert rule_violated(cr.protos(cfg)) is None, what
        if cfg["mode"] in cr.TUNED:
            assert all(0 < abs(o) <= cr._offset_limit(cfg["rate_in"], ro) for o in cfg["offsets"]), what
            assert len(set(cfg["offsets"])) == len(cfg["offsets"]) <= 64, what
        else:
            assert cr.group_size(cfg) == 1, what
        for i in range(cr.group_size(cfg)):
            dec, info = cr.plan(cfg, i)
            h = cr.configure(cfg, i)   # the ABI's own plan, before allocate (no device)
            if info is None:
                with pytest.raises(capi.ErtGpuError):
                    h.resampler()
            else:
                assert h.resampler()[0] == info, what
            if dec is not None:
                assert h.decimator()[0] == dec, what
            if cfg["mode"] in cr.WIDE:
                w = wide_ref.Wide(cfg["rate_in"], ro, cfg["offsets"][i])
                assert w.info == info and (dec is None or w.dec == dec), what
            h.close()
        # the cut plan: increasing, to the end, whole blocks natively, device calls within max_blocks
        ends = [c[0] for c in cfg["cuts"]]
        assert ends == sorted(set(ends)) and ends[0] > 0 and ends[-1] == cfg["nsamples"], what
        assert {c[1] for c in cfg["cuts"]} <= set(cr.PATHS), what
        if cfg["mode"] in ("pass", "convert"):
            assert all(e % cr.geometry(cfg)["BS"] == 0 for e in ends), what
        mb = cr.max_blocks_effective(cfg)
        for x, (y, path) in zip([0] + ends, cfg["cuts"]):
            if path == "device":
                assert cr.blocks_after(cfg, y) - cr.blocks_after(cfg, x) <= mb, what


def test_the_fixed_edges(built):
    cfgs = {c["name"]: c for c in cr.fixed_configs()}
    info = {n: cr.plan(c)[1] for n, c in cfgs.items()}
    dec = {n: cr.plan(c)[0] for n, c in cfgs.items()}
    assert info["untuned_4_to_1_up"]["L"] == 4 * info["untuned_4_to_1_up"]["M"]
    assert info["untuned_1_to_4_down"]["M"] == 4 * info["untuned_1_to_4_down"]["L"]
    co = info["untuned_coprime_2_4M"]
    assert np.gcd(co["L"], co["M"]) == 1 and 2_300_000 < co["L"] < co["M"] < 2_500_000
    assert (info["tuned_10_to_1_T218"]["T"], info["tuned_10_to_1_T218"]["P"]) == (218, 64)
    assert cfgs["tuned_10_to_1_T218"]["rate_in"] == 10 * R72
    for t, p in ((96, 256), (98, 128), (160, 128), (162, 64)):
        assert (info[f"tuned_T{t}"]["T"], info[f"tuned_T{t}"]["P"]) == (t, p)
    assert info["tuned_interpolating_1_to_4"]["L"] == 4 * info["tuned_interpolating_1_to_4"]["M"]
    assert [dec[n]["D"] for n in ("decimating_D64", "decimating_D4", "decimating_D5")] == [64, 4, 5]
    assert cfgs["decimating_cl8"]["cl"] == 8 and dec["decimating_cl8"]["D"] > 1
    w = cfgs["wide_r900_cl32"]
    assert w["mode"] == "wide" and w["cl"] == 32 and "r900" in w["protocols"]


def test_coverage_cells_are_reachable(built):
    missing = cr.all_cells() - cr.planned_cells()
    assert not missing, sorted(missing)


def _first_of(mode, pred=lambda c: True):
    return next(c for c in cr.configs() if c["mode"] == mode and pred(c))


@pytest.mark.parametrize("mode", cr.MODES)
def test_expected_equals_the_per_stage_restatements(built, mode):
    cfg = _first_of(mode, lambda c: c["nsamples"] <= 1_500_000)
    raw = cr.capture(cfg)
    exp = cr.expected(cfg, raw)
    ro, fmt, off = cr.rate_out(cfg), cfg["fmt"], cfg["offsets"][0]
    u8c = convert(raw, fmt, cfg["scale"])
    if mode in ("pass", "convert"):
        want = u8c
    elif mode == "resample":
        want = resample_ref.resample(u8c, cfg["rate_in"], ro)
    elif mode in cr.WIDE:
        want, _ = wide_ref.wide(raw, fmt, cfg["rate_in"], ro, off, exp["members"][0]["k"], cfg["scale"])
    elif cr.plan(cfg)[0] is not None and cr.plan(cfg)[0]["D"] > 1:
        want = decimate_ref.decimate(u8c, cfg["rate_in"], ro, off)
    else:
        want = tune_ref.tune(u8c, cfg["rate_in"], ro, off)
    m = exp["members"][0]
    bs2 = 2 * cr.geometry(cfg)["BS"]
    assert np.array_equal(m["bytes"], want[:want.size // bs2 * bs2])
    # the candidates are the oracle's (helpers.oracle_run), their records signal_ref.record over the whole stream
    geo = cr.geometry(cfg)
    _, cands, _ = oracle_run(cfg["protocols"], cfg["cl"], m["bytes"])
    nbytes = (geo["PK"] + 7) >> 3
    ok = [k for k, _ in m["cands"]]
    want_keys = sorted(cand_key_oracle(c, nbytes, geo["PK"]) for c in cands
                       if not cfg["flags"] or any(k[:4] == cand_key_oracle(c, nbytes, geo["PK"]) for k in ok))
    assert sorted(k[:4] for k in ok) == want_keys
    if cfg["signal"]:
        ps = cr.protos(cfg)
        for key, rec in m["cands"][:40]:
            data = next(c.data[:nbytes] for c in cands if (c.block, c.preamble_id, c.idx) == key[:3])
            whole = signal_ref.record(m["bytes"], key[0], key[2], key[1], key[4], data, ps)
            assert rec == tuple(whole[f] for f in signal_ref.FIELDS)


def _feed_calls(cfg, raw, member=0, k=None):
    """The member's decoder bytes fed to the restatement call by call."""
    ro, fmt, s = cr.rate_out(cfg), cfg["fmt"], cr.sample_bytes(cfg)
    off = cfg["offsets"][member]
    if cfg["mode"] in cr.WIDE:
        st = wide_ref.Wide(cfg["rate_in"], ro, off, k)
        step = lambda part: st.feed(wide_ref.wide_components(part, fmt, cfg["scale"]))[0]  # noqa: E731
    else:
        if cfg["mode"] in ("pass", "convert"):
            st = None
        elif cfg["mode"] == "resample":
            st = resample_ref.Resampler(cfg["rate_in"], ro)
        elif cfg["allow_decimation"]:
            st = decimate_ref.Cascade(cfg["rate_in"], ro, off)
        else:
            st = tune_ref.Tuner(cfg["rate_in"], ro, off)
        step = lambda part: convert(part, fmt, cfg["scale"]) if st is None else st.feed(convert(part, fmt, cfg["scale"]))  # noqa: E731
    out, x = [], 0
    for y, _ in cfg["cuts"]:
        out.append(step(raw[x * s:y * s]))
        x = y
    return out


@pytest.mark.parametrize("name", ["untuned_coprime_2_4M", "tuned_interpolating_1_to_4", "decimating_D4", "decimating_D64",
                                  "wide_r900_cl32", "tuned_T162"])
def test_split_invariance(built, name):
    cfg = next(c for c in cr.fixed_configs() if c["name"] == name)
    raw = cr.capture(cfg)
    exp = cr.expected(cfg, raw)
    bs = cr.geometry(cfg)["BS"]
    for i, m in enumerate(exp["members"]):
        parts = _feed_calls(cfg, raw, i, m["k"])
        outs = np.cumsum([p.size // 2 for p in parts])
        assert [cr.outputs_after(cfg, e) for e in exp["ends"]] == outs.tolist()
        assert np.array_equal(np.concatenate(parts)[:m["bytes"].size], m["bytes"])
        got_b, got_c, got_rows = [], [], []
        for c in range(len(cfg["cuts"])):
            e = cr.call_expectation(cfg, exp, i, c)
            assert e["b1"] == outs[c] // bs
            got_b.append(e["bytes"])
            got_c += e["cands"]
            if "rows" in e:
                got_rows += [r for r in e["rows"][0] if r[1] == cfg["spectrum"][1]]
        assert np.array_equal(np.concatenate(got_b), m["bytes"])
        assert sorted(got_c) == sorted(m["cands"])
        if "spectrum" in m:
            whole = spectrum_ref.rows_of_powers(m["spectrum"], cfg["spectrum"][1])
            assert got_rows == whole[0] and len(whole[0]) >= 2


def _sensitivity_case():
    cfg = cr.make_config("sensitivity", 77, mode="tuned", protocols=["scm", "r900"], cl=72, rate_in=10_000_000,
                         offsets=[-2_000_000], signal=True, fmt=capi.FORMAT_CS16, nsamples=1_000_000)
    raw = cr.capture(cfg)
    return cfg, raw, cr.expected(cfg, raw)


def test_comparisons_reject_wrong_answers(built):
    cfg, raw, exp = _sensitivity_case()
    m = exp["members"][0]
    u8, want = m["bytes"], sorted(m["cands"])
    assert len(want) > 10 and any(k[5] for k, _ in want) and any(k[4] for k, _ in want)
    cr.assert_bytes(u8, u8)
    cr.assert_candidates([k for k, _ in want], [r for _, r in want], want)
    # decoder bytes shifted by one sample: other bytes and other candidates
    shifted = np.concatenate([u8[2:], u8[:2]])
    with pytest.raises(AssertionError):
        cr.assert_bytes(shifted, u8)
    wrong = cr.oracle_candidates(cfg, shifted)
    with pytest.raises(AssertionError):
        cr.assert_candidates([k for k, _ in wrong], None, [(k, None) for k, _ in want])
    # I and Q swapped
    swapped = u8.reshape(-1, 2)[:, ::-1].ravel()
    with pytest.raises(AssertionError):
        cr.assert_bytes(swapped, u8)
    # the NCO's sign flipped
    flipped = dict(cfg, offsets=[-cfg["offsets"][0]])
    with pytest.raises(AssertionError):
        cr.assert_bytes(cr.decoder_bytes(flipped, raw)[:u8.size], u8)
    # a signal record computed with the wrong history in front of its call: the call starts at the candidate's block
    ps = cr.protos(cfg)
    bs = cr.geometry(cfg)["BS"]
    key, rec = next((k, r) for k, r in want if k[0] > 8 and k[4])
    bad = u8.copy()
    bad[:2 * key[0] * bs] = np.roll(bad[:2 * key[0] * bs], 2 * bs)   # the previous call's bytes, one block late
    assert cr.signal_of(bad, key, _data(cfg, key, u8), ps) != rec
    with pytest.raises(AssertionError):
        cr.assert_candidates([k for k, _ in want], [cr.signal_of(bad, k, _data(cfg, k, u8), ps) if k == key else r
                                                    for k, r in want], want)
    # an r900 digit off by one
    i = next(j for j, (k, _) in enumerate(want) if k[5])
    k = want[i][0]
    dig = bytearray(k[6])
    dig[17] = (dig[17] + 1) % 6
    keys = [x for x, _ in want]
    keys[i] = k[:6] + (bytes(dig),)
    with pytest.raises(AssertionError):
        cr.assert_candidates(keys, [r for _, r in want], want)


def _data(cfg, key, u8):
    return next(d for k, d in cr.oracle_candidates(cfg, u8) if k == key)


def test_wide_gain_off_by_one_is_rejected(built):
    cfg = next(c for c in cr.fixed_configs() if c["name"] == "wide_r900_cl32")
    raw = cr.capture(cfg)
    k = cfg["ks"][0]
    u8 = cr.decoder_bytes(cfg, raw, 0, k)
    for other in (k - 1, k + 1):
        with pytest.raises(AssertionError):
            cr.assert_bytes(cr.decoder_bytes(cfg, raw, 0, other), u8)


def test_special_values_reach_every_format(built):
    """The sweep's captures hold every special value of their format, and the restatement maps them inside the byte and
    wide ranges (NaN to 0, the clamps at +-16383)."""
    for fmt in cr.FORMATS:
        raw = cr.special_raw(fmt, 4096, 900 + fmt)
        dt = np.dtype(cr.LAYOUT[fmt][0])
        v, sp = raw.view(dt), cr.special_values(fmt)
        for x in sp:
            assert (np.isnan(v).any() if np.isnan(x) else (v.view(f"u{dt.itemsize}") == np.array([x], dt).view(
                f"u{dt.itemsize}")[0]).any()), (fmt, x)
        sw = wide_ref.wide_components(raw, fmt)
        assert np.abs(sw).max() == (64 * 255 if fmt == capi.FORMAT_CU8 else wide_ref.WIDE_MAX)
