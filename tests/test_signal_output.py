"""CPU tests of the -signal output fields: the parsers' messages with their candidates' signal records through
ertgpu_decode_file's plain line and the csv, json and xml encoders (libertgpu_host.so, no device), against the same
messages without reports."""
import json
import xml.etree.ElementTree as ET

import numpy as np
import pytest

import signal_ref
from rtlamr_b200 import capi, host, synth

CHANNEL, RATE = 912_600_155, 32768 * 72


def _case():
    """Two valid scm candidates: one whose record has a summary, one (a packet before the stream) without."""
    data = synth.encode_scm(12345678, 7, 1, 2, 987654)
    cands = np.zeros(2, dtype=capi.CAND_DTYPE)
    for i, (block, idx) in enumerate([(3, 100), (9, 2000)]):
        cands[i]["block"], cands[i]["idx"], cands[i]["check_mask"] = block, idx, 1
        cands[i]["bytes"][:len(data)] = np.frombuffer(data, dtype=np.uint8)
    sigs = np.zeros(2, dtype=capi.SIGNAL_DTYPE)
    sigs[0] = (3420, 3420 * 20000, 3420, 3420 * 200, 10**9, 2 * 10**8, 3325, 0, 95)
    sigs[1]["symbols"] = 95
    return cands, sigs


def _want(sig):
    return signal_ref.summary({f: int(sig[f]) for f in signal_ref.FIELDS}, CHANNEL, RATE)


@pytest.fixture(scope="module")
def parsers(built):
    p = host.Parsers("scm", 72)
    yield p
    p.close()


def test_plain(parsers):
    cands, sigs = _case()
    lines = parsers.encode_signal(cands, sigs, CHANNEL, RATE, "plain").splitlines()
    s = _want(sigs[0])
    assert lines[0].startswith(f"{{Block:3 Idx:100 Channel:{CHANNEL} Freq:{s['freq']} Level:{s['level']:.2f} "
                               f"Noise:{s['noise']:.2f} SNR:{s['snr']:.2f} SCM:{{ID:")
    assert lines[1].startswith("{Block:9 Idx:2000 Channel:- Freq:- Level:- Noise:- SNR:- SCM:{ID:")
    # the message's own part is the line without reports
    plain = [m.text for m in parsers.parse(cands)]
    assert [ln.split(" SCM:", 1)[1] for ln in lines] == [t + "}" for t in plain]


def test_csv(parsers):
    cands, sigs = _case()
    rows = [ln.split(",") for ln in parsers.encode_signal(cands, sigs, CHANNEL, RATE, "csv").splitlines()]
    base = [ln.split(",") for ln in parsers.encode(cands, "csv").splitlines()]
    s = _want(sigs[0])
    assert rows[0] == base[0] + [str(CHANNEL), str(s["freq"]), f"{s['level']:.2f}", f"{s['noise']:.2f}", f"{s['snr']:.2f}"]
    assert rows[1] == base[1] + [""] * 5


def test_json(parsers):
    cands, sigs = _case()
    got = [json.loads(ln) for ln in parsers.encode_signal(cands, sigs, CHANNEL, RATE, "json").splitlines()]
    base = [json.loads(ln) for ln in parsers.encode(cands, "json").splitlines()]
    assert [list(g) for g in got] == [list(b) + ["Signal"] for b in base]
    s = _want(sigs[0])
    assert got[0]["Signal"] == {"Channel": CHANNEL, "Freq": s["freq"], "Level": round(s["level"], 2),
                                "Noise": round(s["noise"], 2), "SNR": round(s["snr"], 2)}
    assert got[1]["Signal"] is None
    for g, b in zip(got, base):
        del g["Signal"]
        assert g == b


def test_xml(parsers):
    cands, sigs = _case()
    got = [ET.fromstring(ln) for ln in parsers.encode_signal(cands, sigs, CHANNEL, RATE, "xml").splitlines()]
    base = parsers.encode(cands, "xml").splitlines()
    s = _want(sigs[0])
    assert [c.tag for c in got[0]] == ["Message", "Signal"]
    assert got[0].find("Signal").attrib == {"Channel": str(CHANNEL), "Freq": str(s["freq"]), "Level": f"{s['level']:.2f}",
                                            "Noise": f"{s['noise']:.2f}", "SNR": f"{s['snr']:.2f}"}
    assert got[1].find("Signal").attrib == {}
    for g, b in zip(got, base):
        g.remove(g.find("Signal"))
        assert ET.tostring(g) == ET.tostring(ET.fromstring(b))


def test_without_reports_nothing_changes(parsers):
    """The messages of a decoder without reports carry none: every encoder writes exactly what it wrote before."""
    cands, _ = _case()
    for fmt in ("csv", "json", "xml"):
        assert "Signal" not in parsers.encode(cands, fmt) and "912600155" not in parsers.encode(cands, fmt)
    assert all(m.signal is None for m in parsers.parse(cands))
