"""ertgpu_decode_file's -format=json|xml, -samplefile, -single and -duration (rtlamr flags.go:37-58,140-170, main.go:225-287)
on the golden capture and on synthetic streams of every protocol."""
import json
import os
import re
import subprocess
import sys
import time
import xml.etree.ElementTree as ET

import pytest

from conftest import GOLDEN, ROOT
from helpers import synth_stream

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "rtlamr_b200", "ertgpu_decode_file")
SAMPLE = os.path.join(GOLDEN, "sample_cl78.bin")
ID_KEY = {"SCM": "ID", "SCM+": "EndpointID", "IDM": "ERTSerialNumber", "NetIDM": "ERTSerialNumber", "R900": "ID", "R900BCD": "ID"}
CASES = [("sample", "scm", 78), ("synth", "scm", 72), ("synth", "scm+", 72), ("synth", "idm", 72), ("synth", "netidm", 48),
         ("synth", "r900", 72), ("synth", "r900bcd", 32)]


def cli(*args, stdin=None):
    out = subprocess.run([CLI, *args], capture_output=True, text=True, timeout=300, stdin=stdin)
    assert out.returncode == 0, out.stderr
    return out.stdout.splitlines(), out.stderr


def case_file(kind, mt, cl, tmp_path):
    if kind == "sample":
        return SAMPLE
    iq, _, _ = synth_stream(mt, cl, 1 << 21, spacing=1 << 18)
    path = tmp_path / f"{mt}_{cl}.bin"
    iq.tofile(path)
    return str(path)


def plain_key(line):
    """(type, meter id) of a plain line {Block:.. Idx:.. TYPE:{...}}"""
    m = re.match(r"\{Block:\d+ Idx:\d+ ([A-Z0-9+a-z]+):\{(?:.*? )?(?:ID|EndpointID|ERTSerialNumber): *(\d+)", line)
    return m.group(1), int(m.group(2))


def xml_values(line):
    """LogMessage attributes and the message's fields (attributes and children, arrays as lists) of an XML line."""
    root = ET.fromstring(line)
    msg = root.find("Message")
    vals = {k: int(v) for k, v in msg.attrib.items()}
    for c in msg:
        v = c.text or ""
        v = int(v) if v.isdigit() else v
        if c.tag in vals:
            vals[c.tag] = (vals[c.tag] if isinstance(vals[c.tag], list) else [vals[c.tag]]) + [v]
        else:
            vals[c.tag] = v
    return root.attrib, vals


@pytest.mark.parametrize("kind,mt,cl", CASES)
def test_json_and_xml_carry_the_plain_messages(built, tmp_path, kind, mt, cl):
    path = case_file(kind, mt, cl, tmp_path)
    args = [f"-msgtype={mt}", f"-symbollength={cl}"]
    plain, _ = cli(*args, path)
    js, _ = cli(*args, "-format=json", path)
    xs, _ = cli(*args, "-format=xml", path)
    assert len(plain) == len(js) == len(xs) >= (14 if kind == "sample" else 4)
    for p, j, x in zip(plain, js, xs):
        j = json.loads(j)
        assert (j["Offset"], j["Length"]) == (0, 0)
        assert plain_key(p) == (j["Type"], j["Message"][ID_KEY[j["Type"]]])
        attrs, vals = xml_values(x)
        assert (attrs["Type"], attrs["Offset"], attrs["Length"]) == (j["Type"], "0", "0")
        tagged = j["Type"] in ("SCM", "SCM+")     # their checksum field carries the xml name Checksum
        jm = {("Checksum" if tagged and k in ("ChecksumVal", "PacketCRC") else k): v for k, v in j["Message"].items()}
        if j["Type"] == "IDM":      # []byte: base64 in JSON, escaped raw bytes in XML
            for k in ("TamperCounters", "PowerOutageFlags"):
                jm.pop(k), vals.pop(k)
        assert vals == jm
    if kind == "sample":
        assert json.loads(js[0])["Message"] == {"ID": 17580293, "Type": 8, "TamperPhy": 1, "TamperEnc": 1, "Consumption": 111414,
                                                "ChecksumVal": 0xD005}


def _sample_run(path, mt, cl, blocks, tmp_path):
    sf = tmp_path / f"samples_{blocks}.bin"
    lines, _ = cli(f"-msgtype={mt}", f"-symbollength={cl}", f"-blocks={blocks}", "-format=json", f"-samplefile={sf}", path)
    msgs = [json.loads(l) for l in lines]
    for m in msgs:
        m.pop("Time")
    return msgs, sf.read_bytes()


@pytest.mark.parametrize("kind,mt,cl", [("sample", "scm", 78), ("synth", "scm,scm+,idm,r900", 72)])
def test_samplefile_holds_every_message_and_ignores_blocks(built, tmp_path, kind, mt, cl):
    """main.go:225-230,279-284: every reported message points into the sample file at the sampleBuf dumped after its block,
    which decodes alone to the same message; the file and the offsets do not depend on how many blocks one call decodes."""
    path = case_file(kind, mt, cl, tmp_path)
    a, fa = _sample_run(path, mt, cl, 4096, tmp_path)
    b, fb = _sample_run(path, mt, cl, 1, tmp_path)
    c, fc = _sample_run(path, mt, cl, 3, tmp_path)
    assert a == b == c and fa == fb == fc
    assert len(a) >= 4
    spans = sorted({(m["Offset"], m["Length"]) for m in a})
    assert sum(n for _, n in spans) == len(fa)                     # one dump per block with messages, back to back
    assert all(o2 == o1 + n1 for (o1, n1), (o2, _) in zip(spans, spans[1:]))
    for off, n in spans:
        piece = tmp_path / f"piece_{off}.bin"
        piece.write_bytes(fa[off:off + n])
        again, _ = cli(f"-msgtype={mt}", f"-symbollength={cl}", "-format=json", str(piece))
        again = [json.loads(l)["Message"] for l in again]
        for m in a:
            if (m["Offset"], m["Length"]) == (off, n):
                assert m["Message"] in again, (off, n, m)
    # without -samplefile, Offset and Length stay 0 and nothing else changes
    plain, _ = cli(f"-msgtype={mt}", f"-symbollength={cl}", "-format=json", path)
    assert [json.loads(l)["Message"] for l in plain] == [m["Message"] for m in a]


def test_samplefile_offsets_grow_across_a_batch(built, tmp_path):
    """Every file of a batch starts with an empty sampleBuf; the files share one sample file."""
    sf = tmp_path / "batch.bin"
    one, _ = cli("-msgtype=scm", "-symbollength=78", "-format=csv", f"-samplefile={tmp_path / 'one.bin'}", SAMPLE)
    two, _ = cli("-msgtype=scm", "-symbollength=78", "-format=csv", f"-samplefile={sf}", SAMPLE, SAMPLE)
    single = (tmp_path / "one.bin").read_bytes()
    assert sf.read_bytes() == single + single
    strip = lambda l: l.split(",", 3)[1:]
    first = [strip(l) for l in one]
    second = [[str(int(o) + len(single)), n, rest] for o, n, rest in first]
    assert [strip(l) for l in two] == first + second


def test_single_stops_after_one_message(built, tmp_path):
    sf = tmp_path / "s.bin"
    lines, err = cli("-msgtype=scm", "-symbollength=78", "-single", "-format=json", f"-samplefile={sf}", SAMPLE)
    assert len(lines) == 1
    m = json.loads(lines[0])
    assert m["Message"]["ID"] == 17580293 and m["Offset"] == 0 and m["Length"] == sf.stat().st_size > 0
    assert "1 messages" in err


def test_single_with_filterid_waits_for_every_meter(built):
    every, _ = cli("-msgtype=scm", "-symbollength=78", SAMPLE)
    ids = [plain_key(l)[1] for l in every]
    a, b = ids[0], next(i for i in reversed(ids) if i != ids[0])
    lines, _ = cli("-msgtype=scm", "-symbollength=78", "-single", f"-filterid={a},{b}", SAMPLE)
    assert sorted(plain_key(l)[1] for l in lines) == sorted([a, b])
    # a meter that never transmits: every message of the listed ones is printed once, then EOF ends the run
    lines, _ = cli("-msgtype=scm", "-symbollength=78", "-single", f"-filterid={a},1", SAMPLE)
    assert [plain_key(l)[1] for l in lines] == [a]


def test_duration_ends_an_endless_stream(built):
    gen = subprocess.Popen([sys.executable, "-c", "import sys\nb = bytes(range(256)) * 4096\nw = sys.stdout.buffer.write\n"
                                                  "while True:\n    w(b)\n"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
    try:
        t0 = time.monotonic()
        out = subprocess.run([CLI, "-msgtype=scm", "-blocks=64", "-duration=2s", "-"], stdin=gen.stdout, capture_output=True,
                             text=True, timeout=120)
        elapsed = time.monotonic() - t0
    finally:
        gen.kill()
        gen.wait()
    assert out.returncode == 0, out.stderr
    assert 2.0 <= elapsed < 20, elapsed
    assert re.search(r"from [1-9]\d* blocks", out.stderr)


def test_bad_duration_is_a_usage_error(built):
    out = subprocess.run([CLI, "-duration=5 parsecs", SAMPLE], capture_output=True, text=True, timeout=60)
    assert out.returncode == 2 and "-duration" in out.stderr
