"""rtlamr's -format=json and -format=xml (flags.go:140-170) in the C++ mirror (rtlamr_b200/host/filters.hpp), no device:
packets of all six message types from this repository's encoders (rtlamr_b200/synth.py) go through the parse-only host, and
every line is checked against the rules of Go's encoding/json and encoding/xml restated here from the packet bytes."""
import base64
import csv
import glob
import io
import json
import os
import xml.etree.ElementTree as ET

import numpy as np
import pytest

import oracle
from conftest import GOLDEN
from helpers import whole_blocks

T0 = 1700000000   # 2023-11-14T22:13:20Z
TYPES = {"scm": "SCM", "scm+": "SCM+", "idm": "IDM", "netidm": "NetIDM", "r900": "R900", "r900bcd": "R900BCD"}


def _bits(data: bytes) -> str:
    return "".join(f"{b:08b}" for b in data)


def _be(b: bytes) -> int:
    return int.from_bytes(b, "big")


def expected_fields(mt: str, data: bytes):
    """(Go field name, xml attribute name or None, value) in declaration order, read from the packet bytes the way each
    parser does (scm.go:103-119, scmplus.go:105-109, idm.go:121-156, netidm.go:131-160, r900.go:223-242, r900bcd.go:63-65).
    Values are int, bytes ([]byte) or list (array of uint16)."""
    if mt == "scm":
        s = _bits(data)
        u = lambda a, b: int(s[a:b], 2)
        return [("ID", "ID", u(21, 23) << 24 | u(56, 80)), ("Type", "Type", u(26, 30)), ("TamperPhy", "TamperPhy", u(24, 26)),
                ("TamperEnc", "TamperEnc", u(30, 32)), ("Consumption", "Consumption", u(32, 56)), ("ChecksumVal", "Checksum", u(80, 96))]
    if mt == "scm+":
        return [("FrameSync", "FrameSync", _be(data[0:2])), ("ProtocolID", "ProtocolID", data[2]), ("EndpointType", "EndpointType", data[3]),
                ("EndpointID", "EndpointID", _be(data[4:8])), ("Consumption", "Consumption", _be(data[8:12])),
                ("Tamper", "Tamper", _be(data[12:14])), ("PacketCRC", "Checksum", _be(data[14:16]))]
    if mt in ("idm", "netidm"):
        s = _bits(data)
        head = [("Preamble", _be(data[0:4])), ("PacketTypeID" if mt == "idm" else "ProtocolID", data[4]), ("PacketLength", data[5]),
                ("HammingCode", data[6]), ("ApplicationVersion", data[7]), ("ERTType", data[8] & 0x0F),
                ("ERTSerialNumber", _be(data[9:13])), ("ConsumptionIntervalCount", data[13])]
        if mt == "idm":
            body = [("ModuleProgrammingState", data[14]), ("TamperCounters", bytes(data[15:21])), ("AsynchronousCounters", _be(data[21:23])),
                    ("PowerOutageFlags", bytes(data[23:29])), ("LastConsumptionCount", _be(data[29:33])),
                    ("DifferentialConsumptionIntervals", [int(s[264 + 9 * k:273 + 9 * k], 2) for k in range(47)])]
        else:
            body = [("ProgrammingState", data[14]), ("LastGeneration", _be(data[28:31])), ("LastConsumption", _be(data[25:28])),
                    ("LastConsumptionNet", _be(data[34:38])),
                    ("DifferentialConsumptionIntervals", [int(s[304 + 14 * k:318 + 14 * k], 2) for k in range(27)])]
        tail = [("TransmitTimeOffset", _be(data[86:88])), ("SerialNumberCRC", _be(data[88:90])), ("PacketCRC", _be(data[90:92]))]
        return [(n, None, v) for n, v in head + body + tail]
    if mt in ("r900", "r900bcd"):   # data: the 21 symbols
        s = "".join(f"{x:05b}" for x in data[:16])
        u = lambda a, b: int(s[a:b], 2)
        cons = u(48, 72)
        if mt == "r900bcd":
            h = f"{cons:X}"
            cons = int(h) if h.isdigit() else 0
        names = [("ID", 0, 32), ("Unkn1", 32, 40), ("NoUse", 40, 46), ("BackFlow", 46, 48), ("Consumption", 48, 72), ("Unkn3", 72, 74),
                 ("Leak", 74, 78), ("LeakNow", 78, 80)]
        return [(n, n, cons if n == "Consumption" else u(a, b)) for n, a, b in names]
    raise ValueError(mt)


def go_escape_text(b: bytes) -> str:
    """xml.EscapeText: runes decoded like utf8.DecodeRune (an invalid sequence is one byte), markup characters, tab, LF and CR as
    character references, invalid UTF-8 and runes outside XML's Char production as U+FFFD."""
    esc = {'"': "&#34;", "'": "&#39;", "&": "&amp;", "<": "&lt;", ">": "&gt;", "\t": "&#x9;", "\n": "&#xA;", "\r": "&#xD;"}
    out, i = [], 0
    while i < len(b):
        r, w, ok = "�", 1, False
        for n in (1, 2, 3, 4):
            try:
                r, w, ok = b[i:i + n].decode("utf-8"), n, True   # strict: no overlong forms, surrogates or values past U+10FFFF
                break
            except UnicodeDecodeError:
                continue
        c = ord(r)
        in_char = c in (9, 10, 13) or 0x20 <= c <= 0xD7FF or 0xE000 <= c <= 0xFFFD or 0x10000 <= c <= 0x10FFFF
        out.append(esc.get(r) or (r if ok and in_char else "�"))
        i += w
    return "".join(out)


def packets(mt: str, n: int, seed: int = 11):
    """n distinct packets of type mt: (candidate bytes, r900 digits or None)."""
    from rtlamr_b200 import synth
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        if mt == "scm":
            out.append((synth.encode_scm(int(rng.integers(1, 1 << 26)), int(rng.integers(0, 16)), int(rng.integers(0, 4)),
                                         int(rng.integers(0, 4)), int(rng.integers(0, 1 << 24))), None))
        elif mt == "scm+":
            out.append((synth.encode_scmplus(int(rng.integers(0, 256)), int(rng.integers(1, 1 << 32)), int(rng.integers(0, 1 << 32)),
                                             int(rng.integers(0, 1 << 16))), None))
        elif mt in ("idm", "netidm"):
            enc = synth.encode_idm if mt == "idm" else synth.encode_netidm
            out.append((enc(int(rng.integers(0, 16)), int(rng.integers(1, 1 << 32)), bytes(rng.integers(0, 256, 75, dtype=np.uint8))), None))
        else:
            cons = int(rng.integers(0, 1 << 24))
            if mt == "r900bcd" and len(out) % 2 == 0:     # every other one a decimal-looking hex value
                cons = int(str(int(rng.integers(0, 1000000))), 16)
            _, sym = synth.encode_r900(int(rng.integers(1, 1 << 32)), int(rng.integers(0, 256)), int(rng.integers(0, 64)),
                                       int(rng.integers(0, 4)), cons, int(rng.integers(0, 4)), int(rng.integers(0, 16)),
                                       int(rng.integers(0, 4)))
            out.append((bytes(sym), [d for s in sym for d in (s // 6, s % 6)]))
    return out


def records(pkts):
    from rtlamr_b200 import capi
    rec = np.zeros(len(pkts), dtype=capi.CAND_DTYPE)
    for i, (data, digits) in enumerate(pkts):
        rec[i]["block"], rec[i]["idx"] = i, 100 + i      # one packet per block: no parser's per-block `seen` set interferes
        if digits is None:
            rec[i]["bytes"][:len(data)] = np.frombuffer(data, dtype=np.uint8)
        else:
            rec[i]["r900_digits"][:] = digits
            rec[i]["flags"] = capi.CAND_HAS_R900
    return rec


def encode(mt, pkts, fmt, **kw):
    from rtlamr_b200 import host
    p = host.Parsers(mt, 72)
    try:
        return p.encode(records(pkts), fmt, **kw).splitlines(keepends=True)
    finally:
        p.close()


def json_value(v):
    return base64.b64encode(v).decode() if isinstance(v, bytes) else v


@pytest.mark.parametrize("mt", list(TYPES))
def test_json_lines_follow_encoding_json(built, mt):
    pkts = packets(mt, 24)
    kw = dict(unix_seconds=T0, nanos=120000000, offset=123456789012, length=81920)
    lines = encode(mt, pkts, "json", **kw)
    assert len(lines) == len(pkts)
    for line, (data, _) in zip(lines, pkts):
        want = {"Time": "2023-11-14T22:13:20.12Z", "Offset": 123456789012, "Length": 81920, "Type": TYPES[mt],
                "Message": {name: json_value(v) for name, _, v in expected_fields(mt, data)}}
        assert line == json.dumps(want, separators=(",", ":")) + "\n"
        # Go's HTML escaping (<, >, &) has nothing to rewrite in these lines
        assert not set("<>&\\") & set(line)


@pytest.mark.parametrize("mt", list(TYPES))
def test_json_round_trips_to_the_csv_record(built, mt):
    """The same message through -format=json and -format=csv: the same time, offset, length and field values (the CSV
    record renders some of them in hex, and IDM's Interval as one column per item)."""
    pkts = packets(mt, 16, seed=5)
    kw = dict(unix_seconds=T0, nanos=7, offset=42, length=32768)
    js = [json.loads(l) for l in encode(mt, pkts, "json", **kw)]
    cs = list(csv.reader(io.StringIO("".join(encode(mt, pkts, "csv", **kw)))))
    assert len(js) == len(cs) == len(pkts)
    for j, rec in zip(js, cs):
        assert [j["Time"], str(j["Offset"]), str(j["Length"])] == rec[:3] == ["2023-11-14T22:13:20.000000007Z", "42", "32768"]
        flat = []
        for v in j["Message"].values():
            flat += v if isinstance(v, list) else [v]
        assert len(flat) == len(rec) - 3
        for v, r in zip(flat, rec[3:]):
            if isinstance(v, str):
                assert base64.b64decode(v) == bytes.fromhex(r)
            else:
                assert v == int(r, 0)


@pytest.mark.parametrize("mt", list(TYPES))
def test_xml_lines_follow_encoding_xml(built, mt):
    pkts = packets(mt, 24, seed=3)
    lines = encode(mt, pkts, "xml", unix_seconds=T0, nanos=0, offset=0, length=0)
    assert len(lines) == len(pkts)
    for line, (data, _) in zip(lines, pkts):
        assert line.endswith("</Message></LogMessage>\n") and "/>" not in line     # Go never self-closes
        root = ET.fromstring(line)
        assert root.tag == "LogMessage"
        assert root.attrib == {"Time": "2023-11-14T22:13:20Z", "Offset": "0", "Length": "0", "Type": TYPES[mt]}
        assert [c.tag for c in root] == ["Message"]
        fields = expected_fields(mt, data)
        msg = root[0]
        assert msg.attrib == {attr: str(v) for _, attr, v in fields if attr}
        want_children = []
        for name, attr, v in fields:
            if attr:
                continue
            if isinstance(v, list):
                want_children += [(name, str(x)) for x in v]
            elif isinstance(v, bytes):
                want_children.append((name, go_escape_text(v)))
            else:
                want_children.append((name, str(v)))
        got_children = [(c.tag, c.text or "") for c in msg]
        if not any(isinstance(v, bytes) for _, _, v in fields):
            assert got_children == want_children
            continue
        # character data: compare the raw escaped text, which the parser has already turned back into runes
        for name, text in want_children:
            assert f"<{name}>{text}</{name}>" in line
        assert [t for t, _ in got_children] == [t for t, _ in want_children]


def test_one_literal_line_per_format(built):
    """The first message of tests/golden/sample_cl78.bin, rebuilt from its fields: SCM ID 17580293, type 8, tamper 1/1,
    consumption 111414 and (computed by the encoder) CRC 0xD005 = 53253."""
    from rtlamr_b200 import synth
    pkt = [(synth.encode_scm(17580293, 8, 1, 1, 111414), None)]
    kw = dict(unix_seconds=T0, nanos=500000000, offset=4096, length=8192)
    assert encode("scm", pkt, "json", **kw) == [
        '{"Time":"2023-11-14T22:13:20.5Z","Offset":4096,"Length":8192,"Type":"SCM","Message":{"ID":17580293,"Type":8,'
        '"TamperPhy":1,"TamperEnc":1,"Consumption":111414,"ChecksumVal":53253}}\n']
    assert encode("scm", pkt, "xml", **kw) == [
        '<LogMessage Time="2023-11-14T22:13:20.5Z" Offset="4096" Length="8192" Type="SCM"><Message ID="17580293" Type="8" '
        'TamperPhy="1" TamperEnc="1" Consumption="111414" Checksum="53253"></Message></LogMessage>\n']
    assert encode("scm", pkt, "csv", **kw) == ["2023-11-14T22:13:20.5Z,4096,8192,17580293,8,0x1,0x1,111414,0xd005\n"]


@pytest.mark.parametrize("fmt", [-1, 4, 1 << 30])
def test_any_other_format_value_is_the_plain_line(built, fmt):
    """erthost_encode and erthost_encode_signal take 1, 2 and 3 as csv, json and xml, and every other int as plain."""
    import ctypes as C
    from rtlamr_b200 import capi, host, synth
    rec = records([(synth.encode_scm(17580293, 8, 1, 1, 111414), None)])
    sig = np.zeros(len(rec), dtype=capi.SIGNAL_DTYPE)
    p = host.Parsers("scm", 72)
    try:
        L, buf = p._L, C.create_string_buffer(1 << 16)
        n = L.erthost_encode(p._h, rec.ctypes.data, len(rec), fmt, T0, 0, 4096, 8192, 1, buf, len(buf))
        assert buf.raw[:n].decode() == p.encode(rec, "plain", unix_seconds=T0, offset=4096, length=8192)
        n = L.erthost_encode_signal(p._h, rec.ctypes.data, sig.ctypes.data, len(rec), 912_600_000, 2_359_296, fmt, T0, 0,
                                    buf, len(buf))
        assert buf.raw[:n].decode() == p.encode_signal(rec, sig, 912_600_000, 2_359_296, "plain", unix_seconds=T0)
    finally:
        p.close()


def test_scmplus_packet_crc_is_keyed_packetcrc_in_json_and_checksum_in_xml(built):
    """scmplus.go:101: `xml:"Checksum,attr",json:"Checksum"` -- reflect.StructTag.Get("json") stops at the comma, so only the
    xml key takes effect."""
    from rtlamr_b200 import synth
    pkt = [(synth.encode_scmplus(0xAB, 0x12345678, 987654, 0x0102), None)]
    crc = _be(pkt[0][0][14:16])
    j = json.loads(encode("scm+", pkt, "json")[0])
    assert list(j["Message"])[-1] == "PacketCRC" and j["Message"]["PacketCRC"] == crc and "Checksum" not in j["Message"]
    x = ET.fromstring(encode("scm+", pkt, "xml")[0])[0]
    assert x.attrib["Checksum"] == str(crc) and "PacketCRC" not in x.attrib
    # SCM's ChecksumVal: the json key is the Go name, the xml attribute is Checksum
    s = [(synth.encode_scm(99, 1, 0, 0, 5), None)]
    assert "ChecksumVal" in json.loads(encode("scm", s, "json")[0])["Message"]
    assert "Checksum" in ET.fromstring(encode("scm", s, "xml")[0])[0].attrib


def test_idm_byte_fields_with_markup_and_invalid_utf8(built):
    """IDM's []byte fields: standard padded base64 in JSON, escaped character data in XML with U+FFFD for every byte that is
    not valid UTF-8 (0x00 is valid UTF-8 but not an XML Char)."""
    from rtlamr_b200 import synth
    filler = bytearray(75)
    filler[2:8] = b"\x00<\xffA&\n"                    # TamperCounters = bytes 15..20
    filler[10:16] = b"\xe2\x82\xac\xc3(\xed"          # PowerOutageFlags = bytes 23..28: a valid euro sign, then two bad starts
    pkt = [(synth.encode_idm(3, 0xCAFE01, bytes(filler)), None)]
    j = json.loads(encode("idm", pkt, "json")[0])
    assert j["Message"]["TamperCounters"] == "ADz/QSYK" == base64.b64encode(b"\x00<\xffA&\n").decode()
    assert j["Message"]["PowerOutageFlags"] == base64.b64encode(b"\xe2\x82\xac\xc3(\xed").decode()
    line = encode("idm", pkt, "xml")[0]
    assert "<TamperCounters>�&lt;�A&amp;&#xA;</TamperCounters>" in line
    assert "<PowerOutageFlags>€�(�</PowerOutageFlags>" in line
    assert line.count("<DifferentialConsumptionIntervals>") == 47
    assert ET.fromstring(line)[0].find("TamperCounters").text == "�<�A&\n"


# ---- pinning against the stock Go encoders (go/goldengen -format json|xml), when those lines exist ----
# case -> (msgtypes, chip length), the `run` lines of tests/golden/make_go_fmt_golden.sh
GO_FMT_CASES = {"sample_cl78_scm": ("scm", 78), "sample_cl72_scm": ("scm", 72), "synth_cl72_scm": ("scm", 72),
                "synth_cl72_multi": ("scm,scm+,idm", 72), "synth_cl72_r900": ("r900", 72), "synth_cl32_all": ("scm,scm+,idm,r900", 32)}
GO_FMT = sorted(glob.glob(os.path.join(GOLDEN, "go_fmt_*.jsonl")) + glob.glob(os.path.join(GOLDEN, "go_fmt_*.xmll")))


def _oracle_records(msgtypes, cl, iq):
    """The candidates the Go decoder hands its parsers (oracle, Go-faithful Search), one Decode per block, with the r900
    payload digits taken from the oracle's r900 buffer as the GPU attaches them."""
    from rtlamr_b200 import capi
    mts = [m.strip() for m in msgtypes.split(",")]
    o = oracle.Oracle(mts, cl, oracle.SEARCH_GO)
    bs2 = o.cfg.block_size2
    iq = whole_blocks(iq, bs2)
    has_r900 = any(m in ("r900", "r900bcd") for m in mts)
    recs = []
    for b in range(iq.size // bs2):
        cands, _ = o.decode(iq[b * bs2:(b + 1) * bs2])
        rec = np.zeros(len(cands), dtype=capi.CAND_DTYPE)
        q = o.r900_quantized() if has_r900 else None
        for i, c in enumerate(sorted(cands, key=lambda c: (c.preamble_id, c.idx))):
            rec[i]["block"], rec[i]["idx"], rec[i]["preamble_id"] = b, c.idx, c.preamble_id
            rec[i]["bytes"][:len(c.data)] = np.frombuffer(c.data, dtype=np.uint8)
            if has_r900:
                payload = c.idx + o.cfg.preamble_length - o.cfg.symbol_length
                rec[i]["r900_digits"][:] = [int(q[payload + k * 4 * cl]) for k in range(capi.R900_DIGITS)]
                rec[i]["flags"] = capi.CAND_HAS_R900
        recs.append(rec)
    return np.concatenate(recs)


@pytest.mark.skipif(not GO_FMT, reason="no Go encoder lines committed: run tests/golden/make_go_fmt_golden.sh on a machine with Go "
                                       "(the json and xml formats are UNPINNED against Go until then)")
@pytest.mark.parametrize("path", GO_FMT or ["absent"])
def test_encoders_equal_the_go_encoders(built, path):
    from rtlamr_b200 import host
    from test_go_golden import case_input
    name, ext = os.path.splitext(os.path.basename(path)[len("go_fmt_"):])
    fmt = {".jsonl": "json", ".xmll": "xml"}[ext]
    mt, cl = GO_FMT_CASES[name]
    p = host.Parsers(mt, cl)
    got = p.encode(_oracle_records(mt, cl, case_input(name)), fmt, T0, 0, 0, 0).splitlines()
    p.close()
    # the order of a block's messages is unspecified in Go (decode.go:177-187): compare as multisets
    assert sorted(got) == sorted(open(path).read().splitlines())
