"""CPU tests of several channels of one capture in the file receiver: the cross-channel dedup through the host C API
(against a Python restatement of the rule) and the usage errors of a -centerfreq list, none of which needs a device."""
import os
import subprocess

import numpy as np
import pytest

import oracle
from helpers import whole_blocks
from test_host_mirror import _cand_records

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "rtlamr_b200", "ertgpu_decode_file")


def _digest(m):
    return (m.msgtype, m.meter_type, m.meter_id, m.checksum)


def _merge(per_channel, block_dedup):
    """The receiver's print order and dedup restated: ascending block, then channel in the order given; a message is
    dropped when its digest was seen for the previous block in any channel or for the same block in an earlier one."""
    blocks = sorted({m.block for msgs in per_channel for m in msgs})
    out, dropped, prev, prev_block = [], 0, set(), -2
    for b in blocks:
        if b != prev_block + 1:
            prev = set()
        nxt = set()
        for c, msgs in enumerate(per_channel):
            earlier = set(nxt)
            for m in (m for m in msgs if m.block == b):
                d = _digest(m)
                nxt.add(d)
                if block_dedup and (d in prev or d in earlier):
                    dropped += 1
                    continue
                out.append((c, m))
        prev, prev_block = nxt, b
    return out, dropped


def test_cross_channel_dedup_rule(built):
    from rtlamr_b200 import host, synth
    mt, cl = "scm", 72
    o = oracle.Oracle(mt, cl)
    n = 1 << 21
    pk, _ = synth.make_packets(mt, cl, n, seed=17, spacing=1 << 18)
    cands, msgs = o.decode(whole_blocks(synth.host_fill(0, n, 0x5EED0011, pk), o.cfg.block_size2))
    rec = _cand_records(cands)
    assert len(msgs) >= 4
    later, gap = rec.copy(), rec.copy()
    later["block"] += 1                      # the same packets one block later: the previous block of another channel
    gap["block"] += 2                        # two blocks later: not a duplicate
    half = rec[rec["block"] % 2 == 0]        # some of the same packets in the same blocks: an earlier channel's
    p = host.Parsers(mt, cl)
    for channels in ([rec], [rec, rec], [rec, later], [later, rec], [rec, gap, half], [half, rec, later, gap]):
        per = [p.parse(c) for c in channels]
        for block_dedup in (True, False):
            got, dropped = p.parse_dedup_channels(channels, block_dedup=block_dedup)
            want, want_dropped = _merge(per, block_dedup)
            assert [(c, m.block, m.idx, _digest(m)) for c, m in got] == \
                   [(c, m.block, m.idx, _digest(m)) for c, m in want]
            assert dropped == want_dropped
    # one channel is exactly the cross-block dedup of one decoder
    one, dropped = p.parse_dedup_channels([rec])
    alone, dropped_alone = p.parse_dedup(rec)
    assert [m for _, m in one] == alone and dropped == dropped_alone
    # a packet decoded in two overlapping channels is reported once
    both, _ = p.parse_dedup_channels([rec, rec])
    assert [m for _, m in both] == alone and {c for c, _ in both} == {0}
    p.close()


WIDE = ["-sampleformat=cs16", "-samplerate=30720000"]


@pytest.mark.parametrize("args,needle", [
    (["-centerfreq=911000000,912600155"], "-centerfreq needs -capturefreq"),
    (["-capturefreq=915000000", "-centerfreq=911000000,911000000"], "names the channel 911000000 Hz twice"),
    (["-capturefreq=915000000", "-centerfreq=911000000,912.6e6"], "invalid value \"912.6e6\" for flag -centerfreq"),
    (["-capturefreq=915000000", "-centerfreq=911000000,,912600000"], "invalid value \"\" for flag -centerfreq"),
    (["-capturefreq=915000000", "-centerfreq=911000000,930000000"], "channel 930000000 Hz does not fit"),
    (["-capturefreq=915000000", "-centerfreq=911000000,912600000", "-samplefile=out.bin"], "-samplefile takes one channel"),
])
def test_centerfreq_list_usage_errors(built, tmp_path, args, needle):
    r = subprocess.run([CLI] + WIDE + args + [os.devnull], capture_output=True, text=True, timeout=60, cwd=tmp_path)
    assert r.returncode == 2 and needle in r.stderr, r.stderr
    assert r.stdout == "" and not (tmp_path / "out.bin").exists()
