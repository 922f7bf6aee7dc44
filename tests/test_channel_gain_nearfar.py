"""CPU tests of the wide channel path's sensitivity and of -channelgain's usage errors.  The near-far capture
(tests/nearfar_ref.py): on the narrow tuned path at -samplescale=auto the strong carrier sets the gain and the packets
40-50 dB below it are lost in the byte's rounding; the wide path at -channelgain=auto decodes every one, both checked
through the CPU restatements and the oracle."""
import os
import subprocess

import numpy as np
import pytest

import nearfar_ref as nf
import oracle

CLI = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rtlamr_b200", "ertgpu_decode_file")


def _oracle_ids(iq):
    o = oracle.Oracle("scm", 72, oracle.SEARCH_GO)
    bs2 = o.cfg.block_size2
    _, msgs = o.decode(iq[: iq.size // bs2 * bs2])
    return [m.meter_id for m in msgs]


@pytest.mark.parametrize("seed", [3, 8])
def test_near_far_narrow_loses_the_packets_wide_decodes_them(seed):
    raw, truth = nf.capture(seed)
    assert len(truth) >= 6
    narrow = nf.found(_oracle_ids(nf.narrow(raw)), truth)
    wide, k = nf.wide(raw)
    assert narrow <= 1 and nf.found(_oracle_ids(wide), truth) == len(truth), (narrow, k)
    assert k >= 6


def _cli(tmp_path, *args):
    path = tmp_path / "x.cs16"
    np.zeros(4 * 100_000, np.uint8).tofile(path)
    return subprocess.run([CLI, "-msgtype=scm", "-sampleformat=cs16", "-samplerate=10000000", *args, str(path)],
                          capture_output=True, text=True, timeout=60)


def test_cli_channelgain_usage_errors(built, tmp_path):
    for bad in ("0", "3", "-4", "32768", "1.5", "x"):
        r = _cli(tmp_path, "-capturefreq=915000000", f"-channelgain={bad}")
        assert r.returncode == 2 and "-channelgain" in r.stderr, bad
    for good in ("auto", "1", "16"):   # without a capture frequency each is a usage error
        r = _cli(tmp_path, f"-channelgain={good}")
        assert r.returncode == 2 and "-channelgain needs -capturefreq" in r.stderr, good
