"""GPU tests (-m gpu) of the wide channel path above the C ABI: ertgpu_decode_file -channelgain=G|auto, host.Receiver
(channel_gain=), and the near-far capture (tests/nearfar_ref.py) decoded on the GPU, where the narrow path at
-samplescale=auto loses the packets and the wide path at -channelgain=auto decodes all of them."""
import json
import os
import re
import subprocess

import numpy as np
import pytest

from rtlamr_b200 import capi

import nearfar_ref as nf
from test_gpu_resample import _scm_fields

pytestmark = pytest.mark.gpu

CLI = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rtlamr_b200", "ertgpu_decode_file")
CHANNEL = nf.CAPTURE + nf.OFFSET


def _run(path, *args):
    return subprocess.run([CLI, "-msgtype=scm", "-format=json", "-sampleformat=cs16", f"-samplerate={nf.RATE}",
                           "-samplescale=auto", f"-capturefreq={nf.CAPTURE}", f"-centerfreq={CHANNEL}", *args, str(path)],
                          capture_output=True, text=True, timeout=600, check=True)


def _ids(stdout):
    return {json.loads(l)["Message"]["ID"] for l in stdout.splitlines()}


def _strip(stdout):
    return [json.dumps({k: v for k, v in json.loads(l).items() if k != "Time"}) for l in stdout.splitlines()]


def test_cli_near_far_and_auto_equals_the_printed_gain(built, tmp_path):
    raw, truth = nf.capture(3)
    path = tmp_path / "nearfar.cs16"
    raw.tofile(path)
    want = {_scm_fields(t.data)[0] for t in truth}
    narrow = _run(path)
    assert len(_ids(narrow.stdout) & want) <= 1
    auto = _run(path, "-channelgain=auto")
    m = re.search(rf"channel {CHANNEL}: 2\^(\d+) = (\d+)\n", auto.stderr)
    _, k_ref = nf.wide(raw)
    assert m and int(m.group(1)) == k_ref and int(m.group(2)) == 1 << k_ref
    assert _ids(auto.stdout) == want
    fixed = _run(path, f"-channelgain={m.group(2)}")
    assert _strip(auto.stdout) == _strip(fixed.stdout)
    # stdin: nothing is read twice
    with open(path, "rb") as f:
        piped = subprocess.run([CLI, "-msgtype=scm", "-format=json", "-sampleformat=cs16", f"-samplerate={nf.RATE}",
                                "-samplescale=auto", f"-capturefreq={nf.CAPTURE}", f"-centerfreq={CHANNEL}",
                                "-channelgain=auto", "-"], stdin=f, capture_output=True, text=True, timeout=600, check=True)
    assert _strip(piped.stdout) == _strip(auto.stdout)


def test_cli_channel_list_prints_each_channels_gain(built, tmp_path):
    raw, truth = nf.capture(8)
    path = tmp_path / "nearfar.cs16"
    raw.tofile(path)
    other = nf.CAPTURE + nf.STRONG_OFFSET + 300_000   # next to the carrier: a small k
    r = subprocess.run([CLI, "-msgtype=scm", "-format=json", "-sampleformat=cs16", f"-samplerate={nf.RATE}",
                        "-samplescale=auto", f"-capturefreq={nf.CAPTURE}", f"-centerfreq={CHANNEL},{other}",
                        "-channelgain=auto", str(path)], capture_output=True, text=True, timeout=600, check=True)
    ks = {int(f): int(k) for f, k in re.findall(r"channel (\d+): 2\^(\d+) = \d+\n", r.stderr)}
    assert set(ks) == {CHANNEL, other} and ks[other] < ks[CHANNEL]
    assert {_scm_fields(t.data)[0] for t in truth} <= _ids(r.stdout)


def test_host_receiver_channel_gain(built):
    from rtlamr_b200 import host
    raw, truth = nf.capture(3)
    want = {int(t.meter_id) for t in truth}
    _, k_ref = nf.wide(raw)
    g = nf.auto_scale(raw)
    kw = dict(input_rate=nf.RATE, input_format=capi.FORMAT_CS16, input_scale=g, capture_freq=nf.CAPTURE, center_freq=CHANNEL)
    r = host.Receiver("scm", 72, channel_gain="auto", **kw)
    got = r.decode(raw)
    assert r.channel_gain() == k_ref and {m.meter_id for m in got} == want
    r.close()
    r = host.Receiver("scm", 72, channel_gain=k_ref, **kw)
    assert r.channel_gain() == k_ref and sorted(m.meter_id for m in r.decode(raw)) == sorted(m.meter_id for m in got)
    r.close()
    r = host.Receiver("scm", 72, **kw)
    assert r.channel_gain() is None and len({m.meter_id for m in r.decode(raw)} & want) <= 1
    r.close()
    with pytest.raises(RuntimeError):   # untuned
        host.Receiver("scm", 72, input_rate=nf.RATE, input_format=capi.FORMAT_CS16, channel_gain=2)
