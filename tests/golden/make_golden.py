"""Regenerates tests/golden/sample_cl78_scm.json from the reference fixture with the oracle.

sample_cl78.bin is a byte-for-byte copy of the reference's assets/sample.bin (a data capture,
572160 bytes = 15 buffer dumps taken at chip length 78; see SURVEY.md "three facts").  The Go
toolchain is not available in this image, so the vectors come from oracle/ert_oracle.c; they
are self-verifying because every message passes the BCH check of scm/scm.go:76.
Run from the repo root:  python tests/golden/make_golden.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402

here = os.path.dirname(os.path.abspath(__file__))

# synthetic inputs shared with the Go-side generator (tests/golden/make_go_golden.sh, tests/test_go_golden.py):
# name -> (msgtypes, chip length, samples, noise seed, packet seed, spacing)
SYNTH_CASES = {
    "synth_cl72_scm": ("scm", 72, 1 << 21, 0x5EED0101, 21, 1 << 18),
    "synth_cl72_multi": ("scm,scm+,idm", 72, 1 << 22, 0x5EED0102, 22, 1 << 18),
    "synth_cl72_r900": ("r900", 72, 1 << 21, 0x5EED0103, 23, 1 << 18),
    "synth_cl32_all": ("scm,scm+,idm,r900", 32, 1 << 21, 0x5EED0104, 24, 1 << 17),
}


def synth_input(name):
    from rtlamr_b200 import synth
    mt, cl, n, seed, pseed, spacing = SYNTH_CASES[name]
    pk, _ = synth.make_packets(mt, cl, n, seed=pseed, spacing=spacing)
    return synth.host_fill(0, n, seed, pk)


if len(sys.argv) == 3 and sys.argv[1] == "--synthetic-inputs":
    for name in SYNTH_CASES:
        synth_input(name).tofile(os.path.join(sys.argv[2], name + ".bin"))
    sys.exit(0)
if __name__ != "__main__":
    raise ImportError("make_golden is a script; import SYNTH_CASES / synth_input via tests/test_go_golden.py's loader")

iq = np.fromfile(os.path.join(here, "sample_cl78.bin"), dtype=np.uint8)
out = {}
for name, mode in (("exact", oracle.SEARCH_EXACT), ("go_faithful", oracle.SEARCH_GO)):
    o = oracle.Oracle("scm", 78, mode)
    n = iq.size // o.cfg.block_size2
    cands, msgs = o.decode(iq[: n * o.cfg.block_size2])
    if name == "exact":
        out[name] = {"n_candidates": len(cands),
                     "messages": [[m.block, m.idx, m.data.hex(), m.meter_id, m.meter_type, m.consumption] for m in msgs]}
    else:
        out[name] = {"n_candidates": len(cands), "messages": [[m.block, m.idx, m.data.hex()] for m in msgs]}
with open(os.path.join(here, "sample_cl78_scm.json"), "w") as f:
    json.dump(out, f, indent=1)
print({k: (v["n_candidates"], len(v["messages"])) for k, v in out.items()})
