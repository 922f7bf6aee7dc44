"""bench.py's JSON contract, checked on CPU through the reference arm (the GPU arm needs an H100)."""
import json
import os
import subprocess
import sys

from conftest import ROOT

KEYS = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
        "vs_baseline", "dtype", "data", "config", "e2e", "cpu_baseline", "impl"}


def test_reference_arm_prints_one_contract_line(built):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1",
                          "--warmup", "0", "--bytes-per-gpu", str(8 << 20)], capture_output=True, text=True, timeout=300, check=True)
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    j = json.loads(lines[0])
    assert KEYS <= set(j)
    assert j["impl"] == "reference" and j["higher_is_better"] is True and j["vs_baseline"] is None
    assert j["unit"] == "Msamples/s" and j["value"] > 1.0
    assert j["cpu_baseline"]["kind"] == "port" and j["cpu_baseline"]["cores"] >= 1
    assert j["e2e"]["value"] == j["value"] and j["e2e"]["h2d_bytes_per_step"] == 0
    assert "workload" in j["config"] and "model" not in j["config"]
    # the reference arm decodes the workload's own stream (same `config` object as the GPU arm prints), cut over
    # every CPU the process may use, and says how many threads / physical cores that was
    assert j["config"]["bytes_per_gpu"] == 8 << 20 and j["config"]["msgtype"] == "scm" and j["config"]["chip_length"] == 72
    assert j["cpu_baseline"]["cores"] == len(os.sched_getaffinity(0)) and j["cpu_baseline"]["physical_cores"] >= 1
    assert j["cpu_baseline"]["one_core_value"] > 1.0


def test_both_arms_print_the_same_config_object(built):
    import bench
    a = bench.workload_config("scm1g", bench.WORKLOADS["scm1g"], 1 << 30, 8, 4096, 13824)
    assert a["halo_blocks"] == 5 and a["blocks_per_gpu"] == 131072 and a["total_bytes"] == 8 << 30
    assert "configs[1]" in a["workload"]
    m = bench.workload_config("multi8g", bench.WORKLOADS["multi8g"], 8 << 30, 1, 8192, 105984)
    assert m["halo_blocks"] == 0 and m["blocks_per_gpu"] == 524288 and "configs[2]" in m["workload"]


def test_cpu_arm_scales_with_threads(built):
    """The C thread driver behind the CPU arm: T decoders over T shards of one stream run in parallel (no GIL,
    nothing allocated in the timed region) and see the same packets as one decoder."""
    import oracle
    from rtlamr_b200 import synth
    n = 1 << 23
    pk, truth = synth.make_packets("scm", 72, n, seed=1, spacing=1 << 19)
    iq = synth.host_fill(0, n, 3, pk, nthreads=4)
    assert (iq == synth.host_fill(0, n, 3, pk)).all()
    t1, c1, m1, nb = oracle.bench_threads("scm", 72, iq, 1)
    ncpu = min(4, oracle.host_cpus())
    tn, cn, mn, _ = oracle.bench_threads("scm", 72, iq, ncpu)
    assert nb == n // 4096 and m1 >= len(truth) - 2 and abs(mn - m1) <= 2 * ncpu   # a shard seam can cut a packet
    if ncpu >= 4:
        assert tn < t1 / 2.0, (t1, tn)


def test_non_zero_ranks_of_the_reference_arm_do_no_work(built):
    env = dict(os.environ, RANK="1", WORLD_SIZE="2")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2"],
                         capture_output=True, text=True, timeout=60, env=env)
    assert out.returncode == 0 and out.stdout.strip() == ""


def test_dump_outputs_writes_float_arrays_within_the_limit(tmp_path, monkeypatch):
    """--dump-outputs: one float64 / float32 .npy per candidate field; above the size limit a seeded sample of whole
    records in stream order, the same one every run."""
    import numpy as np

    import bench
    from rtlamr_b200 import capi
    got = np.zeros(1000, dtype=capi.CAND_DTYPE)
    got["block"] = np.arange(1000)
    got["bytes"][:, 0] = np.arange(1000) % 256
    bench.dump_outputs(str(tmp_path / "a"), "scm1g", got)
    blk = np.load(tmp_path / "a" / "scm1g_block.npy")
    assert blk.dtype == np.float64 and np.array_equal(blk, np.arange(1000))
    b = np.load(tmp_path / "a" / "scm1g_bytes.npy")
    assert b.dtype == np.float32 and b.shape == (1000, capi.MAX_PACKET_BYTES) and np.array_equal(b[:, 0], np.arange(1000) % 256)
    assert sorted(os.listdir(tmp_path / "a")) == sorted(f"scm1g_{f}.npy" for f in
                                                          ("block", "idx", "preamble_id", "check_mask", "flags", "bytes", "r900_digits"))
    monkeypatch.setattr(bench, "DUMP_LIMIT_BYTES", 100 * 1000)
    for d in ("b", "c"):
        bench.dump_outputs(str(tmp_path / d), "scm1g", got)
    bench.dump_outputs(str(tmp_path / "d"), "scm1g", got, 50 * 1000)
    assert sum(os.path.getsize(tmp_path / "d" / f) for f in os.listdir(tmp_path / "d")) <= 50 * 1000
    total = sum(os.path.getsize(tmp_path / "b" / f) for f in os.listdir(tmp_path / "b"))
    blk_b, blk_c = np.load(tmp_path / "b" / "scm1g_block.npy"), np.load(tmp_path / "c" / "scm1g_block.npy")
    assert 0 < len(blk_b) < 1000 and np.all(np.diff(blk_b) > 0) and np.array_equal(blk_b, blk_c)
    assert total <= 100 * 1000
