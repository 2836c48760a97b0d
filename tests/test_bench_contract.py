"""bench.py's output contract, checked on CPU through the reference arm (the only arm that
runs without a GPU): exactly one JSON line on stdout with the agreed keys."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_json_line():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--entries", "1024",
                        "--prf", "chacha20", "--steps", "2", "--warmup", "1"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-500:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "DPFs/sec" and d["unit"] == "DPFs/sec"
    assert d["value"] > 0 and d["higher_is_better"] is True and d["steps"] == 2 and d["warmup"] == 1
    assert d["cpu_baseline"]["kind"] in ("reference", "port") and d["cpu_baseline"]["cores"] >= 1
    assert d["cpu_baseline"]["value"] == d["value"] and "sample" in d["cpu_baseline"]
    assert d["e2e"] == {"value": d["value"], "unit": "DPFs/sec", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert d["config"]["workload"].startswith("n=1024 entry_size=16 CHACHA20")


def test_non_rank0_reference_arm_is_silent():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2",
                        "--entries", "1024", "--steps", "1", "--warmup", "0"], capture_output=True, text=True,
                       timeout=120, env=env)
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_clock_sampler_parsing(tmp_path):
    sys.path.insert(0, ROOT)
    import bench
    s = bench.ClockSampler(0)
    s.path = str(tmp_path / "c.csv")
    with open(s.path, "w") as f:
        f.write("0, 345, 1965, 140.1, 0x0000000000000001, Not Active, Not Active, Not Active, Not Active\n")
        f.write("0, 1965, 1965, 700.2, 0x0000000000000000, Not Active, Not Active, Not Active, Active\n")
        f.write("0, 1950, 1965, 710.0, 0x0000000000000000, Not Active, Not Active, Not Active, Not Active\n")

    class Dead:
        def terminate(self): pass
        def wait(self, timeout=None): pass
    s.proc = Dead()
    out = s.stop()
    assert out["sm_max_mhz"] == 1965.0 and out["samples"] == 3 and out["sm_mhz"] >= 1950.0
    assert out["reasons"] == ["sw_power_cap"]


def test_key_slices_cover_batch():
    sys.path.insert(0, os.path.join(ROOT, "gpu-dpf_b200"))
    from sharded import key_slice
    for nkeys in (1, 7, 512, 513):
        for world in (1, 2, 8):
            spans = [key_slice(nkeys, r, world) for r in range(world)]
            covered = [i for b, e in spans for i in range(b, e)]
            assert covered == list(range(nkeys))


def test_dump_outputs_sample_is_seeded_and_capped(tmp_path):
    """--dump-outputs: the whole [B, E] result as float64 under the cap; above it the same seeded sample of
    rows every time, with their indices, within the cap."""
    import numpy as np
    sys.path.insert(0, ROOT)
    import bench
    result = (np.arange(40 * 16, dtype=np.int64).reshape(40, 16) * 2654435761 % 2**32 - 2**31).astype(np.int32)
    bench.dump_outputs(str(tmp_path), result)
    out = np.load(tmp_path / "out.npy")
    assert out.dtype == np.float64 and np.array_equal(out, result) and not (tmp_path / "out_rows.npy").exists()
    cap = 10 * (16 * 8 + 8)
    for _ in range(2):
        bench.dump_outputs(str(tmp_path), result, cap_bytes=cap)
        out, rows = np.load(tmp_path / "out.npy"), np.load(tmp_path / "out_rows.npy")
        assert out.nbytes + rows.nbytes <= cap and out.shape == (10, 16)
        assert np.array_equal(out, result[rows.astype(np.int64)]) and np.all(np.diff(rows) > 0)
        if _ == 0:
            first = rows
    assert np.array_equal(rows, first)


def test_reference_arm_rejects_dump_outputs(tmp_path):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--entries", "1024",
                        "--steps", "1", "--warmup", "0", "--dump-outputs", str(tmp_path / "d")],
                       capture_output=True, text=True, timeout=120)
    assert r.returncode != 0 and "--dump-outputs" in r.stderr and not (tmp_path / "d").exists()
