"""CPU: the reference arm of bench.py runs without a GPU and prints one JSON line with the contract's keys."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENV = dict(os.environ, PVB_BENCH_REF_BUDGET_S="3")      # the driver's run uses the full budget; the CPU tier a short one


def test_reference_arm_json_line():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1",
                          "--warmup", "0"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600,
                         cwd=ROOT, env=ENV)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "sdf_grad_queries_per_s" and d["unit"] == "queries/s"
    assert d["higher_is_better"] is True and d["value"] > 0 and d["n_gpus"] == 1
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    # the default line is the C4 RobotSDF headline, with the SAME config object the GPU arm prints ...
    sys.path.insert(0, ROOT)
    import bench
    assert d["config"] == bench.c4_config() and d["scaling"] == "strong"
    assert d["config"]["n_cfg"] == 200 and d["config"]["n_pts"] == 100_000
    # ... and carries every other BASELINE config next to it
    assert set(d["workloads"]) == set(bench.OTHER_WORKLOADS)
    for name, w in d["workloads"].items():
        assert w["value"] > 0 and w["cpu_baseline"]["cores"] >= 1, (name, w)


def test_reference_arm_single_workload():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1",
                          "--warmup", "0", "--workload", "c2"], stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                         text=True, timeout=600, cwd=ROOT, env=ENV)
    assert out.returncode == 0, out.stderr[-2000:]
    d = json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][0])
    assert d["impl"] == "reference" and "C2" in d["config"]["workload"] and "workloads" not in d


def test_reference_arm_other_ranks_exit_quietly():
    env = dict(ENV, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1",
                          "--warmup", "0", "--gpus", "2"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                         timeout=600, cwd=ROOT, env=env)
    assert out.returncode == 0 and out.stdout.strip() == ""


def test_dump_outputs_full_and_sampled(tmp_path):
    """--dump-outputs: small results are written whole in their own shape; large ones as the same seeded rows of value
    and gradient, float32 / float64 only, under 64 MB, identical from run to run."""
    import numpy as np
    import torch
    sys.path.insert(0, ROOT)
    import bench
    val = torch.arange(6, dtype=torch.float32).reshape(2, 3)
    bench.dump_outputs((val, torch.stack([val, -val, 2 * val], -1)), str(tmp_path / "small"))
    assert np.array_equal(np.load(tmp_path / "small" / "value.npy"), val.numpy())
    assert np.load(tmp_path / "small" / "grad.npy").shape == (2, 3, 3)
    assert not (tmp_path / "small" / "sample_index.npy").exists()

    rows = bench.DUMP_MAX_ROWS + 12345
    big_v = torch.randn(rows, generator=torch.Generator().manual_seed(0))
    big_g = torch.randn(rows, 3, generator=torch.Generator().manual_seed(1)).double()
    for d in ("a", "b"):
        bench.dump_outputs((big_v, big_g), str(tmp_path / d))
    files = {p.name for p in (tmp_path / "a").iterdir()}
    assert files == {"value.npy", "grad.npy", "sample_index.npy"}
    assert sum((tmp_path / "a" / f).stat().st_size for f in files) <= bench.DUMP_MAX_BYTES
    idx = np.load(tmp_path / "a" / "sample_index.npy")
    v, g = np.load(tmp_path / "a" / "value.npy"), np.load(tmp_path / "a" / "grad.npy")
    assert idx.dtype == np.float64 and v.dtype == np.float32 and g.dtype == np.float64
    assert len(np.unique(idx)) == len(idx) == len(v) == len(g) <= bench.DUMP_MAX_ROWS
    assert np.array_equal(v, big_v.numpy()[idx.astype(np.int64)])
    assert np.array_equal(g, big_g.numpy()[idx.astype(np.int64)])
    for f in files:
        assert np.array_equal(np.load(tmp_path / "a" / f), np.load(tmp_path / "b" / f))
