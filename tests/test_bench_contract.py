"""CPU: the bench's reference arm prints the contract's JSON line; the GPU arm refuses to run without a GPU."""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def _run(*args, env=None):
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), *args], capture_output=True, text=True, timeout=600,
                          env=dict(os.environ, **(env or {})))


def test_reference_arm_line():
    r = _run("--impl", "reference", "--steps", "2", "--warmup", "1")
    assert r.returncode == 0, r.stderr[-500:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["unit"] == "graphs/s" and line["higher_is_better"] is True
    assert line["steps"] == 2 and line["warmup"] == 1 and line["n_gpus"] == 1 and line["value"] > 0
    assert line["metric"].startswith("graphs/sec") and "workload" in line["config"] and line["data"] == "synthetic"
    cb = line["cpu_baseline"]
    from oracle import reference_runner
    assert cb["kind"] == ("reference" if reference_runner.available() else "port")
    assert cb["cores"] >= 1 and cb["value"] == line["value"] and cb["sample"]
    assert set(line["config"]) == {"workload", "name", "global_batch", "per_gpu_batch", "parallelism", "optimizer_step", "l2"}
    assert line["e2e"] == {"value": line["value"], "unit": "graphs/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}


def test_reference_arm_other_configs():
    for cfg in ("contextpred", "gat"):
        r = _run("--impl", "reference", "--config", cfg, "--steps", "1", "--warmup", "1")
        assert r.returncode == 0, r.stderr[-500:]
        line = json.loads(r.stdout.strip().splitlines()[-1])
        assert line["config"]["name"] == cfg and line["value"] > 0 and cfg in line["metric"]


def test_reference_arm_other_ranks_exit_quietly():
    r = _run("--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "1", env={"RANK": "1", "WORLD_SIZE": "2", "LOCAL_RANK": "1"})
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_b200_arm_needs_a_gpu():
    if torch.cuda.is_available():
        return
    r = _run("--steps", "1", "--warmup", "1")
    assert r.returncode != 0 and "no CPU fallback" in (r.stderr + r.stdout)


def test_dump_outputs_files_dtypes_and_budget(tmp_path, monkeypatch):
    """bench.dump_outputs: loss as float64, one float32 file per gradient; over the byte budget every array becomes a seeded sample
    whose values and int64 indices together stay within it, and the same call gives the same sample."""
    import numpy as np
    import bench
    g = torch.Generator().manual_seed(0)
    loss = torch.tensor(1.25, dtype=torch.float64)
    grads = [("a.weight", torch.randn(300, 200, generator=g)), ("a.bias", torch.randn(300, generator=g)), ("b.weight", None)]
    bench.dump_outputs(str(tmp_path / "full"), loss, grads)
    full = tmp_path / "full"
    assert sorted(p.name for p in full.iterdir()) == ["grad.a.bias.npy", "grad.a.weight.npy", "loss.npy"]
    assert np.load(full / "loss.npy").dtype == np.float64 and float(np.load(full / "loss.npy")[0]) == 1.25
    w = np.load(full / "grad.a.weight.npy")
    assert w.dtype == np.float32 and np.array_equal(w, grads[0][1].numpy())
    monkeypatch.setattr(bench, "DUMP_BYTES", 64 << 10)   # far below the 241 KB of these arrays
    for run in ("s1", "s2"):
        bench.dump_outputs(str(tmp_path / run), loss, grads)
        assert sum(p.stat().st_size for p in (tmp_path / run).iterdir()) <= bench.DUMP_BYTES
    idx = np.load(tmp_path / "s1" / "grad.a.weight.idx.npy")
    vals = np.load(tmp_path / "s1" / "grad.a.weight.npy")
    assert idx.dtype == np.int64 and vals.dtype == np.float32 and idx.size == vals.size > 0
    assert np.array_equal(vals, grads[0][1].numpy().reshape(-1)[idx])
    for f in (tmp_path / "s1").iterdir():
        assert np.array_equal(np.load(f), np.load(tmp_path / "s2" / f.name))
