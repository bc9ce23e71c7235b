# coding=utf-8
"""bench.py's output contract, checked on the arm that needs no GPU (`--impl reference`: the op-for-op torch-CPU port of the
reference's op sequence on a bounded sample).  One JSON line on stdout, the keys the driver reads, and under torchrun only
rank 0 speaks."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REQUIRED = ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
            "dtype", "data", "config", "impl", "cpu_baseline", "e2e")


def _check_line(stdout, n_gpus):
    lines = [l for l in stdout.splitlines() if l.strip()]
    assert len(lines) == 1, "expected exactly one stdout line, got {}: {!r}".format(len(lines), lines[:3])
    rec = json.loads(lines[0])
    for key in REQUIRED:
        assert key in rec, key
    assert rec["impl"] == "reference" and rec["n_gpus"] == n_gpus and rec["steps"] == 1 and rec["warmup"] == 1
    assert rec["unit"] == "edges/s" and rec["higher_is_better"] is True and rec["vs_baseline"] is None
    assert rec["value"] > 0 and rec["ms_per_step"] > 0 and rec["dtype"] == "f32" and rec["data"] == "synthetic"
    assert "workload" in rec["config"] and "model" not in rec["config"]
    cb = rec["cpu_baseline"]
    assert cb["kind"] in ("port", "reference") and cb["cores"] >= 1 and cb["sample"] and cb["value"] == rec["value"]
    e2e = rec["e2e"]
    assert e2e["value"] == rec["value"] and e2e["h2d_bytes_per_step"] == 0 and e2e["d2h_bytes_per_step"] == 0
    return rec


def test_reference_arm_prints_one_contract_line():
    out = subprocess.run([sys.executable, "bench.py", "--impl", "reference", "--steps", "1", "--warmup", "1", "--cpu-sample-div", "400"], cwd=ROOT,
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-2000:]
    _check_line(out.stdout, 1)


def test_reference_arm_under_torchrun_only_rank0_speaks():
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                          "--master-addr", "127.0.0.1", "--master-port", "29731", "bench.py", "--impl", "reference", "--gpus", "2",
                          "--steps", "1", "--warmup", "1", "--cpu-sample-div", "400"], cwd=ROOT, capture_output=True, text=True, timeout=900, env=env)
    assert out.returncode == 0, out.stderr[-2000:]
    _check_line(out.stdout, 2)


def test_reference_arm_covers_every_baseline_config():
    """--config cfg1..cfg5 on the CPU arm: each BASELINE.json configuration has its own op sequence and declares its sample."""
    for name in ("cfg1", "cfg2", "cfg3", "cfg4", "cfg5"):
        out = subprocess.run([sys.executable, "bench.py", "--impl", "reference", "--config", name, "--steps", "1", "--warmup", "1",
                              "--cpu-sample-div", "1" if name == "cfg1" else "2000"], cwd=ROOT, capture_output=True, text=True,
                             timeout=600)
        assert out.returncode == 0, (name, out.stderr[-2000:])
        rec = _check_line(out.stdout, 1)
        assert rec["config"]["name"] == name and "reference_sample" in rec["config"]
        assert rec["metric"].startswith("edges/sec")


def test_gpu_arm_refuses_to_run_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        import pytest
        pytest.skip("a GPU is present")
    out = subprocess.run([sys.executable, "bench.py", "--steps", "1", "--warmup", "1"], cwd=ROOT, capture_output=True,
                         text=True, timeout=300)
    assert out.returncode != 0 and out.stdout.strip() == "" and "no CPU fallback" in out.stderr


def test_dump_outputs_is_refused_where_it_cannot_be_honoured():
    """--dump-outputs writes the single-GPU path's outputs; the CPU arm, several GPUs and cfg5 refuse it instead of ignoring it."""
    for extra in (["--impl", "reference"], ["--gpus", "2"], ["--config", "cfg5"]):
        out = subprocess.run([sys.executable, "bench.py", "--steps", "1", "--dump-outputs", "unused_dir"] + extra, cwd=ROOT,
                             capture_output=True, text=True, timeout=300)
        assert out.returncode != 0 and out.stdout.strip() == "" and "--dump-outputs" in out.stderr, extra
        assert not os.path.exists(os.path.join(ROOT, "unused_dir"))
