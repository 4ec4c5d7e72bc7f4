"""bench.py contract pieces that run without a GPU: the reference arm (the real reference PLMSSampler + UNetModel from
the archive oracle/_ref that build() makes where the original project is available, on the host cores; the oracle port
when it is absent) prints one JSON line with the keys the benchmark consumers read; the product arm refuses to run without CUDA (no CPU fallback)."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_line():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--config", "tiny", "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["higher_is_better"] is True and line["unit"] == "images/s"
    assert line["value"] > 0 and line["e2e"]["value"] == line["value"]
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["e2e"]["d2h_bytes_per_step"] == 0
    cb = line["cpu_baseline"]
    from oracle import build_ref, ref_harness
    have_ref = build_ref.available() or os.path.isdir(ref_harness.REF_DIR)          # the rule ref_harness.mount("auto") uses
    assert cb["kind"] == ("reference" if have_ref else "port") and cb["cores"] >= 1 and cb["value"] == line["value"] and cb["sample"]
    if have_ref:
        assert "PLMSSampler.sample" in cb["sample"] and line["config"]["reference_batch"] >= 1
    assert "workload" in line["config"] and "model" not in line["config"]


def test_reference_arm_other_ranks_are_silent():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--config", "tiny", "--gpus", "2", "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=600, cwd=ROOT, env=env)
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_product_arm_needs_cuda():
    if torch.cuda.is_available():
        return
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1", "--warmup", "0"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode != 0 and "no CPU fallback" in (r.stderr + r.stdout)
