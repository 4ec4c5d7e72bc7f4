import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLD = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: run with -m gpu)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def rel_l2(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def assert_close(got, ref, rel=6e-3, max_rel=3e-2, what=""):
    """relative-L2 and max-abs (scaled by max|ref|) bounds; both printed on failure."""
    got, ref = got.float().cpu(), ref.float().cpu()
    assert torch.isfinite(got).all(), f"{what}: non-finite values"
    r = rel_l2(got, ref)
    m = (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-12)
    assert r <= rel and m <= max_rel, f"{what}: rel_l2={r:.3e} (<= {rel}) max_rel={m:.3e} (<= {max_rel})"
    return r, m
