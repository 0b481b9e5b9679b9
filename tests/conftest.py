import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# Parity bar of BASELINE.json's north_star for floating point: 1e-3 relative fp32.  Two norms, both must hold:
#   max-rel  = max|ours - ref| / max|ref| over the tensor (one outlier anywhere fails it), and
#   rel-RMS  = ||ours - ref||_2 / ||ref||_2 (scale-aware: a tensor whose values are mostly far below its maximum cannot
#              hide a large relative error behind that maximum).
# Mask / index ops are compared bit-exactly (torch.equal).
REL_TOL = 1e-3


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90) GPU")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden():
    from oracle import golden_io
    return golden_io.load(os.path.join(ROOT, "tests", "golden", "reference_vectors.npz"))


def rel_err(ours: torch.Tensor, ref: torch.Tensor) -> float:
    ours = ours.detach().double().cpu()
    ref = ref.detach().double().cpu()
    assert ours.shape == ref.shape, (ours.shape, ref.shape)
    return float((ours - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


def rel_rms(ours: torch.Tensor, ref: torch.Tensor) -> float:
    ours = ours.detach().double().cpu()
    ref = ref.detach().double().cpu()
    assert ours.shape == ref.shape, (ours.shape, ref.shape)
    return float((ours - ref).pow(2).sum().sqrt() / ref.pow(2).sum().sqrt().clamp_min(1e-30))


def assert_close(ours, ref, tol=REL_TOL, what=""):
    if isinstance(ref, np.ndarray):
        ref = torch.from_numpy(ref)
    e = rel_err(ours, ref)
    assert e <= tol, f"{what}: max-rel error {e:.3e} > {tol:.1e}"
    r = rel_rms(ours, ref)
    assert r <= tol, f"{what}: rel-RMS error {r:.3e} > {tol:.1e}"
    return e
