"""GPEN's FullGenerator (SURVEY.md section 8f.2) on the e4s_b200 kernels.

CPU part: oracle/gpen_oracle.py against tests/golden/gpen_vectors.npz - outputs of the UNMODIFIED reference model on
seeded inputs and parameters (oracle/make_golden_gpen.py) - and the state-dict contract.  GPU part: the module of
e4s_b200/gpen/gpen_model.py against the same vectors and, at GPEN-BFR-512's real size, against the oracle.
Tolerance: the path's fp32 bar, max|a - b| / max|b| <= 1e-3 (conftest.REL_TOL).
"""
import os

import numpy as np
import pytest
import torch

from conftest import REL_TOL, ROOT, assert_close
from oracle import golden_io
from oracle import gpen_oracle as GO
from oracle.make_golden_gpen import CASES, case_input


@pytest.fixture(scope="module")
def ggold():
    return golden_io.load(os.path.join(ROOT, "tests", "golden", "gpen_vectors.npz"))


# ------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("tag,size,batch,seed", CASES[:2])
def test_oracle_matches_reference_vectors(ggold, tag, size, batch, seed):
    st = GO.synthetic_state(size, salt=size)
    x = case_input(size, batch, seed)
    with torch.no_grad():
        assert_close(GO.full_generator_forward(st, x, size), ggold[f"gpen/{tag}/image"], 2e-5, tag)
        feats = GO.encode(st, x, size)
    assert_close(feats[-1], ggold[f"gpen/{tag}/ecd_last"], 2e-5, tag + " encoder")
    assert_close(feats[1][:, ::8, ::2, ::2], ggold[f"gpen/{tag}/ecd1_sub"], 2e-5, tag + " ecd1")


def test_state_dict_contract():
    """Parameter / buffer names and shapes equal the reference's (GO.param_shapes is asserted equal to the reference model's
    state_dict by make_golden_gpen.py), so GPEN-BFR checkpoints load."""
    from e4s_b200.gpen.gpen_model import FullGenerator
    for size in (64, 512):
        m = FullGenerator(size, 512, 8, channel_multiplier=2, narrow=1, device="cpu")
        assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == GO.param_shapes(size)
    assert m.generator.n_latent == 16 and len(m.generator.convs) == 14 and m.names == [f"ecd{i}" for i in range(8)]


def test_strided_conv_identity():
    """The encoder trick of e4s_b200/gpen/gpen_model.py: Blur pad (2,2) + 3x3 stride-2 conv without padding equals
    Blur pad (3,2) + 3x3 padding-1 conv sampled at even pixels, first row / column dropped."""
    import torch.nn.functional as F
    from oracle import e4s_oracle as O
    g = torch.Generator().manual_seed(0)
    x, w, fir = torch.randn(2, 5, 12, 16, generator=g), torch.randn(7, 5, 3, 3, generator=g), torch.randn(4, 4, generator=g)
    ref = F.conv2d(O.upfirdn2d(x, fir, pad=(2, 2)), w, stride=2, padding=0)
    ours = F.conv2d(O.upfirdn2d(x, fir, pad=(3, 2)), w, stride=1, padding=1)[:, :, ::2, ::2][:, :, 1:, 1:]
    assert torch.equal(ref, ours)


# ------------------------------------------------------------------------------------------------------- GPU
def _model(size):
    from e4s_b200.gpen.gpen_model import FullGenerator
    st = GO.synthetic_state(size, salt=size)
    m = FullGenerator(size, 512, 8, channel_multiplier=2, narrow=1, device="cuda").eval()
    m.load_state_dict(st)
    return m.cuda(), st


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["auto", "simt"])
@pytest.mark.parametrize("tag,size,batch,seed", CASES)
def test_full_generator_golden(monkeypatch, ggold, path, tag, size, batch, seed):
    monkeypatch.setenv("E4S_B200_CONV", path)                 # generator convs on the tensor-core / exact-fp32 kernel
    m, _ = _model(size)
    x = case_input(size, batch, seed).cuda()
    with torch.no_grad():
        img, none = m(x)
        feats, h = [], x
        for name in m.names:
            h = getattr(m, name)(h)
            feats.append(h)
    assert none is None and img.shape == (batch, 3, size, size)
    assert_close(feats[-1], ggold[f"gpen/{tag}/ecd_last"], REL_TOL, tag + " encoder")
    assert_close(feats[1][:, ::8, ::2, ::2], ggold[f"gpen/{tag}/ecd1_sub"], REL_TOL, tag + " ecd1")
    e = assert_close(img, ggold[f"gpen/{tag}/image"], REL_TOL, tag)
    print(f"gpen {tag} [{path}]: image max-rel err {e:.2e}")


@pytest.mark.gpu
def test_full_generator_512_vs_oracle():
    """GPEN-BFR-512's real configuration (size 512, 8 mapping layers, channel multiplier 2), two faces."""
    m, st = _model(512)
    x = case_input(512, 2, 3)
    with torch.no_grad():
        img, _ = m(x.cuda())
        ref = GO.full_generator_forward(st, x, 512)
    assert_close(img, ref, REL_TOL, "gpen 512")


@pytest.mark.gpu
def test_generator_api_surface():
    """Generator alone (style list in, explicit per-resolution noise maps, return_latents, truncation) keeps the reference's
    surface.  (The reference's `noise=None` branch, gpen_model.py:508-516, draws one map per resolution where the layer loop
    consumes two per resolution, so with isconcat=True it cannot run there either; callers always pass the encoder's maps.)"""
    m, _ = _model(64)
    G = m.generator
    z = torch.randn(3, 512, device="cuda")
    maps = [torch.randn(3, G.channels[4], 4, 4, device="cuda")]
    for r in (8, 16, 32, 64):
        maps += [torch.randn(3, G.channels[r], r, r, device="cuda")] * 2
    with torch.no_grad():
        img, lat = G([z], return_latents=True, noise=maps)
        img2, none = G([G.get_latent(z)], input_is_latent=True, truncation=0.7, truncation_latent=G.mean_latent(64), noise=maps)
    assert img.shape == (3, 3, 64, 64) and lat.shape == (3, G.n_latent, 512) and none is None
    assert torch.isfinite(img).all() and torch.isfinite(img2).all()
    assert [n.shape[-1] for n in G.make_noise()] == [4, 8, 8, 16, 16, 32, 32, 64, 64]
    with pytest.raises(NotImplementedError, match="forward-only"):
        m(torch.randn(1, 3, 64, 64, device="cuda", requires_grad=True))
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        with torch.no_grad():
            m(torch.randn(1, 3, 64, 64))
