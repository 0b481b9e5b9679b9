"""GPEN's RealESRNet x4 (e4s_b200.gpen.sr_model): the oracle and the mirror against the reference's goldens on the CPU.
The kernels' results at the production shape are checked in tests/test_sr_at_scale.py."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT

from oracle import golden_io
from oracle import sr_oracle as SO

CASES = [("s32", 32, 32, 21), ("s20x44", 20, 44, 22)]


@pytest.fixture(scope="module")
def gold():
    return golden_io.load(os.path.join(ROOT, "tests", "golden", "sr_vectors.npz"))


@pytest.mark.parametrize("tag,h,w,seed", CASES)
def test_oracle_matches_reference_golden(gold, tag, h, w, seed):
    img = SO.case_image(h, w, seed)
    assert np.array_equal(img, gold[f"sr/{tag}/image"])
    st = SO.synthetic_state()
    with torch.no_grad():
        out = SO.rrdbnet_forward(st, SO.to_input(img))
    ref = torch.from_numpy(gold[f"sr/{tag}/forward"])
    assert tuple(out.shape) == (1, 3, 4 * h, 4 * w)
    assert float((out - ref).abs().max() / ref.abs().max()) <= 2e-5
    assert np.array_equal(SO.process(st, img), gold[f"sr/{tag}/process"])


def test_golden_images_are_not_degenerate(gold):
    for tag, h, w, _ in CASES:
        out = gold[f"sr/{tag}/process"]
        assert out.shape == (4 * h, 4 * w, 3) and out.dtype == np.uint8
        assert len(np.unique(out)) >= 64, tag              # clamping and rounding are exercised, not one flat value


def test_mirror_state_dict_layout():
    from e4s_b200.gpen.sr_model.rrdbnet_arch import RRDBNet
    with open(os.path.join(ROOT, "tests", "golden", "sr_checkpoint_layout.json")) as f:
        layout = json.load(f)
    net = RRDBNet(num_in_ch=3, num_out_ch=3, num_feat=32, num_block=23, num_grow_ch=32, scale=4)
    assert {k: list(v.shape) for k, v in net.state_dict().items()} == layout
    assert len(layout) == 702
    for scale in (1, 2):                                   # the pixel-unshuffle variants build the reference's tree too
        net = RRDBNet(3, 3, scale=scale, num_feat=32, num_block=2, num_grow_ch=32)
        assert tuple(net.conv_first.weight.shape) == (32, 3 * (16 if scale == 1 else 4), 3, 3)


def test_stand_in_state_matches_oracle_recipe():
    from e4s_b200.synthetic import synthetic_sr_state
    for seed in (0, 5):
        ours, theirs = synthetic_sr_state(seed), SO.synthetic_state(seed)
        assert sorted(ours) == sorted(theirs)
        for k in ours:
            assert ours[k].dtype == theirs[k].dtype and torch.equal(ours[k], theirs[k]), k
    assert all(float(v.abs().sum()) > 0 for k, v in synthetic_sr_state().items() if k.endswith(".bias"))


def test_dense_branches_contribute():
    """The stand-in weights make every residual dense block's branch count: ||0.2 x5|| / ||x|| well above rounding."""
    st = SO.synthetic_state()
    x = SO.to_input(SO.case_image(32, 32, 21))
    with torch.no_grad():
        feat = SO._conv(st, "conv_first", x)
        ratios = []
        for i in range(3):                                 # the first three blocks
            for r in range(1, 4):
                out = SO.rdb_forward(st, f"body.{i}.rdb{r}.", feat)
                ratios.append(float((out - feat).norm() / feat.norm()))
                feat = out
    assert min(ratios) > 0.1, ratios


def test_real_esrnet_checkpoint_rule_and_scale_guard(tmp_path):
    from e4s_b200.gpen.sr_model.real_esrnet import RealESRNet
    from e4s_b200.synthetic import synthetic_sr_state
    os.makedirs(tmp_path / "weights")
    torch.save({"params_ema": synthetic_sr_state()}, tmp_path / "weights" / "realesrnet_x4.pth")
    sr = RealESRNet(str(tmp_path), "realesrnet", 4, device="cpu")
    assert torch.equal(sr.srmodel.conv_last.bias, SO.synthetic_state()["conv_last.bias"])
    with pytest.raises(FileNotFoundError):
        RealESRNet(str(tmp_path), None, 4, device="cpu")   # model None -> weights/realesrnet_x2.pth
    with pytest.raises(ValueError):                        # the kernels need a CUDA tensor
        with torch.no_grad():
            sr.srmodel(torch.zeros(1, 3, 8, 8))


def test_dropin_resolves_sr_model():
    code = ("import e4s_b200.dropin as d; d.install()\n"
            "from src.pretrained.gpen.sr_model.rrdbnet_arch import RRDBNet, RRDB, ResidualDenseBlock\n"
            "from src.pretrained.gpen.sr_model.real_esrnet import RealESRNet\n"
            "assert RRDBNet.__module__ == RRDB.__module__ == ResidualDenseBlock.__module__ == "
            "'e4s_b200.gpen.sr_model.rrdbnet_arch'\n"
            "assert RealESRNet.__module__ == 'e4s_b200.gpen.sr_model.real_esrnet'\n")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True,
                       env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode == 0, r.stderr
