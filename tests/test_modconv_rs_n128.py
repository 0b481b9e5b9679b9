"""128-channel N tiles in the register-operand forward (csrc/wgmma_conv_rs.cu, conv3x3_rs_kernel<128>): the weights stream
through a three-slot ring of three-tap groups instead of whole chunks, but every output is still summed chunk-outer,
tap-inner, K16-slice-inner with the three split products in split_mma's order - so the output must be bitwise identical
to the 64-channel tile (E4S_B200_RS_NTILE=64 against =128).  Also pinned: the automatic choice of the width
(e4s_modconv3x3_tcr_fwd_plan, host only) and that neither variable leaks into the other's kernels."""
import ctypes

import pytest
import torch

from conftest import assert_close
from f64ref import default_kernels, modconv_case  # noqa: F401

DEV = "cuda:0"


def _at_width(monkeypatch, width, fn):
    if width is None:
        monkeypatch.delenv("E4S_B200_RS_NTILE", raising=False)
    else:
        monkeypatch.setenv("E4S_B200_RS_NTILE", str(width))
    out = fn()
    torch.cuda.synchronize()
    return out


def _plan(b, h, w, cout):
    from e4s_b200 import _lib
    nt = ctypes.c_int()
    assert _lib.load().e4s_modconv3x3_tcr_fwd_plan(b, h, w, cout, ctypes.byref(nt)) == 0
    return nt.value


@pytest.mark.gpu
@pytest.mark.parametrize("b,cin,cout,h,w,labels,noise_b,plain", [
    (1, 128, 128, 20, 44, "face", 1, False),      # ragged tiles, one face
    (3, 128, 128, 20, 44, "iid", 3, False),       # every tile mixes regions; noise of batch B
    (3, 128, 128, 64, 96, None, 1, False),        # 144 items: CTAs of the persistent grid walk several
    (1, 256, 256, 37, 21, None, 1, False),
    (3, 256, 256, 4, 4, "iid", 1, False),         # one partial tile per sample
    (3, 256, 256, 20, 44, "face", 3, True),       # no demodulation, noise or bias
    (1, 512, 512, 4, 4, "face", 1, False),
    (3, 512, 512, 40, 44, "iid", 1, False),       # 180 items over four N tiles, sixteen chunks each
    (3, 512, 512, 20, 44, None, 1, True),
    (1, 64, 128, 33, 17, "face", 1, False),       # two chunks, one N tile
    (3, 64, 128, 20, 44, "iid", 3, False),
])
def test_n128_equals_n64(monkeypatch, b, cin, cout, h, w, labels, noise_b, plain):
    from e4s_b200 import kernels as K
    c = modconv_case(b, cin, cout, h, w, 12 if labels else 1, labels, noise_b=noise_b, seed=b + cin + cout + h + w,
                     device=DEV)
    args = (c.s, None, c.label, None, None, None, False, False) if plain else (c.s, c.dm, c.label, c.noise, c.nw, c.bias,
                                                                              False, True)
    run = lambda: K.modconv3x3_tcr_fwd(c.x, c.prep.w_hilo, *args)
    y128 = _at_width(monkeypatch, 128, run)
    y64 = _at_width(monkeypatch, 64, run)
    assert torch.equal(y128, y64)
    assert torch.equal(y128, _at_width(monkeypatch, 128, run)), "two runs of the 128-channel tile differ"


@pytest.mark.gpu
@pytest.mark.parametrize("b,cin,cout,h,w,labels", [(3, 256, 256, 20, 44, "face"), (1, 64, 128, 33, 17, "iid")])
def test_n128_against_simt(monkeypatch, b, cin, cout, h, w, labels):
    from e4s_b200 import kernels as K
    c = modconv_case(b, cin, cout, h, w, 12, labels, noise_b=b, seed=7 + cin + h, device=DEV)
    args = (c.s, c.dm, c.label, c.noise, c.nw, c.bias, False, True)
    y128 = _at_width(monkeypatch, 128, lambda: K.modconv3x3_tcr_fwd(c.x, c.prep.w_hilo, *args))
    assert_close(y128, K.modconv3x3_fwd(c.x, c.prep.wt, *args), 1e-4, "128-channel register-operand forward vs simt")


def test_width_plan(monkeypatch):
    """The automatic width (132 SMs assumed without a device): 128 when the channel count allows it and the 64-channel
    items would need more than one wave of CTAs, else the 64 / 32 rule of the other kernels."""
    # the 16-face batch: c5 @32, c7 @64 (512 channels), c9 @128 (256), c11 @256 (128) and GPEN's 128-channel 512^2 layer
    assert [_plan(16, r, r, c) for r, c in ((32, 512), (64, 512), (128, 256), (256, 128), (512, 128))] == [128] * 5
    assert _plan(16, 512, 512, 64) == 64 and _plan(16, 1024, 1024, 32) == 32
    assert _plan(16, 16, 16, 512) == 128 and _plan(16, 8, 8, 512) == 64     # c3: 128 items of 128 channels; c1: 64
    assert _plan(8, 16, 16, 512) == 64                                      # 128 items of 64 channels: one wave already
    # one face (the inversion loop): c1, c3, c5 keep 32; c7, c9, c11 have 128, 256, 512 items of 128 channels
    assert [_plan(1, r, r, c) for r, c in ((8, 512), (16, 512), (32, 512), (64, 512), (128, 256), (256, 128))] == [32, 32, 32, 128, 128, 128]
    # E4S_B200_RS_NTILE forces 64 or 128 where the channel count allows it, and nothing else
    monkeypatch.setenv("E4S_B200_RS_NTILE", "128")
    assert _plan(1, 4, 4, 512) == 128 and _plan(16, 512, 512, 64) == 64 and _plan(1, 4, 4, 192) == 32
    monkeypatch.setenv("E4S_B200_RS_NTILE", "64")
    assert _plan(16, 64, 64, 512) == 64 and _plan(1, 4, 4, 512) == 64 and _plan(1, 4, 4, 96) == 32
    monkeypatch.setenv("E4S_B200_RS_NTILE", "32")
    assert _plan(16, 64, 64, 512) == 128
    monkeypatch.delenv("E4S_B200_RS_NTILE")
    # a set E4S_B200_NTILE keeps its meaning: 32 | 64 force that width, anything else the 64 / 32 rule
    for v, nt in (("32", 32), ("64", 64), ("128", 64)):
        monkeypatch.setenv("E4S_B200_NTILE", v)
        assert _plan(16, 64, 64, 512) == nt, v
    # the gradient's plan does not know the new variable
    monkeypatch.delenv("E4S_B200_NTILE")
    from e4s_b200 import _lib
    monkeypatch.setenv("E4S_B200_RS_NTILE", "128")
    nt, gs, hs = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    assert _lib.load().e4s_modconv3x3_bwd_tc_plan(16, 64, 64, 512, 12, 0, ctypes.byref(nt), ctypes.byref(gs), ctypes.byref(hs)) == 0
    assert nt.value == 64
    assert _lib.load().e4s_modconv3x3_tcr_fwd_plan(1, 4, 4, 48, None) == -1


@pytest.mark.gpu
@pytest.mark.parametrize("cin,cout,r", [(512, 512, 64), (256, 256, 128)])     # c7, c9 at the benchmark's batch
def test_default_runs_n128_at_batch_16(monkeypatch, cin, cout, r):
    from e4s_b200 import kernels as K
    assert _plan(16, r, r, cout) == 128
    c = modconv_case(16, cin, cout, r, r, 12, "face", noise_b=16, seed=r, device=DEV)
    args = (c.s, c.dm, c.label, c.noise, c.nw, c.bias, False, True)
    run = lambda: K.modconv3x3_tcr_fwd(c.x, c.prep.w_hilo, *args)
    assert torch.equal(_at_width(monkeypatch, None, run), _at_width(monkeypatch, 64, run))


@pytest.mark.gpu
def test_64_channels_ignore_128(monkeypatch):
    from e4s_b200 import kernels as K
    c = modconv_case(2, 64, 64, 43, 51, 12, "iid", seed=3, device=DEV)
    args = (c.s, c.dm, c.label, c.noise, c.nw, c.bias, False, True)
    run = lambda: K.modconv3x3_tcr_fwd(c.x, c.prep.w_hilo, *args)
    assert torch.equal(_at_width(monkeypatch, 128, run), _at_width(monkeypatch, None, run))
