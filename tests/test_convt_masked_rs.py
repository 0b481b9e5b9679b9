"""The masked up-sampling layers' gathered-row GEMM on the register-operand kernel (e4s_modconv3x3_up_masked_tcr_fwd):
every N-tile width the width rule picks, K chains shorter than one ring slot, and outputs that do not depend on the
batch a face is computed in."""
import pytest
import torch

from conftest import assert_close
from f64ref import modconv_case, row_list

DEV = "cuda:0"


def _masked(c):
    from e4s_b200 import kernels as K
    return K.modconv3x3_up_masked_tcr_fwd(c.x, c.prep.w_convt_hilo, c.prep.w_hilo, c.prep.fir, c.s, c.dm, c.label, c.noise, c.nw,
                                          c.bias, True)


def _simt(c):
    from e4s_b200 import kernels as K
    return K.modconv3x3_fwd(c.x, c.prep.wt, c.s, c.dm, c.label, c.noise, c.nw, c.bias, True, True)


# (batch, Cin, Cout, input side): Cout 32 and 96 take 32-channel tiles, 64 takes 64, 128 and 256 take 64 or 128 by the
# launch size; Cin 32 makes class (1, 1) a one-step chain and class (0, 0) a four-step one
WIDTHS = [
    (2, 64, 32, 12),
    (2, 128, 96, 12),
    (2, 96, 64, 20),
    (1, 64, 128, 16),
    (16, 64, 128, 24),
    (2, 128, 256, 16),
    (16, 32, 256, 16),
    (3, 32, 64, 13),
]


@pytest.mark.gpu
@pytest.mark.parametrize("b,cin,cout,hw", WIDTHS)
def test_gathered_gemm_widths_match_simt(b, cin, cout, hw):
    from e4s_b200.kernels import convt_masked_cap
    c = modconv_case(b, cin, cout, hw, hw, 12, "face", up=True, seed=b + cin + cout + hw, device=DEV)
    # every sample's rows fit the cap: the gathered GEMM, not the folded fallback, computes the whole output
    assert all(len(row_list(lab, 12, hw, hw)[2]) <= convt_masked_cap(hw, hw) for lab in c.label.cpu())
    assert_close(_masked(c), _simt(c), 1e-4, f"masked convT {b},{cin},{cout},{hw}")


@pytest.mark.gpu
@pytest.mark.parametrize("cout", [128, 256])
def test_gathered_gemm_64_and_128_channel_tiles_are_bitwise_equal(monkeypatch, cout):
    c = modconv_case(2, 64, cout, 16, 16, 12, "face", up=True, seed=cout, device=DEV)
    outs = []
    for nt in ("64", "128"):
        monkeypatch.setenv("E4S_B200_RS_NTILE", nt)
        outs.append(_masked(c))
    assert torch.equal(outs[0], outs[1])


@pytest.mark.gpu
@pytest.mark.parametrize("cout", [64, 128])
def test_face_alone_equals_face_in_batch(cout):
    """A face's output computed alone equals the same face's output inside a 16-face batch, bit for bit: the launch size
    changes the N-tile width (and the item count), never an output's sum order."""
    c = modconv_case(16, 128, cout, 16, 16, 12, "face", up=True, noise_b=16, seed=11, device=DEV)
    batch = _masked(c)
    for i in (0, 7, 15):
        one = modconv_case(1, 128, cout, 16, 16, 12, "face", up=True, seed=11, device=DEV)
        one.x, one.s, one.label, one.noise = c.x[i:i + 1], c.s[i:i + 1], c.label[i:i + 1], c.noise[i:i + 1]
        one.dm, one.bias = c.dm[i:i + 1], c.bias
        assert torch.equal(_masked(one)[0], batch[i]), f"face {i}"
