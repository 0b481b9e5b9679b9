"""Unmasked up-sampling layers as a transposed-convolution GEMM plus a blur pass (e4s_modconv3x3_up_tcr_fwd).

The host test restates the class-stacked weights and the blur indexing in float64; the GPU tests check the entry point
against the fp32 SIMT kernel (folded parity weights) and the oracle."""
import pytest
import torch
import torch.nn.functional as F

from oracle import e4s_oracle as O
from conftest import assert_close
from f64ref import default_kernels, modconv_case  # noqa: F401

DEV = "cuda:0"


def _convt_then_blur_emulated(x, w, fir):
    """What the two kernels compute, in float64: T' = stride-1 2x2 convolution of x (padded by one pixel) with the
    class-stacked weights, T[2m + a, 2n + c] = T'[m, n, (a, c)], y[Y, X] = sum_{p,q} fir[3-p, 3-q] T[Y-1+p, X-1+q]."""
    from e4s_b200.stylegan2.modconv import convt_class_kernels
    b, cin, h, wd = x.shape
    cout = w.shape[0]
    wc = convt_class_kernels(w)                                           # [9, 4 Cout, Cin]
    assert all(float(wc[t].abs().max()) == 0.0 for t in (2, 5, 6, 7, 8))
    k2 = torch.stack([torch.stack([wc[0], wc[1]], -1), torch.stack([wc[3], wc[4]], -1)], -2)   # [4 Cout, Cin, dy, dx]
    tp = F.conv2d(F.pad(x, (1, 1, 1, 1)), k2)                             # [B, 4 Cout, H+1, W+1]
    assert tp.shape[-2:] == (h + 1, wd + 1)
    t = tp.reshape(b, 2, 2, cout, h + 1, wd + 1).permute(0, 3, 4, 1, 5, 2).reshape(b, cout, 2 * h + 2, 2 * wd + 2)
    tpad = F.pad(t, (1, 0, 1, 0))                                         # T[-1] = 0
    y = torch.zeros(b, cout, 2 * h, 2 * wd, dtype=x.dtype)
    for p in range(4):
        for q in range(4):
            y += fir[3 - p, 3 - q] * tpad[:, :, p:p + 2 * h, q:q + 2 * wd]
    return y


def test_convt_class_kernels_and_blur_indexing_match_convT_plus_blur():
    """e4s_modconv3x3_up_tcr_fwd's decomposition == conv_transpose2d(stride 2) + upfirdn2d(pad 1) (model.py:287-300), for a
    symmetric and an arbitrary FIR and odd H / W."""
    g = torch.Generator().manual_seed(0)
    cin, cout = 5, 7
    w = torch.randn(cout, cin, 3, 3, generator=g, dtype=torch.float64)
    for h, wd in [(6, 7), (5, 3), (1, 4)]:
        x = torch.randn(2, cin, h, wd, generator=g, dtype=torch.float64)
        for fir in (O.make_fir((1, 3, 3, 1), 4.0).double(), torch.rand(4, 4, generator=g, dtype=torch.float64)):
            ref = O.upfirdn2d(F.conv_transpose2d(x, w.transpose(0, 1), stride=2), fir, pad=(1, 1))
            assert_close(_convt_then_blur_emulated(x, w, fir), ref, 1e-5, f"convT + blur emulation {h}x{wd}")


# ------------------------------------------------------------------------------------------------ GPU
def _convt(c, act=True, noise=True):
    """The transposed-convolution GEMM + blur pass on unmasked up-sampling case c."""
    from e4s_b200 import kernels as K
    return K.modconv3x3_up_tcr_fwd(c.x, c.prep.w_convt_hilo, c.prep.fir, c.s, c.dm, c.noise if noise else None,
                                   c.nw if noise else None, c.bias, act)


def _simt(c, act=True, noise=True):
    """The fp32 SIMT kernel on case c (folded parity weights)."""
    from e4s_b200 import kernels as K
    return K.modconv3x3_fwd(c.x, c.prep.wt, c.s, c.dm, None, c.noise if noise else None, c.nw if noise else None, c.bias,
                            True, act)


UNMASKED_UP = [
    (1, 128, 256, 16),        # N tile inside a class of 256 channels
    (1, 64, 32, 16),          # one K chunk of 64, N tile 32
    (2, 128, 64, 20),         # partial tiles in both directions
    (1, 96, 32, 18),          # three K chunks of 32
    (1, 64, 32, 512),         # c14 ^1024
    (1, 128, 64, 256),        # c12 ^512
]


@pytest.mark.gpu
@pytest.mark.parametrize("ntile", ["auto", "32", "64", "128", "256"])
@pytest.mark.parametrize("b,cin,cout,hw", UNMASKED_UP)
def test_convt_up_layer_matches_simt(monkeypatch, ntile, b, cin, cout, hw):
    """Transposed-convolution GEMM + blur pass vs the fp32 SIMT kernel on the folded parity weights, for both N-tile widths
    (a tile inside one class skips the taps the class does not use; one spanning two classes multiplies their union); 128
    and 256 are not accepted and leave the automatic choice."""
    if ntile == "auto":
        monkeypatch.delenv("E4S_B200_NTILE", raising=False)
    else:
        monkeypatch.setenv("E4S_B200_NTILE", ntile)
    c = modconv_case(b, cin, cout, hw, hw, 1, None, up=True, seed=cin + cout + hw, device=DEV)
    out = _convt(c)
    torch.cuda.synchronize()
    e = assert_close(out, _simt(c), 1e-4, f"convT + blur vs simt, N tile {ntile}: {b},{cin},{cout},{hw}")
    print(f"convT-vs-simt rel err {e:.2e}")


@pytest.mark.gpu
@pytest.mark.parametrize("noise_b", ["1", "B"])
@pytest.mark.parametrize("demod,bias,act", [(True, True, True), (False, False, False), (True, False, True), (False, True, False)])
def test_convt_up_layer_epilogue_inputs(noise_b, demod, bias, act):
    """Noise of batch 1 and B, with and without demodulation, bias and activation."""
    b, cin, cout, hw = 3, 64, 64, 24
    c = modconv_case(b, cin, cout, hw, hw, 1, None, up=True, noise_b=1 if noise_b == "1" else b, demod=demod, bias=bias,
                     seed=5, device=DEV)
    out = _convt(c, act)
    torch.cuda.synchronize()
    assert_close(out, _simt(c, act), 1e-4,
                 f"convT + blur vs simt, noise batch {noise_b}, demod {demod}, bias {bias}, act {act}")
    assert_close(_convt(c, act, False), _simt(c, act, False), 1e-4, "convT + blur vs simt, no noise")


@pytest.mark.gpu
def test_convt_up_layer_asymmetric_fir_against_oracle():
    """An asymmetric FIR (true convolution: the flipped taps matter), bare convolution, against conv_transpose2d + upfirdn2d
    of the oracle; odd output tile remainders."""
    from e4s_b200 import kernels as K
    from e4s_b200.stylegan2.modconv import PreparedConv
    g = torch.Generator().manual_seed(11)
    cin, cout, hw = 64, 32, 13
    fir = torch.outer(torch.tensor([1., 2., 4., 3.]), torch.tensor([2., 1., 5., 1.]))
    fir = fir / fir.sum() * 4
    w = torch.randn(1, cout, cin, 3, 3, generator=g)
    prep = PreparedConv().get(w.to(DEV), True, fir.to(DEV))
    x = torch.randn(1, hw, hw, cin, generator=g)
    s = 1.0 + 0.3 * torch.randn(1, 1, cin, generator=g)
    out = K.modconv3x3_up_tcr_fwd(x.to(DEV), prep.w_convt_hilo, prep.fir, s.to(DEV), None, None, None, None, False)
    wt = w[0] / (cin * 9) ** 0.5
    xs = (x * s[:, 0][:, None, None, :]).permute(0, 3, 1, 2).double()
    u = F.conv_transpose2d(xs, wt.double().transpose(0, 1), stride=2)
    ref = O.upfirdn2d(u.float(), fir, pad=(1, 1)).permute(0, 2, 3, 1)
    assert_close(out, ref, 1e-4, "convT + blur, asymmetric FIR, bare conv")


@pytest.mark.gpu
@pytest.mark.parametrize("b,cin,cout,hw", [(2, 128, 64, 40), (1, 64, 32, 64)])
def test_convt_up_layer_is_bit_reproducible(b, cin, cout, hw):
    c = modconv_case(b, cin, cout, hw, hw, 1, None, up=True, seed=7, device=DEV)
    outs = [_convt(c) for _ in range(3)]
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


@pytest.mark.gpu
def test_styled_conv_dispatch_by_mask(monkeypatch):
    """StyledConvFn: an up-sampling layer without a label map runs the transposed-convolution entry, one with a label map
    the masked one (from MASKED_CONVT_MIN_RES on; test_convt_masked covers the folded kernel below it); the unmasked one
    agrees with the SIMT kernel."""
    from e4s_b200 import kernels as K
    from e4s_b200.stylegan2 import modconv as MC
    calls = []
    for name in ("modconv3x3_up_tcr_fwd", "modconv3x3_up_masked_tcr_fwd", "modconv3x3_tcr_fwd"):
        fn = getattr(K, name)
        monkeypatch.setattr(K, name, lambda *a, _fn=fn, _n=name: (calls.append(_n), _fn(*a))[1])
    c = modconv_case(2, 64, 32, 16, 16, 1, None, up=True, seed=3, device=DEV)
    y = MC.StyledConvFn.apply(c.x, c.s, c.noise, c.nw, c.bias, None, c.prep, True, True, True)
    assert calls == ["modconv3x3_up_tcr_fwd"]
    assert_close(y, _simt(c), 1e-4)
    label = torch.zeros(2, 32, 32, dtype=torch.uint8, device=DEV)
    MC.StyledConvFn.apply(c.x, c.s, c.noise, c.nw, c.bias, label, c.prep, True, True, True)
    assert calls == ["modconv3x3_up_tcr_fwd", "modconv3x3_up_masked_tcr_fwd"]
