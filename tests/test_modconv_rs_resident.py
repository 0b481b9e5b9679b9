"""Resident weights in the register-operand forward (csrc/modconv_tc.cu, conv3x3_rs_kernel): when an N tile's whole
weight block fits in shared memory beside the two halo slots, a CTA copies it once instead of with every (item, chunk).
The MMAs read the same bytes in the same order, so the output must be bitwise identical to the streamed form
(E4S_B200_RS_STREAM=1) - for every shape class that goes resident: the plain 32 -> 32 layer at N = 32, 64 -> 64, and the
transposed-convolution GEMMs of the 512^2 and 1024^2 up-sampling layers (tap groups of 4 / 2 and of 4 / 2 / 2 / 1 taps)."""
import pytest
import torch
import torch.nn.functional as F

from conftest import assert_close

DEV = "cuda:0"
KC, HALO_BYTES = 32, 10 * 18 * 32 * 4


def _is_resident(cin, nt, maxtaps, ncls):
    """The host's fit rule: two ring slots (halo + one chunk's styles of every region) and the N tile's weight block
    (every chunk, every tap of its group, hi and lo bf16 planes)."""
    slot = HALO_BYTES + ncls * KC * 4
    block = (cin // KC) * maxtaps * 2 * nt * KC * 2
    return 128 + 2 * slot + block <= torch.cuda.get_device_properties(0).shared_memory_per_block_optin


def _crosses_ntile(items_per_ntile, n_tiles, grid):
    """Some CTA of a persistent grid walks items of two N tiles (the N tile is the outermost item index)."""
    items = items_per_ntile * n_tiles
    return any(len({i // items_per_ntile for i in range(c, items, grid)}) > 1 for c in range(min(grid, items)))


def _tiles(mh, mw):
    return -(-mh // 8) * -(-mw // 16)


def _inputs(b, cin, cout, h, w, ncls, noise_b, up, seed):
    from e4s_b200.stylegan2.modconv import PreparedConv
    from oracle import e4s_oracle as O
    g = torch.Generator().manual_seed(seed)
    wt = torch.randn(1, cout, cin, 3, 3, generator=g)
    prep = PreparedConv().get(wt.to(DEV), up, O.make_fir((1, 3, 3, 1), 4.0).to(DEV) if up else None)
    x = torch.randn(b, h, w, cin, generator=g).to(DEV)
    s = (1.0 + 0.3 * torch.randn(b, ncls, cin, generator=g)).to(DEV)
    label = None
    if ncls > 1:
        coarse = torch.randint(0, ncls, (b, 1, 5, 5), generator=g).float()
        label = F.interpolate(coarse, size=(h, w), mode="nearest")[:, 0].to(torch.uint8).to(DEV)
    ho, wo = (2 * h, 2 * w) if up else (h, w)
    noise = torch.randn(noise_b, 1, ho, wo, generator=g).to(DEV)
    nw = torch.tensor([0.37], device=DEV)
    bias = (0.1 * torch.randn(cout, generator=g)).to(DEV)
    return prep, x, s, label, noise, nw, bias


def _resident_and_streamed(monkeypatch, fn):
    monkeypatch.delenv("E4S_B200_RS_STREAM", raising=False)
    res = fn()
    monkeypatch.setenv("E4S_B200_RS_STREAM", "1")
    strm = fn()
    monkeypatch.delenv("E4S_B200_RS_STREAM")
    torch.cuda.synchronize()
    return res, strm


@pytest.mark.gpu
@pytest.mark.parametrize("b,cin,cout,h,w,ncls,nt,noise_b", [
    (2, 32, 32, 37, 45, 1, 32, 1),        # c15's channels, ragged tiles
    (3, 32, 32, 21, 29, 5, 32, 3),        # masked, noise of batch B
    (1, 32, 32, 19, 23, 1, 32, 1),        # B = 1 (the inversion's batch)
    (2, 64, 64, 43, 51, 4, 64, 1),        # c13's channels, ragged tiles
    (1, 64, 64, 67, 75, 3, 64, 1),        # B = 1
    (16, 64, 64, 40, 40, 12, 32, 16),     # two 32-channel N tiles: CTAs cross from the first to the second
])
def test_plain_layer_resident_equals_streamed(monkeypatch, b, cin, cout, h, w, ncls, nt, noise_b):
    from e4s_b200 import kernels as K
    monkeypatch.setenv("E4S_B200_NTILE", str(nt))
    assert _is_resident(cin, nt, 9, ncls)
    prep, x, s, label, noise, nw, bias = _inputs(b, cin, cout, h, w, ncls, noise_b, False, seed=b + cin + h + w)
    args = (s, K.demod(s, prep.wsq), label, noise, nw, bias, False, True)
    res, strm = _resident_and_streamed(monkeypatch, lambda: K.modconv3x3_tcr_fwd(x, prep.w_hilo, *args))
    assert torch.equal(res, strm)
    if cout // nt > 1:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        assert all(_crosses_ntile(_tiles(h, w) * b, cout // nt, g) for g in (sms, 2 * sms))
        assert_close(res, K.modconv3x3_fwd(x, prep.wt, *args), 1e-4, "resident register-operand forward vs simt")


@pytest.mark.gpu
@pytest.mark.parametrize("b,cin,cout,h,w,noise_b,maxtaps", [
    (2, 64, 32, 23, 29, 1, 4),            # c14's GEMM: N = 128 in two 64-channel tiles, tap groups of 4 and 2
    (1, 64, 32, 17, 13, 1, 4),            # B = 1
    (2, 128, 64, 21, 27, 2, 4),           # c12's GEMM: N = 256 in four tiles, tap groups of 4, 2, 2 and 1
    (1, 128, 64, 29, 35, 1, 4),           # B = 1
    (16, 128, 64, 40, 40, 16, 4),         # CTAs cross N tiles (and tap groups) part-way through their items
])
def test_convt_gemm_resident_equals_streamed(monkeypatch, b, cin, cout, h, w, noise_b, maxtaps):
    """The GEMM runs on the (H + 1) x (W + 1) row grid; its output is compared through the (deterministic) blur pass."""
    from e4s_b200 import kernels as K
    monkeypatch.delenv("E4S_B200_NTILE", raising=False)
    assert _is_resident(cin, 64, maxtaps, 1)
    prep, x, s, _, noise, nw, bias = _inputs(b, cin, cout, h, w, 1, noise_b, True, seed=b + cin + h + w)
    dm = K.demod(s, prep.wsq)
    res, strm = _resident_and_streamed(
        monkeypatch, lambda: K.modconv3x3_up_tcr_fwd(x, prep.w_convt_hilo, prep.fir, s, dm, noise, nw, bias, True))
    assert torch.equal(res, strm)
    if b == 16:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        assert _crosses_ntile(_tiles(h + 1, w + 1) * b, 4 * cout // 64, sms)


@pytest.mark.gpu
def test_full_size_c15_resident_equals_streamed(monkeypatch):
    """The 1024 x 1024 32 -> 32 layer at B = 2: resident at N = 32, two CTAs per SM."""
    from e4s_b200 import kernels as K
    monkeypatch.delenv("E4S_B200_NTILE", raising=False)
    assert _is_resident(32, 32, 9, 1)
    prep, x, s, _, noise, nw, bias = _inputs(2, 32, 32, 1024, 1024, 1, 1, False, seed=15)
    args = (s, K.demod(s, prep.wsq), None, noise, nw, bias, False, True)
    res, strm = _resident_and_streamed(monkeypatch, lambda: K.modconv3x3_tcr_fwd(x, prep.w_hilo, *args))
    assert torch.equal(res, strm)
