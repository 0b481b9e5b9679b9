"""Work items of the up-sampling layers' transposed-convolution GEMMs (csrc/wgmma_convt.cu).

Masked layers (the gathered-row GEMM): one batch holds a single-region sample (exactly (H+1)(W+1) rows), a face-mask
sample, an iid sample over the cap (left to the folded kernel) and a sample whose row count is a multiple of 128 (no
partial 128-row block).  Unmasked layers (convt_rs_kernel): the four classes of a
32-channel slice in one item, at Cout = 32 (one slice: c14's shape class), resident and streamed.  Both against the fp32 SIMT kernel on the folded parity
weights."""
import pytest
import torch
import torch.nn.functional as F

from conftest import assert_close
from f64ref import default_kernels, labels, modconv_case, row_list  # noqa: F401

DEV = "cuda:0"


def _row_count(label, ncls, h, w):
    """Rows of one sample's list: per T' pixel (m, n), the regions of the clipped output window [2m-2, 2m+2]^2."""
    onehot = F.one_hot(label.long().clamp(max=ncls - 1), ncls).permute(2, 0, 1)[None].float()     # [1, ncls, 2H, 2W]
    present = F.max_pool2d(F.pad(onehot, (2, 3, 2, 3)), 5, stride=2)                             # [1, ncls, H+1, W+1]
    assert present.shape[-2:] == (h + 1, w + 1)
    return int(present.sum())


def _multiple_of_128(h, w, ncls):
    """A blob label map (a random coarse map of random size, nearest-upsampled, and one pixel of a random region; the first
    seed that fits) whose row list is a multiple of 128 long and within the cap."""
    from e4s_b200.kernels import convt_masked_cap
    for seed in range(10000):
        g = torch.Generator().manual_seed(seed)
        cy, cx = (int(v) for v in torch.randint(2, 9, (2,), generator=g))
        coarse = torch.randint(0, ncls, (1, 1, cy, cx), generator=g).float()
        lab = F.interpolate(coarse, size=(2 * h, 2 * w), mode="nearest")[0, 0].to(torch.uint8)
        y, x, r = (int(v) for v in torch.randint(0, 1 << 16, (3,), generator=g))
        lab[y % (2 * h), x % (2 * w)] = r % ncls        # one odd pixel: the counts of blob maps alone are all odd
        n = _row_count(lab, ncls, h, w)
        if n % 128 == 0 and n <= convt_masked_cap(h, w):
            return lab
    raise AssertionError("no seed gives a multiple of 128 rows")


def test_row_count_helper_matches_row_list():
    g = torch.Generator().manual_seed(2)
    for h, w, ncls in [(5, 7, 12), (6, 3, 5)]:
        lab = torch.randint(0, ncls, (2 * h, 2 * w), generator=g, dtype=torch.uint8)
        need, base, rows = row_list(lab, ncls, h, w)
        assert _row_count(lab, ncls, h, w) == len(rows)
    lab = _multiple_of_128(16, 16, 12)
    assert len(row_list(lab, 12, 16, 16)[2]) % 128 == 0


@pytest.mark.gpu
@pytest.mark.parametrize("cin,cout,hw", [
    (512, 512, 16),           # c4 ^32
    (256, 128, 128),          # c10 ^256
    (64, 96, 13),             # partial pixel tiles, three channel slices
])
def test_masked_item_walk_matches_simt(cin, cout, hw):
    from e4s_b200 import kernels as K
    ncls = 12
    c = modconv_case(4, cin, cout, hw, hw, ncls, "face", up=True, noise_b=4, seed=cin + hw, device=DEV)
    cap = K.convt_masked_cap(hw, hw)
    c.label[0] = 5                                                         # one region: (H+1)(W+1) rows
    c.label[2] = labels("iid", 1, c.ho, c.wo, ncls, torch.Generator().manual_seed(hw))[0].to(DEV)
    c.label[3] = _multiple_of_128(hw, hw, ncls).to(DEV)
    counts = [_row_count(c.label[i].cpu(), ncls, hw, hw) for i in range(4)]
    assert counts[0] == (hw + 1) ** 2 and counts[1] <= cap and counts[2] > cap
    assert counts[3] <= cap and counts[3] % 128 == 0
    out = K.modconv3x3_up_masked_tcr_fwd(c.x, c.prep.w_convt_hilo, c.prep.w_hilo, c.prep.fir, c.s, c.dm, c.label, c.noise,
                                         c.nw, c.bias, True)
    ref = K.modconv3x3_fwd(c.x, c.prep.wt, c.s, c.dm, c.label, c.noise, c.nw, c.bias, True, True)
    torch.cuda.synchronize()
    for i in range(4):
        assert_close(out[i], ref[i], 1e-4, f"masked item walk vs simt, sample {i} ({counts[i]} rows): {cin},{cout},{hw}")


@pytest.mark.gpu
@pytest.mark.parametrize("b,hw", [(3, 40), (2, 23)])
def test_unmasked_single_slice_matches_simt_and_resident_equals_streamed(monkeypatch, b, hw):
    from e4s_b200 import kernels as K
    c = modconv_case(b, 64, 32, hw, hw, 1, None, up=True, seed=hw, device=DEV)

    def run():
        return K.modconv3x3_up_tcr_fwd(c.x, c.prep.w_convt_hilo, c.prep.fir, c.s, c.dm, c.noise, c.nw, c.bias, True)
    res = run()
    monkeypatch.setenv("E4S_B200_RS_STREAM", "1")
    strm = run()
    monkeypatch.delenv("E4S_B200_RS_STREAM")
    ref = K.modconv3x3_fwd(c.x, c.prep.wt, c.s, c.dm, None, c.noise, c.nw, c.bias, True, True)
    torch.cuda.synchronize()
    assert torch.equal(res, strm)
    assert_close(res, ref, 1e-4, f"unmasked Cout 32 vs simt: {b},{hw}")
