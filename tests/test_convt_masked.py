"""Masked up-sampling layers as a transposed-convolution GEMM over (T' pixel, region) rows plus a region-aware blur pass
(e4s_modconv3x3_up_masked_tcr_fwd).

The host test checks the row list (f64ref.row_list) and a restatement of the blur's row lookup in float64 against the mask-sum form of the reference; the GPU
tests check the entry point against the fp32 SIMT kernel (folded parity weights)."""
import pytest
import torch
import torch.nn.functional as F

from oracle import e4s_oracle as O
from conftest import assert_close
from f64ref import face_labels, row_list

DEV = "cuda:0"


def _gathered_forward(x, w, fir, s, label, ncls):
    """What the kernels compute, in float64: T'c[i] = the 2 x 2 transposed-convolution block (m, n) of x * s[region] for row
    i = (m, n, region); y[Y, X] = sum_{p,q} fir[3-p, 3-q] T(u = Y-1+p, v = X-1+q) read from row
    base[m, n] + popcount(need[m, n] & ((1 << r) - 1)) with r = label[Y, X] (zero for u < 0 or v < 0)."""
    b, cin, h, wd = x.shape
    cout = w.shape[0]
    y = torch.zeros(b, cout, 2 * h, 2 * wd, dtype=x.dtype)
    for bi in range(b):
        need, base, rows = row_list(label[bi], ncls, h, wd)
        tr = {}
        for r in {r for _, _, r in rows}:
            t = F.conv_transpose2d((x[bi:bi + 1] * s[bi, r][None, :, None, None]), w.transpose(0, 1), stride=2)[0]
            tr[r] = F.pad(t, (0, 1, 0, 1))                                   # [Cout, 2H+2, 2W+2]
        tc = torch.stack([tr[r][:, 2 * m:2 * m + 2, 2 * n:2 * n + 2] for m, n, r in rows])   # [rows, Cout, 2, 2]
        for Y in range(2 * h):
            for X in range(2 * wd):
                r = min(int(label[bi, Y, X]), ncls - 1)
                for p in range(4):
                    for q in range(4):
                        u, v = Y - 1 + p, X - 1 + q
                        if u < 0 or v < 0:
                            continue
                        m, n = u >> 1, v >> 1
                        assert (need[m][n] >> r) & 1, "an output reads a (pixel, region) row that was not computed"
                        i = base[m][n] + bin(need[m][n] & ((1 << r) - 1)).count("1")
                        assert rows[i] == (m, n, r)
                        y[bi, :, Y, X] += fir[3 - p, 3 - q] * tc[i, :, u & 1, v & 1]
    return y


def _mask_sum_reference(x, w, fir, s, label, ncls):
    """The reference form: every region's modulated up-sampling convolution, mask-summed (model.py:287-300, 395-398)."""
    y = 0
    for r in range(ncls):
        u = F.conv_transpose2d(x * s[:, r][:, :, None, None], w.transpose(0, 1), stride=2)
        y = y + (label.clamp(max=ncls - 1) == r)[:, None].to(x.dtype) * O.upfirdn2d(u, fir, pad=(1, 1))
    return y


def test_row_list_and_region_lookup_match_mask_sum():
    """Face-like, iid and single-region labels, odd sizes, a symmetric and an asymmetric FIR: the gathered rows and the
    blur's lookup give the per-region mask-sum of the reference, and no output reads a row that was not computed."""
    g = torch.Generator().manual_seed(0)
    cin, cout = 4, 3
    w = torch.randn(cout, cin, 3, 3, generator=g, dtype=torch.float64)
    asym = torch.outer(torch.tensor([1., 2., 4., 3.]), torch.tensor([2., 1., 5., 1.])).double()
    for h, wd, kind, ncls in [(5, 7, "face", 12), (6, 3, "iid", 5), (4, 4, "one", 3), (3, 5, "iid", 32)]:
        x = torch.randn(2, cin, h, wd, generator=g, dtype=torch.float64)
        s = 1.0 + 0.3 * torch.randn(2, ncls, cin, generator=g, dtype=torch.float64)
        if kind == "face":
            label = face_labels(2, 2 * h, 2 * wd)
        elif kind == "iid":
            label = torch.randint(0, ncls, (2, 2 * h, 2 * wd), generator=g, dtype=torch.uint8)
        else:
            label = torch.full((2, 2 * h, 2 * wd), 2, dtype=torch.uint8)
        for fir in (O.make_fir((1, 3, 3, 1), 4.0).double(), asym / asym.sum() * 4):
            ref = _mask_sum_reference(x, w, fir, s, label, ncls)
            assert_close(_gathered_forward(x, w, fir, s, label, ncls), ref, 1e-10, f"gathered rows {kind} {h}x{wd}")


def test_face_masks_fit_the_row_cap_from_the_min_resolution():
    """Face masks need no more rows than convt_masked_cap reserves from an output side of MASKED_CONVT_MIN_RES on, and
    more below it, where the layer stays on the folded kernel."""
    from e4s_b200.kernels import convt_masked_cap
    from e4s_b200.stylegan2.modconv import MASKED_CONVT_MIN_RES
    for ho in (8, 16, 32):
        h = ho // 2
        rows = [len(row_list(lab, 12, h, h)[2]) for lab in face_labels(4, ho, ho)]
        fits = all(r <= convt_masked_cap(h, h) for r in rows)
        assert fits == (ho >= MASKED_CONVT_MIN_RES), (ho, rows, convt_masked_cap(h, h))


# ------------------------------------------------------------------------------------------------ GPU
def _case(b, cin, cout, hw, seed, ncls=12, labels="face", noise_b=1, demod=True, bias=True):
    from e4s_b200 import kernels as K
    from e4s_b200.stylegan2.modconv import PreparedConv
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(1, cout, cin, 3, 3, generator=g)
    prep = PreparedConv().get(w.to(DEV), True, O.make_fir((1, 3, 3, 1), 4.0).to(DEV))
    x = torch.randn(b, hw, hw, cin, generator=g).to(DEV)
    s = (1.0 + 0.3 * torch.randn(b, ncls, cin, generator=g)).to(DEV)
    label = face_labels(b, 2 * hw, 2 * hw)
    if labels != "face":                              # sample 0 iid (falls back), the others face masks
        label[0] = torch.randint(0, ncls, (2 * hw, 2 * hw), generator=g, dtype=torch.uint8)
    if ncls == 32:
        label[label == 3] = 31
    noise = torch.randn(noise_b, 1, 2 * hw, 2 * hw, generator=g).to(DEV)
    nw = torch.tensor([0.37], device=DEV)
    bv = (0.1 * torch.randn(cout, generator=g)).to(DEV) if bias else None
    dm = K.demod(s, prep.wsq) if demod else None
    return K, prep, x, s, dm, label.to(DEV), noise, nw, bv


def _masked(K, prep, x, s, dm, label, noise, nw, bv, act=True):
    return K.modconv3x3_up_masked_tcr_fwd(x, prep.w_convt_hilo, prep.w_hilo, prep.fir, s, dm, label, noise, nw, bv, act)


MASKED_UP = [
    (2, 512, 512, 16),        # c4 ^32
    (2, 512, 512, 32),        # c6 ^64
    (2, 512, 256, 64),        # c8 ^128
    (2, 256, 128, 128),       # c10 ^256
    (3, 64, 32, 13),          # partial tiles
]


@pytest.mark.gpu
@pytest.mark.parametrize("b,cin,cout,hw", MASKED_UP)
def test_masked_convt_matches_simt(b, cin, cout, hw):
    K, prep, x, s, dm, label, noise, nw, bv = _case(b, cin, cout, hw, seed=cin + cout + hw)
    ref = K.modconv3x3_fwd(x, prep.wt, s, dm, label, noise, nw, bv, True, True)
    out = _masked(K, prep, x, s, dm, label, noise, nw, bv)
    torch.cuda.synchronize()
    e = assert_close(out, ref, 1e-4, f"masked convT + blur vs simt: {b},{cin},{cout},{hw}")
    print(f"masked-convT-vs-simt rel err {e:.2e}")


@pytest.mark.gpu
@pytest.mark.parametrize("ncls", [12, 32])
def test_masked_convt_mixed_fallback_batch(ncls):
    """Sample 0 has iid labels (more rows than the cap: the folded kernel computes it), the others face masks (gathered);
    ncls 32 puts pixels in region 31."""
    from e4s_b200 import kernels as K
    b, cin, cout, hw = 3, 128, 64, 24
    K, prep, x, s, dm, label, noise, nw, bv = _case(b, cin, cout, hw, seed=9, ncls=ncls, labels="mixed", noise_b=b)
    if ncls == 32:
        assert int(label.max()) == 31
    ref = K.modconv3x3_fwd(x, prep.wt, s, dm, label, noise, nw, bv, True, True)
    out = _masked(K, prep, x, s, dm, label, noise, nw, bv)
    assert_close(out, ref, 1e-4, f"mixed fallback batch, ncls {ncls}")


@pytest.mark.gpu
@pytest.mark.parametrize("noise_b", ["1", "B"])
@pytest.mark.parametrize("demod,bias,act", [(True, True, True), (False, False, False), (True, False, True), (False, True, False)])
def test_masked_convt_epilogue_inputs(noise_b, demod, bias, act):
    b, cin, cout, hw = 3, 64, 64, 24
    K, prep, x, s, dm, label, noise, nw, bv = _case(b, cin, cout, hw, seed=5, noise_b=1 if noise_b == "1" else b,
                                                    demod=demod, bias=bias)
    ref = K.modconv3x3_fwd(x, prep.wt, s, dm, label, noise, nw, bv, True, act)
    out = _masked(K, prep, x, s, dm, label, noise, nw, bv, act)
    assert_close(out, ref, 1e-4, f"noise batch {noise_b}, demod {demod}, bias {bias}, act {act}")
    ref = K.modconv3x3_fwd(x, prep.wt, s, dm, label, None, None, bv, True, act)
    out = _masked(K, prep, x, s, dm, label, None, None, bv, act)
    assert_close(out, ref, 1e-4, "no noise")


@pytest.mark.gpu
def test_masked_convt_is_bit_reproducible():
    K, prep, x, s, dm, label, noise, nw, bv = _case(3, 128, 64, 40, seed=7, labels="mixed")
    outs = [_masked(K, prep, x, s, dm, label, noise, nw, bv) for _ in range(3)]
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


@pytest.mark.gpu
def test_styled_conv_takes_masked_convt_path(monkeypatch):
    """StyledConvFn runs the gathered entry for a masked up-sampling layer from MASKED_CONVT_MIN_RES on, the folded one
    below it."""
    from e4s_b200 import kernels as K
    from e4s_b200.stylegan2 import modconv as MC
    names = []
    call = K._call
    monkeypatch.setattr(K, "_call", lambda name, *a, **kw: (names.append(name), call(name, *a, **kw))[1])
    for hw, entry in [(8, "e4s_modconv3x3_up_masked_tcr_fwd"), (4, "e4s_modconv3x3_tcr_fwd")]:
        K_, prep, x, s, dm, label, noise, nw, bv = _case(2, 64, 32, hw, seed=3)
        names.clear()
        y = MC.StyledConvFn.apply(x, s, noise, nw, bv, label, prep, True, True, True)
        assert entry in names and ("e4s_modconv3x3_up_masked_tcr_fwd" in names) == (2 * hw >= MC.MASKED_CONVT_MIN_RES)
        ref = K.modconv3x3_fwd(x, prep.wt, s, K.demod(s, prep.wsq), label, noise, nw, bv, True, True)
        assert_close(y, ref, 1e-4, f"StyledConvFn masked up-sampling {hw}")


@pytest.mark.gpu
def test_graphed_synthesis_replay_with_new_labels():
    """A CUDA-graph replay after the label maps change (face-like blocks, then iid labels that overflow the row cap) equals
    the eager forward on the new labels: the row lists and the fallback are decided on the device."""
    from types import SimpleNamespace
    from e4s_b200.networks import Net3
    from e4s_b200.pipeline import GraphedSynthesis
    from e4s_b200.stylegan2.modconv import LabelPyramid
    from e4s_b200.synthetic import load_synthetic
    opts = SimpleNamespace(num_seg_cls=6, remaining_layer_idx=13, out_size=64, train_G=False, start_from_latent_avg=False,
                           learn_in_w=False, fsencoder_type="psp")
    net = Net3(opts).eval()
    load_synthetic(net.G, salt=3)
    net = net.to(DEV)
    g = torch.Generator().manual_seed(4)
    synth = GraphedSynthesis(net, 6, (2, 6, 18, 512), (2, 1, 128, 128), randomize_noise=False)
    blocks = torch.randint(0, 6, (2, 1, 4, 4), generator=g).to(torch.uint8).repeat_interleave(32, 2).repeat_interleave(32, 3)
    for labels in (blocks, torch.randint(0, 6, (2, 1, 128, 128), generator=g).to(torch.uint8)):
        codes = torch.randn(2, 6, 18, 512, generator=g).to(DEV)
        labels = labels.to(DEV)
        with torch.no_grad():
            ref = net.gen_img(None, codes, LabelPyramid(labels[:, 0], 6), randomize_noise=False)[0]
        out = synth(codes, labels)
        assert_close(out, ref, 1e-5, "replay vs the eager forward on the new labels")
