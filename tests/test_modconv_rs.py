"""The forward modulated convolution on register operands (csrc/modconv_tc.cu, conv3x3_rs_kernel): plain layers of any
mask and the transposed-convolution GEMM of the unmasked up-sampling layers.

The host tests restate the kernel's indexing in float64 - the halo tile with zero fill, its XOR swizzle, the wgmma
fragment rows and channels, and the fragment-row -> output-pixel -> region mapping - and check it against conv2d of the
region-scaled input, and that every warp's fragment read is served in the minimal number of shared-memory wavefronts.
The GPU tests check the kernel against the fp32 SIMT kernel."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import assert_close

TH, TW, KC = 8, 16, 32
HALO_H, HALO_W = TH + 2, TW + 2
HALO_PIX = HALO_H * HALO_W
WARPS = 8


def _halo_word(hp, c):
    """fp32 word index of channel c (0..31) of halo pixel hp: 16-byte quad c // 4 stored at quad (c // 4) ^ (hp % 8)."""
    return hp * KC + (((c >> 2) ^ (hp & 7)) << 2) + (c & 3)


# per lane of a warp and fragment register r of a K16 slice ks: row g + 8 (r & 1), channels 16 ks + 8 (r >> 1) + 2 q, + 1
LANE = np.arange(32)
G, Q = LANE >> 2, LANE & 3


def _emulate(x, w, s, label, mh, mw, taps):
    """What conv3x3_rs_kernel computes, in float64.  x [B, H, W, Cin], w [9, N, Cin], s [B, ncls, Cin],
    label [B, mh, mw] or None; output rows on the mh x mw grid; source pixel of row (iy, ix) at tap t:
    (iy + t // 3 - 1, ix + t % 3 - 1)."""
    b_, h, wd, cin = x.shape
    n = w.shape[1]
    out = np.zeros((b_, mh, mw, n))
    for b in range(b_):
        for ty in range(-(-mh // TH)):
            for tx in range(-(-mw // TW)):
                y0, x0 = ty * TH, tx * TW
                # region of each fragment row's own output pixel: cls[warp, h, g]
                cls = np.zeros((WARPS, 2, 8), dtype=np.int64)
                for wp in range(WARPS):
                    for hh in range(2):
                        iy, ix = y0 + wp, x0 + G[::4] + 8 * hh
                        ok = (iy < mh) & (ix < mw)
                        if label is not None and iy < mh:
                            cls[wp, hh][ok] = label[b, iy, ix[ok]]
                acc = np.zeros((WARPS, 2, 8, n))                       # [warp, row half, g, n]
                for kc in range(cin // KC):
                    halo = np.full(HALO_PIX * KC, np.nan)
                    for hp in range(HALO_PIX):                         # fill: zero outside the image
                        sy, sx = y0 - 1 + hp // HALO_W, x0 - 1 + hp % HALO_W
                        v = x[b, sy, sx, kc * KC:(kc + 1) * KC] if (0 <= sy < h and 0 <= sx < wd) else np.zeros(KC)
                        for c in range(KC):
                            halo[_halo_word(hp, c)] = v[c]
                    assert not np.isnan(halo).any()
                    for t in taps:
                        dy, dx = t // 3, t % 3
                        for wp in range(WARPS):
                            for ks in range(2):
                                for r in range(4):
                                    hh, j = r & 1, 2 * ks + (r >> 1)
                                    hp = (wp + dy) * HALO_W + G + 8 * hh + dx
                                    for e in range(2):
                                        c = 8 * j + 2 * Q + e                 # channel within the chunk, per lane
                                        a = halo[_halo_word(hp, c)] * s[b, cls[wp, hh][G], kc * KC + c]
                                        # lane (g, q) holds A[row g + 8 hh, k = c]: the MMA sums over the four q lanes
                                        np.add.at(acc[wp, hh], G, a[:, None] * w[t][:, kc * KC + c].T)
                for wp in range(WARPS):
                    for hh in range(2):
                        for gg in range(8):
                            iy, ix = y0 + wp, x0 + gg + 8 * hh
                            if iy < mh and ix < mw:
                                out[b, iy, ix] = acc[wp, hh, gg]
    return out


def _region_scaled_conv(x, w, s, label, ncls):
    """sum_r [label == r] conv2d(x * s_r, w), pad 1: the region-selected modulated convolution without demodulation."""
    xt = torch.from_numpy(x).permute(0, 3, 1, 2)
    wt = torch.from_numpy(w).reshape(3, 3, w.shape[1], w.shape[2]).permute(2, 3, 0, 1)
    out = 0
    for r in range(ncls):
        y = F.conv2d(xt * torch.from_numpy(s[:, r])[:, :, None, None], wt, padding=1).permute(0, 2, 3, 1).numpy()
        m = np.ones(y.shape[:3]) if label is None else (label == r).astype(np.float64)
        out = out + y * m[..., None]
    return out


@pytest.mark.parametrize("b,cin,n,h,w,ncls,kind", [
    (1, 64, 8, 11, 21, 1, "none"),      # odd sizes, ragged tiles in both directions, two chunks
    (2, 32, 8, 9, 17, 4, "iid"),        # iid labels: every row its own region
    (1, 32, 16, 4, 4, 3, "blobs"),      # smaller than one tile
])
def test_rs_indexing_matches_region_scaled_conv2d(b, cin, n, h, w, ncls, kind):
    rng = np.random.default_rng(cin + n + h + w)
    x = rng.standard_normal((b, h, w, cin))
    wts = rng.standard_normal((9, n, cin))
    s = 1.0 + 0.3 * rng.standard_normal((b, ncls, cin))
    if kind == "none":
        label = None
    elif kind == "iid":
        label = rng.integers(0, ncls, (b, h, w))
    else:
        label = np.repeat(np.repeat(rng.integers(0, ncls, (b, 2, 2)), 2, 1), 2, 2)[:, :h, :w]
    got = _emulate(x, wts, s, label, h, w, range(9))
    ref = _region_scaled_conv(x, wts, s, label, ncls)
    np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-10)


@pytest.mark.parametrize("h,w", [(5, 7), (8, 16), (3, 20)])
def test_rs_indexing_transposed_convolution_row_grid(h, w):
    """The transposed-convolution GEMM: rows on the (H+1) x (W+1) grid, taps {0, 1, 3, 4}, against conv2d of the
    one-pixel-padded input with the 2 x 2 kernel of those taps."""
    rng = np.random.default_rng(h * w)
    cin, n = 32, 8
    x = rng.standard_normal((1, h, w, cin))
    wts = rng.standard_normal((9, n, cin))
    s = 1.0 + 0.3 * rng.standard_normal((1, 1, cin))
    got = _emulate(x, wts, s, None, h + 1, w + 1, (0, 1, 3, 4))
    xs = torch.from_numpy(x * s[:, 0][:, None, None, :]).permute(0, 3, 1, 2)
    k2 = torch.from_numpy(np.stack([np.stack([wts[0], wts[1]], -1), np.stack([wts[3], wts[4]], -1)], -2))   # [n, cin, dy, dx]
    ref = F.conv2d(F.pad(xs, (1, 1, 1, 1)), k2).permute(0, 2, 3, 1).numpy()
    assert ref.shape[1:3] == (h + 1, w + 1)
    np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-10)


def _wavefronts(word_addrs):
    """Shared-memory wavefronts of one warp access: the largest number of distinct 4-byte words any bank must serve."""
    words = np.unique(np.asarray(word_addrs).ravel())
    return int(np.bincount(words % 32, minlength=32).max())


def test_rs_halo_reads_and_fills_are_conflict_free():
    """Every warp-wide float2 fragment read (32 lanes x 8 bytes) is served in 2 wavefronts, the minimum for 256 bytes; an
    unswizzled [pixel][32] layout would need 8.  The fill's 16-byte cp.async writes (8 consecutive threads per pixel) hit
    each bank once per 128 bytes."""
    for t in range(9):
        dy, dx = t // 3, t % 3
        for wp in range(WARPS):
            for r in range(4):
                for ks in range(2):
                    hh, j = r & 1, 2 * ks + (r >> 1)
                    hp = (wp + dy) * HALO_W + G + 8 * hh + dx
                    c = 8 * j + 2 * Q
                    words = np.stack([_halo_word(hp, c), _halo_word(hp, c + 1)])
                    assert _wavefronts(words) == 2, (t, wp, r, ks)
                    assert _wavefronts(np.stack([hp * KC + c, hp * KC + c + 1])) == 8      # without the swizzle
    for e0 in range(0, HALO_PIX * 8, 8):
        e = np.arange(e0, e0 + 8)
        hp, c = e >> 3, e & 7
        quads = hp * KC + ((c ^ (hp & 7)) << 2)
        words = quads[:, None] + np.arange(4)[None, :]
        assert _wavefronts(words) == 1


# ------------------------------------------------------------------------------------------------ GPU
DEV = "cuda:0"


def _case(b, cin, cout, h, w, ncls, kind, seed, noise_b=1):
    from e4s_b200 import kernels as K
    from e4s_b200.stylegan2.modconv import PreparedConv
    g = torch.Generator().manual_seed(seed)
    wt = torch.randn(1, cout, cin, 3, 3, generator=g)
    prep = PreparedConv().get(wt.to(DEV), False, None)
    x = torch.randn(b, h, w, cin, generator=g).to(DEV)
    s = (1.0 + 0.3 * torch.randn(b, ncls, cin, generator=g)).to(DEV)
    if ncls == 1:
        label = None
    elif kind == "iid":
        label = torch.randint(0, ncls, (b, h, w), generator=g, dtype=torch.uint8).to(DEV)
    else:
        coarse = torch.randint(0, ncls, (b, 1, 3, 3), generator=g).float()
        label = F.interpolate(coarse, size=(h, w), mode="nearest")[:, 0].to(torch.uint8).to(DEV)
    noise = torch.randn(noise_b, 1, h, w, generator=g).to(DEV)
    nw = torch.tensor([0.37], device=DEV)
    bias = (0.1 * torch.randn(cout, generator=g)).to(DEV)
    return K, prep, x, s, label, noise, nw, bias


@pytest.mark.gpu
@pytest.mark.parametrize("b,cin,cout,h,w,ncls,kind", [
    (2, 32, 64, 24, 40, 3, "blobs"),      # Cin = 32: one chunk per item
    (1, 512, 128, 16, 32, 5, "iid"),      # Cin = 512: 16 chunks per item
    (2, 64, 64, 13, 37, 4, "blobs"),      # H, W not multiples of the tile
    (16, 512, 512, 4, 4, 12, "iid"),      # smaller than the tile: the 4x4 / 8x8 layers of a 16-face batch
    (16, 512, 512, 8, 8, 12, "blobs"),
    (1, 64, 32, 16, 16, 1, "none"),       # two items, far fewer than the grid
    (2, 96, 128, 56, 72, 2, "iid"),       # 140 items of 64 channels: a ragged last wave of the persistent loop
    (3, 32, 32, 40, 40, 1, "none"),       # c15's channels: 32-channel N tile, stacked hi / lo weights
])
def test_rs_kernel_matches_simt(b, cin, cout, h, w, ncls, kind):
    K, prep, x, s, label, noise, nw, bias = _case(b, cin, cout, h, w, ncls, kind, seed=cin + cout + h + w)
    dm = K.demod(s, prep.wsq)
    args = (s, dm, label, noise, nw, bias, False, True)
    ref = K.modconv3x3_fwd(x, prep.wt, *args)
    out = K.modconv3x3_tcr_fwd(x, prep.w_hilo, *args)
    torch.cuda.synchronize()
    assert_close(out, ref, 1e-4, f"register-operand forward vs simt {b},{cin},{cout},{h}x{w},{ncls},{kind}")


@pytest.mark.gpu
@pytest.mark.parametrize("ntile", ["32", "64"])
def test_rs_kernel_every_instantiation(monkeypatch, ntile):
    """Both instantiations (N tile 32 with stacked hi / lo weights, N tile 64 with three products) on a masked layer with
    ragged tiles, and on the transposed-convolution GEMM of an unmasked up-sampling layer."""
    monkeypatch.setenv("E4S_B200_NTILE", ntile)
    K, prep, x, s, label, noise, nw, bias = _case(2, 128, 128, 20, 27, 6, "iid", seed=3)
    dm = K.demod(s, prep.wsq)
    args = (s, dm, label, noise, nw, bias, False, True)
    assert_close(K.modconv3x3_tcr_fwd(x, prep.w_hilo, *args), K.modconv3x3_fwd(x, prep.wt, *args), 1e-4,
                 f"N tile {ntile}")
    from e4s_b200.stylegan2.modconv import PreparedConv
    from oracle import e4s_oracle as O
    g = torch.Generator().manual_seed(4)
    cin, cout, hw = 64, 32, 19
    wt = torch.randn(1, cout, cin, 3, 3, generator=g)
    pu = PreparedConv().get(wt.to(DEV), True, O.make_fir((1, 3, 3, 1), 4.0).to(DEV))
    xu = torch.randn(2, hw, hw, cin, generator=g).to(DEV)
    su = (1.0 + 0.3 * torch.randn(2, 1, cin, generator=g)).to(DEV)
    nu = torch.randn(1, 1, 2 * hw, 2 * hw, generator=g).to(DEV)
    dmu = K.demod(su, pu.wsq)
    ref = K.modconv3x3_fwd(xu, pu.wt, su, dmu, None, nu, nw, None, True, True)
    out = K.modconv3x3_up_tcr_fwd(xu, pu.w_convt_hilo, pu.fir, su, dmu, nu, nw, None, True)
    assert_close(out, ref, 1e-4, f"convT GEMM, N tile {ntile}")


@pytest.mark.gpu
@pytest.mark.parametrize("noise_b", ["1", "B"])
@pytest.mark.parametrize("demod,bias,act", [(True, True, True), (False, False, False), (True, False, True), (False, True, False)])
def test_rs_kernel_epilogue_inputs(noise_b, demod, bias, act):
    """Noise of batch 1 and B, with and without demodulation, bias and activation."""
    b = 3
    K, prep, x, s, label, noise, nw, bv = _case(b, 64, 64, 20, 24, 4, "blobs", seed=9, noise_b=1 if noise_b == "1" else b)
    dm = K.demod(s, prep.wsq) if demod else None
    bv = bv if bias else None
    for nz, w_ in ((noise, nw), (None, None)):
        args = (s, dm, label, nz, w_, bv, False, act)
        assert_close(K.modconv3x3_tcr_fwd(x, prep.w_hilo, *args), K.modconv3x3_fwd(x, prep.wt, *args), 1e-4,
                     f"noise batch {noise_b}, noise {nz is not None}, demod {demod}, bias {bias}, act {act}")


@pytest.mark.gpu
def test_rs_kernel_is_bit_reproducible():
    K, prep, x, s, label, noise, nw, bias = _case(2, 128, 64, 30, 44, 5, "iid", seed=12)
    args = (s, K.demod(s, prep.wsq), label, noise, nw, bias, False, True)
    outs = [K.modconv3x3_tcr_fwd(x, prep.w_hilo, *args) for _ in range(3)]
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


@pytest.mark.gpu
def test_plain_layer_and_convt_gemm_run_on_register_operand_kernel():
    """torch.profiler: a plain layer and the unmasked up-sampling layer's GEMM launch conv3x3_rs_kernel, not the
    shared-memory-operand kernel."""
    from torch.profiler import ProfilerActivity, profile
    from e4s_b200.stylegan2.modconv import PreparedConv
    from oracle import e4s_oracle as O
    K, prep, x, s, label, noise, nw, bias = _case(2, 64, 64, 32, 32, 3, "blobs", seed=1)
    args = (s, K.demod(s, prep.wsq), label, noise, nw, bias, False, True)
    pu = PreparedConv().get(torch.randn(1, 32, 64, 3, 3).to(DEV), True, O.make_fir((1, 3, 3, 1), 4.0).to(DEV))
    su = s[:, :1].contiguous()
    nu = torch.randn(1, 1, 64, 64, device=DEV)
    for fn in (lambda: K.modconv3x3_tcr_fwd(x, prep.w_hilo, *args),
               lambda: K.modconv3x3_up_tcr_fwd(x, pu.w_convt_hilo, pu.fir, su, K.demod(su, pu.wsq), nu, nw, None, True)):
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = [ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA]
        assert any("conv3x3_rs_kernel" in n for n in names), names
        assert not any("conv3x3_wgmma_kernel" in n for n in names), names
