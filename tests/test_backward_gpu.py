"""GPU parity of the backward kernels (input/style gradients) and of the inversion loop against the CPU oracle's autograd."""
import types

import pytest
import torch

from oracle import e4s_oracle as O
from conftest import REL_TOL, assert_close

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def cu(t):
    return t.to(DEV)


def _load(module, salt):
    st = O.synthetic_state({k: tuple(v.shape) for k, v in module.state_dict().items()}, salt)
    module.load_state_dict(st)
    for p in module.parameters():
        p.requires_grad = False
    return st


@pytest.mark.parametrize("kind", ["blobs", "iid"])
@pytest.mark.parametrize("tag,cin,cout,up,hw,masked", [
    ("plain", 16, 24, False, 8, True), ("up", 24, 16, True, 8, True), ("wide", 72, 40, False, 12, True),
    ("global", 32, 32, False, 10, False), ("global_up", 16, 8, True, 6, False)])
def test_styled_conv_gradients(kind, tag, cin, cout, up, hw, masked):
    from e4s_b200.stylegan2.model import StyledConv
    g = torch.Generator().manual_seed(17 + hw)
    ncls = 5
    codes, mask, _, _ = O.synthetic_inputs(2, ncls, 16, 32, seed=3, kind=kind)
    m = StyledConv(cin, cout, 3, 512, upsample=up, mask_op=masked)
    st = _load(m, 7 + len(tag))
    x = torch.randn(2, cin, hw, hw, generator=g)
    style = codes[:, :, 0] if masked else codes[:, 0, 0]
    hout = 2 * hw if up else hw
    nz = torch.randn(2, 1, hout, hout, generator=g)
    go = torch.randn(2, cout, hout, hout, generator=g)
    # oracle autograd (CPU)
    xr, sr = x.clone().requires_grad_(True), style.clone().requires_grad_(True)
    O.styled_conv(xr, sr, mask, nz, st, "", up, masked).backward(go)
    # ours
    xg, sg = cu(x).requires_grad_(True), cu(style).requires_grad_(True)
    y = m.to(DEV)(xg, sg, cu(mask), noise=cu(nz))
    y.backward(cu(go))
    assert_close(xg.grad, xr.grad, 1e-4, f"{kind}/{tag} d/dx")
    assert_close(sg.grad, sr.grad, 1e-4, f"{kind}/{tag} d/dstyle")


def test_styled_conv_noise_gradient():
    from e4s_b200.stylegan2.model import StyledConv
    g = torch.Generator().manual_seed(5)
    m = StyledConv(16, 24, 3, 512, mask_op=False)
    st = _load(m, 3)
    x, style = torch.randn(2, 16, 8, 8, generator=g), torch.randn(2, 512, generator=g)
    nz, go = torch.randn(2, 1, 8, 8, generator=g), torch.randn(2, 24, 8, 8, generator=g)
    nr = nz.clone().requires_grad_(True)
    O.styled_conv(x, style, None, nr, st, "", False, False).backward(go)
    ng = cu(nz).requires_grad_(True)
    m.to(DEV)(cu(x), cu(style), None, noise=ng).backward(cu(go))
    assert_close(ng.grad, nr.grad, 1e-4, "d/dnoise")


@pytest.mark.parametrize("masked", [True, False])
def test_torgb_gradients(masked):
    from e4s_b200.stylegan2.model import ToRGB
    g = torch.Generator().manual_seed(23)
    codes, mask, _, _ = O.synthetic_inputs(2, 5, 16, 32, seed=3, kind="iid")
    m = ToRGB(24, 512, upsample=True, mask_op=masked)
    st = _load(m, 11)
    x, skip = torch.randn(2, 24, 16, 16, generator=g), torch.randn(2, 3, 8, 8, generator=g)
    style = codes[:, :, 1] if masked else codes[:, 0, 1]
    go = torch.randn(2, 3, 16, 16, generator=g)
    xr, sr, kr = x.clone().requires_grad_(True), style.clone().requires_grad_(True), skip.clone().requires_grad_(True)
    O.to_rgb(xr, sr, mask, kr, st, "", masked).backward(go)
    xg, sg, kg = cu(x).requires_grad_(True), cu(style).requires_grad_(True), cu(skip).requires_grad_(True)
    m.to(DEV)(xg, sg, cu(mask), kg).backward(cu(go))
    assert_close(xg.grad, xr.grad, 1e-4, "d/dx")
    assert_close(sg.grad, sr.grad, 1e-4, "d/dstyle")
    assert_close(kg.grad, kr.grad, 1e-4, "d/dskip")


def _generator_dcodes():
    from e4s_b200.stylegan2.model import Generator
    size, K = 32, 13
    G = Generator(size, 512, 8, split_layer_idx=5, remaining_layer_idx=K).eval()
    _load(G, size)
    G = G.to(DEV)
    codes, mask, _, noise = O.synthetic_inputs(1, 12, size, 64, seed=size + K, kind="iid")
    cg = cu(codes).requires_grad_(True)
    img, _, _ = G([cg], None, cu(mask), input_is_latent=True, noise=[cu(n) for n in noise])
    R = torch.randn(img.shape, generator=torch.Generator().manual_seed(99))
    (img * cu(R)).sum().backward()
    return cg.grad


def test_generator_gradient_golden_exact_path(golden, monkeypatch):
    """d<image, R>/d(codes) for the 32x32, K=13, iid-mask case against the reference's own autograd result, with the
    forward on the exact-fp32 kernels: max-norm parity at the 1e-3 bar."""
    monkeypatch.setenv("E4S_B200_CONV", "simt")
    monkeypatch.setenv("E4S_B200_BWD", "simt")
    assert_close(_generator_dcodes(), golden["generator/g32_k13_iid/dcodes"], REL_TOL, "dcodes (fp32 path)")


def test_generator_gradient_golden_tensor_core_path(golden, monkeypatch):
    """Same gradient with the forward on the tensor-core kernels.  The backward is exact given the forward's
    activations, but leaky-ReLU's derivative is discontinuous: a forward that differs by 1e-5 (split-bf16) flips the
    sign of a few dozen near-zero pre-activations per layer, each moving its share of the gradient by O(1).  In
    max-norm that is ~1e-2 for this case (any non-bit-exact forward - e.g. the reference's own default TF32 convs -
    shows the same effect, larger); the direction and norm of the gradient are what the optimiser consumes."""
    monkeypatch.setenv("E4S_B200_CONV", "tcr")
    monkeypatch.setenv("E4S_B200_BWD", "tc")
    g = _generator_dcodes().double().cpu().flatten()
    ref = torch.from_numpy(golden["generator/g32_k13_iid/dcodes"]).double().flatten()
    rel_l2 = float((g - ref).norm() / ref.norm())
    cos = float(torch.dot(g, ref) / (g.norm() * ref.norm()))
    print(f"tensor-core path gradient: rel-L2 {rel_l2:.2e}, cosine {cos:.6f}")
    assert rel_l2 < 3e-2 and cos > 0.9995, (rel_l2, cos)


def test_inversion_loop_matches_oracle(monkeypatch):
    """Three Adam steps of the texture-vector optimisation (scripts/optimization.py:209-232, l2 term, fixed noise):
    losses and the updated latent against the same loop run through the CPU oracle."""
    from e4s_b200.networks import Net3
    from e4s_b200.optimization import invert
    monkeypatch.setenv("E4S_B200_CONV", "simt")          # strict step-by-step comparison on the exact-fp32 kernels
    monkeypatch.setenv("E4S_B200_BWD", "simt")
    size, ncls, K = 32, 12, 13
    opts = types.SimpleNamespace(fsencoder_type="psp", remaining_layer_idx=K, num_seg_cls=ncls, out_size=size,
                                 train_G=False, start_from_latent_avg=True, learn_in_w=False)
    net = Net3(opts).eval()
    st = O.synthetic_state({k: tuple(v.shape) for k, v in net.state_dict().items()}, salt=5)
    net.load_state_dict(st)
    for p in net.parameters():
        p.requires_grad = False
    net = net.to(DEV)
    lat = 0.1 * torch.randn(18, 512, generator=torch.Generator().manual_seed(77))
    net.latent_avg = cu(lat)
    g = torch.Generator().manual_seed(8)
    sv0 = 0.5 * torch.randn(1, ncls, 1280, generator=g)
    _, mask, _, noise = O.synthetic_inputs(1, ncls, size, 64, seed=12)
    gst = {k[2:]: v for k, v in st.items() if k.startswith("G.")}
    with torch.no_grad():
        target, _ = O.generator_forward(gst, O.cal_style_codes(st, 0.5 * torch.randn(1, ncls, 1280, generator=g), lat, K),
                                        mask, noise, size, K)
    # oracle loops: Adam for the loss trajectory (its sign-like first steps amplify 1e-7 gradient noise on
    # near-zero-gradient coordinates, so latents are compared under plain SGD, which is linear in the gradient)
    def oracle_loop(opt_name, lr):
        latent = sv0.clone().requires_grad_(True)
        opt = (torch.optim.Adam if opt_name == "adam" else torch.optim.SGD)([latent], lr=lr)
        losses = []
        for _ in range(3):
            opt.zero_grad()
            rec, _ = O.generator_forward(gst, O.cal_style_codes(st, latent, lat, K), mask, noise, size, K)
            loss = torch.nn.functional.mse_loss(rec, target)
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
        return latent.detach(), losses

    for opt_name, lr in (("adam", 1e-2), ("sgd", 2.0)):
        ref_latent, ref_losses = oracle_loop(opt_name, lr)
        out_latent, recon, hist = invert(net, cu(target), cu(mask), style_vectors=cu(sv0), steps=3, lr=lr, opt_name=opt_name,
                                         noise=[cu(n) for n in noise])
        ours = [float(h) for h in hist]
        for a, b in zip(ours, ref_losses):
            assert abs(a - b) <= 1e-3 * abs(b), (opt_name, ours, ref_losses)
        if opt_name == "sgd":
            assert_close(out_latent - cu(sv0), ref_latent - sv0, 5e-3, "SGD update of the texture vectors after 3 steps")
        assert ours[-1] < ours[0], (opt_name, ours)
    # and the same loop on the tensor-core forward: the loss trajectory must still track the oracle's
    monkeypatch.setenv("E4S_B200_CONV", "tcr")
    monkeypatch.setenv("E4S_B200_BWD", "tc")
    ref_latent, ref_losses = oracle_loop("adam", 1e-2)
    _, _, hist = invert(net, cu(target), cu(mask), style_vectors=cu(sv0), steps=3, lr=1e-2, opt_name="adam",
                        noise=[cu(n) for n in noise])
    for a, b in zip([float(h) for h in hist], ref_losses):
        assert abs(a - b) <= 5e-3 * abs(b), ([float(h) for h in hist], ref_losses)


def test_graphed_inversion_equals_eager():
    """invert(cuda_graph=True) makes exactly `steps` optimiser updates and follows the eager loop (same fixed noise): the
    capture itself does not execute a step (round-1 review: the graphed path ran one update short and logged a stale loss)."""
    from e4s_b200.networks import Net3
    from e4s_b200.optimization import invert
    size, ncls, K = 32, 12, 13
    opts = types.SimpleNamespace(fsencoder_type="psp", remaining_layer_idx=K, num_seg_cls=ncls, out_size=size,
                                 train_G=False, start_from_latent_avg=True, learn_in_w=False)
    net = Net3(opts).eval()
    st = O.synthetic_state({k: tuple(v.shape) for k, v in net.state_dict().items()}, salt=5)
    net.load_state_dict(st)
    for p in net.parameters():
        p.requires_grad = False
    net = net.to(DEV)
    net.latent_avg = cu(0.1 * torch.randn(18, 512, generator=torch.Generator().manual_seed(77)))
    g = torch.Generator().manual_seed(8)
    sv0 = cu(0.5 * torch.randn(1, ncls, 1280, generator=g))
    _, mask, _, noise = O.synthetic_inputs(1, ncls, size, 64, seed=12)
    noise = [cu(n) for n in noise]
    with torch.no_grad():
        target, _, _ = net.gen_img(None, net.cal_style_codes(cu(0.5 * torch.randn(1, ncls, 1280, generator=g))), cu(mask), noise=noise)
    steps = 7
    lat_e, _, hist_e = invert(net, target, cu(mask), style_vectors=sv0, steps=steps, noise=noise)
    lat_g, _, hist_g = invert(net, target, cu(mask), style_vectors=sv0, steps=steps, noise=noise, cuda_graph=True)
    assert len(hist_e) == len(hist_g) == steps
    he, hg = [float(h) for h in hist_e], [float(h) for h in hist_g]
    for a, b in zip(hg, he):
        assert abs(a - b) <= 2e-3 * abs(b), (hg, he)
    assert len(set(hg)) == steps, hg                          # no duplicated (stale) entry
    # same number of Adam updates: the latent moved as far as the eager one (Adam's first steps are ~lr per coordinate)
    de, dg = (lat_e - sv0).abs().mean(), (lat_g - sv0).abs().mean()
    assert abs(float(dg) - float(de)) <= 0.05 * float(de), (float(dg), float(de))
    with pytest.raises(ValueError):
        invert(net, target, cu(mask), style_vectors=sv0, steps=2, opt_name="sgd", cuda_graph=True)
    with pytest.raises(ValueError):
        invert(net, target, cu(mask), style_vectors=sv0, steps=2, callback=lambda *a: None, cuda_graph=True)


# ------------------------------------------------------------------ tensor-core dgrad vs the fp32 SIMT dgrad
@pytest.mark.parametrize("b,cin,cout,hw,up,ncls,kind,act", [
    (1, 64, 64, 16, False, 1, "blobs", True),
    (2, 128, 64, 24, False, 1, "blobs", False),
    (1, 64, 128, 16, True, 1, "blobs", True),
    (2, 96, 160, 20, False, 5, "blobs", True),
    (1, 128, 64, 16, False, 6, "iid", True),
    (2, 64, 96, 12, True, 4, "blobs", True),
    (1, 256, 512, 16, True, 3, "iid", True),
    (1, 32, 32, 40, False, 1, "blobs", True),
    (1, 512, 512, 4, False, 12, "iid", True),      # the 4x4 / 8x8 layers of a one-face inversion
    (1, 512, 512, 4, True, 3, "iid", True),
    (2, 256, 256, 8, False, 12, "blobs", True),
])
def test_dgrad_tc_matches_simt(b, cin, cout, hw, up, ncls, kind, act):
    _dgrad_case(b, cin, cout, hw, up, ncls, kind, act)


@pytest.mark.parametrize("ntile", ["32", "64", "128", "256"])
@pytest.mark.parametrize("b,cin,cout,hw,up,ncls,kind,act", [
    (1, 512, 512, 8, False, 12, "iid", True),
    (1, 512, 512, 8, True, 3, "iid", True),
    (2, 256, 128, 16, True, 4, "blobs", True),
])
def test_dgrad_tc_every_n_tile_width(monkeypatch, ntile, b, cin, cout, hw, up, ncls, kind, act):
    """csrc/modconv_tc.cu:pick_ntile (input channels per work item, 32 or 64 by occupancy): both widths give the same
    gradients, and a width E4S_B200_NTILE does not accept (128, 256) leaves the automatic choice."""
    monkeypatch.setenv("E4S_B200_NTILE", ntile)
    _dgrad_case(b, cin, cout, hw, up, ncls, kind, act)


@pytest.mark.parametrize("split", ["1,1", "3,1", "2,2", "12,4", "5,4"])
@pytest.mark.parametrize("b,cin,cout,hw,up,ncls,kind,act", [
    (1, 512, 512, 4, False, 12, "iid", True),
    (1, 512, 512, 8, True, 12, "iid", True),
    (2, 128, 64, 20, True, 5, "blobs", True),        # tiles with fewer regions than the split: some work items are empty
    (1, 64, 64, 24, False, 1, "blobs", False),       # single region: the region split degenerates, the parity split does not apply
    (1, 64, 32, 24, True, 1, "blobs", True),         # single region, up-sampling: parity split only
])
def test_dgrad_tc_split_work_items(monkeypatch, split, b, cin, cout, hw, up, ncls, kind, act):
    """csrc/modconv_tc.cu:choose_split cuts a tile's chain of region passes / parity planes into several work items whose
    partial sums meet in gx and gs (atomics): every split gives the same gradients."""
    monkeypatch.setenv("E4S_B200_DGRAD_SPLIT", split)
    _dgrad_case(b, cin, cout, hw, up, ncls, kind, act)


def _dgrad_case(b, cin, cout, hw, up, ncls, kind, act):
    from e4s_b200 import kernels as K
    from e4s_b200.stylegan2.modconv import PreparedConv
    from e4s_b200.stylegan2 import modconv_bwd as MB
    g = torch.Generator().manual_seed(cin + cout + hw)
    w = torch.randn(1, cout, cin, 3, 3, generator=g)
    prep = PreparedConv().get(cu(w), up, cu(O.make_fir((1, 3, 3, 1), 4.0)) if up else None)
    ho = 2 * hw if up else hw
    x = cu(torch.randn(b, hw, hw, cin, generator=g))
    s = cu(1.0 + 0.3 * torch.randn(b, ncls, cin, generator=g))
    dm = K.demod(s, prep.wsq)
    gy = cu(torch.randn(b, ho, ho, cout, generator=g))
    y = cu(torch.randn(b, ho, ho, cout, generator=g))
    if kind == "iid":
        label = torch.randint(0, ncls, (b, ho, ho), generator=g, dtype=torch.uint8)
    else:
        coarse = torch.randint(0, ncls, (b, 1, max(2, ho // 8), max(2, ho // 8)), generator=g).float()
        label = torch.nn.functional.interpolate(coarse, size=(ho, ho), mode="nearest")[:, 0].to(torch.uint8)
    label = cu(label) if ncls > 1 else None
    gx0, gs0 = K.modconv3x3_bwd(gy, y if act else None, x, MB._dgrad_weights(prep), s, dm, label, up, act, True, True)
    gx1, gs1 = K.modconv3x3_bwd_tc(gy, y if act else None, x, MB._dgrad_planes(prep), s, dm, label, up, act, True, True)
    torch.cuda.synchronize()
    assert_close(gx1, gx0, 1e-4, "gx tc vs simt")
    assert_close(gs1, gs0, 1e-4, "gs tc vs simt")
