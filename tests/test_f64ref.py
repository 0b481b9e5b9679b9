"""The shared float64 references of f64ref.py against the CPU oracle (and through it the goldens), in float64 on the CPU,
<= 1e-10; and the 1024 generator's layer table against the oracle's layer plan."""
import pytest
import torch

import f64ref as F64
from oracle import e4s_oracle as O
from conftest import assert_close


def _oracle_styled(x, style, mask, noise, p, up, masked, demod):
    """O.styled_conv, or its demodulation-free variant assembled from the oracle's modulated_conv2d."""
    if demod:
        return O.styled_conv(x, style, mask, noise, p, "", up, masked)
    wk = dict(weight=p["conv.weight"], mod_weight=p["conv.modulation.weight"], mod_bias=p["conv.modulation.bias"],
              demodulate=False, upsample=up)
    if masked:
        out = sum(O.modulated_conv2d(x, style[:, c], **wk) * mask[:, c:c + 1] for c in range(style.shape[1]))
    else:
        out = O.modulated_conv2d(x, style, **wk)
    return O.fused_leaky_relu(out + p["noise.weight"] * noise, p["activate.bias"])


def _styled_inputs(up, masked):
    """Seeded StyledConv parameters p, label map, x, style, noise and output gradient; one region (1) may be absent, the
    last one is not.  The oracle resizes masks to squares."""
    g = torch.Generator().manual_seed(11 + 2 * up + masked)
    b, cin, cout, h, w, ncls, sdim = 2, 6, 5, 6, 6, 4, 16
    ho, wo = (2 * h, 2 * w) if up else (h, w)
    dd = dict(generator=g, dtype=torch.float64)
    p = {"conv.weight": torch.randn(1, cout, cin, 3, 3, **dd), "conv.modulation.weight": torch.randn(cin, sdim, **dd),
         "conv.modulation.bias": 1.0 + 0.1 * torch.randn(cin, **dd), "noise.weight": torch.tensor([0.37], dtype=torch.float64),
         "activate.bias": 0.1 * torch.randn(cout, **dd)}
    label = torch.randint(0, ncls, (b, ho, wo), generator=g)
    label[:, 0, 0] = ncls - 1
    label[label == 1] = 2
    x = torch.randn(b, cin, h, w, **dd)
    style = torch.randn(b, ncls, sdim, **dd) if masked else torch.randn(b, sdim, **dd)
    noise = torch.randn(1, 1, ho, wo, **dd)
    go = torch.randn(b, cout, ho, wo, **dd)
    return p, label, ncls, x, style, noise, go


def _style(p, style, masked):
    s = F64.equal_linear(style, p["conv.modulation.weight"], p["conv.modulation.bias"])
    return s if masked else s[:, None]


@pytest.mark.parametrize("demod", [True, False])
@pytest.mark.parametrize("masked", [True, False])
@pytest.mark.parametrize("up", [False, True])
def test_ref_styled_matches_oracle(up, masked, demod):
    """act(styled_preact) against the oracle's StyledConv, forward and autograd (x, style, noise), <= 1e-10."""
    p, label, ncls, x, style, noise, go = _styled_inputs(up, masked)
    for t in (x, style, noise):
        t.requires_grad_(True)
    ref = _oracle_styled(x, style, F64.onehot(label, ncls, torch.float64) if masked else None, noise, p, up, masked, demod)
    gref = torch.autograd.grad(ref, (x, style, noise), go)
    ours = F64.act(F64.styled_preact(x, _style(p, style, masked), p["conv.weight"][0], label if masked else None, noise,
                                     p["noise.weight"], p["activate.bias"], up, demod))
    gours = torch.autograd.grad(ours, (x, style, noise), go)
    assert_close(ours, ref, 1e-10, "forward")
    for a, r, what in zip(gours, gref, ("d/dx", "d/dstyle", "d/dnoise")):
        assert_close(a, r, 1e-10, what)


@pytest.mark.parametrize("masked", [True, False])
@pytest.mark.parametrize("up", [False, True])
def test_per_pixel_form_matches_region_sum_and_oracle(up, masked):
    """styled_conv_per_pixel (parity kernels and the unfold DGEMM for masked layers) against act(styled_preact) and the
    oracle's StyledConv, forward, <= 1e-10."""
    p, label, ncls, x, style, noise, _ = _styled_inputs(up, masked)
    s, lab = _style(p, style, masked), (label if masked else None)
    w, nw, bias = p["conv.weight"][0], p["noise.weight"], p["activate.bias"]
    ours = F64.styled_conv_per_pixel(x, s, w, lab, noise, nw, bias, up)
    assert_close(ours, F64.act(F64.styled_preact(x, s, w, lab, noise, nw, bias, up, True)), 1e-10, "region sum")
    ref = O.styled_conv(x, style, F64.onehot(label, ncls, torch.float64) if masked else None, noise, p, "", up, masked)
    assert_close(ours, ref, 1e-10, "oracle")


@pytest.mark.parametrize("skip", [True, False])
@pytest.mark.parametrize("masked", [True, False])
def test_ref_to_rgb_matches_oracle(masked, skip):
    """to_rgb against the oracle's ToRGB, forward and autograd (x, style, skip), <= 1e-10."""
    g = torch.Generator().manual_seed(5 + masked)
    b, cin, h, w, ncls, sdim = 2, 8, 6, 6, 5, 16
    dd = dict(generator=g, dtype=torch.float64)
    p = {"conv.weight": torch.randn(1, 3, cin, 1, 1, **dd), "conv.modulation.weight": torch.randn(cin, sdim, **dd),
         "conv.modulation.bias": 1.0 + 0.1 * torch.randn(cin, **dd), "bias": 0.1 * torch.randn(1, 3, 1, 1, **dd)}
    label = torch.randint(0, ncls, (b, h, w), generator=g)
    x = torch.randn(b, cin, h, w, **dd).requires_grad_(True)
    style = (torch.randn(b, ncls, sdim, **dd) if masked else torch.randn(b, sdim, **dd)).requires_grad_(True)
    sk = torch.randn(b, 3, h // 2, w // 2, **dd).requires_grad_(True) if skip else None
    go = torch.randn(b, 3, h, w, **dd)
    inputs = (x, style) + ((sk,) if skip else ())

    ref = O.to_rgb(x, style, F64.onehot(label, ncls, torch.float64) if masked else None, sk, p, "", masked)
    gref = torch.autograd.grad(ref, inputs, go)
    ours = F64.to_rgb(x, _style(p, style, masked), p["conv.weight"], label if masked else None, p["bias"], sk)
    gours = torch.autograd.grad(ours, inputs, go)
    assert_close(ours, ref, 1e-10, "forward")
    for a, r, what in zip(gours, gref, ("d/dx", "d/dstyle", "d/dskip")):
        assert_close(a, r, 1e-10, what)


def test_layer_table_matches_the_oracle_plan():
    """The masked flags of the table are the oracle's generator_layer_plan(1024, 13)."""
    log_size, conv_mask, rgb_mask = O.generator_layer_plan(F64.RES, F64.K_LAYERS)
    rows = {r.module: r for r in F64.layer_table()}
    assert len(rows) == 2 + 3 * (log_size - 2)
    assert rows["conv1"].masked and rows["to_rgb1"].masked
    for r in range(log_size - 2):
        assert rows[f"convs.{2 * r}"].masked == conv_mask[r] and rows[f"convs.{2 * r + 1}"].masked == conv_mask[r], r
        assert rows[f"to_rgbs.{r}"].masked == rgb_mask[r], r
        assert rows[f"convs.{2 * r}"].up and not rows[f"convs.{2 * r + 1}"].up
    assert rows[f"convs.{2 * (log_size - 3) + 1}"].side == F64.RES


# ============================================================================ the whole chain against the CPU oracle
def _small_net(size=32, k_layers=5, ncls=4):
    """Generator(size, K = k_layers) and ncls LocalMLPs with seeded parameters, the oracle's parameter dicts of both, and
    a latent_avg of n_latent rows: the 1024 inversion's structure at a size the CPU differentiates in float64."""
    from types import SimpleNamespace
    from e4s_b200.networks import LocalMLP
    from e4s_b200.stylegan2.model import Generator
    G = Generator(size, 512, 8, split_layer_idx=5, remaining_layer_idx=k_layers)
    state = O.synthetic_state({k: tuple(v.shape) for k, v in G.state_dict().items()}, salt=size)
    G.load_state_dict(state)
    mlps = torch.nn.ModuleList([LocalMLP(dim_component=1280, dim_style=512, num_w_layers=k_layers) for _ in range(ncls)])
    mstate = O.synthetic_state(O.mlp_param_shapes(ncls, k_layers), salt=size)
    mlps.load_state_dict({k[len("MLPs."):]: v for k, v in mstate.items()})
    avg = 0.1 * torch.randn(G.n_latent, 512, generator=torch.Generator().manual_seed(77))
    net = SimpleNamespace(G=G, MLPs=mlps, latent_avg=avg, remaining_layer_idx=k_layers)
    return net, {k: v.double() for k, v in state.items()}, {k: v.double() for k, v in mstate.items()}


def _chain_inputs(size, ncls, b):
    g = torch.Generator().manual_seed(19)
    sv = 0.5 * torch.randn(b, ncls, 1280, generator=g, dtype=torch.float64)
    _, mask, label, noise = O.synthetic_inputs(b, ncls, size, 64, seed=7)
    w = torch.randn(b, 3, size, size, generator=g, dtype=torch.float64)
    return sv, mask.double(), label[:, 0].to(torch.uint8), [n.double() for n in noise], w


def _chain_gradient(net, sv, label, noise, w, act_from=None):
    """(image, codes, d<image, w>/d codes, d<image, w>/d style vectors, StyledConv outputs) of style_codes + RefChain."""
    v = sv.clone().requires_grad_(True)
    codes = F64.style_codes(net, v)
    codes.retain_grad()
    chain = F64.RefChain(net.G, codes, label, noise, act_from)
    ys = []
    for i in range(len(chain.sched)):
        out = chain.step()
        if chain.is_conv[i]:
            ys.append(out.detach())
    img = chain.skip
    (img * w).sum().backward()
    return img.detach(), codes.detach(), codes.grad, v.grad, ys


def test_reference_matches_oracle_per_unit_and_end_to_end():
    """RefChain against O.styled_conv / O.to_rgb on the same input, layer by layer, and against O.generator_forward, in
    float64 on the CPU at 32 x 32, K = 5, B = 2, 4 regions, to 1e-10.  K = 5 gives masked and unmasked StyledConvs (both
    up-sampling) and masked and global ToRGBs."""
    from e4s_b200.stylegan2.model import Generator
    size, k_layers, b, ncls = 32, 5, 2, 4
    G = Generator(size, 512, 8, split_layer_idx=5, remaining_layer_idx=k_layers)
    state = O.synthetic_state({k: tuple(v.shape) for k, v in G.state_dict().items()}, salt=size)
    G.load_state_dict(state)
    p = {k: v.double() for k, v in state.items()}
    codes, mask, label, noise = O.synthetic_inputs(b, ncls, size, 64, seed=7)
    codes, mask, noise = codes.double(), mask.double(), [n.double() for n in noise]
    chain = F64.RefChain(G, codes, label[:, 0].to(torch.uint8), noise)
    names = {id(m): n for n, m in G.named_modules()}
    kinds = set()
    for i, (m, idx, per_region) in enumerate(chain.sched):
        x, skip = chain.seek(i)
        style = codes[:, :, idx] if per_region else codes[:, 0, idx]
        prefix = names[id(m)] + "."
        if chain.is_conv[i]:
            kinds.add(("conv", m.conv.upsample, m.mask_op))
            ref = O.styled_conv(x, style, mask, noise[chain.noise_index[i]], p, prefix, m.conv.upsample, m.mask_op)
        else:
            kinds.add(("rgb", m.mask_op))
            ref = O.to_rgb(x, style, mask, skip, p, prefix, m.mask_op)
        assert_close(chain.step(), ref, 1e-10, names[id(m)])
    assert kinds >= {("conv", True, True), ("conv", True, False), ("conv", False, True), ("conv", False, False),
                     ("rgb", True), ("rgb", False)}, kinds
    img, _ = O.generator_forward(p, codes, mask, noise, size, k_layers)
    assert_close(chain.image(), img, 1e-10, "image")


def test_chain_gradient_matches_oracle_autograd():
    """style_codes + RefChain under autograd against O.cal_style_codes + O.generator_forward: codes, image and the
    gradient of <image, w> with respect to the codes and to the texture vectors, float64 on the CPU at 32 x 32, K = 5,
    B = 2, 4 regions, to 1e-10."""
    size, k_layers, b, ncls = 32, 5, 2, 4
    net, p, mp = _small_net(size, k_layers, ncls)
    sv, mask, label, noise, w = _chain_inputs(size, ncls, b)
    img, codes, gcodes, gsv, _ = _chain_gradient(net, sv, label, noise, w)

    v = sv.clone().requires_grad_(True)
    codes_ref = O.cal_style_codes(mp, v, net.latent_avg.double(), k_layers)
    codes_ref.retain_grad()
    img_ref, _ = O.generator_forward(p, codes_ref, mask, noise, size, k_layers)
    (img_ref * w).sum().backward()
    assert_close(codes, codes_ref, 1e-10, "codes")
    assert_close(img, img_ref, 1e-10, "image")
    assert_close(gcodes, codes_ref.grad, 1e-10, "d/dcodes")
    assert_close(gsv, v.grad, 1e-10, "d/dstyle vectors")
    assert bool((gsv.abs().amax(-1) > 0).all()), "every region of every sample should receive a gradient here"


def test_branch_pins_at_own_signs_change_nothing():
    """act_from = the chain's own StyledConv outputs (same signs as the pre-activations) gives the same image and
    texture-vector gradient to 1e-12; the opposite signs at one layer change the gradient, so the pins are used."""
    size, k_layers, b, ncls = 32, 5, 2, 4
    net, _, _ = _small_net(size, k_layers, ncls)
    sv, _, label, noise, w = _chain_inputs(size, ncls, b)
    img, _, _, gsv, ys = _chain_gradient(net, sv, label, noise, w)
    assert all(bool((y > 0).any()) and bool((y < 0).any()) for y in ys)
    img_pin, _, _, gsv_pin, _ = _chain_gradient(net, sv, label, noise, w, act_from=ys)
    assert_close(img_pin, img, 1e-12, "image, pinned")
    assert_close(gsv_pin, gsv, 1e-12, "d/dstyle vectors, pinned")
    flipped = list(ys)
    flipped[3] = -ys[3]
    _, _, _, gsv_flip, _ = _chain_gradient(net, sv, label, noise, w, act_from=flipped)
    assert float((gsv_flip - gsv).norm() / gsv.norm()) > 1e-2
