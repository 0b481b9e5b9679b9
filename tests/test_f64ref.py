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
