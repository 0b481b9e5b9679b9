"""Input-, style- and noise-gradients of the synthesis layers at the layer shapes of the 1024x1024 generator (K = 13, 12
regions), against a float64 reference that shares no code with the kernels or their weight preparation.

The inversion loop (optimization.invert) runs StyledConvFn / ToRGBFn backward for every layer at every step.  Here each
layer of the 1024 schedule - read from Generator._schedule(), not typed in - runs forward and backward through the default
kernel selection, and the kernels behind its backward (tensor-core and SIMT dgrad, class_reduce, torgb_bwd) are also
called directly at the same shapes.  The reference is per-region F.conv2d / F.conv_transpose2d + blur in float64 with the
demodulation computed from s inside the graph, so autograd differentiates the demodulation path as well.  Leaky-ReLU's
derivative is taken from the kernel's own forward output y (act_from), as the backward does: a 1e-5 forward difference
then cannot flip a near-zero branch and the per-layer bars stay tight.

The reference itself is pinned to the CPU oracle (and through it to the goldens) by the host-only tests at the top.
"""
import ctypes
import functools
import math
import os
import zlib
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F

from oracle import e4s_oracle as O
from oracle import golden_io
from conftest import ROOT, assert_close

DEV = "cuda:0"
SQRT2 = math.sqrt(2.0)
TOL_TC = 1e-4          # tensor-core (split-bf16) outputs
TOL_F32 = 2e-5         # exact-fp32 kernels: SIMT dgrad, class_reduce, torgb, the noise gradient
RES, K_LAYERS, NCLS = 1024, 13, 12


# ============================================================================ float64 reference (plain torch ops)
def _blur(ref):
    return O.make_fir((1, 3, 3, 1), 4.0, dtype=torch.float64).to(ref.device)


def _act(v, act_from=None):
    """sqrt(2) * leaky_relu(v, 0.2); with act_from the branch is taken from act_from > 0 instead of from v."""
    if act_from is None:
        return F.leaky_relu(v, 0.2) * SQRT2
    return torch.where(act_from > 0, v * SQRT2, v * (0.2 * SQRT2))


def ref_preact(x, s, w, label, noise, noise_w, bias, up, demod, s_demod=None):
    """Pre-activation of StyledConv in float64: sum over the regions r present of [label == r] * d_r * conv(x * s_r, W)
    + noise_w * noise + bias.

    x [B, Cin, H, W]; s [B, R, Cin]; w the raw weight [Cout, Cin, 3, 3] (scaled here by 1/sqrt(9 Cin)); label [B, Ho, Wo]
    or None (R == 1); noise [B | 1, 1, Ho, Wo] or None.  Up-sampling layers: conv_transpose2d(stride 2) then the 4x4 blur
    with pad (1, 1).  d_r = rsqrt(sum_i s_r,i^2 Wsq[:, i] + 1e-8) is computed from ``s_demod`` (default: s) inside the
    graph; passing a separate leaf there splits the style gradient into its convolution and demodulation parts."""
    x, s, w = x.double(), s.double(), w.double()
    sd = s if s_demod is None else s_demod.double()
    b, cin, h, wd = x.shape
    ws = w * (1.0 / math.sqrt(9 * cin))
    wsq = ws.pow(2).sum((2, 3))                                   # [Cout, Cin]
    ho, wo = (2 * h, 2 * wd) if up else (h, wd)
    regions = [0] if label is None else torch.unique(label).tolist()
    out = x.new_zeros(b, w.shape[0], ho, wo)
    for r in regions:
        xs = x * s[:, r, :, None, None]
        if up:
            t = O.upfirdn2d(F.conv_transpose2d(xs, ws.transpose(0, 1), stride=2), _blur(x), pad=(1, 1))
        else:
            t = F.conv2d(xs, ws, padding=1)
        if demod:
            t = t * torch.rsqrt(sd[:, r].pow(2) @ wsq.t() + 1e-8)[:, :, None, None]
        if label is not None:
            t = t * (label == r)[:, None].to(t.dtype)
        out = out + t
    if noise is not None:
        out = out + noise_w.double() * noise.double()
    if bias is not None:
        out = out + bias.double()[None, :, None, None]
    return out


def ref_styled(x, s, w, label, noise, noise_w, bias, up, demod, act_from=None):
    """StyledConv forward in float64 (see ref_preact); act_from: take leaky-ReLU's branch from act_from > 0."""
    return _act(ref_preact(x, s, w, label, noise, noise_w, bias, up, demod), act_from)


def ref_to_rgb(x, s, wrgb, label, bias, skip, fir):
    """ToRGB in float64: sum_r [label == r] * conv1x1(x * s_r, W / sqrt(Cin)) + bias + upfirdn2d(skip, up 2, pad (2, 1)).
    x [B, Cin, H, W]; s [B, R, Cin]; wrgb the raw weight (any shape holding [3, Cin]); bias [3]; skip [B, 3, H/2, W/2]."""
    x, s = x.double(), s.double()
    b, cin, h, wd = x.shape
    ws = wrgb.double().reshape(3, cin, 1, 1) * (1.0 / math.sqrt(cin))
    regions = [0] if label is None else torch.unique(label).tolist()
    out = x.new_zeros(b, 3, h, wd)
    for r in regions:
        t = F.conv2d(x * s[:, r, :, None, None], ws)
        if label is not None:
            t = t * (label == r)[:, None].to(t.dtype)
        out = out + t
    if bias is not None:
        out = out + bias.double().reshape(1, 3, 1, 1)
    if skip is not None:
        out = out + O.upfirdn2d(skip.double(), fir.double(), up=2, pad=(2, 1))
    return out


def ref_class_reduce(gy, y, label, noise, noise_w, bias, ncls, act):
    """gdu[b, r, o] = sum over the pixels of region r of act'(y) gy * (act^-1(y) - noise_w noise - bias), in float64 with
    index_add.  gy, y pixel-major [B, Ho, Wo, Cout]; noise [B | 1, 1, Ho, Wo]."""
    gy, y = gy.double(), y.double()
    b, ho, wo, cout = gy.shape
    if act:
        slope = torch.where(y > 0, y.new_tensor(SQRT2), y.new_tensor(0.2 * SQRT2))
        gv, u = gy * slope, y / slope
    else:
        gv, u = gy, y
    if noise is not None:
        u = u - noise_w.double() * noise.double()[:, 0, :, :, None]
    if bias is not None:
        u = u - bias.double()
    idx = torch.arange(b, device=gy.device)[:, None, None] * ncls
    if label is not None:
        idx = idx + label.long()
    idx = idx.expand(b, ho, wo).reshape(-1)
    out = torch.zeros(b * ncls, cout, dtype=torch.float64, device=gy.device)
    return out.index_add_(0, idx, (gv * u).reshape(-1, cout)).reshape(b, ncls, cout)


# ============================================================================ the reference against the CPU oracle
def _onehot(label, ncls):
    return F.one_hot(label.long(), ncls).permute(0, 3, 1, 2).double()


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


@pytest.mark.parametrize("demod", [True, False])
@pytest.mark.parametrize("masked", [True, False])
@pytest.mark.parametrize("up", [False, True])
def test_ref_styled_matches_oracle(up, masked, demod):
    """ref_styled against the oracle's StyledConv in float64 on the CPU, forward and autograd (x, style, noise), <= 1e-10."""
    g = torch.Generator().manual_seed(11 + 2 * up + masked)
    b, cin, cout, h, w, ncls, sdim = 2, 6, 5, 6, 6, 4, 16          # the oracle resizes masks to squares
    ho, wo = (2 * h, 2 * w) if up else (h, w)
    dd = dict(generator=g, dtype=torch.float64)
    p = {"conv.weight": torch.randn(1, cout, cin, 3, 3, **dd), "conv.modulation.weight": torch.randn(cin, sdim, **dd),
         "conv.modulation.bias": 1.0 + 0.1 * torch.randn(cin, **dd), "noise.weight": torch.tensor([0.37], dtype=torch.float64),
         "activate.bias": 0.1 * torch.randn(cout, **dd)}
    label = torch.randint(0, ncls, (b, ho, wo), generator=g)
    label[:, 0, 0] = ncls - 1                                    # one region (1) may be absent, the last one is not
    label[label == 1] = 2
    x = torch.randn(b, cin, h, w, **dd).requires_grad_(True)
    style = torch.randn(b, ncls, sdim, **dd) if masked else torch.randn(b, sdim, **dd)
    style.requires_grad_(True)
    noise = torch.randn(1, 1, ho, wo, **dd).requires_grad_(True)
    go = torch.randn(b, cout, ho, wo, **dd)

    ref = _oracle_styled(x, style, _onehot(label, ncls) if masked else None, noise, p, up, masked, demod)
    gref = torch.autograd.grad(ref, (x, style, noise), go)
    s = O.equal_linear(style, p["conv.modulation.weight"], p["conv.modulation.bias"])
    s = s if masked else s[:, None]
    ours = ref_styled(x, s, p["conv.weight"][0], label if masked else None, noise, p["noise.weight"], p["activate.bias"],
                      up, demod)
    gours = torch.autograd.grad(ours, (x, style, noise), go)
    assert_close(ours, ref, 1e-10, "forward")
    for a, r, what in zip(gours, gref, ("d/dx", "d/dstyle", "d/dnoise")):
        assert_close(a, r, 1e-10, what)


@pytest.mark.parametrize("skip", [True, False])
@pytest.mark.parametrize("masked", [True, False])
def test_ref_to_rgb_matches_oracle(masked, skip):
    """ref_to_rgb against the oracle's ToRGB in float64 on the CPU, forward and autograd (x, style, skip), <= 1e-10."""
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

    ref = O.to_rgb(x, style, _onehot(label, ncls) if masked else None, sk, p, "", masked)
    gref = torch.autograd.grad(ref, inputs, go)
    s = O.equal_linear(style, p["conv.modulation.weight"], p["conv.modulation.bias"])
    ours = ref_to_rgb(x, s if masked else s[:, None], p["conv.weight"], label if masked else None, p["bias"].reshape(3), sk,
                      O.make_fir((1, 3, 3, 1), 4.0, dtype=torch.float64))
    gours = torch.autograd.grad(ours, inputs, go)
    assert_close(ours, ref, 1e-10, "forward")
    for a, r, what in zip(gours, gref, ("d/dx", "d/dstyle", "d/dskip")):
        assert_close(a, r, 1e-10, what)


# ============================================================================ the layer table of the 1024 generator
Layer = namedtuple("Layer", "name module kind cin cout side up masked")     # side: input side of the layer


@functools.lru_cache(maxsize=None)
def layer_table():
    """Every StyledConv and ToRGB of Generator(1024, K = 13) in execution order, read from Generator._schedule()."""
    from e4s_b200.stylegan2.model import Generator, StyledConv
    G = Generator(RES, 512, 8, split_layer_idx=5, remaining_layer_idx=K_LAYERS)
    modules = {id(m): n for n, m in G.named_modules()}
    side, rows = 4, []
    for m, _, per_region in G._schedule():
        assert per_region == m.mask_op, modules[id(m)]
        if isinstance(m, StyledConv):
            up = m.conv.upsample
            out_side = 2 * side if up else side
            name = "conv1" if modules[id(m)] == "conv1" else f"{'up' if up else 'c'}{out_side}"
            rows.append(Layer(name, modules[id(m)], "conv", m.conv.in_channel, m.conv.out_channel, side, up, m.mask_op))
            side = out_side
        else:
            rows.append(Layer(f"rgb{side}", modules[id(m)], "rgb", m.conv.in_channel, 3, side, False, m.mask_op))
    return tuple(rows)


def test_layer_table_matches_the_oracle_plan():
    """The masked flags of the table are the oracle's generator_layer_plan(1024, 13)."""
    log_size, conv_mask, rgb_mask = O.generator_layer_plan(RES, K_LAYERS)
    rows = {r.module: r for r in layer_table()}
    assert len(rows) == 2 + 3 * (log_size - 2)
    assert rows["conv1"].masked and rows["to_rgb1"].masked
    for r in range(log_size - 2):
        assert rows[f"convs.{2 * r}"].masked == conv_mask[r] and rows[f"convs.{2 * r + 1}"].masked == conv_mask[r], r
        assert rows[f"to_rgbs.{r}"].masked == rgb_mask[r], r
        assert rows[f"convs.{2 * r}"].up and not rows[f"convs.{2 * r + 1}"].up
    assert rows[f"convs.{2 * (log_size - 3) + 1}"].side == RES


# StyledConv case: b, channels, input h x w, up, regions (1 = no label map), labels: face | iid | face32 (region 3 -> 31),
# noise batch, need: which inputs require grad (xs | s: the gs-only call of conv1 | x: the gx-only call)
Case = namedtuple("Case", "id b cin cout h w up ncls labels noise_b need")


def _styled_cases():
    cases = []
    convs = [r for r in layer_table() if r.kind == "conv"]
    for r in convs:
        ncls = NCLS if r.masked else 1
        need = "s" if r.name == "conv1" else "xs"       # conv1's input is the constant input: a gs-only call
        cases.append(Case(f"{r.name}-b1", 1, r.cin, r.cout, r.side, r.side, r.up, ncls, "face", 1, need))
    for i, r in enumerate(c for c in convs if c.side * (2 if c.up else 1) <= 128):
        ncls = NCLS if r.masked else 1
        cases.append(Case(f"{r.name}-b8", 8, r.cin, r.cout, r.side, r.side, r.up, ncls, "face", 8 if i % 2 else 1,
                          "s" if r.name == "conv1" else "xs"))
    cases += [
        Case("c32-gx_only-b1", 1, 512, 512, 32, 32, False, NCLS, "face", 1, "x"),       # split plan (32, 5, 1), x NULL
        Case("c8-iid-b1", 1, 512, 512, 8, 8, False, NCLS, "iid", 1, "xs"),
        Case("up16-iid-b2", 2, 512, 512, 8, 8, True, NCLS, "iid", 2, "xs"),
        Case("c16-r32-b2", 2, 512, 512, 16, 16, False, 32, "face32", 1, "xs"),
        Case("c20x44-b2", 2, 512, 512, 20, 44, False, NCLS, "face", 2, "xs"),
        Case("up26x74-b1", 1, 512, 256, 13, 37, True, NCLS, "face", 1, "xs"),          # masked transposed convolution
        Case("up26x74-global-b2", 2, 128, 64, 13, 37, True, 1, "face", 2, "xs"),
        Case("up14x10-b2", 2, 256, 128, 7, 5, True, NCLS, "face", 1, "xs"),            # below 16: folded parity kernel
    ]
    return cases


STYLED_CASES = _styled_cases()


def _plan(lib, b, h, w, cin, ncls, up):
    nt, gs, hs = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    assert lib.e4s_modconv3x3_bwd_tc_plan(b, h, w, cin, ncls, int(up), ctypes.byref(nt), ctypes.byref(gs), ctypes.byref(hs)) == 0
    return nt.value, gs.value, hs.value


def test_gpu_cases_cover_every_production_plan(monkeypatch):
    """Every work-list plan (N-tile width, region split, parity split) the tensor-core gradient takes for a layer of the
    1024 schedule at 1, 8 or 16 faces is taken by at least one GPU case of this file.  A heuristic change that brings in
    a new plan fails here until a case covers it."""
    from e4s_b200 import _lib
    lib = _lib.load()
    for var in ("E4S_B200_NTILE", "E4S_B200_DGRAD_SPLIT"):
        monkeypatch.delenv(var, raising=False)
    production = {}
    for b in (1, 8, 16):
        for r in layer_table():
            if r.kind == "conv":
                production.setdefault(_plan(lib, b, r.side, r.side, r.cin, NCLS if r.masked else 1, r.up), []).append(f"{r.name}@B{b}")
    covered = {}
    for c in STYLED_CASES:
        covered.setdefault(_plan(lib, c.b, c.h, c.w, c.cin, c.ncls, c.up), []).append(c.id)
    for plan in sorted(production):
        print(f"plan {plan}: production {' '.join(production[plan])}; covered by {' '.join(covered.get(plan, ['NOTHING']))}")
    missing = sorted(set(production) - set(covered))
    assert not missing, f"production plans without a GPU case: {missing}"


# ============================================================================ GPU checks
_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _error_report():
    yield
    if _WORST:
        print("\nlargest observed error per output kind (max-rel, rel-RMS, case):")
        for kind in sorted(_WORST):
            e, r, what = _WORST[kind]
            print(f"  {kind:24s} {e:.2e}  {r:.2e}  {what}")


def _check(ours, ref, tol, kind, case):
    ours, ref = ours.detach().double(), ref.detach().double().to(ours.device)
    e = float((ours - ref).abs().max() / ref.abs().max().clamp_min(1e-30))
    r = float((ours - ref).norm() / ref.norm().clamp_min(1e-30))
    print(f"{case}: {kind} max-rel {e:.2e} rel-RMS {r:.2e} (bar {tol:.0e})")
    if kind not in _WORST or e > _WORST[kind][0]:
        _WORST[kind] = (e, r, case)
    assert_close(ours, ref, tol, f"{case} {kind}")


@pytest.fixture
def default_kernels(monkeypatch):
    """The default kernel selection (no forced path, tile width or split)."""
    for var in ("E4S_B200_CONV", "E4S_B200_BWD", "E4S_B200_NTILE", "E4S_B200_DGRAD_SPLIT", "E4S_B200_UP2"):
        monkeypatch.delenv(var, raising=False)


@functools.lru_cache(maxsize=None)
def _faces():
    gold = golden_io.load(os.path.join(ROOT, "tests", "golden", "reference_vectors.npz"))
    return [torch.from_numpy(gold[k]) for k in ("mask/source_cls12", "mask/target_cls12")]


def _face_labels(b, ho, wo):
    """Face-like 12-region maps (the committed parsing masks, alternately mirrored) nearest-resized to ho x wo."""
    faces = _faces()
    lab = torch.stack([faces[i % 2] if i % 4 < 2 else faces[i % 2].flip(-1) for i in range(b)])
    idx_y = (torch.arange(ho) * lab.shape[1]) // ho
    idx_x = (torch.arange(wo) * lab.shape[2]) // wo
    return lab[:, idx_y][:, :, idx_x].contiguous()


def _labels(kind, b, ho, wo, ncls, g):
    if kind == "iid":
        return torch.randint(0, ncls, (b, ho, wo), generator=g, dtype=torch.uint8)
    lab = _face_labels(b, ho, wo)
    if kind == "face32":
        lab[lab == 3] = 31
    return lab


@pytest.mark.gpu
@pytest.mark.parametrize("case", STYLED_CASES, ids=[c.id for c in STYLED_CASES])
def test_styled_conv_gradients_at_scale(case, default_kernels):
    """StyledConvFn forward and backward (default entry selection) against the float64 reference: y, gx, the total gs
    and gnoise; then the backward kernels at the same shape - tensor-core and SIMT dgrad (gx, conv-path gs) and
    class_reduce (gdu) for act 0 / 1, noise NULL / 1 / B and bias NULL / given."""
    from e4s_b200 import kernels as K
    from e4s_b200.stylegan2 import modconv as MC
    from e4s_b200.stylegan2 import modconv_bwd as MB
    c = case
    g = torch.Generator().manual_seed(zlib.crc32(c.id.encode()))
    ho, wo = (2 * c.h, 2 * c.w) if c.up else (c.h, c.w)
    w = torch.randn(c.cout, c.cin, 3, 3, generator=g).to(DEV)
    x = torch.randn(c.b, c.h, c.w, c.cin, generator=g).to(DEV)
    s = (1.0 + 0.3 * torch.randn(c.b, c.ncls, c.cin, generator=g)).to(DEV)
    noise = torch.randn(c.noise_b, 1, ho, wo, generator=g).to(DEV)
    nw = torch.tensor([0.37], device=DEV)
    bias = (0.1 * torch.randn(c.cout, generator=g)).to(DEV)
    gy = torch.randn(c.b, ho, wo, c.cout, generator=g).to(DEV)
    label = _labels(c.labels, c.b, ho, wo, c.ncls, g).to(DEV) if c.ncls > 1 else None
    blur = O.make_fir((1, 3, 3, 1), 4.0).to(DEV)
    prep = MC.PreparedConv().get(w[None], c.up, blur if c.up else None)

    # ours, through autograd
    xg = x.clone().requires_grad_("x" in c.need)
    sg = s.clone().requires_grad_("s" in c.need)
    ng = noise.clone().requires_grad_(True)
    y = MC.StyledConvFn.apply(xg, sg, ng, nw, bias, label, prep, c.up, True, True)
    y.backward(gy)
    torch.cuda.synchronize()

    # float64 reference: separate leaves for the style in the convolution and in the demodulation
    xr = x.double().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    s_conv = s.double().requires_grad_(True)
    s_dem = s.double().requires_grad_(True)
    nr = noise.double().requires_grad_(True)
    v = ref_preact(xr, s_conv, w, label, nr, nw, bias, c.up, True, s_demod=s_dem)
    y_nchw = y.detach().permute(0, 3, 1, 2)
    _act(v, act_from=y_nchw).backward(gy.double().permute(0, 3, 1, 2))
    pm = lambda t: t.permute(0, 2, 3, 1)                          # NCHW -> pixel-major
    gs_conv_ref = s_conv.grad

    _check(y, pm(_act(v.detach())), TOL_TC, "y", c.id)
    if "x" in c.need:
        _check(xg.grad, pm(xr.grad), TOL_TC, "gx (autograd)", c.id)
    else:
        assert xg.grad is None
    if "s" in c.need:
        _check(sg.grad, s_conv.grad + s_dem.grad, TOL_TC, "gs total (autograd)", c.id)
    else:
        assert sg.grad is None
    _check(ng.grad, nr.grad, TOL_F32, "gnoise (autograd)", c.id)
    del v, s_dem, nr

    # the dgrad kernels, both outputs, against the convolution path of the reference
    y32 = y.detach()
    dm = K.demod(s, prep.wsq)
    gx_tc, gs_tc = K.modconv3x3_bwd_tc(gy, y32, x, MB._dgrad_planes(prep), s, dm, label, c.up, True, True, True)
    _check(gx_tc, pm(xr.grad), TOL_TC, "gx tc kernel", c.id)
    _check(gs_tc, gs_conv_ref, TOL_TC, "gs_conv tc kernel", c.id)
    del gx_tc, gs_tc
    gx_f32, gs_f32 = K.modconv3x3_bwd(gy, y32, x, MB._dgrad_weights(prep), s, dm, label, c.up, True, True, True)
    _check(gx_f32, pm(xr.grad), TOL_F32, "gx simt kernel", c.id)
    _check(gs_f32, gs_conv_ref, TOL_F32, "gs_conv simt kernel", c.id)
    del gx_f32, gs_f32

    # class_reduce: activation on / off, noise absent / batch 1 / batch B, bias absent / given
    noise_1 = noise[:1]
    noise_b = torch.randn(c.b, 1, ho, wo, generator=g).to(DEV)
    for act, nz, bv in ((True, noise_1, bias), (True, noise_b, None), (False, None, bias), (False, noise_b, bias),
                        (True, None, None)):
        gdu = K.class_reduce(gy, y32, label, nz, nw if nz is not None else None, bv, c.ncls, act)
        ref = ref_class_reduce(gy, y32, label, nz, nw, bv, c.ncls, act)
        tag = f"act={int(act)} noise={'-' if nz is None else nz.shape[0]} bias={'-' if bv is None else 'y'}"
        _check(gdu, ref, TOL_F32, "gdu class_reduce", f"{c.id} {tag}")


# ToRGB case: b, Cin, side h x w, regions, skip?, x offset in floats (4: 16-byte aligned only)
RgbCase = namedtuple("RgbCase", "id b cin h w ncls skip offset")


def _rgb_cases():
    cases = []
    rgbs = [r for r in layer_table() if r.kind == "rgb"]
    for r in rgbs:
        cases.append(RgbCase(f"{r.name}-b1", 1, r.cin, r.side, r.side, NCLS if r.masked else 1, r.module != "to_rgb1", 0))
    for r in rgbs:
        if r.side <= 128:
            cases.append(RgbCase(f"{r.name}-b8", 8, r.cin, r.side, r.side, NCLS if r.masked else 1, r.module != "to_rgb1", 0))
    # the warp-per-pixel forward: Cin not a multiple of 8 (4 / 8 / 16 lanes per pixel), and x not 32-byte aligned (32 lanes)
    cases += [RgbCase("cin12-lpp4-b2", 2, 12, 40, 24, NCLS, True, 0),
              RgbCase("cin36-lpp8-b2", 2, 36, 24, 40, NCLS, True, 0),
              RgbCase("cin100-lpp16-b2", 2, 100, 30, 18, NCLS, True, 0),
              RgbCase("cin128-offset16-b2", 2, 128, 64, 64, NCLS, True, 4)]
    return cases


RGB_CASES = _rgb_cases()


@pytest.mark.gpu
@pytest.mark.parametrize("case", RGB_CASES, ids=[c.id for c in RGB_CASES])
def test_to_rgb_at_scale(case, default_kernels):
    """ToRGBFn forward and backward (torgb_fwd, torgb_bwd, the skip's adjoint) against ref_to_rgb in float64."""
    from e4s_b200.stylegan2 import modconv as MC
    c = case
    g = torch.Generator().manual_seed(zlib.crc32(c.id.encode()))
    w = torch.randn(1, 3, c.cin, 1, 1, generator=g).to(DEV)
    n = c.b * c.h * c.w * c.cin
    buf = torch.empty(n + c.offset, device=DEV)
    x = buf[c.offset:].view(c.b, c.h, c.w, c.cin)
    x.copy_(torch.randn(c.b, c.h, c.w, c.cin, generator=g))
    s = (1.0 + 0.3 * torch.randn(c.b, c.ncls, c.cin, generator=g)).to(DEV)
    bias = (0.1 * torch.randn(3, generator=g)).to(DEV)
    skip = torch.randn(c.b, 3, c.h // 2, c.w // 2, generator=g).to(DEV) if c.skip else None
    go = torch.randn(c.b, 3, c.h, c.w, generator=g).to(DEV)
    label = _labels("face", c.b, c.h, c.w, c.ncls, g).to(DEV) if c.ncls > 1 else None
    fir = O.make_fir((1, 3, 3, 1), 4.0).to(DEV)
    prep = MC.PreparedConv().get(w, False, None)

    x.requires_grad_(True)
    sg = s.clone().requires_grad_(True)
    kg = skip.clone().requires_grad_(True) if c.skip else None
    out = MC.ToRGBFn.apply(x, sg, kg, bias, label, prep, fir if c.skip else None)
    out.backward(go)
    torch.cuda.synchronize()

    xr = x.detach().double().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    sr = s.double().requires_grad_(True)
    kr = skip.double().requires_grad_(True) if c.skip else None
    ref = ref_to_rgb(xr, sr, w, label, bias, kr, fir)
    ref.backward(go.double())
    _check(out, ref, TOL_F32, "rgb", c.id)
    _check(x.grad, xr.grad.permute(0, 2, 3, 1), TOL_F32, "rgb gx", c.id)
    _check(sg.grad, sr.grad, TOL_F32, "rgb gs", c.id)
    if c.skip:
        _check(kg.grad, kr.grad, TOL_F32, "rgb gskip", c.id)
