"""Input-, style- and noise-gradients of the synthesis layers at the layer shapes of the 1024x1024 generator (K = 13, 12
regions), against a float64 reference that shares no code with the kernels or their weight preparation.

The inversion loop (optimization.invert) runs StyledConvFn / ToRGBFn backward for every layer at every step.  Here each
layer of the 1024 schedule - read from Generator._schedule(), not typed in - runs forward and backward through the default
kernel selection, and the kernels behind its backward (tensor-core and SIMT dgrad, class_reduce, torgb_bwd) are also
called directly at the same shapes.  The reference (f64ref.styled_preact / to_rgb) is per-region F.conv2d /
F.conv_transpose2d + blur in float64 with the demodulation computed from s inside the graph, so autograd differentiates the
demodulation path as well.  Leaky-ReLU's derivative is taken from the kernel's own forward output y (act_from), as the
backward does: a 1e-5 forward difference then cannot flip a near-zero branch and the per-layer bars stay tight.

The reference itself is pinned to the CPU oracle (and through it to the goldens) by tests/test_f64ref.py.
"""
import ctypes
import zlib
from collections import namedtuple

import pytest
import torch

import f64ref as F64
from oracle import e4s_oracle as O
from f64ref import SQRT2, layer_table, pm

DEV = "cuda:0"
TOL_TC = 1e-4          # tensor-core (split-bf16) outputs
TOL_F32 = 2e-5         # exact-fp32 kernels: SIMT dgrad, class_reduce, torgb, the noise gradient
NCLS = 12


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
    F64.clear_kernel_selection(monkeypatch)
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
LEDGER = F64.Ledger(24)
_check = LEDGER.check


@pytest.fixture(scope="module", autouse=True)
def _error_report():
    yield
    LEDGER.report()


@pytest.fixture
def default_kernels(monkeypatch):
    F64.clear_kernel_selection(monkeypatch)


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
    label = F64.labels(c.labels, c.b, ho, wo, c.ncls, g).to(DEV) if c.ncls > 1 else None
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
    v = F64.styled_preact(xr, s_conv, w, label, nr, nw, bias, c.up, True, s_demod=s_dem)
    y_nchw = y.detach().permute(0, 3, 1, 2)
    F64.act(v, act_from=y_nchw).backward(gy.double().permute(0, 3, 1, 2))
    gs_conv_ref = s_conv.grad

    _check(y, pm(F64.act(v.detach())), TOL_TC, "y", c.id)
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
    """ToRGBFn forward and backward (torgb_fwd, torgb_bwd, the skip's adjoint) against f64ref.to_rgb."""
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
    label = F64.labels("face", c.b, c.h, c.w, c.ncls, g).to(DEV) if c.ncls > 1 else None
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
    ref = F64.to_rgb(xr, sr, w, label, bias, kr)
    ref.backward(go.double())
    _check(out, ref, TOL_F32, "rgb", c.id)
    _check(x.grad, xr.grad.permute(0, 2, 3, 1), TOL_F32, "rgb gx", c.id)
    _check(sg.grad, sr.grad, TOL_F32, "rgb gs", c.id)
    if c.skip:
        _check(kg.grad, kr.grad, TOL_F32, "rgb gskip", c.id)
