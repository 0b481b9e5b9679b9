"""The inversion step with the reference's default loss (e4s_b200.criteria.InversionLoss: 0.1 ID + 1.0 l2 + 0.8 LPIPS at
1024 / 512 / 256 + 0.1 parsing) at 1024 x 1024 on the default kernels, at bench.py's one face and at 4 faces, against
float64: the fused pooling pyramid those networks start from, the loss and its image gradient term by term, one step
through the generator, and the eager, graphed and TF32 invert legs that bench.py times.

The benchmark's configuration is imported, not restated: bench.build_net gives the generator, bench.face_label_maps the
label maps, the texture vectors and targets are drawn as bench.run_ours draws them, and the criterion is built as
bench.py builds it (InversionLoss() with load_synthetic_losses(crit, 11)); the noise is fixed.  Faces 1-3 of the 4-face
leg take f64ref.labels("one-pixel") maps, so region 11 is present at every level, at none and at some next to each other.

The float64 loss is oracle/loss_oracle.calc_loss with loss_states(11) moved to the device in float64, unchanged: it
shares no code with e4s_b200.criteria, and tests/test_losses.py pins it to the reference's goldens and to the product's
seeded weights.  It is evaluated one face at a time and divided by the batch size, so the reference gradient of face f
depends on face f alone, as every mean of calc_loss over the batch makes it.

The step's reference is f64ref.style_codes + f64ref.RefChain with the leaky-ReLU branches pinned to our StyledConv
outputs (as tests/test_inversion_at_scale.py pins them), seeded with the float64 loss gradient taken at OUR image: the
loss networks' ReLU, PReLU and max-pool kinks then sit in the same place on both sides.  The float64 end-to-end gradient
(the loss at the reference's own image) is reported beside it under a looser bar.
"""
import contextlib
import time
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

import f64ref as F64
from f64ref import layer_table
from oracle import loss_oracle as LO

DEV = "cuda:0"
RES, NCLS = 1024, 12                       # bench.py defaults: --size 1024 --ncls 12
B_LABELS, B_BENCH, B_INV = 16, 8, 4        # --batch 16 label maps, --inversion-batch 8 draws; this file's batch: 4 faces
LABEL_SEED, SV_SEED, NOISE_SEED = 200, 300, 400          # bench.run_ours at rank 0: labels 200, texture vectors 300
SALT = 11                                  # bench.py: load_synthetic_losses(crit, 11)
N_OPT = 13                                 # codes from this index on are latent_avg rows (K = 13), not optimised
LAMBDAS = {"id": 0.1, "l2": 1.0, "lpips": 0.8, "face_parsing": 0.1}     # InversionLoss's and calc_loss's defaults
TERMS = tuple(LAMBDAS)
LAYERS = layer_table()

# Bars.  The largest error observed on an H100 80GB HBM3 (700 W power limit) is in the comment; each bar sits 2-3x
# above it.  Pyramid: every output element within PYR_ULPS fp32 ulps (eps = 2^-23) of the float64 sum of its terms'
# magnitudes.  The 4x4 means are two levels of a fixed-order 4-term sum, within 2 such ulps by the rounding bound, the
# 2x2 means and the gradient within 1.5: largest observed 0.99 (4x4 means).
PYR_ULPS = 2.5
# The rest in max-rel (against the face's or slice's own maximum) and rel-RMS; both must hold everywhere.
TOL_LOSS = 4e-7         # the loss and each term against calc_loss in float64 at our image: 1.5e-7 (B = 4, the loss)
# d loss / d recon per face, (max-rel, rel-RMS) apart: the loss networks evaluated in fp32 put some ReLU and max-pool
# decisions on the other side of their kink, which moves a few hundred of the 3M pixels' gradient (the oracle's own
# calc_loss in fp32 on a CPU does the same against float64: parsing 5.5e-2 / 1.1e-3 on 284 pixels, LPIPS 3.7e-3 /
# 2.0e-4), so max-rel is the loose norm and rel-RMS the tight one.  Largest observed, all at B = 4:
TOL_GIMG = {"all": (2e-2, 2e-3),           # 8.7e-3 / 8.2e-4
            "id": (6e-4, 4e-4),            # 2.3e-4 / 1.4e-4
            "l2": (3e-7, 1.5e-7),          # 1.1e-7 / 4.7e-8
            "lpips": (4e-2, 4e-3),         # 1.7e-2 / 1.4e-3
            "face_parsing": (2e-1, 1.2e-2)}  # 9.3e-2 / 4.6e-3
TOL_GIMG_TF32 = (7.5e-2, 3.5e-2)  # the whole gradient with the loss networks' convolutions in TF32: 3.0e-2 / 1.4e-2
TOL_GIMG_FACE = (5e-4, 1e-4)  # face f of the 4-face batch x 4 against face f alone: 1.8e-4 / 3.8e-5 (face 3)
TOL_GCODES = 4e-4       # d loss / d codes, every (face, region, latent index) slice: 1.4e-4 (B = 4, rgb32/up64)
TOL_GSV = 3e-4          # d loss / d texture vectors, every (face, region) slice: 1.1e-4 (B = 4)
# d loss / d texture vectors per face, float64 loss at the float64 image (ours and the reference's images differ by the
# generator's forward error, which moves the loss networks' kinks; held per face, not per slice): 1.2e-4 (B = 4)
TOL_E2E = 3.5e-4
TOL_SGD = 3e-4          # one SGD step of invert, (initial - final) / lr per face, against the float64 gradient: 1.0e-4
TOL_SGD_OURS = 5e-6     # the same against our own gradient of the checked step: 1.9e-6 (B = 4)
TOL_GRAPH_LOSS = 3e-5   # the graphed loss trajectory against the eager one, step by step: 1.3e-5 (B = 4)
TOL_TF32_LOSS = 5e-5    # the TF32 graphed trajectory against the exact graphed one, step by step: 1.9e-5

LEDGER = F64.Ledger(44)
_PEAKS = []


@pytest.fixture(scope="module", autouse=True)
def _error_report():
    t0 = time.perf_counter()
    yield
    LEDGER.report()
    if LEDGER.worst:
        print(f"file wall time {time.perf_counter() - t0:.1f} s; largest peaks of device memory (reserved, allocated):")
        for res, alloc, name in sorted(_PEAKS, reverse=True)[:4]:
            print(f"  {res / 2 ** 30:5.1f} GiB  {alloc / 2 ** 30:5.1f} GiB  {name}")


@pytest.fixture(autouse=True)
def default_kernels(monkeypatch):
    F64.clear_kernel_selection(monkeypatch)


@pytest.fixture(autouse=True)
def _release_cached_memory(request):
    """Hand the allocator's cached blocks back after every test (the GPU is shared) and record each test's peak."""
    if torch.cuda.is_available():
        torch.cuda.reset_peak_memory_stats()
    yield
    if torch.cuda.is_available():
        _PEAKS.append((torch.cuda.max_memory_reserved(), torch.cuda.max_memory_allocated(), request.node.name))
        torch.cuda.empty_cache()


# ============================================================================ inputs
def _criterion(**lambdas):
    """InversionLoss with bench.py's seeded loss networks; lambdas (id=, l2=, ...) override the defaults."""
    from e4s_b200.criteria import InversionLoss
    from e4s_b200.synthetic import load_synthetic_losses
    crit = InversionLoss(**{f"{k}_lambda": v for k, v in lambdas.items()})
    load_synthetic_losses(crit, SALT)
    return crit.to(DEV)


def _only(term):
    """The lambdas of a criterion that keeps term alone, at its default weight."""
    return {t: (LAMBDAS[t] if t == term else 0.0) for t in TERMS}


@pytest.fixture(scope="module")
def inv():
    """The benchmark's network (every parameter frozen), its label maps, texture vectors and targets for the one-face and
    the 4-face legs, fixed per-face noise, the benchmark's criterion, one criterion per loss term and the float64 states
    of the loss networks."""
    import bench
    from e4s_b200 import kernels as K
    net = bench.build_net(RES, NCLS, torch.device(DEV))
    for p in net.parameters():
        p.requires_grad = False
    G = net.G
    labels = bench.face_label_maps(B_LABELS, NCLS, "faces", seed=LABEL_SEED)
    g2 = torch.Generator().manual_seed(SV_SEED)
    draw = lambda b: (0.5 * torch.randn(b, NCLS, 1280, generator=g2)).to(DEV)
    sv1, tv1 = draw(1), draw(1)                        # run_ours: sv, then the target's texture vectors
    svb, tvb = draw(B_BENCH)[:B_INV], draw(B_BENCH)[:B_INV]      # then the batched leg's (its first 4 faces)
    lab_b = labels[:B_INV].clone()
    lab_b[1:4, 0] = F64.labels("one-pixel", 3, 512, 512, NCLS, None)
    gn = torch.Generator().manual_seed(NOISE_SEED)
    sides = [4] + [2 ** (i // 2 + 3) for i in range(2 * (G.log_size - 2))]
    noise_b = [torch.randn(B_INV, 1, s, s, generator=gn).to(DEV) for s in sides]
    names = {}
    for r, (_, idx, _) in zip(LAYERS, G._schedule()):
        names.setdefault(idx, []).append(r.name)
    legs = {}
    for b, sv, tv, lab, noise in ((1, sv1, tv1, labels[:1], [n[:1] for n in noise_b]), (B_INV, svb, tvb, lab_b, noise_b)):
        lab = lab.to(DEV)
        onehot = K.label_to_onehot(lab, NCLS)
        with torch.no_grad():
            target = net.gen_img(None, net.cal_style_codes(tv), onehot, noise=noise)[0]
        legs[b] = SimpleNamespace(b=b, sv=sv, target=target, label=lab[:, 0], onehot=onehot, noise=noise)
    states = {k: {n: (t.double() if t.is_floating_point() else t).to(DEV) for n, t in sd.items()}
              for k, sd in LO.loss_states(SALT).items()}
    return SimpleNamespace(net=net, G=G, names=names, legs=legs, crit=_criterion(),
                           crit_term={t: _criterion(**_only(t)) for t in TERMS}, states=states)


def switches():
    """cuDNN's fp32 precision switches: the per-operator ones where this torch has them, else the legacy allow_tf32
    (reading the legacy one while the new ones differ raises)."""
    cd = torch.backends.cudnn
    mods = [getattr(cd, n, None) for n in ("conv", "rnn")]
    new = tuple(m.fp32_precision for m in mods if m is not None and hasattr(m, "fp32_precision"))
    return new or (cd.allow_tf32,)


def precision_of(exact):
    """switches() inside the criterion's conv_precision(exact)."""
    from e4s_b200.criteria.inversion_loss import conv_precision
    with conv_precision(exact):
        return switches()


@contextlib.contextmanager
def backward_switches(crit):
    """Yields a list that receives switches() each time a backward pass reaches the input of one of crit's convolutions,
    that is right after that convolution's input gradient has been computed."""
    seen = []

    def pre(mod, inp):
        if torch.is_grad_enabled() and inp[0].requires_grad:
            inp[0].register_hook(lambda g: seen.append(switches()))

    hooks = [m.register_forward_pre_hook(pre) for m in crit.modules() if isinstance(m, torch.nn.Conv2d)]
    try:
        yield seen
    finally:
        for h in hooks:
            h.remove()


# ============================================================================ the float64 loss
def ref_loss(states, recon, target, **lambdas):
    """calc_loss in float64, one face at a time: (loss, {term: value}, {"all" and each term: d (lambda * term) / d recon})
    of the batch, each face's loss divided by the batch size.  lambdas: calc_loss's, default its own."""
    b = recon.shape[0]
    lam = {t: lambdas.get(t, LAMBDAS[t]) for t in TERMS}
    loss, terms, grads = 0.0, {}, {}
    for f in range(b):
        r = recon[f:f + 1].detach().double().requires_grad_(True)
        lf, tf = LO.calc_loss(states, target[f:f + 1].double(), r, **{f"{t}_lambda": v for t, v in lam.items()})
        parts = {"all": lf, **{t: lam[t] * tf[f"loss_{t}"] for t in TERMS if lam[t] > 0}}
        for k, v in parts.items():
            (g,) = torch.autograd.grad(v / b, r, retain_graph=True)
            grads.setdefault(k, []).append(g)
        loss = loss + float(lf.detach()) / b
        for k, v in tf.items():
            terms[k] = terms.get(k, 0.0) + float(v.detach()) / b
        del r, lf, tf, parts
    return loss, terms, {k: torch.cat(v) for k, v in grads.items()}


def our_loss(crit, recon, target):
    """(loss, terms, d loss / d recon) of the criterion at recon, the backward inside crit.conv_precision() as invert
    runs it."""
    crit.set_target(target)
    r = recon.detach().clone().requires_grad_(True)
    loss, terms = crit(r, return_terms=True)
    with crit.conv_precision():
        loss.backward()
    return float(loss.detach()), {k: float(v.detach()) for k, v in terms.items()}, r.grad


# ============================================================================ one step, ours and float64
def _ours(inv, leg):
    """One loop body of invert with the benchmark's criterion on the default kernels: the image, its gradient, the codes'
    and the texture vectors' gradients and every StyledConv's output."""
    from e4s_b200.stylegan2.model import StyledConv
    acts = []
    hooks = [m.register_forward_hook(lambda mod, inp, out: acts.append(out.detach()))
             for m in inv.G.modules() if isinstance(m, StyledConv)]
    try:
        inv.crit.set_target(leg.target)
        latent = leg.sv.clone().requires_grad_(True)
        codes = inv.net.cal_style_codes(latent)
        codes.retain_grad()
        img = inv.net.gen_img(None, codes, leg.onehot, noise=leg.noise)[0]
        img.retain_grad()
        loss = inv.crit(img)
        with inv.crit.conv_precision():
            loss.backward()
        torch.cuda.synchronize()
    finally:
        for h in hooks:
            h.remove()
    return SimpleNamespace(img=img.detach(), gimg=img.grad, gcodes=codes.grad, gsv=latent.grad, acts=acts)


def _reference(inv, leg, ours):
    """style_codes + RefChain in float64 one face at a time, leaky-ReLU branches pinned to our activations, back-propagated
    twice: from the float64 loss gradient at our image (gcodes, gsv) and from the one at the chain's own image (gsv_e2e)."""
    _, _, gimg = ref_loss(inv.states, ours.img, leg.target)
    outs = []
    for f in range(leg.b):
        v = leg.sv[f:f + 1].double().requires_grad_(True)
        codes = F64.style_codes(inv.net, v)
        chain = F64.RefChain(inv.G, codes, leg.label[f:f + 1], [n[f:f + 1] for n in leg.noise],
                             [a[f:f + 1] for a in ours.acts])
        img = chain.image()
        gc, gv = torch.autograd.grad(img, (codes, v), gimg["all"][f:f + 1], retain_graph=True)
        _, _, ge = ref_loss(inv.states, img, leg.target[f:f + 1])
        (gv_e2e,) = torch.autograd.grad(img, v, ge["all"] / leg.b)
        outs.append((gc, gv, gv_e2e))
        del chain, img, codes, v
    return SimpleNamespace(gimg=gimg["all"], **{k: torch.cat([o[i] for o in outs])
                                                 for i, k in enumerate(("gcodes", "gsv", "gsv_e2e"))})


_RUNS = {}


def step_and_reference(inv, b):
    """(ours, reference) of one step at b faces, computed once per module."""
    if b not in _RUNS:
        leg = inv.legs[b]
        t0 = time.perf_counter()
        ours = _ours(inv, leg)
        t1 = time.perf_counter()
        torch.cuda.reset_peak_memory_stats()
        ref = _reference(inv, leg, ours)
        torch.cuda.synchronize()
        print(f"B={b}: our step {t1 - t0:.1f} s, float64 reference {time.perf_counter() - t1:.1f} s "
              f"(peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB allocated)")
        del ours.acts
        torch.cuda.empty_cache()
        _RUNS[b] = (ours, ref)
    return _RUNS[b]


B_CASES = [1, B_INV]
B_IDS = ["b1", f"b{B_INV}"]


# ============================================================================ 1. the fused pooling pyramid
def _pyr_ref(x):
    """(2x2, 4x4 block means) in float64 and the float64 means of |x| over the same blocks."""
    x = x.double()
    return F.avg_pool2d(x, 2), F.avg_pool2d(x, 4), F.avg_pool2d(x.abs(), 2), F.avg_pool2d(x.abs(), 4)


def _pyr_bwd_ref(g1, g2, g4, shape):
    """g1 + up2(g2) / 4 + up4(g4) / 16 in float64 (absent gradients are 0)."""
    out = torch.zeros(shape, dtype=torch.float64, device=DEV)
    for g, k in ((g1, 1), (g2, 2), (g4, 4)):
        if g is not None:
            out = out + g.double().repeat_interleave(k, -2).repeat_interleave(k, -1) / (k * k)
    return out


def _ulps(ours, ref, mag, kind, case):
    """|ours - ref| in fp32 ulps of mag (the float64 sum of the terms' magnitudes), elementwise; the largest against
    PYR_ULPS.  An element whose terms are all 0 must be exactly 0."""
    d = (ours.double() - ref).abs()
    assert bool(torch.isfinite(ours).all()), f"{case} {kind}: non-finite values"
    assert not bool((d[mag == 0] != 0).any()), f"{case} {kind}: non-zero where every term is 0"
    u = float((d / (torch.finfo(torch.float32).eps * mag).clamp_min(1e-300)).max())
    rms = float(d.norm() / ref.norm().clamp_min(1e-300))
    print(f"{case}: {kind} {u:.2f} ulp of sum|terms| at most, rel-RMS {rms:.2e} (bar {PYR_ULPS} ulp)")
    LEDGER.note(kind + " (ulp of sum|terms|)", u, rms, case)
    assert u <= PYR_ULPS, f"{case} {kind}: {u:.2f} ulp over the bar {PYR_ULPS}"


def _wrap_shape():
    """A shape whose 4x4 blocks outnumber the kernel's grid (SMs x 16 blocks of 256 threads) more than twice over, not
    a multiple of it: the grid-stride loop wraps."""
    cap = torch.cuda.get_device_properties(0).multi_processor_count * 16 * 256
    shape = (7, 3, 1024, 1032)
    assert shape[0] * shape[1] * (shape[2] // 4) * (shape[3] // 4) > 2 * cap
    return shape


# the benchmark's one face and 4 faces; h / 4 = 11 and w / 8 = 7 odd (w % 8 == 0 makes w / 4 even); a wrapping grid
PYR_SHAPES = [(1, 3, 1024, 1024), (4, 3, 1024, 1024), (3, 5, 44, 56), "wrap"]
PYR_IDS = ["1x3x1024", "4x3x1024", "3x5x44x56", "wrap"]
SUBSETS = [(1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (1, 0, 1), (0, 1, 1), (1, 1, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", PYR_SHAPES, ids=PYR_IDS)
def test_pyramid_against_float64(shape):
    """K.avgpool_pyramid against float64 block means, and K.avgpool_pyramid_bwd for every non-empty subset of
    {g1, g2, g4} against float64 g1 + up2(g2) / 4 + up4(g4) / 16; then all three gradients as non-contiguous views."""
    from e4s_b200 import kernels as K
    shape = _wrap_shape() if shape == "wrap" else shape
    n, c, h, w = shape
    case = "x".join(map(str, shape))
    x = F64.randn(*shape, seed=1)
    y2, y4 = K.avgpool_pyramid(x)
    r2, r4, m2, m4 = _pyr_ref(x)
    _ulps(y2, r2, m2, "pyramid fwd 2x2", case)
    _ulps(y4, r4, m4, "pyramid fwd 4x4", case)
    del x, y2, y4, r2, r4, m2, m4
    gs = [F64.randn(n, c, h // k, w // k, seed=2 + k) for k in (1, 2, 4)]
    for sub in SUBSETS:
        g = [t if on else None for t, on in zip(gs, sub)]
        gx = K.avgpool_pyramid_bwd(*g, shape)
        mag = _pyr_bwd_ref(*[None if t is None else t.abs() for t in g], shape)
        _ulps(gx, _pyr_bwd_ref(*g, shape), mag, "pyramid bwd", f"{case} g1/g2/g4 = {sub}")
        del gx, mag
    # non-contiguous views: every other column of a wider tensor, a transposed tensor, a channels-last tensor
    g1 = F64.randn(n, c, h, 2 * w, seed=6)[..., ::2]
    g2 = F64.randn(n, c, w // 2, h // 2, seed=7).transpose(-1, -2)
    g4 = F64.randn(n, h // 4, w // 4, c, seed=8).permute(0, 3, 1, 2)
    assert not any(t.is_contiguous() for t in (g1, g2, g4))
    gx = K.avgpool_pyramid_bwd(g1, g2, g4, shape)
    assert torch.equal(gx, K.avgpool_pyramid_bwd(g1.contiguous(), g2.contiguous(), g4.contiguous(), shape))
    _ulps(gx, _pyr_bwd_ref(g1, g2, g4, shape), _pyr_bwd_ref(g1.abs(), g2.abs(), g4.abs(), shape), "pyramid bwd",
          f"{case} non-contiguous gradients")


@pytest.mark.gpu
def test_pyramid_c_entry_writes_only_its_output():
    """The C entries, called directly, write their outputs placed inside NaN-filled buffers longer than them: every
    element around the outputs stays NaN, every element of them is written."""
    from e4s_b200 import _lib
    from e4s_b200._lib import check, ptr, stream_ptr
    n, c, h, w = 2, 3, 44, 56
    pad = 64                                           # floats before and after each output (keeps 16-byte alignment)
    lib = _lib.load()

    def placed(numel):
        buf = torch.full((numel + 2 * pad,), float("nan"), device=DEV)
        return buf, buf[pad:pad + numel]

    x = F64.randn(n, c, h, w, seed=11)
    b2, y2 = placed(n * c * h * w // 4)
    b4, y4 = placed(n * c * h * w // 16)
    check(lib.e4s_avgpool_pyramid_f32(ptr(x), ptr(y2), ptr(y4), n * c, h, w, stream_ptr()), "e4s_avgpool_pyramid_f32")
    g1, g2, g4 = (F64.randn(n, c, h // k, w // k, seed=12 + k) for k in (1, 2, 4))
    bx, gx = placed(n * c * h * w)
    check(lib.e4s_avgpool_pyramid_bwd_f32(ptr(g1), ptr(g2), ptr(g4), ptr(gx), n * c, h, w, stream_ptr()),
          "e4s_avgpool_pyramid_bwd_f32")
    torch.cuda.synchronize()
    for what, buf, out in (("2x2 means", b2, y2), ("4x4 means", b4, y4), ("gradient", bx, gx)):
        assert bool(buf[:pad].isnan().all()) and bool(buf[-pad:].isnan().all()), f"{what}: written outside the output"
        assert bool(torch.isfinite(out).all()), f"{what}: element not written"
    r2, r4, m2, m4 = _pyr_ref(x)
    _ulps(y2.view(n, c, h // 2, w // 2), r2, m2, "pyramid fwd 2x2", "C entry")
    _ulps(y4.view(n, c, h // 4, w // 4), r4, m4, "pyramid fwd 4x4", "C entry")
    _ulps(gx.view(n, c, h, w), _pyr_bwd_ref(g1, g2, g4, (n, c, h, w)),
          _pyr_bwd_ref(g1.abs(), g2.abs(), g4.abs(), (n, c, h, w)), "pyramid bwd", "C entry")


@pytest.mark.gpu
def test_pyramid_rejects_illegal_widths():
    """A width that is not a multiple of 8 is refused by the kernel's shape check, not computed."""
    from e4s_b200 import kernels as K
    with pytest.raises(Exception, match="SHAPE"):
        K.avgpool_pyramid(F64.randn(1, 3, 36, 36, seed=1))


# (shape, dtype, device, sizes, fused?)
DISPATCH = [((1, 3, 1024, 1024), torch.float32, DEV, (1024, 512, 256), True),
            ((2, 3, 64, 64), torch.float32, DEV, (64, 32, 16), True),
            ((2, 3, 64, 64), "channels_last", DEV, (64, 32, 16), True),
            ((1, 3, 64, 96), torch.float32, DEV, (64, 32, 16), False),        # not square
            ((1, 3, 36, 36), torch.float32, DEV, (36, 18, 9), False),         # w % 8 != 0
            ((1, 3, 64, 64), torch.float32, DEV, (64, 32, 8), False),         # not (H, H / 2, H / 4)
            ((1, 3, 64, 64), torch.float32, DEV, (64, 32), False),
            ((1, 3, 64, 64), torch.float64, DEV, (64, 32, 16), False),
            ((1, 3, 64, 64), torch.float32, "cpu", (64, 32, 16), False)]
DISPATCH_IDS = ["1024", "64", "64-channels-last", "non-square", "w36", "sizes-64-32-8", "two-sizes", "float64", "cpu"]


@pytest.mark.gpu
@pytest.mark.parametrize("shape,dtype,device,sizes,fused", DISPATCH, ids=DISPATCH_IDS)
def test_pyramid_dispatch(shape, dtype, device, sizes, fused):
    """criteria.inversion_loss.pyramid() launches the fused kernels exactly when its conditions hold, and equals
    F.adaptive_avg_pool2d: its values within the ulp bar of the float64 pooling on the fused path and bit for bit on the
    other (which is F.adaptive_avg_pool2d), its gradient within the ulp bar of the float64 one on both."""
    from e4s_b200 import kernels as K
    from e4s_b200.criteria.inversion_loss import pyramid
    x = F64.randn(*shape, seed=21, device=device)
    if dtype == "channels_last":
        x = x.contiguous(memory_format=torch.channels_last)
    elif dtype == torch.float64:
        x = x.double()
    ws = [F64.randn(*shape[:2], s, s, seed=22 + i, device=device).to(x.dtype) for i, s in enumerate(sizes)]

    def pooled(fn, x):
        """fn's poolings of a leaf copy of x and the gradient of sum_i <pooling_i, ws_i>."""
        x = x.detach().clone().requires_grad_(True)
        outs = fn(x)
        sum((o * wi).sum() for o, wi in zip(outs, ws)).backward()
        return [o.detach() for o in outs], x.grad

    launches, call = [], K._call
    K._call = lambda name, *a, **kw: (launches.append(name), call(name, *a, **kw))[1]
    try:
        outs, grad = pooled(lambda t: pyramid(t, sizes), x)
    finally:
        K._call = call
    assert launches == (["e4s_avgpool_pyramid_f32", "e4s_avgpool_pyramid_bwd_f32"] if fused else []), launches
    plain = lambda t: [F.adaptive_avg_pool2d(t, (s, s)) for s in sizes]
    refs, ref_grad = pooled(plain, x.double())
    mags = [F.adaptive_avg_pool2d(x.double().abs(), (s, s)) for s in sizes]
    ws = [wi.abs() for wi in ws]
    _, mag_grad = pooled(plain, x.double())             # the same adjoint applied to |ws|
    case = f"{'x'.join(map(str, shape))} {dtype} {device}"
    for s, o, r, m in zip(sizes, outs, refs, mags):
        assert o.shape == r.shape and o.dtype == x.dtype, (o.shape, o.dtype)
        if fused:
            _ulps(o, r, m, "pyramid() values", f"{case} size {s}")
        else:
            assert torch.equal(o, F.adaptive_avg_pool2d(x, (s, s))), s
    _ulps(grad, ref_grad, mag_grad, "pyramid() gradient", case)


# ============================================================================ 2. the loss and its image gradient
def image_gradient_errors(ours, ref):
    """(max-rel, rel-RMS) of the worst face for each norm, every face against its own maximum."""
    errs = [F64.Ledger._errors(ours[f:f + 1], ref[f:f + 1], 1e-30, "d / d recon") for f in range(ours.shape[0])]
    return max(e for e, _ in errs), max(r for _, r in errs)


def check_image_gradient(ours, ref, bars, kind, case):
    """Every face's max-rel <= bars[0] and rel-RMS <= bars[1]."""
    e, r = image_gradient_errors(ours, ref)
    print(f"{case}: {kind} max-rel {e:.2e} rel-RMS {r:.2e} (bars {bars[0]:.1e} / {bars[1]:.1e})")
    LEDGER.note(kind, e, r, case)
    assert e <= bars[0] and r <= bars[1], f"{case} {kind}: max-rel {e:.3e} rel-RMS {r:.3e} over the bars {bars}"


def _loss_case(inv, b):
    """Our fp32 reconstruction (the grad-mode forward of the checked step) and the leg's target."""
    ours, _ = step_and_reference(inv, b)
    return ours.img, inv.legs[b].target


@pytest.mark.gpu
@pytest.mark.parametrize("b", B_CASES, ids=B_IDS)
def test_loss_and_terms(b, inv):
    """The benchmark's criterion at our reconstruction: the loss and each of its four terms against calc_loss in
    float64 on the same two images, and the criterion's defaults are calc_loss's."""
    crit = inv.crit
    assert {t: getattr(crit, f"{t}_lambda") for t in TERMS} == LAMBDAS and crit.exact
    assert crit.lpips_sizes == (1024, 512, 256)
    recon, target = _loss_case(inv, b)
    loss, terms, _ = our_loss(crit, recon, target)
    with torch.no_grad():
        rl, rt = LO.calc_loss(inv.states, target.double(), recon.double())
    assert set(terms) == set(rt), (terms, rt)
    case = f"B={b}"
    for k, ours, ref in [("loss", loss, float(rl))] + [(k, terms[k], float(rt[k])) for k in sorted(rt)]:
        e = abs(ours - ref) / abs(ref)
        print(f"{case}: {k} {ours:.8g} float64 {ref:.8g} rel {e:.2e} (bar {TOL_LOSS:.0e})")
        LEDGER.note(f"loss value: {k}", e, e, case)
        assert e <= TOL_LOSS, (k, ours, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("b", B_CASES, ids=B_IDS)
def test_image_gradient(b, inv):
    """d loss / d recon per face against the float64 calc_loss gradient at the same image: the whole loss, then each term
    alone through a criterion that keeps only its lambda, so that a 0.1-weighted term cannot hide under the others.
    The reference is computed face by face and divided by the batch size."""
    recon, target = _loss_case(inv, b)
    _, _, ref = ref_loss(inv.states, recon, target)
    case = f"B={b}"
    _, _, g = our_loss(inv.crit, recon, target)
    check_image_gradient(g, ref["all"], TOL_GIMG["all"], "d loss / d recon", case)
    for t in TERMS:
        _, _, g = our_loss(inv.crit_term[t], recon, target)
        check_image_gradient(g, ref[t], TOL_GIMG[t], f"d {LAMBDAS[t]} {t} / d recon", case)


@pytest.mark.gpu
def test_image_gradient_faces_are_independent(inv):
    """Face f's image gradient at 4 faces is face f's gradient at one face divided by 4: our criterion mixes no faces and
    carries the 1/B of its means."""
    recon, target = _loss_case(inv, B_INV)
    _, _, g = our_loss(inv.crit, recon, target)
    for f in range(B_INV):
        _, _, g1 = our_loss(inv.crit, recon[f:f + 1], target[f:f + 1])
        check_image_gradient(B_INV * g[f:f + 1], g1, TOL_GIMG_FACE, "d loss / d recon, face of 4 x 4 vs alone",
                             f"face {f}")


@pytest.mark.gpu
def test_tf32_loss_networks_exceed_the_exact_bar(inv):
    """Negative control: with crit.exact = False the loss networks' convolutions run in TF32, and the same image-gradient
    check must then exceed the exact-mode bar (so that bar can see a TF32 backward); the error is held to its own looser
    bar.  The cuDNN precision switches are the same after the criterion as before, in either mode."""
    recon, target = _loss_case(inv, 1)
    _, _, ref = ref_loss(inv.states, recon, target)
    before = switches()
    crit = inv.crit
    try:
        crit.exact = False
        _, _, g = our_loss(crit, recon, target)
    finally:
        crit.exact = True
    assert switches() == before, (switches(), before)
    e, r = image_gradient_errors(g, ref["all"])
    exact = TOL_GIMG["all"]
    assert e > exact[0] or r > exact[1], f"the exact-mode bars {exact} do not see TF32 convolutions: {e:.2e} / {r:.2e}"
    check_image_gradient(g, ref["all"], TOL_GIMG_TF32, "d loss / d recon, TF32 loss networks", "B=1")


# ============================================================================ 3. one full-loss step through the generator
@pytest.mark.gpu
@pytest.mark.parametrize("b", B_CASES, ids=B_IDS)
def test_codes_gradient(b, inv):
    """d loss / d codes, every (face, region, latent index) slice against its own maximum."""
    ours, ref = step_and_reference(inv, b)
    LEDGER.check_slices(ours.gcodes, ref.gcodes, TOL_GCODES, "d loss / d codes", f"B={b}", inv.names)


@pytest.mark.gpu
@pytest.mark.parametrize("b", B_CASES, ids=B_IDS)
def test_texture_vector_gradient(b, inv):
    """d loss / d texture vectors, every (face, region) slice; and the float64 end-to-end gradient (loss and generator
    both in float64, the loss at the reference's own image) per face under its looser bar: the two images differ by the
    generator's forward error, which moves the loss networks' kinks."""
    ours, ref = step_and_reference(inv, b)
    LEDGER.check_slices(ours.gsv, ref.gsv, TOL_GSV, "d loss / d texture vectors", f"B={b}")
    LEDGER.check(ours.gsv, ref.gsv_e2e, TOL_E2E, "d loss / d texture vectors, float64 end to end", f"B={b}",
                 per_face=True)


@pytest.mark.gpu
def test_absent_regions_have_exactly_zero_gradients(inv):
    """The zero slices of d loss / d codes and d loss / d texture vectors are exactly those of regions without a pixel at
    every level that reads them, in the reference and in ours, and the 4-face leg has region 11 present and absent side
    by side."""
    leg = inv.legs[B_INV]
    ours, ref = step_and_reference(inv, B_INV)
    present = F64.present_pattern(inv.G, leg.label, NCLS)
    assert torch.equal((ref.gcodes == 0).all(-1).cpu(), ~present)
    assert torch.equal((ours.gcodes == 0).all(-1).cpu(), ~present)
    zero_sv = ~present[:, :, :N_OPT].any(-1)
    assert torch.equal((ref.gsv == 0).all(-1).cpu(), zero_sv)
    assert torch.equal((ours.gsv == 0).all(-1).cpu(), zero_sv)
    assert bool(zero_sv[2, 11]) and not bool(zero_sv[1, 11]) and not bool(zero_sv[3, 11]), zero_sv[:, 11]


# ============================================================================ 4. the invert legs bench.py times
def invert_inside(inv, leg, outside_exact, **kw):
    """invert with the benchmark's criterion and the leg's inputs, called inside conv_precision(outside_exact), so that
    only invert's own precision context can give the loss networks' backward the criterion's precision.  Returns the
    texture vectors, the loss history and the set of switches() the backward passes met at the loss networks'
    convolutions; the switches after invert are those before it."""
    from e4s_b200.criteria.inversion_loss import conv_precision
    from e4s_b200.optimization import invert
    with conv_precision(outside_exact):
        before = switches()
        with backward_switches(inv.crit) as seen:
            latent, _, hist = invert(inv.net, leg.target, leg.onehot, style_vectors=leg.sv, noise=leg.noise,
                                     criterion=inv.crit, **kw)
        torch.cuda.synchronize()
        assert switches() == before, (switches(), before)
    return latent, [float(h) for h in hist], set(seen)


@pytest.mark.gpu
@pytest.mark.parametrize("b", B_CASES, ids=B_IDS)
def test_sgd_step_moves_texture_vectors_by_the_gradient(b, inv):
    """invert(steps=1, opt_name="sgd", criterion=crit), called with cuDNN in TF32, runs the loss networks' backward in
    full fp32 and moves the texture vectors by -lr times the gradient checked above: against the float64 gradient and
    against our own gradient of the same step, per face; bit-unchanged where the gradient is exactly 0.  lr makes the
    largest move a tenth of the largest texture-vector entry, so fp32 rounding of the update stays far below the bars."""
    leg = inv.legs[b]
    ours, ref = step_and_reference(inv, b)
    lr = 0.1 * float(leg.sv.abs().max()) / float(ref.gsv.abs().max())
    latent, hist, seen = invert_inside(inv, leg, False, steps=1, lr=lr, opt_name="sgd")
    assert seen == {precision_of(True)}, seen
    moved = (leg.sv.double() - latent.double()) / lr
    zero = (ref.gsv == 0).all(-1)
    assert torch.equal(latent[zero], leg.sv[zero])
    LEDGER.check(moved, ref.gsv, TOL_SGD, "SGD step / -lr", f"B={b} lr {lr:.3g}", per_face=True)
    LEDGER.check(moved, ours.gsv, TOL_SGD_OURS, "SGD step / -lr against our gradient", f"B={b}", per_face=True)
    assert len(hist) == 1


_TRAJ = {}


def _graphed(inv, b):
    """invert(criterion=crit, cuda_graph=True, steps=6) with the exact criterion, called with cuDNN in TF32, once per
    module: (texture vectors, losses, switches the backward met)."""
    if b not in _TRAJ:
        _TRAJ[b] = invert_inside(inv, inv.legs[b], False, steps=6, cuda_graph=True)
    return _TRAJ[b]


@pytest.mark.gpu
@pytest.mark.parametrize("b", B_CASES, ids=B_IDS)
def test_adam_eager_and_graphed(b, inv):
    """Adam with the benchmark's criterion, eager and invert(cuda_graph=True) (3 eager warm-up steps, then 3 replays),
    both called with cuDNN in TF32: the loss networks' backward runs in full fp32 in both, the graphed loss trajectory
    follows the eager one step by step, and the texture vectors of absent regions stay bit-identical while the others
    move."""
    leg = inv.legs[b]
    _, ref = step_and_reference(inv, b)
    absent = (ref.gsv == 0).all(-1)
    steps = 6
    lat_e, he, seen_e = invert_inside(inv, leg, False, steps=steps)
    torch.cuda.empty_cache()
    lat_g, hg, seen_g = _graphed(inv, b)
    assert seen_e == seen_g == {precision_of(True)}, (seen_e, seen_g)
    for what, lat in (("eager", lat_e), ("graphed", lat_g)):
        assert torch.equal(lat[absent], leg.sv[absent]), what
        assert bool((lat[~absent] != leg.sv[~absent]).any(-1).all()), what
    print(f"Adam B={b}: eager losses {he}, graphed {hg}")
    assert len(he) == len(hg) == steps and len(set(hg)) == steps, (he, hg)
    e = max(abs(a - c) / abs(c) for a, c in zip(hg, he))
    LEDGER.note("graphed loss trajectory vs eager", e, e, f"B={b}")
    assert e <= TOL_GRAPH_LOSS, (hg, he)
    assert he[-1] < he[0], he


@pytest.mark.gpu
def test_tf32_graphed_trajectory(inv):
    """bench.py's ms_per_replayed_step_tf32_loss_networks configuration (one face, crit.exact = False, graphed, 6 steps),
    called with cuDNN in full fp32: the loss networks' backward runs in TF32, the loss trajectory differs from the exact
    graphed one but stays within TOL_TF32_LOSS of it step by step, invert leaves crit.exact as it found it, and the test
    restores it."""
    _, hx, _ = _graphed(inv, 1)
    try:
        inv.crit.exact = False
        _, ht, seen = invert_inside(inv, inv.legs[1], True, steps=6, cuda_graph=True)
        assert inv.crit.exact is False
    finally:
        inv.crit.exact = True
    assert seen == {precision_of(False)}, seen
    print(f"TF32 graphed losses {ht}, exact {hx}")
    e = max(abs(a - c) / abs(c) for a, c in zip(ht, hx))
    LEDGER.note("TF32 graphed loss trajectory vs exact", e, e, "B=1")
    assert len(ht) == 6 and e <= TOL_TF32_LOSS, (ht, hx)
    assert ht != hx, "TF32 trajectory identical to the exact one: the switch did not reach the loss networks"
