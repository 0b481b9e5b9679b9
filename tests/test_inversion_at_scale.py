"""One step of the 1024x1024 inversion (optimization.invert: cal_style_codes -> gen_img -> l2 loss -> backward) on the
default kernels, at one face and at bench.py's 8-face batch, against a float64 reference that shares no code with the
kernels or their weight preparation.

The benchmark's configuration is imported, not restated: bench.build_net gives the weights, bench.face_label_maps the label
maps, and the texture vectors and targets are drawn as bench.run_ours draws them at rank 0; the noise is fixed, as invert
accepts it.  Faces 5-7 of the batch take f64ref.labels("one-pixel") maps: region 11 is a single pixel (the first, the last
or an inner one) that survives the nearest-resized label pyramid at some levels and not at others, so those faces have
exactly-zero style gradients at some layers and the next face has the region elsewhere - a gradient that leaks across
faces or regions shows as a non-zero where the reference has an exact 0.

Under grad mode Generator._layer_styles hands every layer its latent slice, so each layer runs its own modulation
(LinearFn on e4s_linear_f32) and demodulation, and the LocalMLPs run as two more LinearFn launches: the path checked here
is not the no-grad forward of tests/test_synthesis_at_scale.py.

The reference is f64ref.style_codes + f64ref.RefChain under autograd, one face at a time.  Each StyledConv's leaky-ReLU
branch is pinned to the sign of our own output of that layer (recorded with forward hooks), as the backward kernels take
it: a near-zero pre-activation that the split-bf16 forward puts on the other branch then moves the reference with it,
and the reference's gradient is a smooth function of its inputs.  That is what lets the whole gradient be held, slice by
slice, to a bar a few times the per-layer ones instead of a cosine.  tests/test_f64ref.py pins the chain, its gradient
and the pins to the CPU oracle.
"""
import time
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

import f64ref as F64
from f64ref import layer_table

DEV = "cuda:0"
RES, NCLS = 1024, 12                       # bench.py defaults: --size 1024 --ncls 12
B_LABELS, B_INV = 16, 8                    # --batch 16 (the label maps the inversion takes its faces from), --inversion-batch 8
LABEL_SEED, SV_SEED, NOISE_SEED = 200, 300, 400          # bench.run_ours at rank 0: labels 200, texture vectors 300
N_OPT = 13                                 # codes from this index on are latent_avg rows (K = 13), not optimised
ONE_PIXEL = {5: "first", 6: "last", 7: "inner"}          # faces of the batch with a one-pixel region 11
LAYERS = layer_table()

# Bars, in max-rel (against the slice's or face's own maximum) and rel-RMS; both must hold everywhere.  The largest error
# observed on an H100 80GB HBM3 (700 W power limit) is in the comment; each bar sits 2-3x above it.
TOL_CODES = 3e-6        # codes from the two LocalMLP GEMMs, exact fp32: 1.2e-6 (B = 8)
TOL_IMAGE = 2.5e-4      # the image after the grad-mode forward (per-layer modulation and demodulation launches): 9.8e-5
# d loss / d codes, each (face, region, latent index) slice against its own maximum: 4.0e-4 (B = 8, region 0 at latent 17,
# rgb1024: the ToRGB style gradient sums g * x over the image, and x carries the 17 stacked StyledConvs' forward error);
# 1.6e-4 at one face (c256)
TOL_GCODES = 1e-3
TOL_GSV = 7.5e-4        # d loss / d texture vectors, each (face, region) slice against its own maximum: 2.9e-4 (B = 8)
TOL_SGD = 7e-4          # one SGD step of invert, (initial - final) / lr per face, against the float64 gradient: 2.7e-4
# The graphed Adam loop's loss against the eager one on the same inputs, step by step: 6.8e-6 at most over 6 steps (the
# capturable Adam's arithmetic differs from the eager one's from the first update on).
TOL_GRAPH_LOSS = 2e-5

LEDGER = F64.Ledger(34)
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
@pytest.fixture(scope="module")
def inv():
    """The benchmark's network (every parameter frozen, as bench.py freezes it before the inversion legs), its label maps,
    texture vectors and targets for the one-face and the 8-face legs, fixed per-face noise, and the layers that read each
    latent index."""
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
    svb, tvb = draw(B_INV), draw(B_INV)                # then the batched leg's
    lab_b = labels[:B_INV].clone()
    lab_b[5:8, 0] = F64.labels("one-pixel", 3, 512, 512, NCLS, None)
    gn = torch.Generator().manual_seed(NOISE_SEED)
    sides = [4] + [2 ** (i // 2 + 3) for i in range(2 * (G.log_size - 2))]
    noise_b = [torch.randn(B_INV, 1, s, s, generator=gn).to(DEV) for s in sides]
    sched = G._schedule()
    names = {}
    for r, (_, idx, _) in zip(LAYERS, sched):
        names.setdefault(idx, []).append(r.name)
    legs = {}
    for b, sv, tv, lab, noise in ((1, sv1, tv1, labels[:1], [n[:1] for n in noise_b]), (B_INV, svb, tvb, lab_b, noise_b)):
        lab = lab.to(DEV)
        onehot = K.label_to_onehot(lab, NCLS)
        with torch.no_grad():
            target = net.gen_img(None, net.cal_style_codes(tv), onehot, noise=noise)[0]
        legs[b] = SimpleNamespace(b=b, sv=sv, target=target, label=lab[:, 0], onehot=onehot, noise=noise)
    return SimpleNamespace(net=net, G=G, sched=sched, names=names, legs=legs)


# ============================================================================ one step, ours and float64
def _ours(inv, leg):
    """One loop body of invert on the default kernels: the codes (read with retain_grad), the image, the gradients, the
    kernel launches of the forward and every StyledConv's output."""
    from e4s_b200 import kernels as K
    from e4s_b200.stylegan2.model import StyledConv
    launches, acts, call = [], [], K._call
    hooks = [m.register_forward_hook(lambda mod, inp, out: acts.append(out.detach()))
             for m in inv.G.modules() if isinstance(m, StyledConv)]
    K._call = lambda name, *a, **kw: (launches.append(name), call(name, *a, **kw))[1]
    try:
        latent = leg.sv.clone().requires_grad_(True)
        codes = inv.net.cal_style_codes(latent)
        codes.retain_grad()
        img = inv.net.gen_img(None, codes, leg.onehot, noise=leg.noise)[0]
        fwd = list(launches)
        loss = F.mse_loss(img, leg.target)
        loss.backward()
        torch.cuda.synchronize()
    finally:
        K._call = call
        for h in hooks:
            h.remove()
    return SimpleNamespace(codes=codes.detach(), img=img.detach(), gcodes=codes.grad, gsv=latent.grad, launches=fwd,
                           acts=acts)


def _reference(inv, leg, acts):
    """style_codes + RefChain in float64 for one face at a time, leaky-ReLU branches pinned to acts; face f's l2 loss is
    divided by the batch size, as F.mse_loss averages over the batch."""
    outs = []
    for f in range(leg.b):
        v = leg.sv[f:f + 1].double().requires_grad_(True)
        codes = F64.style_codes(inv.net, v)
        codes.retain_grad()
        chain = F64.RefChain(inv.G, codes, leg.label[f:f + 1], [n[f:f + 1] for n in leg.noise], [a[f:f + 1] for a in acts])
        img = chain.image()
        loss = (img - leg.target[f:f + 1].double()).pow(2).sum() / (leg.b * img.numel())
        loss.backward()
        outs.append((codes.detach(), img.detach(), codes.grad, v.grad))
        del chain, img, loss, codes, v
    return SimpleNamespace(**{k: torch.cat([o[i] for o in outs]) for i, k in enumerate(("codes", "img", "gcodes", "gsv"))})


_RUNS = {}


def step_and_reference(inv, b):
    """(ours, reference) of one step at b faces, computed once per module."""
    if b not in _RUNS:
        leg = inv.legs[b]
        t0 = time.perf_counter()
        ours = _ours(inv, leg)
        t1 = time.perf_counter()
        torch.cuda.reset_peak_memory_stats()
        ref = _reference(inv, leg, ours.acts)
        torch.cuda.synchronize()
        print(f"B={b}: our step {t1 - t0:.1f} s, float64 reference {time.perf_counter() - t1:.1f} s "
              f"(peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB allocated)")
        del ours.acts
        torch.cuda.empty_cache()
        _RUNS[b] = (ours, ref)
    return _RUNS[b]


B_CASES = [1, B_INV]
B_IDS = ["b1", f"b{B_INV}"]


# ============================================================================ GPU checks
@pytest.mark.gpu
@pytest.mark.parametrize("b", B_CASES, ids=B_IDS)
def test_grad_mode_forward(b, inv):
    """The forward under grad mode: no batched linear_multi launch, one e4s_linear_f32 per modulation (17 StyledConvs, 9
    ToRGBs) plus the two LocalMLP GEMMs, one demodulation per StyledConv; the codes and the image against float64."""
    ours, ref = step_and_reference(inv, b)
    n_conv = sum(r.kind == "conv" for r in LAYERS)
    assert "e4s_linear_multi_f32" not in ours.launches, ours.launches
    assert ours.launches.count("e4s_linear_f32") == len(LAYERS) + 2, ours.launches
    assert ours.launches.count("e4s_demod_gemm_f32") == n_conv, ours.launches
    case = f"B={b}"
    LEDGER.check(ours.codes, ref.codes, TOL_CODES, "codes", case, per_face=True)
    LEDGER.check(ours.img, ref.img, TOL_IMAGE, "image (grad-mode forward)", case, per_face=True)


@pytest.mark.gpu
@pytest.mark.parametrize("b", B_CASES, ids=B_IDS)
def test_codes_gradient(b, inv):
    """d loss / d codes, every (face, region, latent index) slice against its own maximum: a slice is the style gradient
    of the one or two layers that read that latent index, so a wrong region, layer or face shows in its own slice.  Codes
    from index 13 on are latent_avg rows; their region-0 slices carry the global layers' style gradients."""
    ours, ref = step_and_reference(inv, b)
    LEDGER.check_slices(ours.gcodes, ref.gcodes, TOL_GCODES, "d loss / d codes", f"B={b}", inv.names)


@pytest.mark.gpu
@pytest.mark.parametrize("b", B_CASES, ids=B_IDS)
def test_texture_vector_gradient(b, inv):
    """d loss / d texture vectors (through LinearFn's backward of both LocalMLP GEMMs), every (face, region) slice."""
    ours, ref = step_and_reference(inv, b)
    LEDGER.check_slices(ours.gsv, ref.gsv, TOL_GSV, "d loss / d texture vectors", f"B={b}")


@pytest.mark.gpu
def test_absent_regions_have_exactly_zero_gradients(inv):
    """The zero slices of d loss / d codes are exactly those of regions without a pixel at every level that reads them, in
    the reference and in ours; the one-pixel faces have the intended pattern (region 11 everywhere, nowhere, and only at
    the 256 x 256 layers), so the batch does exercise zero slices next to non-zero ones of the same region."""
    leg = inv.legs[B_INV]
    ours, ref = step_and_reference(inv, B_INV)
    present = F64.present_pattern(inv.G, leg.label, NCLS)
    zero_ref = (ref.gcodes == 0).all(-1).cpu()
    zero_ours = (ours.gcodes == 0).all(-1).cpu()
    assert torch.equal(zero_ref, ~present), (zero_ref != ~present).nonzero().tolist()[:12]
    assert torch.equal(zero_ours, ~present), (zero_ours != ~present).nonzero().tolist()[:12]
    opt = present[:, 11, :N_OPT]
    assert bool(opt[5].all()), "first pixel: every level"
    assert not bool(opt[6].any()), "last pixel: no masked level"
    inner = [i for i in range(N_OPT) if opt[7, i]]
    assert inner and all(LAYERS[k].side >= 128 for k, (_, idx, _) in enumerate(inv.sched) if idx in inner), inner
    assert not bool(opt[7].all())
    zero_sv = (ref.gsv == 0).all(-1).cpu()
    assert torch.equal(zero_sv, ~present[:, :, :N_OPT].any(-1)) and bool(zero_sv[6, 11])
    assert torch.equal((ours.gsv == 0).all(-1).cpu(), zero_sv)


@pytest.mark.gpu
@pytest.mark.parametrize("b", B_CASES, ids=B_IDS)
def test_sgd_step_moves_texture_vectors_by_the_gradient(b, inv):
    """invert(steps=1, opt_name="sgd", lr) moves the texture vectors by -lr times the gradient checked above: (initial -
    final) / lr against the float64 gradient per face, and bit-unchanged where that gradient is exactly 0.  lr makes the
    largest move a tenth of the largest texture-vector entry, so fp32 rounding of the update stays far below the bar."""
    from e4s_b200.optimization import invert
    leg = inv.legs[b]
    _, ref = step_and_reference(inv, b)
    lr = 0.1 * float(leg.sv.abs().max()) / float(ref.gsv.abs().max())
    latent, _, hist = invert(inv.net, leg.target, leg.onehot, style_vectors=leg.sv, steps=1, lr=lr, opt_name="sgd",
                             noise=leg.noise)
    moved = (leg.sv.double() - latent.double()) / lr
    zero = (ref.gsv == 0).all(-1)
    assert torch.equal(latent[zero], leg.sv[zero])
    LEDGER.check(moved, ref.gsv, TOL_SGD, "SGD step / -lr", f"B={b} lr {lr:.3g}", per_face=True)
    assert len(hist) == 1


@pytest.mark.gpu
def test_adam_eager_and_graphed_batch(inv):
    """Adam at the 8-face batch, eager and invert(cuda_graph=True) (the benchmark's batched leg): the texture vectors of
    regions absent from a face stay bit-identical over every step, the others move, and the graphed loss trajectory
    follows the eager one step by step."""
    from e4s_b200.optimization import invert
    leg = inv.legs[B_INV]
    _, ref = step_and_reference(inv, B_INV)
    absent = (ref.gsv == 0).all(-1)
    assert bool(absent.any()) and bool((~absent).any())
    steps = 6                                          # 3 eager warm-up steps + 3 replays on the graphed path
    lat_e, _, hist_e = invert(inv.net, leg.target, leg.onehot, style_vectors=leg.sv, steps=steps, noise=leg.noise)
    torch.cuda.empty_cache()
    lat_g, _, hist_g = invert(inv.net, leg.target, leg.onehot, style_vectors=leg.sv, steps=steps, noise=leg.noise,
                              cuda_graph=True)
    torch.cuda.synchronize()
    for what, lat in (("eager", lat_e), ("graphed", lat_g)):
        assert torch.equal(lat[absent], leg.sv[absent]), what
        assert bool((lat[~absent] != leg.sv[~absent]).any(-1).all()), what
    he, hg = [float(h) for h in hist_e], [float(h) for h in hist_g]
    print(f"Adam B={B_INV}: eager losses {he}, graphed {hg}")
    assert len(he) == len(hg) == steps and len(set(hg)) == steps, (he, hg)
    for a, b in zip(hg, he):
        assert abs(a - b) <= TOL_GRAPH_LOSS * abs(b), (hg, he)
    assert he[-1] < he[0], he
    de, dg = (lat_e - leg.sv).abs().mean(), (lat_g - leg.sv).abs().mean()
    assert abs(float(dg) - float(de)) <= 0.05 * float(de), (float(dg), float(de))
