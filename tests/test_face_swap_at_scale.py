"""The batched face swap of bench.py (face_swap.swap_faces, 16 pairs at 1024 x 1024, 12 regions) against float64, stage by
stage and per pair: encoder, shape swap and blending masks, texture swap, MLP codes, generator.

The benchmark's configuration is imported, not restated: bench.build_net gives the weights, bench.face_label_maps the label
maps, and the images and labels are drawn as the benchmark's face-swap leg draws them at rank 0.  That draw gives 16 copies
of two label configurations in which every driven face has ears and teeth, so a few pairs are changed to make the batch
mix every branch of the texture swap and both paths of the masked up-sampling layers:

    pair NO_EAR    driven map without ears (class 7 relabelled as skin)
    pair NO_TEETH  driven map without teeth (class 9 relabelled as skin)
    pair NEITHER   both
    pair IID       iid labels on both sides: fragmented holes, and swapped maps whose row lists overflow the row cap

swap_comp_style_vector takes its two empty-region decisions per pair on the device; the reference takes them for its one
pair on the host.  Only a batch whose pairs disagree tells the two apart, so the texture swap is checked by applying the
reference (oracle.mask_oracle) to each pair's own vectors alone.  The encoder is f64ref.ref_get_style_vectors on the 32
faces, the codes f64ref.style_codes, the generator f64ref.RefChain on the host-swapped maps; tests/test_f64ref.py pins all
three to the CPU oracle.  Pairs must not see each other: reversing the pair order, running a pair alone, or making one
pair's images non-finite must leave every other pair's results where a second run of the same batch leaves them.
"""
import functools
import time
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import f64ref as F64
from f64ref import RefChain, layer_table, row_counts
from oracle import mask_oracle as MO

DEV = "cuda:0"
RES, NCLS, P, MASK_SIDE = 1024, 12, 16, 512       # bench.py defaults: --size 1024 --ncls 12, 16 face-swap pairs
IMAGE_SEED, LABEL_SEED = 400, 500                 # bench.py's face-swap leg at rank 0: driven / target images, label maps
NOISE_SEED, IID_SEED = 600, 700
NO_EAR, NO_TEETH, NEITHER, IID = 2, 5, 13, 7      # the pairs changed from the benchmark's draw
EAR, TEETH, SKIN = 7, 9, 6
OUTER_DILATION = 5                                # swap_faces' default
ALONE = (0, IID, 15)                              # pairs also run on their own
NAN_PAIR, INF_PAIR = 4, 11                        # the bad-pair run: driven image of NAN_PAIR NaN, target of INF_PAIR +Inf
LAYERS = layer_table()

# Bars, in max-rel and rel-RMS, each pair (or face) against its own maximum; both must hold for every pair.  The largest
# error observed on an H100 80GB HBM3 (700 W power limit) is in the comment; each bar sits 2-3x above it.
TOL_CODE = 1e-4       # texture vectors of the 32 faces against the float64 encoder (test_encoder_at_scale's bar): 3.7e-5
TOL_CODES = 3e-6      # MLP codes of the swapped vectors, exact fp32 GEMMs, against float64 on the same vectors: 9.9e-7
TOL_IMAGE = 3e-4      # the image against the float64 generator on our own codes (test_synthesis_at_scale's bar): 1.2e-4
# The image against float64 all the way from the faces: 1.35e-4.  The encoder's 4e-5 error in the texture vectors adds
# about 1e-5 to the generator's own 1.2e-4, so the bar is TOL_IMAGE's.
TOL_E2E = 3e-4
# Two runs of the same batch differ: instnorm_affine accumulates its sums with atomics, whose order varies from run to
# run, and the encoder's split-bf16 convolutions re-round what that changes.  The same bars hold the batch in reversed
# pair order and the clean faces of a batch with one bad pair; over all three, vectors 1.6e-5, codes 1.2e-5, image 2.9e-5.
TOL_RUN = (4e-5, 4e-5, 8e-5)      # vectors, codes, image
# A pair alone against the same pair inside the batch: the vectors at the encoder's batch bar (1.3e-5), the codes 1.2e-5,
# the image at the synthesis file's batch bar (6.9e-5).
TOL_BATCH = (5e-5, 3e-5, 1.5e-4)  # vectors, codes, image

LEDGER = F64.Ledger(42)
_PEAKS = []


def _check(ours, ref, tol, kind, case):
    LEDGER.check(ours, ref, tol, kind, case, per_face=True)


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


# ============================================================================ inputs and host references
@functools.lru_cache(maxsize=None)
def _pair_labels():
    import bench
    labs = bench.face_label_maps(2 * P, NCLS, "faces", seed=LABEL_SEED)[:, 0]
    d, t = labs[0::2].clone(), labs[1::2].clone()             # source / target example masks, alternating
    for p, classes in ((NO_EAR, (EAR,)), (NO_TEETH, (TEETH,)), (NEITHER, (EAR, TEETH))):
        for c in classes:
            d[p][d[p] == c] = SKIN
    g = torch.Generator().manual_seed(IID_SEED)
    d[IID], t[IID] = torch.randint(0, NCLS, (2, MASK_SIDE, MASK_SIDE), generator=g, dtype=torch.uint8)
    return d, t


def pair_labels():
    """Driven and target label maps [P, 512, 512] uint8: the benchmark's, with the changed pairs."""
    return tuple(x.clone() for x in _pair_labels())


def tap_sides():
    """Side of each tap unit's output at the encoder's 256 x 256 input."""
    from e4s_b200.encoders.psp_encoders import TAP_UNITS
    side, out = 256, []
    for i, (_, _, stride) in enumerate(F64.ENCODER_SPECS):
        side //= stride
        if i in TAP_UNITS:
            out.append(side)
    return out


def empty_regions(labels):
    """[B, ncls] bool: the region is absent at every tap level of the float64 encoder (labels_at of the one-hot map),
    which is when its float64 texture vector is all zero.  Present at any one level, it gets a non-zero mean there."""
    mask = F64.onehot(labels, NCLS, torch.float32)
    seen = torch.zeros(labels.shape[0], NCLS, dtype=torch.bool)
    for side in tap_sides():
        lab = F64.labels_at(mask, side, side)
        seen |= F.one_hot(lab.long(), NCLS).sum((1, 2)).cpu() > 0
    return ~seen


BRANCHES = {(False, False): "both", (True, False): "no ear", (False, True): "no teeth", (True, True): "neither"}


def intended_branches():
    want = ["both"] * P
    want[NO_EAR], want[NO_TEETH], want[NEITHER] = "no ear", "no teeth", "neither"
    return want


def branches_of(empty):
    """The texture-swap branch of every pair from the empty regions [P, ncls] of its driven face."""
    return [BRANCHES[(bool(e[EAR]), bool(e[TEETH]))] for e in empty]


@functools.lru_cache(maxsize=None)
def host_masks(hair_first=True, operation="dilation"):
    """The mask stage of every pair alone on the host (oracle.mask_oracle): swapped labels, holes, content, border and
    full masks, each [P, 512, 512] uint8."""
    d, t = _pair_labels()
    out = []
    for p in range(P):
        res, hole = MO.swap_head_mask(d[p].numpy(), t[p].numpy(), hair_first)
        fg = MO.foreground_mask(res, hole)
        _, border, full = MO.create_masks(fg, OUTER_DILATION, operation)
        out.append((res, hole, fg, border, full))
    return tuple(np.stack(x) for x in zip(*out))


def resize_labels(labels, side):
    return F.interpolate(labels[:, None].float(), size=(side, side), mode="nearest")[:, 0].to(torch.uint8)


def gathered_layers():
    """The masked up-sampling layers that run the gathered entry (row list, or the folded kernel past the row cap)."""
    from e4s_b200.stylegan2.modconv import MASKED_CONVT_MIN_RES
    return [r for r in LAYERS if r.kind == "conv" and r.up and r.masked and 2 * r.side >= MASKED_CONVT_MIN_RES]


@functools.lru_cache(maxsize=None)
def host_row_counts():
    """{layer name: (cap, rows of every pair's swapped map at the layer's output side)}."""
    from e4s_b200.kernels import convt_masked_cap
    swapped = torch.from_numpy(host_masks()[0])
    return {r.name: (convt_masked_cap(r.side, r.side), row_counts(resize_labels(swapped, 2 * r.side), NCLS))
            for r in gathered_layers()}


# ============================================================================ host-only
def test_constructed_batch_takes_every_branch():
    """The benchmark's own draw takes one branch in every pair; the constructed batch takes the intended branch in each
    pair and all four kinds occur.  Decided as the float64 vectors decide it: a region is empty when it is absent at
    every tap level."""
    import bench
    labs = bench.face_label_maps(2 * P, NCLS, "faces", seed=LABEL_SEED)[:, 0]
    assert set(branches_of(empty_regions(labs[0::2]))) == {"both"}
    d, _ = pair_labels()
    got = branches_of(empty_regions(d))
    print(f"branches: {got}")
    assert got == intended_branches()
    assert set(got) == set(BRANCHES.values())


def test_swapped_maps_take_both_masked_paths():
    """Some swapped map overflows the row cap of some masked up-sampling layer (its samples run the folded kernel) and
    some fit it at every such layer (the gathered transposed convolution): both paths run inside the one swap.  The
    constructed batch has holes (refilled with skin) in more than one pair."""
    counts = host_row_counts()
    over = {name: [p for p in range(P) if int(rows[p]) > cap] for name, (cap, rows) in counts.items()}
    for name, (cap, rows) in counts.items():
        print(f"{name}: cap {cap}, rows {rows.min()}..{rows.max()}, over the cap: pairs {over[name]}")
    assert any(over.values()), over
    assert any(all(p not in o for o in over.values()) for p in range(P)), over
    holes = host_masks()[1].reshape(P, -1).max(1)
    assert int((holes == 255).sum()) >= 2, holes


# ============================================================================ GPU checks
def run_swap(net, driven, target, d_lab, t_lab, noise, **opts):
    """swap_faces, with the texture vectors of its encoder pass (split into driven and target halves) and the codes it
    handed the generator."""
    from e4s_b200.face_swap import swap_faces
    seen = {}

    def get_style_vectors(img, mask):
        out = type(net).get_style_vectors(net, img, mask)
        seen["vectors"] = out[0].clone()
        return out

    def cal_style_codes(vec):
        seen["codes"] = type(net).cal_style_codes(net, vec)
        return seen["codes"]

    net.get_style_vectors, net.cal_style_codes = get_style_vectors, cal_style_codes
    try:
        res = swap_faces(net, driven, target, d_lab, t_lab, noise=noise, **opts)
    finally:
        del net.get_style_vectors, net.cal_style_codes
    b = driven.shape[0]
    return SimpleNamespace(res=res, d_vec=seen["vectors"][:b], t_vec=seen["vectors"][b:], codes=seen["codes"].clone())


@pytest.fixture(scope="module")
def S():
    """The benchmark's network, the 16 pairs (images as the benchmark draws them, the constructed label maps), fixed
    per-pair noise, and two runs of the clean batch."""
    import bench
    net = bench.build_net(RES, NCLS, torch.device(DEV))
    g = torch.Generator().manual_seed(IMAGE_SEED)
    driven, target = torch.randn(P, 3, RES, RES, generator=g).to(DEV), torch.randn(P, 3, RES, RES, generator=g).to(DEV)
    d_lab, t_lab = (x.to(DEV) for x in pair_labels())
    gn = torch.Generator().manual_seed(NOISE_SEED)
    sides = [4] + [2 ** (i // 2 + 3) for i in range(2 * (net.G.log_size - 2))]
    noise = [torch.randn(P, 1, s, s, generator=gn).to(DEV) for s in sides]
    s = SimpleNamespace(net=net, driven=driven, target=target, d_lab=d_lab, t_lab=t_lab, noise=noise)
    s.swap = lambda **kw: run_swap(net, driven, target, d_lab, t_lab, noise, **kw)
    s.clean = s.swap()
    s.again = s.swap()
    torch.cuda.empty_cache()
    return s


@pytest.fixture(scope="module")
def V64(S):
    """Texture vectors of the 32 faces (driven, then target) from the float64 encoder, on the device."""
    from e4s_b200.encoders.psp_encoders import TAP_UNITS
    p = {k[len("encoder."):]: v.double() for k, v in S.net.state_dict().items() if k.startswith("encoder.")}
    mask = F64.onehot(torch.cat([S.d_lab, S.t_lab]), NCLS, torch.float64)
    t0 = time.perf_counter()
    with torch.no_grad():
        vec = F64.ref_get_style_vectors(p, torch.cat([S.driven, S.target]), mask, TAP_UNITS)
    torch.cuda.synchronize()
    print(f"\nfloat64 encoder, B = {2 * P}: {time.perf_counter() - t0:.1f} s")
    del p, mask
    torch.cuda.empty_cache()
    return vec


def _host(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _check_masks(res, hair_first, operation, case):
    """Labels, holes and the three blending masks of a SwapResult bit for bit against the host mask stage, pair by pair."""
    want = dict(zip(("swapped label", "hole map", "content mask", "border mask", "full mask"),
                    host_masks(hair_first, operation)))
    got = {"swapped label": res.swapped_label, "hole map": res.hole_map, "content mask": res.content_mask[:, 0],
           "border mask": res.border_mask[:, 0], "full mask": res.full_mask[:, 0]}
    for kind, ours in got.items():
        ref = _host(want[kind]).to(ours.dtype)
        bad = [p for p in range(P) if not torch.equal(ours[p], ref[p])]
        assert not bad, f"{case}: {kind} differs on pairs {bad}"


def _same_masks(a, b, pairs, case):
    for kind in ("swapped_label", "hole_map", "content_mask", "border_mask", "full_mask"):
        x, y = getattr(a, kind), getattr(b, kind)
        bad = [p for p in pairs if not torch.equal(x[p], y[p])]
        assert not bad, f"{case}: {kind} differs on pairs {bad}"


@pytest.mark.gpu
def test_encoder_stage(S, V64):
    """The driven and target texture vectors of all 16 pairs (the swap's one encoder pass over 32 faces) against the
    float64 encoder, each face against its own maximum; the regions whose vector is exactly zero are the host's empty
    regions, in ours and in float64."""
    ours = torch.cat([S.clean.d_vec, S.clean.t_vec])
    _check(S.clean.d_vec, V64[:P], TOL_CODE, "texture vectors (driven)", f"encoder B={2 * P}")
    _check(S.clean.t_vec, V64[P:], TOL_CODE, "texture vectors (target)", f"encoder B={2 * P}")
    empty = empty_regions(torch.cat([S.d_lab, S.t_lab]).cpu())
    assert torch.equal((V64 == 0).all(-1).cpu(), empty)
    assert torch.equal((ours == 0).all(-1).cpu(), empty)
    assert branches_of((S.clean.d_vec == 0).all(-1)) == intended_branches()


MASK_VARIANTS = {"default": dict(), "hair_first=False": dict(hair_first=False), "lap_bld": dict(lap_bld=True)}


@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(MASK_VARIANTS))
def test_mask_stage(S, variant):
    """swapped_label and hole_map against MO.swap_head_mask, the content, border and full masks against
    MO.foreground_mask + MO.create_masks, each pair alone on the host, bit for bit: swap_faces' defaults, hair after the
    inner face, and the expansion border of Laplacian blending."""
    opts = MASK_VARIANTS[variant]
    res = S.clean.res if not opts else S.swap(**opts).res
    _check_masks(res, opts.get("hair_first", True), "expansion" if opts.get("lap_bld") else "dilation", variant)


@pytest.mark.gpu
@pytest.mark.parametrize("interp", [False, True], ids=["plain", "belowFace_interpolation"])
def test_texture_swap_per_pair(S, interp):
    """Each pair alone through the reference's texture swap (MO.swap_comp_style_vector at B = 1, its host-side empty-region
    tests), applied to the vectors our encoder pass gave that pair, equals the pair's row of SwapResult.style_vectors bit
    for bit."""
    from e4s_b200.face_swap import TARGET_KEPT_REGIONS
    run = S.clean if not interp else S.swap(belowFace_interpolation=True)
    comp = sorted(set(range(NCLS)) - set(TARGET_KEPT_REGIONS))
    d, t, got = (x.cpu().numpy() for x in (run.d_vec, run.t_vec, run.res.style_vectors))
    assert branches_of(torch.from_numpy(d == 0).all(-1)) == intended_branches()
    bad = [p for p in range(P) if not np.array_equal(MO.swap_comp_style_vector(t[p:p + 1], d[p:p + 1], comp, interp)[0],
                                                     got[p])]
    assert not bad, f"swapped texture vectors differ on pairs {bad}"


@pytest.mark.gpu
def test_codes(S):
    """The codes the swap handed the generator (Net3.cal_style_codes on the swapped vectors) against f64ref.style_codes on
    the same vectors in float64."""
    with torch.no_grad():
        ref = F64.style_codes(S.net, S.clean.res.style_vectors.double())
    _check(S.clean.codes, ref, TOL_CODES, "codes", f"P={P}")


ENTRIES = {"e4s_modconv3x3_up_masked_tcr_fwd": "gathered", "e4s_modconv3x3_up_tcr_fwd": "convt",
           "e4s_modconv3x3_fwd_f32": "simt", "e4s_torgb_fwd_f32": "torgb"}


def _spy(monkeypatch):
    """Record the forward entry of every modulated-convolution launch (as tests/test_synthesis_at_scale.py does) and, for
    the gathered entry, the row count the device reached for each sample: the entry's count buffer is replaced by one the
    spy keeps.  Returns (entries, [(input side, cap, count [B])])."""
    from e4s_b200 import kernels as K
    from e4s_b200._lib import ptr
    taken, counts, call = [], [], K._call

    def spy(name, fn, *args, **kw):
        if name == "e4s_modconv3x3_tcr_fwd":
            taken.append("folded" if args[15] else "rs")
        elif name in ENTRIES:
            taken.append(ENTRIES[name])
        if name == "e4s_modconv3x3_up_masked_tcr_fwd":
            count = torch.empty(args[16], device=DEV, dtype=torch.int32)
            args = args[:12] + (ptr(count),) + args[13:]
            counts.append((args[17], args[22], count))
        return call(name, fn, *args, **kw)
    monkeypatch.setattr(K, "_call", spy)
    return taken, counts


def _expected_entry(r):
    from e4s_b200.stylegan2.modconv import MASKED_CONVT_MIN_RES
    if r.kind == "rgb":
        return "torgb"
    if not r.up:
        return "rs"
    if not r.masked:
        return "convt"
    return "gathered" if 2 * r.side >= MASKED_CONVT_MIN_RES else "folded"


def _ref_image(S, codes64):
    swapped = _host(host_masks()[0])
    with torch.no_grad():
        img = RefChain(S.net.G, codes64, swapped, S.noise).image()
    torch.cuda.empty_cache()
    return img


@pytest.mark.gpu
def test_image(S, monkeypatch):
    """SwapResult.image against f64ref.RefChain on the float64 cast of our own codes and the host-swapped maps, every pair
    against its own maximum.  Every layer takes its expected entry, and at each masked up-sampling layer the device's
    row count of every sample is the host's (or past the cap where the host's is): the pairs over the cap ran on the
    folded kernel, the others on the gathered transposed convolution."""
    taken, counts = _spy(monkeypatch)
    run = S.swap()
    assert taken == [_expected_entry(r) for r in LAYERS], taken
    host = host_row_counts()
    assert [(2 * h, cap) for h, cap, _ in counts] == [(2 * r.side, host[r.name][0]) for r in gathered_layers()]
    paths = set()
    for r, (_, cap, dev) in zip(gathered_layers(), counts):
        dev, rows = dev.cpu().long(), host[r.name][1]
        fits = rows <= cap
        assert torch.equal(dev[fits], rows[fits]) and bool((dev[~fits] > cap).all()), (r.name, dev.tolist(), rows.tolist())
        paths |= {"gathered" if f else "folded" for f in fits.tolist()}
        print(f"{r.name}: pairs on the folded kernel {(~fits).nonzero().flatten().tolist()}")
    assert paths == {"gathered", "folded"}
    _check_masks(run.res, True, "dilation", "spied run")
    ref = _ref_image(S, run.codes.double())
    _check(run.res.image, ref, TOL_IMAGE, "image (our codes)", f"P={P}")


@pytest.mark.gpu
def test_image_from_float64_faces(S, V64):
    """SwapResult.image against float64 all the way from the faces: float64 vectors, the texture swap of each pair alone,
    float64 codes, RefChain.  This measures what the encoder's error does to the swapped face."""
    from e4s_b200.face_swap import TARGET_KEPT_REGIONS
    comp = sorted(set(range(NCLS)) - set(TARGET_KEPT_REGIONS))
    d, t = V64[:P].cpu().numpy(), V64[P:].cpu().numpy()
    vec = np.concatenate([MO.swap_comp_style_vector(t[p:p + 1], d[p:p + 1], comp) for p in range(P)])
    with torch.no_grad():
        codes = F64.style_codes(S.net, _host(vec))
    _check(S.clean.res.image, _ref_image(S, codes), TOL_E2E, "image (float64 from the faces)", f"P={P}")


def _compare_runs(a, b, pairs, tols, what, case):
    """Texture vectors (driven, target, swapped), codes and images of run a against run b on the given pairs (rows of
    both runs), with the bars tols = (vectors, codes, image)."""
    idx = torch.tensor(pairs, device=DEV)
    _check(a.d_vec[idx], b.d_vec[idx], tols[0], f"texture vectors ({what})", case + " driven")
    _check(a.t_vec[idx], b.t_vec[idx], tols[0], f"texture vectors ({what})", case + " target")
    _check(a.res.style_vectors[idx], b.res.style_vectors[idx], tols[0], f"swapped vectors ({what})", case)
    _check(a.codes[idx], b.codes[idx], tols[1], f"codes ({what})", case)
    _check(a.res.image[idx], b.res.image[idx], tols[2], f"image ({what})", case)


def _flipped(run):
    """A run's per-pair outputs in reversed pair order."""
    r = run.res
    res = SimpleNamespace(**{k: getattr(r, k).flip(0) for k in ("image", "swapped_label", "hole_map", "content_mask",
                                                                  "border_mask", "full_mask", "style_vectors")})
    return SimpleNamespace(res=res, d_vec=run.d_vec.flip(0), t_vec=run.t_vec.flip(0), codes=run.codes.flip(0))


@pytest.mark.gpu
def test_pair_order_reversed(S):
    """Two runs of the clean batch differ only by the encoder's atomic sums (the run-to-run bars); the batch in reversed
    pair order gives every output in reversed order, labels and masks bit for bit, the rest within the same bars."""
    every = list(range(P))
    _compare_runs(S.again, S.clean, every, TOL_RUN, "run to run", "second run")
    _same_masks(S.again.res, S.clean.res, every, "second run")
    rev = run_swap(S.net, S.driven.flip(0), S.target.flip(0), S.d_lab.flip(0), S.t_lab.flip(0),
                   [n.flip(0) for n in S.noise])
    back = _flipped(rev)
    del rev
    _same_masks(back.res, S.clean.res, every, "reversed pairs")
    _compare_runs(back, S.clean, every, TOL_RUN, "run to run", "reversed pairs")


@pytest.mark.gpu
@pytest.mark.parametrize("pair", ALONE)
def test_pair_alone(S, pair):
    """A pair swapped on its own (P = 1) against the same pair inside the 16-pair batch."""
    sl = slice(pair, pair + 1)
    one = run_swap(S.net, S.driven[sl], S.target[sl], S.d_lab[sl], S.t_lab[sl], [n[sl] for n in S.noise])
    case = f"pair {pair} alone"
    for kind in ("swapped_label", "hole_map", "content_mask", "border_mask", "full_mask"):
        assert torch.equal(getattr(one.res, kind)[0], getattr(S.clean.res, kind)[pair]), (case, kind)
    clean = SimpleNamespace(res=SimpleNamespace(style_vectors=S.clean.res.style_vectors[sl], image=S.clean.res.image[sl]),
                            d_vec=S.clean.d_vec[sl], t_vec=S.clean.t_vec[sl], codes=S.clean.codes[sl])
    _compare_runs(one, clean, [0], TOL_BATCH, "alone vs batch", case)


@pytest.mark.gpu
def test_one_bad_pair(S):
    """Pair NAN_PAIR's driven face all NaN, pair INF_PAIR's target face all +Inf: every other face's texture vectors and
    every other pair's swapped vectors, codes and image are finite and match the clean run within the run-to-run bars;
    labels and masks, which do not depend on the images, are bit-identical for all 16 pairs."""
    driven, target = S.driven.clone(), S.target.clone()
    driven[NAN_PAIR] = float("nan")
    target[INF_PAIR] = float("inf")
    bad = run_swap(S.net, driven, target, S.d_lab, S.t_lab, S.noise)
    del driven, target
    _same_masks(bad.res, S.clean.res, list(range(P)), "one bad pair")
    good = [p for p in range(P) if p not in (NAN_PAIR, INF_PAIR)]
    case = "one bad pair"
    for half, skip in (("t_vec", NAN_PAIR), ("d_vec", INF_PAIR)):     # the clean face of each bad pair
        _check(getattr(bad, half)[skip:skip + 1], getattr(S.clean, half)[skip:skip + 1], TOL_RUN[0],
               "texture vectors (run to run)", f"{case}, clean face of pair {skip}")
    _compare_runs(bad, S.clean, good, TOL_RUN, "run to run", case)
    finite = {k: [bool(torch.isfinite(getattr(bad.res, k)[p]).all()) for p in (NAN_PAIR, INF_PAIR)]
              for k in ("style_vectors", "image")}
    print(f"bad pairs {NAN_PAIR}, {INF_PAIR}: finite outputs {finite}")
