"""The 1024x1024 mask-guided synthesis forward of bench.py (Net3.gen_img, K = 13, 12 regions, 16 faces) against a float64
reference that shares no code with the kernels, their weight preparation (PreparedConv, fold_upsample_kernels,
convt_class_kernels) or e4s_b200.kernels.

The benchmark's configuration is imported, not restated: bench.build_net gives the weights, bench.face_label_maps the label
maps, and the codes are drawn as bench.run_ours draws them.  Every layer runs through its module's own forward, with the
PrecomputedStyle that Generator._layer_styles hands it, the LabelPyramid of the bench labels and per-sample noise, and
starts from the float64 activation of the layer before it, cast to fp32.  All 16 faces are compared, each against its
own maximum.

The reference (f64ref.RefChain) computes the modulations and demodulations from each module's own parameters.  Its StyledConvs
are f64ref.styled_conv_per_pixel: a masked layer gives each output pixel the style of its own region (unfold x, scale the
patch of pixel p by s[label[p]], one DGEMM with the weight, scale by d[label[p]]; masked up-sampling layers with one
effective 3x3 kernel per output parity, derived as float64 impulse responses of conv_transpose2d(stride 2) + blur), an
unmasked one is F.conv2d / conv_transpose2d + blur on x * s_b.  Its ToRGBs are f64ref.to_rgb.  tests/test_f64ref.py pins
those and the chain to the CPU oracle.  The chain runs here under torch.no_grad().

The masked up-sampling entry decides on the device, per sample, between the gathered transposed-convolution GEMM (at most
`cap` (pixel, region) rows) and the folded parity kernel (more).  A vectorised host row counter, pinned to the restated
row list f64ref.row_list, builds label maps with exactly cap and cap + 1 rows to test that boundary.
"""
import functools
import time
import zlib
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

import f64ref as F64
from f64ref import SQRT2, RefChain, layer_table, row_list

DEV = "cuda:0"
RES, NCLS, B = 1024, 12, 16                       # bench.py defaults: --size 1024 --ncls 12 --batch 16
CODE_SEED, LABEL_SEED = 100, 200                  # bench.run_ours at rank 0
LAYERS = layer_table()

# Bars, in max-rel (per face, against that face's maximum) and rel-RMS; both must hold for every face.  The largest error
# observed on an H100 80GB HBM3 (400 W power limit) is in the comment; each bar sits 2-3x above it.
TOL_CONV = 6e-5       # StyledConv output on the split-bf16 tensor-core kernels: 2.3e-5 (conv1; row-cap batches 2.0e-5)
TOL_RGB = 2e-6        # ToRGB, exact fp32 with the fused skip up-sampling: 7.6e-7 (rgb1024)
TOL_STYLE = 2.5e-6    # modulation s and demodulation dm, exact fp32 products of 512 terms: 1.0e-6
TOL_IMAGE = 3e-4      # the 1024 image after 26 layers: 1.4e-4 (face maps), 9.9e-5 (iid maps)
# A face alone against the same face inside the 16-face batch: 6.6e-5.  The N-tile width of the tensor-core kernels is
# picked from the work-item count, so one face and sixteen can run a layer on different tiles and sum in another order.
TOL_BATCH = 1.5e-4
# Graph replay and the pipeline's host images against the eager forward on the same inputs: bit-identical (0) so far;
# the bar leaves room for a kernel that reorders its sums between launches.
TOL_GRAPH = 1e-5


# ============================================================================ host-only: the gathered path's row count
def row_counts(label, ncls):
    """Rows of each sample's gathered list: T' pixel (m, n) needs every region of the clipped output window
    [2m - 2, 2m + 2] x [2n - 2, 2n + 2].  One-hot, a 5 x 5 window OR at stride 2, then the popcount summed.
    label [B, 2h, 2w] -> int64 [B]."""
    oh = F64.onehot(F64.region_of(label, ncls), ncls, torch.float32)
    win = F.max_pool2d(F.pad(oh, (2, 3, 2, 3)), 5, stride=2)     # [B, ncls, h + 1, w + 1]
    return win.sum((1, 2, 3)).long()


def _resize(labels, side):
    return F.interpolate(labels[:, None].float(), size=(side, side), mode="nearest")[:, 0].to(torch.uint8)


@functools.lru_cache(maxsize=None)
def _bench_labels(kind):
    import bench
    return bench.face_label_maps(B, NCLS, kind, seed=LABEL_SEED)[:, 0]


def _gathered_layers():
    return [r for r in LAYERS if r.kind == "conv" and r.up and r.masked and 2 * r.side >= 16]


def test_row_counter_matches_row_list():
    """row_counts against f64ref.row_list on face, iid and single-region maps of odd and even sizes."""
    g = torch.Generator().manual_seed(3)
    faces = _resize(_bench_labels("faces")[:4], 32)
    for h, w, kind, ncls in [(16, 16, "face", 12), (5, 7, "iid", 12), (6, 3, "iid", 5), (4, 4, "one", 3), (3, 5, "iid", 32)]:
        if kind == "face":
            lab = faces
        elif kind == "iid":
            lab = torch.randint(0, ncls, (3, 2 * h, 2 * w), generator=g, dtype=torch.uint8)
        else:
            lab = torch.full((2, 2 * h, 2 * w), 2, dtype=torch.uint8)
        want = [len(row_list(l, ncls, h, w)[2]) for l in lab]
        assert row_counts(lab, ncls).tolist() == want, (kind, h, w)


def test_bench_face_masks_take_the_gathered_path():
    """Every one of the benchmark's 16 face maps fits the row cap at every masked up-sampling layer from 16 to 256, so the
    headline figure runs them all on the gathered transposed convolution; iid maps overflow it at every one of them."""
    from e4s_b200.kernels import convt_masked_cap
    layers = _gathered_layers()
    assert [r.name for r in layers] == ["up16", "up32", "up64", "up128", "up256"]
    for r in layers:
        cap = convt_masked_cap(r.side, r.side)
        faces = row_counts(_resize(_bench_labels("faces"), 2 * r.side), NCLS)
        iid = row_counts(_resize(_bench_labels("iid"), 2 * r.side), NCLS)
        print(f"{r.name}: cap {cap}, face rows {faces.min()}..{faces.max()}, iid rows {iid.min()}..{iid.max()}")
        assert int(faces.max()) <= cap, (r.name, faces.tolist(), cap)
        assert int(iid.min()) > cap, (r.name, iid.tolist(), cap)


def map_with_rows(face, target, ncls, seed):
    """A label map of face's shape whose gathered list has exactly `target` rows: the first p pixels in raster order are
    replaced by iid labels (the largest p that stays at or below the target, by bisection), then single pixels below them
    are relabelled until the count is exact."""
    g = torch.Generator().manual_seed(seed)
    iid = torch.randint(0, ncls, face.shape, generator=g, dtype=torch.uint8)
    count = lambda lab: int(row_counts(lab[None], ncls)[0])

    def with_prefix(p):
        out = face.clone().reshape(-1)
        out[:p] = iid.reshape(-1)[:p]
        return out.view_as(face)

    lo, hi = 0, face.numel()
    assert count(with_prefix(lo)) <= target < count(with_prefix(hi))
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if count(with_prefix(mid)) <= target else (lo, mid)
    lab, (ho, wo) = with_prefix(lo), face.shape
    c = count(lab)
    for _ in range(500):
        if c == target:
            break
        best = None
        for t in range(32):
            y = int(torch.randint(lo // wo + 1, ho, (1,), generator=g))
            x = int(torch.randint(0, wo, (1,), generator=g))
            r = int(lab[y, min(x + 1, wo - 1)]) if t % 2 else int(torch.randint(0, ncls, (1,), generator=g))
            trial = lab.clone()
            trial[y, x] = r
            ct = count(trial)
            if c < ct <= target and (best is None or ct > best[0]):
                best = (ct, trial)
        if best is not None:
            c, lab = best
    assert c == target, (c, target)
    return lab


@functools.lru_cache(maxsize=None)
def _boundary_batch(name, order):
    from e4s_b200.kernels import convt_masked_cap
    side = next(r.side for r in LAYERS if r.name == name)
    cap = convt_masked_cap(side, side)
    first, last = (cap, cap + 1) if order == "cap_first" else (cap + 1, cap)
    lab = _resize(_bench_labels("faces"), 2 * side)
    lab[0] = map_with_rows(lab[0], first, NCLS, seed=1)
    lab[15] = map_with_rows(lab[15], last, NCLS, seed=2)
    lab[7] = _resize(_bench_labels("iid")[7:8], 2 * side)[0]
    return lab, cap


def boundary_batch(name, order):
    """16 label maps at the output side of layer `name`: with order cap_first, sample 0 has exactly cap rows and sample 15
    cap + 1; overflow_first swaps the two.  Sample 7 is iid, the others are the bench face maps."""
    lab, cap = _boundary_batch(name, order)
    return lab.clone(), cap


BOUNDARY_LAYERS = ["up32", "up256"]
BOUNDARY_ORDERS = ["cap_first", "overflow_first"]


def _boundary_counts(cap, order):
    want = [None] * B
    want[0], want[15] = (cap, cap + 1) if order == "cap_first" else (cap + 1, cap)
    return want


@pytest.mark.parametrize("order", BOUNDARY_ORDERS)
@pytest.mark.parametrize("name", BOUNDARY_LAYERS)
def test_boundary_batch_row_counts(name, order):
    lab, cap = boundary_batch(name, order)
    counts = row_counts(lab, NCLS).tolist()
    want = _boundary_counts(cap, order)
    assert counts[0] == want[0] and counts[15] == want[15] and counts[7] > cap, counts
    assert all(counts[i] <= cap for i in range(1, 15) if i != 7), counts


# ============================================================================ GPU checks
LEDGER = F64.Ledger(32)


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


_PEAKS = []


@pytest.fixture(autouse=True)
def _release_cached_memory(request):
    """Hand the allocator's cached blocks back after every test (the shapes change from layer to layer, and the GPU is
    shared), and record each test's peak device memory."""
    if torch.cuda.is_available():
        torch.cuda.reset_peak_memory_stats()
    yield
    if torch.cuda.is_available():
        _PEAKS.append((torch.cuda.max_memory_reserved(), torch.cuda.max_memory_allocated(), request.node.name))
        torch.cuda.empty_cache()


def _to_pm32(x64):
    """float64 NCHW -> fp32 pixel-major storage, returned as its NCHW view (what the modules pass between layers)."""
    b, c, h, w = x64.shape
    y = torch.empty((b, h, w, c), device=x64.device, dtype=torch.float32)
    y.copy_(x64.permute(0, 2, 3, 1))
    return y.permute(0, 3, 1, 2)


def _renoise(y64, nw, n_from, n_to):
    """act(pre + nw n_to) from y64 = act(pre + nw n_from): the leaky ReLU is inverted exactly in float64."""
    nw = nw.double()
    pre = y64 / torch.where(y64 > 0, y64.new_tensor(SQRT2), y64.new_tensor(0.2 * SQRT2))
    return F64.act(pre - nw * n_from.double() + nw * n_to.double())


ENTRIES = {"e4s_modconv3x3_up_masked_tcr_fwd": "gathered", "e4s_modconv3x3_up_tcr_fwd": "convt",
           "e4s_modconv3x3_fwd_f32": "simt", "e4s_torgb_fwd_f32": "torgb"}


def _spy(monkeypatch):
    """Record the forward entry of every modulated-convolution launch: rs (register-operand), folded (four parity kernels),
    gathered (masked transposed convolution), convt (unmasked transposed convolution), simt, torgb."""
    from e4s_b200 import kernels as K
    taken, call = [], K._call

    def spy(name, fn, *args, **kw):
        if name == "e4s_modconv3x3_tcr_fwd":
            taken.append("folded" if args[15] else "rs")
        elif name in ENTRIES:
            taken.append(ENTRIES[name])
        return call(name, fn, *args, **kw)
    monkeypatch.setattr(K, "_call", spy)
    return taken


def _expected_entry(r):
    if r.kind == "rgb":
        return "torgb"
    if not r.up:
        return "rs"
    if not r.masked:
        return "convt"
    return "gathered" if 2 * r.side >= 16 else "folded"


@pytest.fixture(scope="module")
def bench_setup():
    """The benchmark's network, codes, label maps (faces and iid), one-hot masks, label pyramids, per-sample noise, the
    styles of Generator._layer_styles and a float64 RefChain per label kind."""
    import bench
    from e4s_b200 import kernels as K
    from e4s_b200.stylegan2.modconv import LabelPyramid
    net = bench.build_net(RES, NCLS, torch.device(DEV))
    G = net.G
    codes = torch.randn(B, NCLS, 18, 512, generator=torch.Generator().manual_seed(CODE_SEED)).to(DEV)
    labels = {k: bench.face_label_maps(B, NCLS, k, seed=LABEL_SEED).to(DEV) for k in ("faces", "iid")}
    gn = torch.Generator().manual_seed(300)
    sides = [4] + [2 ** (i // 2 + 3) for i in range(2 * (G.log_size - 2))]
    noise = [torch.randn(B, 1, s, s, generator=gn).to(DEV) for s in sides]
    names = {id(m): n for n, m in G.named_modules()}
    sched = G._schedule()
    assert [names[id(m)] for m, _, _ in sched] == [r.module for r in LAYERS]
    with torch.no_grad():
        styles = G._layer_styles(codes, sched)
    return SimpleNamespace(
        net=net, G=G, codes=codes, labels=labels, noise=noise, sched=sched, styles=styles,
        onehot={k: K.label_to_onehot(v, NCLS) for k, v in labels.items()},
        pyramids={k: LabelPyramid(v[:, 0], NCLS) for k, v in labels.items()},
        chains={k: RefChain(G, codes, v[:, 0], noise) for k, v in labels.items()})


@pytest.mark.gpu
def test_style_stage_at_bench_batch(bench_setup, monkeypatch):
    """Generator._layer_styles at B = 16: every modulation in one linear_multi launch, every demodulation in a second, and
    each PrecomputedStyle (s, dm) against float64 - the per-region layers (latent[:, :, i]) and the global ones
    (latent[:, 0, i], rows ncls * n_latent * 512 floats apart)."""
    from e4s_b200 import kernels as K
    from e4s_b200.stylegan2.modconv import PrecomputedStyle
    bs = bench_setup
    launches, call = [], K._call
    monkeypatch.setattr(K, "_call", lambda name, *a, **kw: (launches.append(name), call(name, *a, **kw))[1])
    with torch.no_grad():
        styles = bs.G._layer_styles(bs.codes, bs.sched)
    assert launches == ["e4s_linear_multi_f32"] * 2, launches
    chain = bs.chains["faces"]
    kinds = set()
    for i, r in enumerate(LAYERS):
        st = styles[i]
        assert isinstance(st, PrecomputedStyle)
        with torch.no_grad():
            s64, d64 = chain.style(i)
        kinds.add(bs.sched[i][2])
        _check(st.s, s64, TOL_STYLE, "s (modulation)", r.name)
        if r.kind == "conv":
            _check(st.dm, d64, TOL_STYLE, "dm (demodulation)", r.name)
        else:
            assert st.dm is None
    assert kinds == {True, False}


def _run_layer(bs, kind, i, monkeypatch):
    """Layer i through its module's forward on the fp32 cast of the float64 state of chain `kind`; checks the entry it
    took and its output against the float64 layer, then (StyledConv) repeats it with the registered noise buffer."""
    r = LAYERS[i]
    m = bs.sched[i][0]
    chain = bs.chains[kind]
    with torch.no_grad():
        x64, skip64 = chain.seek(i)
    x_in = _to_pm32(x64)
    skip_in = None if skip64 is None else skip64.float()
    taken = _spy(monkeypatch)
    case = f"{r.name} {kind} B={B}"
    with torch.no_grad():
        if r.kind == "conv":
            k = chain.noise_index[i]
            ours = m(x_in, bs.styles[i], bs.pyramids[kind], noise=bs.noise[k])
        else:
            ours = m(x_in, bs.styles[i], bs.pyramids[kind], skip=skip_in)
    assert taken == [_expected_entry(r)], (r.name, taken)
    del x64, skip64
    with torch.no_grad():
        ref = chain.step()
    if r.kind == "rgb":
        _check(ours, ref, TOL_RGB, "rgb", case)
        return
    _check(ours, ref, TOL_CONV, "y", case)
    del ours
    buf = getattr(bs.G.noises, f"noise_{k}")                  # [1, 1, Ho, Wo]: randomize_noise=False and the graph use it
    with torch.no_grad():
        ours = m(x_in, bs.styles[i], bs.pyramids[kind], noise=buf)
    _check(ours, lambda sl: _renoise(ref[sl], m.noise.weight, bs.noise[k][sl], buf), TOL_CONV, "y (broadcast noise)", case)


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(LAYERS)), ids=[r.name for r in LAYERS])
def test_layer_at_bench_batch(i, bench_setup, monkeypatch):
    """Every StyledConv (17) and ToRGB (9) of the 1024 generator at B = 16 on the bench face maps, all 16 faces."""
    _run_layer(bench_setup, "faces", i, monkeypatch)


IID_LAYERS = [i for i, r in enumerate(LAYERS) if r.name in ("up16", "up32", "up64", "up128", "up256", "c256")]


@pytest.mark.gpu
@pytest.mark.parametrize("i", IID_LAYERS, ids=[LAYERS[i].name for i in IID_LAYERS])
def test_iid_layer_at_bench_batch(i, bench_setup, monkeypatch):
    """bench.py --mask iid: every sample of every gathered masked up-sampling layer overflows the row cap and runs on the
    folded kernel inside the gathered entry; c256 on the rs kernel with every region in every tile."""
    from e4s_b200.kernels import convt_masked_cap
    r = LAYERS[i]
    if r.up:
        lab = bench_setup.pyramids["iid"].at(2 * r.side, 2 * r.side).cpu()
        assert int(row_counts(lab, NCLS).min()) > convt_masked_cap(r.side, r.side)
    _run_layer(bench_setup, "iid", i, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("order", BOUNDARY_ORDERS)
@pytest.mark.parametrize("name", BOUNDARY_LAYERS)
def test_row_cap_boundary(name, order, bench_setup):
    """e4s_modconv3x3_up_masked_tcr_fwd on a batch with exactly cap rows (gathered) and cap + 1 rows (folded) at samples 0
    and 15, in both orders, an iid sample 7 (folded) and face maps: the device count matches the host count and all 16
    outputs match float64.  The output starts as NaN, so a sample that neither path writes fails.  The folded kernel runs
    after the blur pass and overwrites what the blur wrote for its samples, so a count check that consults the wrong sample
    shows only when that sample's decision differs in the direction that skips a gathered sample: the two orders cover
    sample 0 and sample 15 either way."""
    from e4s_b200 import _lib
    from e4s_b200._lib import ptr, stream_ptr
    r = next(r for r in LAYERS if r.name == name)
    m = bench_setup.G.get_submodule(r.module)
    h, cin, cout = r.side, r.cin, r.cout
    label, cap = boundary_batch(name, order)
    host = row_counts(label, NCLS)
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    x = torch.randn(B, h, h, cin, generator=g).to(DEV)
    s = (1.0 + 0.3 * torch.randn(B, NCLS, cin, generator=g)).to(DEV)
    dm = F64.demod(s, m.conv.weight[0]).float()
    noise = torch.randn(B, 1, 2 * h, 2 * h, generator=g).to(DEV)
    label = label.to(DEV)
    prep = m.conv.prepared()
    nw, bias = m.noise.weight, m.activate.bias
    i32 = dict(device=DEV, dtype=torch.int32)
    # zeroed lists and one spare sample of rows past the end: a wrong count check in the blur pass then reads stale rows of
    # this buffer, and the test fails instead of the kernel reading past its allocation
    need, base = torch.zeros((B, h + 1, h + 1), **i32), torch.zeros((B, h + 1, h + 1), **i32)
    count, rows = torch.full((B,), -1, **i32), torch.zeros((B, cap), **i32)
    t = torch.zeros((B + 1, cap, 4 * cout), device=DEV)
    y = torch.full((B, 2 * h, 2 * h, cout), float("nan"), device=DEV)
    rc = _lib.load().e4s_modconv3x3_up_masked_tcr_fwd(
        ptr(x), ptr(prep.w_convt_hilo), ptr(prep.w_hilo), ptr(prep.fir), ptr(s), ptr(dm), ptr(label), ptr(noise), ptr(nw),
        ptr(bias), ptr(need), ptr(base), ptr(count), ptr(rows), ptr(t), ptr(y), B, h, h, cin, cout, NCLS, cap, B, 1,
        stream_ptr())
    _lib.check(rc, "e4s_modconv3x3_up_masked_tcr_fwd")
    torch.cuda.synchronize()
    dev_count = count.cpu()
    want = _boundary_counts(cap, order)
    assert int(host[0]) == want[0] and int(host[15]) == want[15], host.tolist()
    assert all(int(dev_count[i]) == int(host[i]) for i in range(B) if i != 7), (dev_count.tolist(), host.tolist())
    assert cap < int(dev_count[7]) <= int(host[7])      # an overflowing list stops counting after the chunk that passes cap
    ref = F64.styled_conv_per_pixel(x.permute(0, 3, 1, 2), s, m.conv.weight[0], label, noise, nw, bias, True)
    _check(y.permute(0, 3, 1, 2), ref, TOL_CONV, "y (row-cap boundary)", f"{name} {order} cap {cap}")


def _gen(net, codes, mask, **kw):
    """gen_img's image; the allocator's cached blocks are handed back after it (the forward's activations are several GB,
    and a GraphedSynthesis built next allocates its own pool)."""
    with torch.no_grad():
        img = net.gen_img(None, codes, mask, **kw)[0]
    torch.cuda.empty_cache()
    return img


@pytest.mark.gpu
def test_generator_at_bench_batch(bench_setup):
    """Eager gen_img at B = 16 with explicit per-sample noise against the float64 chain, all 16 faces; then every face
    alone against the same face inside the batch."""
    bs = bench_setup
    with torch.no_grad():
        ref = bs.chains["faces"].image()
    torch.cuda.empty_cache()
    img = _gen(bs.net, bs.codes, bs.onehot["faces"], noise=bs.noise)
    _check(img, ref, TOL_IMAGE, "image", f"faces B={B}")
    for f in range(B):
        one = _gen(bs.net, bs.codes[f:f + 1], bs.onehot["faces"][f:f + 1], noise=[n[f:f + 1] for n in bs.noise])
        _check(one, img[f:f + 1], TOL_BATCH, "face alone vs in the batch", f"face {f}")


@pytest.mark.gpu
def test_graphed_synthesis_and_pipeline_match_eager(bench_setup, monkeypatch):
    """GraphedSynthesis(randomize_noise=False) on uint8 labels equals eager gen_img(randomize_noise=False) on the one-hot
    mask; so do the host images of SynthesisPipeline(cuda_graph=True) for two batches in flight."""
    from e4s_b200 import pipeline as PL
    bs = bench_setup
    labels, onehot = bs.labels["faces"], bs.onehot["faces"]
    eager = _gen(bs.net, bs.codes, onehot, randomize_noise=False)
    synth = PL.GraphedSynthesis(bs.net, NCLS, bs.codes.shape, labels.shape, randomize_noise=False)
    _check(synth(bs.codes, labels), eager, TOL_GRAPH, "graph replay vs eager", f"faces B={B}")
    del synth
    torch.cuda.empty_cache()
    codes2 = bs.codes.flip(0).contiguous()
    eager2 = _gen(bs.net, codes2, onehot, randomize_noise=False)
    monkeypatch.setattr(PL, "GraphedSynthesis", functools.partial(PL.GraphedSynthesis, randomize_noise=False))
    pipe = PL.SynthesisPipeline(bs.net, NCLS, depth=2, cuda_graph=True)
    labels_host = labels.cpu().pin_memory()
    tickets = [pipe.submit(c.cpu().pin_memory(), labels_host) for c in (bs.codes, codes2)]
    for tk, ref in zip(tickets, (eager, eager2)):
        out = pipe.result(tk)
        assert not out.is_cuda
        _check(out, ref, TOL_GRAPH, "pipeline host image vs eager", f"faces B={B} ticket {tk}")
    pipe.drain()
    torch.cuda.synchronize()


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.mark.gpu
def test_random_noise_is_drawn_per_face(bench_setup):
    """Faces 3 and 11 get the same codes and label map: with randomize_noise=True (eager and the graph) they differ, as
    the reference draws noise per sample (model.py:333); with the registered buffers they agree."""
    from e4s_b200.pipeline import GraphedSynthesis
    bs = bench_setup
    labels, onehot = bs.labels["faces"], bs.onehot["faces"]
    assert torch.equal(labels[3], labels[11])
    codes = bs.codes.clone()
    codes[11] = codes[3]
    fixed = _gen(bs.net, codes, onehot, randomize_noise=False)
    _check(fixed[11:12], fixed[3:4], TOL_BATCH, "same face, same noise buffer", "faces 3 / 11")
    fresh = _gen(bs.net, codes, onehot, randomize_noise=True)
    assert _rel(fresh[11], fresh[3]) > 1e-3, _rel(fresh[11], fresh[3])
    synth = GraphedSynthesis(bs.net, NCLS, codes.shape, labels.shape)
    a = synth(codes, labels).clone()
    b = synth(codes, labels).clone()
    print(f"fresh noise: eager faces 3 / 11 differ by {_rel(fresh[11], fresh[3]):.2e}, graph {_rel(a[11], a[3]):.2e}, "
          f"two replays {_rel(a, b):.2e}")
    assert _rel(a[11], a[3]) > 1e-3 and _rel(a, b) > 1e-3


@pytest.mark.gpu
def test_generator_iid_masks_at_bench_batch(bench_setup):
    """bench.py --mask iid: eager gen_img at B = 16 against the float64 chain on the iid maps, all 16 faces."""
    bs = bench_setup
    with torch.no_grad():
        ref = bs.chains["iid"].image()
    torch.cuda.empty_cache()
    img = _gen(bs.net, bs.codes, bs.onehot["iid"], noise=bs.noise)
    _check(img, ref, TOL_IMAGE, "image (iid masks)", f"iid B={B}")
