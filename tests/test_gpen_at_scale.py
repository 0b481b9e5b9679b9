"""GPEN-BFR-512's FullGenerator at the benchmark's 16-face batch: every encoder layer, the heads and every StyledConv and
ToRGB of the generator at B = 1 and B = 16, against a float64 reference that shares no code with e4s_b200.

GPEN drives the shared kernels at shapes the E4S generator never produces: 1024 input channels (the concatenated encoder
maps) in the register-operand forward, the transposed-convolution GEMM, the warp-per-pixel ToRGB and the K-split
modulation / demodulation products; the encoder's blur with pad (3, 2) and the stride-2 tensor-core convolution on sides
that are not multiples of the tile (514 ... 6); the 3 -> 32 zero-padded 1x1 input convolution; the concatenated "noise"
half with its own bias; the 8192-deep final linear and the mapping MLP.  A one-image end-to-end comparison at 1e-3 dilutes
a defect in any of them, so each layer here takes the float64 activation of the layer before it, cast to fp32, and the
kernels behind it are then called directly at the same shapes.

The reference covers all 16 faces for outputs up to 128 x 128 and faces SUB above that (the network is per-face, so a
slice of the batch is exact); the encoder's maps are computed for all 16 faces, as every later layer of the batch reads
them.  Where a B = 16 run needs an input the reference holds for SUB only, the other faces carry mirrored copies of those
three, so the kernels still run the whole batch on distinct data.  Layer shapes come from the module tree (layer_table),
which the host-only tests pin to oracle/gpen_oracle.param_shapes; the reference itself is pinned to the oracle there too.
"""
import functools
import math
import time
import types
import zlib
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F

import f64ref as F64
from oracle import e4s_oracle as O
from oracle import gpen_oracle as GO
from conftest import assert_close
from f64ref import nchw, pm

DEV = "cuda:0"
SIZE, STYLE_DIM, N_MLP = 512, 512, 8
B_FULL = 16                     # bench.py --gpen-batch default
SUB = [0, 7, 15]                # faces the reference covers above FULL_UPTO
FULL_UPTO = 128                 # largest output side the reference computes for all 16 faces
ONE = 7                         # the face the B = 1 cases run alone

# Bars, in conftest.assert_close's norms (max-rel and rel-RMS, both must hold).  The largest error observed on an H100
# 80GB HBM3 (700 W power limit) is in the comment; each bar sits 2-3x above it.
# StyledConv conv half and the modulated-convolution kernels: 5.1e-5 (convs.1, Cin 1024, B = 16).  The 64-channel N tile
# sums x_lo w_hi, x_hi w_lo and x_hi w_hi in one fp32 accumulator and measured 4.7e-5 on the layer where the 32-channel
# tile, which keeps the three in separate accumulators, measured 1.8e-5.
TOL_CONV = 1e-4
TOL_ENC = 5e-5                  # the encoder's tensor-core convolution (ConvLayer, conv3x3_tc): 2.4e-5
# exact-fp32 kernels: final_linear 3.3e-7, upfirdn2d 2.2e-7, ToRGB 2.1e-7, demod 1.8e-7, the noise half 1.2e-7,
# bias_act 9.7e-8, linear 4.9e-8
TOL_F32 = 1e-6
TOL_SIMT = 1.5e-5               # the SIMT modulated convolution (exact fp32, 9216-term sums at Cin 1024): 6.1e-6
TOL_IMAGE = 1e-4                # the image against float64 4.3e-5; the default path against the SIMT path 1.8e-5
TOL_IMAGE_SIMT = 2e-5           # the image on the SIMT path against float64: 6.1e-6
# A face alone against the same face inside the 16-face batch: 2.6e-5.  The N-tile width is picked from the work-item
# count, so one face and sixteen can run a layer on different tile widths (see TOL_CONV).
TOL_BATCH = 5e-5


# ============================================================================ float64 reference (plain torch ops)
def ref_ecd(p, n, x):
    """Encoder layer ecd{n}: a 1x1 conv (n = 0) or blur pad (2, 2) -> 3x3 stride-2 conv without padding, then
    FusedLeakyReLU.  Equalised learning rate: the weight is scaled by 1 / sqrt(fan_in)."""
    if n == 0:
        w, bias = p["ecd0.0.0.weight"], p["ecd0.0.1.bias"]
        y = F.conv2d(x, w / math.sqrt(w.shape[1]))
    else:
        w, bias = p[f"ecd{n}.0.1.weight"], p[f"ecd{n}.0.2.bias"]
        y = F.conv2d(O.upfirdn2d(x, p[f"ecd{n}.0.0.kernel"], pad=(2, 2)), w / math.sqrt(9 * w.shape[1]), stride=2)
    return F64.act(y + bias[None, :, None, None])


def ref_final_linear(p, flat):
    """final_linear: EqualLinear(8192, 512) with FusedLeakyReLU on the channel-major flatten of the 4 x 4 map."""
    return F64.act(F64.equal_linear(flat, p["final_linear.0.weight"], p["final_linear.0.bias"]))


def ref_pixel_norm(z):
    return z * torch.rsqrt(z.pow(2).mean(dim=1, keepdim=True) + 1e-8)


def ref_mapping_layer(p, i, h):
    """generator.style.{i}: EqualLinear(512, 512, lr_mul 0.01) with FusedLeakyReLU."""
    return F64.act(F64.equal_linear(h, p[f"generator.style.{i}.weight"], p[f"generator.style.{i}.bias"], lr_mul=0.01))


def ref_modulation(p, prefix, style):
    """ModulatedConv2d.modulation: EqualLinear(512, Cin) (lr_mul 1) of the latent, [B, Cin]."""
    return F64.equal_linear(style, p[prefix + ".conv.modulation.weight"], p[prefix + ".conv.modulation.bias"])


def ref_styled(p, prefix, x, style, noise, up):
    """StyledConv with the concatenated noise: cat(f64ref.styled_preact of one region, noise_w * noise) ->
    FusedLeakyReLU over 2 Cout."""
    s = ref_modulation(p, prefix, style)[:, None]
    t = F64.styled_preact(x, s, p[prefix + ".conv.weight"][0], None, None, None, None, up, True)
    t = torch.cat((t, p[prefix + ".noise.weight"] * noise), 1)
    return F64.act(t + p[prefix + ".activate.bias"][None, :, None, None])


def ref_rgb(p, prefix, x, style, skip):
    """ToRGB: f64ref.to_rgb of one region."""
    s = ref_modulation(p, prefix, style)[:, None]
    return F64.to_rgb(x, s, p[prefix + ".conv.weight"], None, p[prefix + ".bias"], skip)


def ref_chain(p, img, size, full_upto=None, keep=None):
    """Every activation of FullGenerator.forward in img's dtype, chained: ({layer name: output}, {layer name: faces it
    covers}).  Names: ecd0 ..., final_linear, style (the mapping's output), the generator's conv1, to_rgb1, convs.i,
    to_rgbs.j and image.  Generator layers whose output side exceeds full_upto run on the faces `keep` only."""
    acts, faces = {}, {}
    everyone = list(range(img.shape[0]))

    def put(name, t, f):
        acts[name], faces[name] = t, f

    log_size = int(math.log2(size))
    feats, h = [], img
    for n in range(log_size - 1):
        h = ref_ecd(p, n, h)
        put(f"ecd{n}", h, everyone)
        feats.append(h)
    z = ref_final_linear(p, h.reshape(h.shape[0], -1))
    put("final_linear", z, everyone)
    w = ref_pixel_norm(z)
    for i in range(1, N_MLP + 1):
        w = ref_mapping_layer(p, i, w)
    put("style", w, everyone)

    cur = everyone
    out = p["generator.input.input"].repeat(img.shape[0], 1, 1, 1)
    out = ref_styled(p, "generator.conv1", out, w, feats[-1], False)
    put("conv1", out, cur)
    skip = ref_rgb(p, "generator.to_rgb1", out, w, None)
    put("to_rgb1", skip, cur)
    for j in range(log_size - 2):
        if full_upto is not None and 2 ** (j + 3) > full_upto and cur is everyone:
            out, skip, w, cur = out[keep], skip[keep], w[keep], keep
        noise = feats[log_size - 3 - j]
        noise = noise if cur is everyone else noise[cur]
        out = ref_styled(p, f"generator.convs.{2 * j}", out, w, noise, True)
        put(f"convs.{2 * j}", out, cur)
        out = ref_styled(p, f"generator.convs.{2 * j + 1}", out, w, noise, False)
        put(f"convs.{2 * j + 1}", out, cur)
        skip = ref_rgb(p, f"generator.to_rgbs.{j}", out, w, skip)
        put(f"to_rgbs.{j}", skip, cur)
    put("image", skip, cur)
    return acts, faces


# ============================================================================ the layer table of FullGenerator(512)
Layer = namedtuple("Layer", "name kind cin cout side resample")     # side: input side; resample: down | up | ""


def out_side(r):
    if r.kind == "conv" and r.resample == "up":
        return 2 * r.side
    return r.side // 2 if r.resample == "down" else r.side


@functools.lru_cache(maxsize=None)
def layer_table(size=SIZE):
    """Every layer of FullGenerator(size, 512, 8) in execution order, read from the module tree.  Encoder ConvLayers
    (kind ecd; down = blur + stride-2 conv), the final linear (head), StyledConvs (conv; up = up-sampling) and ToRGBs (rgb;
    up = with an up-sampled skip).  cin counts the concatenated encoder maps."""
    from e4s_b200.gpen.gpen_model import FullGenerator
    m = FullGenerator(size, STYLE_DIM, N_MLP)
    rows, side = [], size
    for name in m.names:
        layer = getattr(m, name)[0]
        conv = layer[1] if layer._downsample else layer[0]
        cout, cin = conv.weight.shape[:2]
        rows.append(Layer(name, "ecd", cin, cout, side, "down" if layer._downsample else ""))
        side = out_side(rows[-1])
    fl = m.final_linear[0]
    rows.append(Layer("final_linear", "head", fl.weight.shape[1], fl.weight.shape[0], side, ""))
    G = m.generator

    def styled(name, mod, side):
        return Layer(name, "conv", mod.conv.in_channel, mod.conv.out_channel, side, "up" if mod.conv.upsample else "")

    def rgb(name, mod, side):
        return Layer(name, "rgb", mod.conv.in_channel, mod.conv.out_channel, side, "up" if hasattr(mod, "upsample") else "")

    rows += [styled("conv1", G.conv1, 4), rgb("to_rgb1", G.to_rgb1, 4)]
    side = 4
    for j, to_rgb in enumerate(G.to_rgbs):
        rows.append(styled(f"convs.{2 * j}", G.convs[2 * j], side))
        side = out_side(rows[-1])
        rows.append(styled(f"convs.{2 * j + 1}", G.convs[2 * j + 1], side))
        rows.append(rgb(f"to_rgbs.{j}", to_rgb, side))
    return tuple(rows)


@functools.lru_cache(maxsize=None)
def wiring(size=SIZE):
    """{layer: (input activation, skip or noise map)} in the names of ref_chain: a StyledConv reads the previous StyledConv
    (None: the constant input) and the encoder map of its output side; a ToRGB reads the StyledConv before it and the
    previous ToRGB's image."""
    rows = layer_table(size)
    ecd_at = {out_side(r): r.name for r in rows if r.kind == "ecd"}
    wires, last_conv, last_rgb = {}, None, None
    for r in rows:
        if r.kind == "conv":
            wires[r.name] = (last_conv, ecd_at[out_side(r)])
            last_conv = r.name
        elif r.kind == "rgb":
            wires[r.name] = (last_conv, last_rgb)
            last_rgb = r.name
    return wires


def test_layer_table_matches_param_shapes():
    """The table read from the module tree equals the one oracle/gpen_oracle.param_shapes(512) implies (itself asserted
    equal to the reference model's state_dict by make_golden_gpen.py): names, order, channels with the concatenation,
    input sides, and which layers down- or up-sample."""
    ps = GO.param_shapes(SIZE)
    log_size = int(math.log2(SIZE))
    want = []
    for n in range(log_size - 1):
        if n == 0:
            cout, cin, k, _ = ps["ecd0.0.0.weight"]
            assert k == 1 and "ecd0.0.0.kernel" not in ps
            want.append(Layer("ecd0", "ecd", cin, cout, SIZE, ""))
        else:
            cout, cin, k, _ = ps[f"ecd{n}.0.1.weight"]
            assert k == 3 and ps[f"ecd{n}.0.0.kernel"] == (4, 4)
            want.append(Layer(f"ecd{n}", "ecd", cin, cout, SIZE >> (n - 1), "down"))
    out_dim, in_dim = ps["final_linear.0.weight"]
    want.append(Layer("final_linear", "head", in_dim, out_dim, 4, ""))

    def styled(name, side):
        _, cout, cin, k, _ = ps[f"generator.{name}.conv.weight"]
        assert k == 3 and ps[f"generator.{name}.activate.bias"] == (2 * cout,)
        return Layer(name, "conv", cin, cout, side, "up" if f"generator.{name}.conv.blur.kernel" in ps else "")

    def rgb(name, side):
        _, cout, cin, _, _ = ps[f"generator.{name}.conv.weight"]
        return Layer(name, "rgb", cin, cout, side, "up" if f"generator.{name}.upsample.kernel" in ps else "")

    want += [styled("conv1", 4), rgb("to_rgb1", 4)]
    for j in range(log_size - 2):
        want += [styled(f"convs.{2 * j}", 2 ** (j + 2)), styled(f"convs.{2 * j + 1}", 2 ** (j + 3)),
                 rgb(f"to_rgbs.{j}", 2 ** (j + 3))]
    assert layer_table() == tuple(want)

    def module_of(key):
        parts = key.split(".")
        if parts[0] != "generator":
            return parts[0]
        return ".".join(parts[1:3]) if parts[1] in ("convs", "to_rgbs") else parts[1]

    # every module of the state dict is one row, the mapping MLP and the constant input aside
    assert {module_of(k) for k in ps} - {"style", "input"} == {r.name for r in want}
    assert all(r.cout % 32 == 0 for r in want if r.kind in ("ecd", "conv"))


def test_reference_matches_the_oracle():
    """The restated reference against oracle/gpen_oracle.py in float64 on the CPU at size 64 with B = 2: every encoder
    map, the final linear, the mapping, every StyledConv and ToRGB from the same input, and the whole forward, <= 1e-10.
    The oracle is pinned to the unmodified reference model by tests/golden/gpen_vectors.npz."""
    size = 64
    p = {k: v.double() for k, v in GO.synthetic_state(size, salt=size).items()}
    x = torch.randn(2, 3, size, size, generator=torch.Generator().manual_seed(zlib.crc32(b"gpen64")), dtype=torch.float64)
    acts, faces = ref_chain(p, x, size)
    assert all(f == [0, 1] for f in faces.values())
    for n, f in enumerate(GO.encode(p, x, size)):
        assert_close(acts[f"ecd{n}"], f, 1e-10, f"ecd{n}")
    z = O.equal_linear(acts[f"ecd{int(math.log2(size)) - 2}"].reshape(2, -1), p["final_linear.0.weight"],
                       p["final_linear.0.bias"], activation=True)
    assert_close(acts["final_linear"], z, 1e-10, "final_linear")
    w = z * torch.rsqrt(z.pow(2).mean(dim=1, keepdim=True) + 1e-8)
    for i in range(1, N_MLP + 1):
        w = O.equal_linear(w, p[f"generator.style.{i}.weight"], p[f"generator.style.{i}.bias"], lr_mul=0.01, activation=True)
    assert_close(acts["style"], w, 1e-10, "mapping")
    wires = wiring(size)
    for r in layer_table(size):
        if r.kind not in ("conv", "rgb"):
            continue
        src, aux = wires[r.name]
        xin = p["generator.input.input"].repeat(2, 1, 1, 1) if src is None else acts[src]
        if r.kind == "conv":
            want = GO.styled_conv(p, "generator." + r.name, xin, acts["style"], acts[aux], r.resample == "up")
            got = ref_styled(p, "generator." + r.name, xin, acts["style"], acts[aux], r.resample == "up")
        else:
            sk = None if aux is None else acts[aux]
            want = GO.to_rgb(p, "generator." + r.name, xin, acts["style"], sk)
            got = ref_rgb(p, "generator." + r.name, xin, acts["style"], sk)
        assert tuple(got.shape[1:]) == ((2 * r.cout if r.kind == "conv" else 3), out_side(r), out_side(r)), r
        assert_close(got, want, 1e-10, r.name)
    assert_close(acts["image"], GO.full_generator_forward(p, x, size), 1e-10, "full_generator_forward")


# ============================================================================ GPU checks
LEDGER = F64.Ledger(36)
_check = LEDGER.check


@pytest.fixture(scope="module", autouse=True)
def _error_report():
    yield
    LEDGER.report()


@pytest.fixture(autouse=True)
def default_kernels(monkeypatch):
    """The default kernel selection; GPEN's modules are forward-only."""
    F64.clear_kernel_selection(monkeypatch)
    with torch.no_grad():
        yield


@pytest.fixture(scope="module")
def R():
    """GPEN-BFR-512 on the device with the bench's weights (GO.synthetic_state(512, salt=512)), 16 seeded 512 x 512
    inputs, and the chained float64 reference of that batch (computed once)."""
    from e4s_b200.gpen.gpen_model import FullGenerator
    st = GO.synthetic_state(SIZE, salt=SIZE)
    m = FullGenerator(SIZE, STYLE_DIM, N_MLP, channel_multiplier=2, narrow=1).eval()
    m.load_state_dict(st)
    m = m.to(DEV).requires_grad_(False)
    p = {k: v.to(DEV, torch.float64) for k, v in st.items()}
    g = torch.Generator().manual_seed(zlib.crc32(b"gpen512-b16"))
    img = torch.randn(B_FULL, 3, SIZE, SIZE, generator=g).to(DEV)
    t0 = time.perf_counter()
    acts, faces = ref_chain(p, img.double(), SIZE, full_upto=FULL_UPTO, keep=SUB)
    torch.cuda.synchronize()
    print(f"\nfloat64 reference GPEN-512, B = {B_FULL}: {time.perf_counter() - t0:.1f} s")
    return types.SimpleNamespace(m=m, p=p, img=img, acts=acts, faces=faces)


def _feed(R, name, b, planar=False):
    """Reference activation `name` cast to fp32 as the input of a b-face run, in channels_last storage like the model's
    own activations (planar: contiguous NCHW, like a ToRGB image).  At b = 16, where the reference holds faces SUB only,
    those faces sit in place and every other face is a mirrored copy of one of them."""
    t, cover = R.acts[name], R.faces[name]
    if b == 1:
        t = t[cover.index(ONE)][None]
    elif len(cover) < b:
        t = torch.stack([t[cover.index(k)] if k in cover else t[k % len(cover)].flip(-1) for k in range(b)])
    t = t.float()
    if t.ndim == 4 and not planar:
        return t.contiguous(memory_format=torch.channels_last)
    return t.contiguous()


def _want(R, name, b):
    """(rows of a b-face run that the reference covers, the reference output on those faces)."""
    t, cover = R.acts[name], R.faces[name]
    if b == 1:
        return [0], t[cover.index(ONE)][None]
    return (slice(None) if len(cover) == b else cover), t


def _sel(r, b):
    """Rows of a b-face run on which a test recomputes float64 references: SUB above FULL_UPTO at b = 16, else all."""
    return SUB if (b == B_FULL and out_side(r) > FULL_UPTO) else slice(None)


ECDS = [r for r in layer_table() if r.kind == "ecd"]
CONVS = [r for r in layer_table() if r.kind == "conv"]
RGBS = [r for r in layer_table() if r.kind == "rgb"]


# ---------------------------------------------------------------------------- encoder
@pytest.mark.gpu
@pytest.mark.parametrize("b", [1, B_FULL])
@pytest.mark.parametrize("row", ECDS, ids=[r.name for r in ECDS])
def test_encoder_layer(R, row, b):
    """ConvLayer.forward of ecd{n}, then its kernels on the same input: the blur with pad (3, 2) (upfirdn2d), the
    padded 3x3 convolution stored at the even pixels (conv3x3_tc out_stride 2) before and after the first row and column
    are cropped, and bias + leaky ReLU on the channels_last map.  ecd0: the 1x1 conv as the centre tap of a 3x3 on the
    input zero-padded 3 -> 32 channels."""
    from e4s_b200 import kernels as K
    case = f"{row.name}-b{b}"
    layer = getattr(R.m, row.name)[0]
    n = int(row.name[3:])
    x = R.img[ONE:ONE + 1] if (n == 0 and b == 1) else (R.img if n == 0 else _feed(R, f"ecd{n - 1}", b))
    rows, want = _want(R, row.name, b)
    out = layer(x)
    assert out.shape == (b, row.cout, out_side(row), out_side(row))
    _check(out[rows], want, TOL_ENC, "ConvLayer out", case)
    del out, want

    sel = _sel(row, b)
    xd = x[sel].double()
    if n == 0:
        conv, act = layer[0], layer[1]
        planes = layer._prepared(conv)
        assert planes.shape == (2, 1, 9, row.cout, 32)
        taps = torch.arange(9, device=planes.device) != 4
        assert int(torch.count_nonzero(planes[:, :, :, :, row.cin:])) == 0, "padded input channels carry weights"
        assert int(torch.count_nonzero(planes[:, :, taps])) == 0, "the 1x1 conv has weights off the centre tap"
        xp = x.new_zeros(b, SIZE, SIZE, 32)
        xp[..., :row.cin] = pm(x)
        y = K.conv3x3_tc(xp, planes)
        w0 = R.p["ecd0.0.0.weight"]
        _check(nchw(y)[sel], F.conv2d(xd, w0 / math.sqrt(row.cin)), TOL_ENC, "conv3x3_tc 1x1 (Cin 3 -> 32)", case)
        bias_key = "ecd0.0.1.bias"
    else:
        blur, conv, act = layer
        assert tuple(blur.pad) == (2, 2)
        fir = R.p[f"{row.name}.0.0.kernel"]
        z = K.upfirdn2d_raw(x.contiguous(), blur.kernel, 1, 1, 1, 1, 3, 2, 3, 2)
        assert z.shape == (b, row.cin, row.side + 2, row.side + 2)
        _check(z[sel], O.upfirdn2d(xd, fir, pad=(3, 2)), TOL_F32, "upfirdn2d pad (3, 2)", case)
        wk = R.p[f"{row.name}.0.1.weight"] / math.sqrt(9 * row.cin)
        y = K.conv3x3_tc(K.to_pixel_major(z), layer._prepared(conv), out_stride=2)
        assert y.shape == (b, row.side // 2 + 1, row.side // 2 + 1, row.cout)
        _check(nchw(y)[sel], F.conv2d(z[sel].double(), wk, stride=2, padding=1), TOL_ENC, "conv3x3_tc out_stride 2", case)
        del z
        y = y[:, 1:, 1:, :].contiguous()
        ref = F.conv2d(O.upfirdn2d(xd, fir, pad=(2, 2)), wk, stride=2)
        _check(nchw(y)[sel], ref, TOL_ENC, "conv3x3_tc out_stride 2, cropped", case)
        del ref
        bias_key = f"{row.name}.0.2.bias"
    a = K.bias_act_fwd(nchw(y), act.bias, 0.2, F64.SQRT2)
    assert pm(a).is_contiguous()                       # channels_last in and out: the pixel-major bias path
    _check(a[sel], F64.act(nchw(y)[sel].double() + R.p[bias_key][None, :, None, None]), TOL_F32, "bias_act (channels_last)", case)


# ---------------------------------------------------------------------------- heads
@pytest.mark.gpu
@pytest.mark.parametrize("b", [1, B_FULL])
def test_heads(R, b, monkeypatch):
    """final_linear (8192 deep, on the channel-major flatten of ecd7), then PixelNorm and each of the 8 mapping layers,
    each from the float64 output of the one before.  F.linear runs in plain fp32 (TF32 off)."""
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    case = f"heads-b{b}"
    last = ECDS[-1].name
    head = [r for r in layer_table() if r.kind == "head"][0]
    flat = _feed(R, last, b).contiguous().reshape(b, -1)          # channel-major, as the reference flattens
    assert flat.shape == (b, head.cin)
    rows, want = _want(R, "final_linear", b)
    z = R.m.final_linear(flat)
    _check(z[rows], want, TOL_F32, "final_linear", case)
    G = R.m.generator
    zr = want.double()
    h = ref_pixel_norm(zr)
    _check(G.style[0](zr.float()), h, TOL_F32, "PixelNorm", case)
    for i in range(1, N_MLP + 1):
        nxt = ref_mapping_layer(R.p, i, h)
        _check(G.style[i](h.float()), nxt, TOL_F32, "mapping layer", f"{case} style.{i}")
        h = nxt
    _check(G.style(zr.float()), _want(R, "style", b)[1], TOL_F32, "mapping (PixelNorm + 8 layers)", case)


# ---------------------------------------------------------------------------- generator
@pytest.mark.gpu
@pytest.mark.parametrize("b", [1, B_FULL])
@pytest.mark.parametrize("row", CONVS, ids=[r.name for r in CONVS])
def test_styled_conv(R, row, b, monkeypatch):
    """StyledConv.forward with its encoder map as the concatenated noise: the conv half (the kernel's fused epilogue with
    bias[:C]) and the noise half (bias_act with bias[C:]) each against float64.  Then, at the same shape, the modulation
    (K.linear, K-split), the demodulation (K.demod) and the modulated convolution (modconv3x3_tcr_fwd, or the
    transposed-convolution GEMM + blur of modconv3x3_up_tcr_fwd for up-sampling layers).  At B = 1 also the exact-fp32
    SIMT path and every N-tile width the channel count allows."""
    from e4s_b200 import kernels as K
    case = f"{row.name}-b{b}"
    layer = R.m.generator.get_submodule(row.name)
    prefix = "generator." + row.name
    src, ecd = wiring()[row.name]
    x = R.m.generator.input.input.repeat(b, 1, 1, 1) if src is None else _feed(R, src, b)
    assert x.shape == (b, row.cin, row.side, row.side)
    noise = _feed(R, ecd, b)
    style = _feed(R, "style", b)
    rows, want = _want(R, row.name, b)
    c, up = row.cout, row.resample == "up"
    out = layer(x, style, noise=noise)
    assert out.shape == (b, 2 * c, out_side(row), out_side(row))
    _check(out[rows][:, :c], want[:, :c], TOL_CONV, "styled conv half", case)
    _check(out[rows][:, c:], want[:, c:], TOL_F32, "styled noise half", case)
    del out

    mw, mb = layer.conv.modulation._frozen()
    s = K.linear(style, mw, mb)
    _check(s, ref_modulation(R.p, prefix, style.double()), TOL_F32, "modulation (linear, K-split)", case)
    s = s[:, None]                                               # [B, 1 region, Cin]
    prep = layer.conv.prepared()
    dm = K.demod(s, prep.wsq)
    _check(dm, F64.demod(s.double(), R.p[prefix + ".conv.weight"][0]), TOL_F32, "demod", case)
    x_pm, bias = K.to_pixel_major(x), layer.activate.bias[:c]
    if up:
        y = K.modconv3x3_up_tcr_fwd(x_pm, prep.w_convt_hilo, prep.fir, s, dm, None, None, bias, True)
        kind = "modconv3x3_up_tcr_fwd"
    else:
        y = K.modconv3x3_tcr_fwd(x_pm, prep.w_hilo, s, dm, None, None, None, bias, False, True)
        kind = "modconv3x3_tcr_fwd"
    _check(nchw(y)[rows], want[:, :c], TOL_CONV, kind, case)
    del y
    if b != 1:
        return

    monkeypatch.setenv("E4S_B200_CONV", "simt")
    _check(layer(x, style, noise=noise)[:, :c], want[:, :c], TOL_SIMT, "styled conv half (simt)", case)
    monkeypatch.delenv("E4S_B200_CONV")
    for nt in (32, 64):
        if (4 * c if up else c) % nt:
            continue
        monkeypatch.setenv("E4S_B200_NTILE", str(nt))
        _check(layer(x, style, noise=noise)[:, :c], want[:, :c], TOL_CONV, f"styled conv half (NTILE {nt})", case)
    monkeypatch.delenv("E4S_B200_NTILE", raising=False)


@pytest.mark.gpu
@pytest.mark.parametrize("b", [1, B_FULL])
@pytest.mark.parametrize("row", RGBS, ids=[r.name for r in RGBS])
def test_to_rgb(R, row, b):
    """ToRGB.forward with the fused up-sampled skip (warp-per-pixel kernel at Cin 1024 / 512, thread-per-pixel at 256 /
    128) and its modulation, against float64."""
    from e4s_b200 import kernels as K
    case = f"{row.name}-b{b}"
    layer = R.m.generator.get_submodule(row.name)
    src, prev = wiring()[row.name]
    x = _feed(R, src, b)
    assert x.shape == (b, row.cin, row.side, row.side)
    skip = None if prev is None else _feed(R, prev, b, planar=True)
    style = _feed(R, "style", b)
    rows, want = _want(R, row.name, b)
    out = layer(x, style, skip)
    _check(out[rows], want, TOL_F32, "rgb", case)
    mw, mb = layer.conv.modulation._frozen()
    _check(K.linear(style, mw, mb), ref_modulation(R.p, "generator." + row.name, style.double()), TOL_F32,
           "modulation (linear, K-split)", case)


# ---------------------------------------------------------------------------- whole network
@pytest.mark.gpu
def test_full_generator_b16(R, monkeypatch):
    """FullGenerator.forward on the 16-face batch: the routing (channel-major flatten into final_linear, each encoder map
    handed to the StyledConv of its side), the image against the chained float64 reference on faces SUB, every face
    alone against the same face in the batch, and the default path against the SIMT path at B = 1."""
    m = R.m
    seen = {}
    hooks = [getattr(m, n).register_forward_hook(lambda mod, a, out, n=n: seen.__setitem__(n, out)) for n in m.names]
    hooks.append(m.final_linear.register_forward_pre_hook(lambda mod, a: seen.__setitem__("flat", a[0])))
    hooks.append(m.generator.register_forward_pre_hook(lambda mod, a, kw: seen.__setitem__("noise", kw["noise"]),
                                                       with_kwargs=True))
    try:
        img, none = m(R.img)
    finally:
        for h in hooks:
            h.remove()
    assert none is None and img.shape == (B_FULL, 3, SIZE, SIZE)
    last = seen[m.names[-1]]
    assert torch.equal(seen["flat"].view(last.shape), last), "final_linear must see the channel-major flatten"
    wires = wiring()
    assert [id(t) for t in seen["noise"]] == [id(seen[wires[r.name][1]]) for r in CONVS]
    del seen, last

    rows, want = _want(R, "image", B_FULL)
    _check(img[rows], want, TOL_IMAGE, "image vs float64", "forward-b16")
    for k in range(B_FULL):
        alone, _ = m(R.img[k:k + 1])
        _check(alone[0], img[k], TOL_BATCH, "image batch invariance", f"face {k}")
        if k == ONE:
            auto = alone
    monkeypatch.setenv("E4S_B200_CONV", "simt")
    simt, _ = m(R.img[ONE:ONE + 1])
    _check(auto, simt, TOL_IMAGE, "image auto vs simt (B = 1)", f"face {ONE}")
    _check(simt, _want(R, "image", 1)[1], TOL_IMAGE_SIMT, "image simt vs float64", f"face {ONE}")


# ---------------------------------------------------------------------------- edges
@pytest.mark.gpu
@pytest.mark.parametrize("hw", [(40, 72), (24, 40)], ids=["40x72", "24x40"])
def test_down_conv_layer_non_square(hw):
    """A down-sampling ConvLayer (64 -> 128 channels) on non-square even inputs - blurred to 42 x 74 (wide upfirdn2d
    tile) and 26 x 42 (narrow tile) - against float64; odd sides are refused before any kernel runs."""
    from e4s_b200.gpen.gpen_model import ConvLayer
    h, w = hw
    case = f"down-2x64x{h}x{w}"
    g = torch.Generator().manual_seed(zlib.crc32(case.encode()))
    layer = ConvLayer(64, 128, 3, downsample=True)
    with torch.no_grad():
        layer[1].weight.copy_(torch.randn(128, 64, 3, 3, generator=g))
        layer[2].bias.copy_(0.1 * torch.randn(128, generator=g))
    layer = layer.to(DEV).requires_grad_(False)
    x = torch.randn(2, 64, h, w, generator=g).to(DEV)
    xd = x.double()
    ref = F.conv2d(O.upfirdn2d(xd, layer[0].kernel.double(), pad=(2, 2)), layer[1].weight.double() / math.sqrt(9 * 64),
                   stride=2)
    ref = F64.act(ref + layer[2].bias.double()[None, :, None, None])
    out = layer(x)
    assert out.shape == (2, 128, h // 2, w // 2)
    _check(out, ref, TOL_ENC, "ConvLayer out (non-square)", case)
    for hh, ww in ((h + 1, w), (h, w + 1)):
        with pytest.raises(NotImplementedError, match="even-sized"):
            layer(torch.zeros(1, 64, hh, ww, device=DEV))
