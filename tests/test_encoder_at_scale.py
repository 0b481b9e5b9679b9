"""The RGI encoder (FSEncoder_PSP) at the face-swap batch: every unit of the 256x256 encoder at B = 1 and B = 32, against a
float64 reference that shares no code with e4s_b200.kernels or the weight preparation (_conv_planes, _conv_planes_s2d).

The face swap encodes the driven and target faces of 16 pairs in one call: B = 32 at 256 x 256 with 12-class face masks.
The reference is the oracle's encoder_unit / _instance_norm in float64 on the GPU, so the SE gate is computed, not assumed
to be 0.5.  Each unit takes the reference activation of the unit before it, cast to fp32, so its error is measured on its
own; the kernels behind the unit (instnorm_affine, conv1 with the folded InstanceNorm and PReLU, conv2 as four taps over
the space-to-depth tensor or plain, the centre-tap shortcut and its InstanceNorm, norm_residual) are then called directly
at the same shapes.  The whole encoder, Net3.get_style_vectors on 1024 x 1024 images, batch invariance and the edges of
the streaming kernels follow.  Unit shapes are read from O.encoder_unit_specs(), which the host-only tests pin to the
module tree; the few restated reference pieces are pinned to the oracle there too.
"""
import functools
import time
import types
import zlib

import pytest
import torch
import torch.nn.functional as F
from torch import nn

import f64ref as F64
from oracle import e4s_oracle as O
from conftest import assert_close
from f64ref import nchw, pm

DEV = "cuda:0"
B_FULL, NCLS, SIDE, MASK_SIDE = 32, 12, 256, 512
ONE = 31                  # the sample the B = 1 cases encode alone
SPECS = O.encoder_unit_specs()

# Bars: the largest error observed on an H100 80GB HBM3 (400 W power limit) is in the comment; each bar sits above it with
# headroom.  Shifts are measured against max(|shift|, 1): the normalised values have unit spread, so an absolute error in
# the shift is a relative error of the normalised output (a zero-mean channel has a shift of ~0).
TOL_CONV = 5e-5           # one split-bf16 tensor-core convolution (conv1, conv2, shortcut) on its own inputs: 2.0e-5
TOL_UNIT = 3e-5           # one unit (or the input layer) through FSEncoder_PSP, from the reference input cast to fp32: 8.6e-6
TOL_F32 = 5e-6            # exact-fp32 kernels: instnorm_affine 1.4e-6, norm_residual 7.7e-8, region_mean 1.9e-7
TOL_CODE = 1e-4           # the 1280-wide code of the whole encoder against the float64 encoder: 2.8e-5
# A face alone against the same face inside the 32-face batch.  Only the InstanceNorm sums are split differently (the
# split count depends on B), but a 1e-7 change of the normalised operand re-rounds its bf16 hi/lo split, so the two runs
# differ by about the convolution's own error: 4.0e-6 per unit, 1.9e-5 over the whole encoder.
TOL_UNIT_BATCH = 1.5e-5
TOL_BATCH = 5e-5
# instnorm_affine sums (x - x[pixel 0]) and its square in one pass: a pixel 0 d sigma away from the mean amplifies the fp32
# rounding of those sums by about d^2 in the variance.  At d = 20 over 65536 pixels the scale was off by up to 3.1e-4
# (the atomic accumulation order varies from run to run).
TOL_OUTLIER = 1e-3


# ============================================================================ float64 reference (plain torch ops)
def ref_in_stats(x):
    """InstanceNorm2d (biased variance, eps 1e-5) of NCHW x as the affine (scale, shift), each [B, C]."""
    var, mean = torch.var_mean(x, dim=(2, 3), unbiased=False)
    scale = torch.rsqrt(var + 1e-5)
    return scale, -mean * scale


def _affine(x, scale, shift):
    return x * scale.double()[:, :, None, None] + shift.double()[:, :, None, None]


def to_s2d(t):
    """NCHW [B, C, H, W] -> space-to-depth pixel-major [B, H/2, W/2, 4C], channel (y & 1, x & 1, c)."""
    b, c, h, w = t.shape
    return t.reshape(b, c, h // 2, 2, w // 2, 2).permute(0, 2, 4, 3, 5, 1).reshape(b, h // 2, w // 2, 4 * c)


def from_s2d(t):
    """The inverse of to_s2d: [B, H/2, W/2, 4C] -> NCHW [B, C, H, W]."""
    b, h2, w2, c4 = t.shape
    return t.reshape(b, h2, w2, 2, 2, c4 // 4).permute(0, 5, 1, 3, 2, 4).reshape(b, c4 // 4, 2 * h2, 2 * w2)


def ref_input_layer(p, x):
    """input_layer: PReLU(IN(conv3x3(x))), x [B, 3, H, W]."""
    return F.prelu(O._instance_norm(F.conv2d(x, p["input_layer.0.weight"], padding=1)), p["input_layer.2.weight"])


def labels_at(mask, h, w):
    """One-hot mask [B, ncls, Hm, Wm] -> label map [B, h, w] (nearest resize, psp_encoders.py:265)."""
    return F.interpolate(mask, size=(h, w), mode="nearest").argmax(1)


def ref_region_mean(feats, label, ncls):
    """Per (sample, region) mean of feats [B, C, h, w] over the pixels of label [B, h, w]; zero for an empty region."""
    b, c = feats.shape[:2]
    idx = (label.long() + ncls * torch.arange(b, device=label.device)[:, None, None]).reshape(-1)
    sums = feats.new_zeros(b * ncls, c).index_add_(0, idx, pm(feats).reshape(-1, c))
    cnt = feats.new_zeros(b * ncls).index_add_(0, idx, feats.new_ones(idx.numel()))
    return (sums / cnt.clamp_min(1)[:, None]).reshape(b, ncls, c), cnt.reshape(b, ncls)


def ref_encoder(p, x, mask, tap_units):
    """Every activation (input layer, then units 0..23, NCHW) and the [B, ncls, 1280] code of the encoder in x's dtype."""
    acts = [ref_input_layer(p, x)]
    for i, (cin, depth, stride) in enumerate(SPECS):
        acts.append(O.encoder_unit(acts[-1], p, f"body.{i}.", cin, depth, stride))
    codes = [ref_region_mean(acts[i + 1], labels_at(mask, *acts[i + 1].shape[2:]), mask.shape[1])[0] for i in tap_units]
    return acts, torch.cat(codes, 2)


# ============================================================================ host-only: module tree and the reference
@functools.lru_cache(maxsize=None)
def _cpu_encoder():
    from e4s_b200.encoders.psp_encoders import FSEncoder_PSP
    return FSEncoder_PSP().eval()


def _encoder_state(enc):
    """Seeded encoder weights with the conventions of the oracle's synthetic_state for the "encoder." keys."""
    st = O.synthetic_state({"encoder." + k: tuple(v.shape) for k, v in enc.state_dict().items()}, salt=5)
    return {k[len("encoder."):]: v for k, v in st.items()}


def test_module_tree_matches_the_oracle_specs():
    """Each unit's channels, stride and shortcut kind, the input layer and the tap units equal the oracle's table."""
    from e4s_b200.encoders import psp_encoders as PE
    enc = _cpu_encoder()
    conv0, norm0, prelu0 = enc.input_layer
    assert (conv0.in_channels, conv0.out_channels, conv0.kernel_size, conv0.padding) == (3, 64, (3, 3), (1, 1))
    assert isinstance(norm0, nn.InstanceNorm2d) and not norm0.affine and prelu0.num_parameters == 64
    assert len(enc.body) == len(SPECS) == 24
    for i, (unit, (cin, depth, stride)) in enumerate(zip(enc.body, SPECS)):
        c1, c2 = unit.res_layer[1], unit.res_layer[3]
        assert (c1.in_channels, c1.out_channels, c1.stride) == (cin, depth, (1, 1)), i
        assert (c2.in_channels, c2.out_channels, c2.stride) == (depth, depth, (stride, stride)), i
        assert isinstance(unit.res_layer[0], nn.InstanceNorm2d) and isinstance(unit.res_layer[4], nn.InstanceNorm2d), i
        if cin == depth:
            assert isinstance(unit.shortcut_layer, nn.MaxPool2d) and unit.shortcut_layer.stride == stride, i
        else:
            sc, sn = unit.shortcut_layer
            assert (sc.in_channels, sc.out_channels, sc.kernel_size, sc.stride) == (cin, depth, (1, 1), (stride, stride)), i
            assert isinstance(sn, nn.InstanceNorm2d), i
    block_ends = [i for i in range(len(SPECS)) if i + 1 == len(SPECS) or SPECS[i + 1][2] == 2]
    assert PE.TAP_UNITS == tuple(block_ends[1:]) == (6, 20, 23)
    assert sum(SPECS[i][1] for i in PE.TAP_UNITS) == 1280


def test_reference_matches_the_oracle():
    """ref_in_stats, the space-to-depth layout, ref_input_layer and ref_region_mean against the oracle, float64 on the
    CPU at 32 x 32 with B = 2, <= 1e-10."""
    from e4s_b200.encoders import psp_encoders as PE
    g = torch.Generator().manual_seed(3)
    x = 3.0 + torch.randn(2, 24, 10, 12, generator=g, dtype=torch.float64)
    s, t = ref_in_stats(x)
    assert_close(_affine(x, s, t), O._instance_norm(x), 1e-10, "ref_in_stats")
    q = to_s2d(x)
    assert torch.equal(from_s2d(q), x)
    for py in (0, 1):
        for px in (0, 1):
            k = py * 2 + px
            assert torch.equal(q[..., k * 24:(k + 1) * 24], pm(x[:, :, py::2, px::2])), (py, px)

    p = {k: v.double() for k, v in _encoder_state(_cpu_encoder()).items()}
    img = torch.randn(2, 3, 32, 32, generator=g, dtype=torch.float64)
    _, mask, _, _ = O.synthetic_inputs(2, NCLS, 32, 64, seed=3, kind="blobs")
    want, _ = O.encoder_forward(p, img, mask.double(), prefix="")
    acts, got = ref_encoder(p, img, mask.double(), PE.TAP_UNITS)
    side = 32
    for a, (_, depth, stride) in zip(acts[1:], SPECS):
        side //= stride
        assert tuple(a.shape[1:]) == (depth, side, side)
    assert_close(got, want, 1e-10, "ref_encoder codes")


@pytest.mark.parametrize("h,w", [(248, 256), (256, 200), (250, 250)])
def test_forward_rejects_sides_not_multiple_of_16(h, w):
    """Each of the four stride-2 units needs an even side: anything but multiples of 16 is refused up front."""
    with torch.no_grad(), pytest.raises(ValueError, match="multiples of 16"):
        _cpu_encoder()(torch.zeros(1, 3, h, w), torch.zeros(1, NCLS, h, w))


# ============================================================================ GPU checks
LEDGER = F64.Ledger(28)
_check = LEDGER.check


@pytest.fixture(scope="module", autouse=True)
def _error_report():
    yield
    LEDGER.report()


@pytest.fixture(autouse=True)
def _forward_only(monkeypatch):
    """The encoder kernels are forward-only; the default kernel selection (the space-to-depth stride-2 form) unless a test
    asks otherwise."""
    F64.clear_kernel_selection(monkeypatch)
    with torch.no_grad():
        yield


@pytest.fixture(scope="module")
def R():
    """The encoder on the device with seeded weights, 32 seeded 1024 x 1024 images, their 256 x 256 bilinear resize, 32 face
    masks, and every float64 reference activation and the reference code of that batch (computed once: ~7 TFLOP)."""
    from e4s_b200.encoders import psp_encoders as PE
    enc = PE.FSEncoder_PSP().eval()
    st = _encoder_state(enc)
    enc.load_state_dict(st)
    enc = enc.to(DEV).requires_grad_(False)
    p = {k: v.to(DEV, torch.float64) for k, v in st.items()}
    g = torch.Generator().manual_seed(1024)
    img1024 = torch.randn(B_FULL, 3, 1024, 1024, generator=g).to(DEV)
    mask = F64.onehot(F64.face_labels(B_FULL, MASK_SIDE, MASK_SIDE, roll=True).to(DEV), NCLS, torch.float32)
    img256 = F.interpolate(img1024.double(), (SIDE, SIDE), mode="bilinear")
    t0 = time.perf_counter()
    acts, codes = ref_encoder(p, img256, mask, PE.TAP_UNITS)
    torch.cuda.synchronize()
    print(f"\nfloat64 reference encoder, B = {B_FULL}: {time.perf_counter() - t0:.1f} s")
    return types.SimpleNamespace(PE=PE, enc=enc, p=p, img1024=img1024, img256=img256, mask=mask, acts=acts, codes=codes)


def _batch(b):
    return slice(0, B_FULL) if b == B_FULL else slice(ONE, ONE + 1)


# ---------------------------------------------------------------------------- per unit
UNITS = ["input"] + list(range(len(SPECS)))


@pytest.mark.gpu
@pytest.mark.parametrize("b", [1, B_FULL])
def test_input_layer(R, b):
    """The input layer (Cin padded 3 -> 32, norm_residual with alpha 1, PReLU and no shortcut) and its kernels."""
    from e4s_b200 import kernels as K
    case, sl = f"input-b{b}", _batch(b)
    x = R.img256[sl].float()
    out = R.enc._input_layer(x)
    _check(out, pm(R.acts[0][sl]), TOL_UNIT, "unit out", case)

    xd = x.double()
    xp = torch.zeros(x.shape[0], SIDE, SIDE, 32, device=DEV)
    xp[..., :3] = pm(x)
    y = K.conv3x3_tc(xp, R.enc._prepared("in", R.enc.input_layer[0].weight, pad_cin_to=32))
    _check(y, pm(F.conv2d(xd, R.p["input_layer.0.weight"], padding=1)), TOL_CONV, "conv (input layer)", case)
    s0, t0 = K.instnorm_affine(y)
    rs, rt = ref_in_stats(nchw(y).double())
    _check(s0, rs, TOL_F32, "instnorm scale", case)
    _check(t0, rt, TOL_F32, "instnorm shift", case, floor=1.0)
    slope = R.p["input_layer.2.weight"]
    nr = K.norm_residual(y, s0, t0, 1.0, prelu=R.enc.input_layer[2].weight)
    _check(nr, pm(F.prelu(_affine(nchw(y).double(), s0, t0), slope)), TOL_F32, "norm_residual", case)


@pytest.mark.gpu
@pytest.mark.parametrize("b", [1, B_FULL])
@pytest.mark.parametrize("i", list(range(len(SPECS))), ids=[f"u{i}" for i in range(len(SPECS))])
def test_unit(R, i, b, monkeypatch):
    """Unit i through FSEncoder_PSP._unit, then each kernel behind it on the same input: instnorm_affine, conv1 (IN fold +
    PReLU; space-to-depth store at stride 2), conv2 (four taps or plain), the centre-tap shortcut and its IN, and
    norm_residual in the unit's form.  Stride-2 units also run the E4S_B200_ENC_S2D=0 form."""
    from e4s_b200 import kernels as K
    PE, enc, p = R.PE, R.enc, R.p
    cin, depth, stride = SPECS[i]
    case, sl, pre = f"u{i}-b{b}", _batch(b), f"body.{i}."
    unit = enc.body[i]
    x = pm(R.acts[i][sl]).float().contiguous()        # the reference input of the unit, cast to fp32
    want = pm(R.acts[i + 1][sl])
    out = enc._unit(i, unit, x)
    _check(out, want, TOL_UNIT, "unit out", case)
    if b == B_FULL:
        _check(enc._unit(i, unit, x[ONE:ONE + 1].contiguous())[0], out[ONE], TOL_UNIT_BATCH, "unit batch invariance", case)
    if i in PE.TAP_UNITS:
        lab = labels_at(R.mask[sl], out.shape[1], out.shape[2])
        got, area = K.region_mean(out, lab.to(torch.uint8).contiguous(), NCLS)
        ref, cnt = ref_region_mean(nchw(out).double(), lab, NCLS)
        _check(got, ref, TOL_F32, "region_mean", case)
        assert torch.equal(area.long(), cnt.long())
    del out
    if stride == 2:
        monkeypatch.setenv("E4S_B200_ENC_S2D", "0")
        _check(enc._unit(i, unit, x), want, TOL_UNIT, "unit out (no s2d)", case)
        monkeypatch.delenv("E4S_B200_ENC_S2D")
    del want

    xd = nchw(x).double()
    sx, tx = K.instnorm_affine(x)
    rs, rt = ref_in_stats(xd)
    _check(sx, rs, TOL_F32, "instnorm scale", case)
    _check(tx, rt, TOL_F32, "instnorm shift", case, floor=1.0)

    # conv1 on the folded InstanceNorm, PReLU in the epilogue; at stride 2 stored space-to-depth
    conv1, prelu, conv2 = unit.res_layer[1], unit.res_layer[2], unit.res_layer[3]
    planes1 = enc._prepared(f"{i}.c1", conv1.weight)
    r1 = F.prelu(F.conv2d(_affine(xd, sx, tx), p[pre + "res_layer.1.weight"], padding=1), p[pre + "res_layer.2.weight"])
    y1 = K.conv3x3_tc(x, planes1, sx, tx, prelu.weight, out_stride=4 if stride == 2 else 1)
    _check(y1, to_s2d(r1) if stride == 2 else pm(r1), TOL_CONV, "conv1", case)
    del r1

    w2 = p[pre + "res_layer.3.weight"]
    if stride == 2:
        y2 = K.conv3x3_tc(y1, enc._prepared(f"{i}.c2s", conv2.weight, s2d=True), tap_mask=PE.TAPS_S2D)
        _check(y2, pm(F.conv2d(from_s2d(y1).double(), w2, stride=2, padding=1)), TOL_CONV, "conv2 (four taps)", case)
        # the E4S_B200_ENC_S2D=0 form: conv1 at full resolution, conv2 computed everywhere and stored at the even pixels
        y1f = K.conv3x3_tc(x, planes1, sx, tx, prelu.weight)
        y2f = K.conv3x3_tc(y1f, enc._prepared(f"{i}.c2", conv2.weight), out_stride=2)
        _check(y2f, pm(F.conv2d(nchw(y1f).double(), w2, stride=2, padding=1)), TOL_CONV, "conv2 (out_stride 2)", case)
        del y1f, y2f
    else:
        y2 = K.conv3x3_tc(y1, enc._prepared(f"{i}.c2", conv2.weight))
        _check(y2, pm(F.conv2d(nchw(y1).double(), w2, padding=1)), TOL_CONV, "conv2", case)
    del y1
    s2, t2 = K.instnorm_affine(y2)
    y2d = nchw(y2).double()
    rs, rt = ref_in_stats(y2d)
    _check(s2, rs, TOL_F32, "instnorm scale", case)
    _check(t2, rt, TOL_F32, "instnorm shift", case, floor=1.0)
    res = 0.5 * _affine(y2d, s2, t2)

    if cin == depth:
        nr = K.norm_residual(y2, s2, t2, 0.5, shortcut=x, sc_stride=stride)
        ref = res + xd[:, :, ::stride, ::stride]
    else:
        xs = x[:, ::stride, ::stride].contiguous()
        sc = K.conv3x3_tc(xs, enc._prepared(f"{i}.sc", unit.shortcut_layer[0].weight), tap_mask=PE.TAP_CENTRE)
        _check(sc, pm(F.conv2d(nchw(xs).double(), p[pre + "shortcut_layer.0.weight"])), TOL_CONV, "shortcut conv", case)
        ss, ts = K.instnorm_affine(sc)
        rs, rt = ref_in_stats(nchw(sc).double())
        _check(ss, rs, TOL_F32, "instnorm scale", case)
        _check(ts, rt, TOL_F32, "instnorm shift", case, floor=1.0)
        nr = K.norm_residual(y2, s2, t2, 0.5, shortcut=sc, sc_scale=ss, sc_shift=ts, sc_stride=1)
        ref = res + _affine(nchw(sc).double(), ss, ts)
    _check(nr, pm(ref), TOL_F32, "norm_residual", case)


# ---------------------------------------------------------------------------- whole encoder
def _code_blocks(codes):
    """The 1280-wide code split into its three tap blocks (units 6, 20, 23: 256, 512, 512 channels)."""
    return {"code u6": codes[..., :256], "code u20": codes[..., 256:768], "code u23": codes[..., 768:]}


@pytest.mark.gpu
def test_encoder_forward_b32_and_batch_invariance(R):
    """FSEncoder_PSP.forward on the 32-face batch against the float64 encoder on all 32 samples, each tap block on its own;
    then faces 0, 15 and 31 alone against the same faces inside the batch."""
    codes, struct = R.enc(R.img256.float(), R.mask)
    assert codes.shape == (B_FULL, NCLS, 1280) and struct.shape == (B_FULL, 512, 16, 16)
    assert float(struct.abs().max()) == 0.0
    ours, ref = _code_blocks(codes), _code_blocks(R.codes)
    for kind in ours:
        _check(ours[kind], ref[kind], TOL_CODE, kind, "forward-b32")
    for k in (0, 15, 31):
        alone, _ = R.enc(R.img256[k:k + 1].float(), R.mask[k:k + 1])
        _check(alone[0], codes[k], TOL_BATCH, "batch invariance", f"sample {k}")
        _check(alone[0], R.codes[k], TOL_CODE, "code (B = 1)", f"sample {k}")


@pytest.mark.gpu
def test_get_style_vectors_1024_b32(R):
    """Net3.get_style_vectors on the 1024 x 1024 images (bilinear resize to 256 included) at B = 32."""
    from e4s_b200.networks import Net3
    opts = types.SimpleNamespace(fsencoder_type="psp", remaining_layer_idx=13, num_seg_cls=NCLS, out_size=64,
                                 train_G=False, start_from_latent_avg=True, learn_in_w=False)
    net = Net3(opts).eval()
    net.encoder = R.enc
    vec, _ = net.get_style_vectors(R.img1024, R.mask)
    ours, ref = _code_blocks(vec), _code_blocks(R.codes)
    for kind in ours:
        _check(ours[kind], ref[kind], TOL_CODE, kind, "get_style_vectors-1024-b32")


@pytest.mark.gpu
def test_encoder_non_square_and_rejected_sizes(R):
    """A valid non-square input (256 x 192) against the float64 encoder; sides that are not multiples of 16 are refused
    before any kernel runs."""
    g = torch.Generator().manual_seed(192)
    h, w = 256, 192
    img = torch.randn(2, 3, h, w, generator=g).to(DEV)
    mask = F64.onehot(F64.face_labels(2, 2 * h, 2 * w, roll=True).to(DEV), NCLS, torch.float32)
    _, ref = ref_encoder(R.p, img.double(), mask, R.PE.TAP_UNITS)
    codes, struct = R.enc(img, mask)
    assert struct.shape == (2, 512, h // 16, w // 16)
    ours, ref = _code_blocks(codes), _code_blocks(ref)
    for kind in ours:
        _check(ours[kind], ref[kind], TOL_CODE, kind, "non-square 256x192")
    for hh, ww in ((256, 248), (250, 256)):
        with pytest.raises(ValueError, match="multiples of 16"):
            R.enc(torch.zeros(1, 3, hh, ww, device=DEV), torch.zeros(1, NCLS, hh, ww, device=DEV))


# ---------------------------------------------------------------------------- edges of the streaming kernels
@pytest.mark.gpu
@pytest.mark.parametrize("b", [1, B_FULL])
@pytest.mark.parametrize("hw", [(256, 256), (16, 16)], ids=["hw65536", "hw256"])
def test_instnorm_affine_edges(b, hw):
    """instnorm_affine at C = 48 (a partial 32-channel chunk) on channel groups: plain; DC offset 1e3 x the spread; constant
    (variance 0: scale = rsqrt(eps)); pixel 0 (the shift the kernel subtracts) 20 sigma out; spreads from 1e-3 to 1e3."""
    from e4s_b200 import kernels as K
    h, w = hw
    case = f"instnorm-{h * w}px-b{b}"
    g = torch.Generator().manual_seed(zlib.crc32(case.encode()))
    x = torch.randn(b, 48, h, w, generator=g, dtype=torch.float64)
    groups = {"plain": slice(0, 12), "dc offset": slice(12, 24), "constant": slice(24, 30), "pixel-0 outlier": slice(30, 36),
              "spread 1e-3..1e3": slice(36, 48)}
    x[:, groups["plain"]] += torch.randn(b, 12, 1, 1, generator=g, dtype=torch.float64)
    x[:, groups["dc offset"]] = 1e3 * (1.0 + torch.rand(b, 12, 1, 1, generator=g, dtype=torch.float64)) + x[:, groups["dc offset"]]
    x[:, groups["constant"]] = torch.randn(b, 6, 1, 1, generator=g, dtype=torch.float64).expand(b, 6, h, w)
    x[:, groups["pixel-0 outlier"], 0, 0] = 20.0
    x[:, groups["spread 1e-3..1e3"]] *= torch.logspace(-3, 3, 12, dtype=torch.float64)[None, :, None, None]
    x = x.float()
    scale, shift = K.instnorm_affine(pm(x).contiguous().to(DEV))
    rs, rt = ref_in_stats(x.double().to(DEV))
    for name, sl in groups.items():
        tol = TOL_OUTLIER if name == "pixel-0 outlier" else TOL_F32
        if name == "spread 1e-3..1e3":           # one bar per channel: the scales span six decades
            for c in range(sl.start, sl.stop):
                _check(scale[:, c], rs[:, c], tol, f"instnorm scale ({name})", f"{case} c{c}")
                _check(shift[:, c], rt[:, c], tol, f"instnorm shift ({name})", f"{case} c{c}", floor=1.0)
            continue
        _check(scale[:, sl], rs[:, sl], tol, f"instnorm scale ({name})", case)
        _check(shift[:, sl], rt[:, sl], tol, f"instnorm shift ({name})", case, floor=1.0)


@pytest.mark.gpu
@pytest.mark.parametrize("b", [1, B_FULL])
def test_norm_residual_forms(b):
    """Every form of norm_residual: shortcut none / stride 1 / stride 2, sc_scale + sc_shift absent / given, PReLU absent /
    given, alpha 0.5 and 1."""
    from e4s_b200 import kernels as K
    h, w, c = 24, 20, 96
    g = torch.Generator().manual_seed(96 + b)
    rnd = lambda *s: torch.randn(*s, generator=g).to(DEV)
    y = rnd(b, h, w, c)
    sy, ty = 0.5 + rnd(b, c).abs(), rnd(b, c)
    ss, ts = 0.5 + rnd(b, c).abs(), rnd(b, c)
    slope = 0.25 + 0.05 * rnd(c)
    shorts = {1: rnd(b, h, w, c), 2: rnd(b, 2 * h, 2 * w, c)}
    for sc_stride in (None, 1, 2):
        for affine in (False, True):
            for act in (False, True):
                for alpha in (0.5, 1.0):
                    tag = f"b{b} shortcut={sc_stride or '-'} sc_affine={int(affine)} prelu={int(act)} alpha={alpha}"
                    sh = shorts[sc_stride] if sc_stride else None
                    out = K.norm_residual(y, sy, ty, alpha, shortcut=sh, sc_scale=ss if affine else None,
                                          sc_shift=ts if affine else None, sc_stride=sc_stride or 1,
                                          prelu=slope if act else None)
                    ref = alpha * _affine(nchw(y).double(), sy, ty)
                    if sh is not None:
                        s = nchw(sh).double()[:, :, ::sc_stride, ::sc_stride]
                        ref = ref + (_affine(s, ss, ts) if affine else s)
                    if act:
                        ref = F.prelu(ref, slope.double())
                    _check(out, pm(ref), TOL_F32, "norm_residual forms", tag)


REGION_CASES = [  # id, b, h, w, c, ncls, labels
    ("tap-u6-face-b32", B_FULL, 64, 64, 256, NCLS, "face"),
    ("tap-u20-face-b32", B_FULL, 32, 32, 512, NCLS, "face"),
    ("tap-u23-face-b32", B_FULL, 16, 16, 512, NCLS, "face"),
    ("tap-u23-face-b1", 1, 16, 16, 512, NCLS, "face"),
    ("one-pixel-b32", B_FULL, 32, 32, 512, NCLS, "one-pixel"),
    ("iid32-b32", B_FULL, 32, 32, 512, 32, "iid"),
    ("c70-face-b32", B_FULL, 16, 16, 70, NCLS, "face"),
    ("ncls46", 2, 16, 16, 64, 46, "iid"),
    ("ncls47", 2, 16, 16, 64, 47, "iid"),
    ("ncls64", 2, 16, 16, 64, 64, "iid"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", REGION_CASES, ids=[c[0] for c in REGION_CASES])
def test_region_mean_edges(case):
    """region_mean (means and areas) against float64 index_add: the three tap shapes at B = 32 with face masks (empty
    regions), a one-pixel region at the first / last / an inner pixel, 32 iid regions, C = 70 (a partial 32-channel
    chunk), and 46, 47 and 64 regions (47 and up need more than 48 KB of shared memory)."""
    from e4s_b200 import kernels as K
    cid, b, h, w, c, ncls, kind = case
    g = torch.Generator().manual_seed(zlib.crc32(cid.encode()))
    lab = F64.labels(kind, b, h, w, ncls, g, roll=True).to(DEV)
    feats = (torch.randn(b, h, w, c, generator=g) + torch.randn(b, 1, 1, c, generator=g)).to(DEV)
    got, area = K.region_mean(feats, lab, ncls)
    ref, cnt = ref_region_mean(nchw(feats).double(), lab, ncls)
    _check(got, ref, TOL_F32, "region_mean", cid)
    assert torch.equal(area.long(), cnt.long()), cid
    if kind != "iid":
        assert int((cnt == 0).sum()) > 0, "the face masks should leave some regions empty"
        assert float(got[cnt == 0].abs().max()) == 0.0
    if kind == "one-pixel":
        assert torch.equal(cnt[:, 11], torch.ones_like(cnt[:, 11]))
