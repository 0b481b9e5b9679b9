"""Shared pieces of the at-scale kernel checks: float64 references built from plain torch ops (they share no code with
e4s_b200.kernels or the weight preparation) up to the whole generator (RefChain) and the texture-vector stage in front of
it (style_codes), the inputs those checks draw, the 1024 generator's layer table, the list of kernel-selection
variables, and the ledger of the largest error per output kind.

The references are pinned to the CPU oracle by tests/test_f64ref.py.  Test modules import this one as they import conftest.
"""
import functools
import math
import os
from collections import namedtuple

import torch
import torch.nn.functional as F

from oracle import e4s_oracle as O
from oracle import golden_io

SQRT2 = math.sqrt(2.0)
CHUNK_BYTES = 2e9         # float64 working set of one chunk of faces in styled_conv_per_pixel

# Every variable that forces a kernel path, tile width, split or batching away from the default selection.
SELECTION_VARS = ("E4S_B200_CONV", "E4S_B200_BWD", "E4S_B200_NTILE", "E4S_B200_RS_NTILE", "E4S_B200_DGRAD_SPLIT",
                  "E4S_B200_UP2", "E4S_B200_RS_STREAM", "E4S_B200_ENC_S2D", "E4S_B200_STYLE_BATCH")


def clear_kernel_selection(monkeypatch):
    """The default kernel selection, whatever the caller's environment forces."""
    for var in SELECTION_VARS:
        monkeypatch.delenv(var, raising=False)


# ============================================================================ error ledger
class Ledger:
    """max-rel (max|ours - ref| / max|ref|) and rel-RMS (||ours - ref|| / ||ref||), conftest.assert_close's norms, computed
    on the device; the largest error per output kind is kept for report()."""

    def __init__(self, width):
        self.width = width        # of the kind column in report()
        self.worst = {}

    @staticmethod
    def _errors(ours, ref, floor, what):
        ours, ref = ours.detach(), ref.detach()
        dev = ours.device if ours.is_cuda else ref.device
        ours, ref = ours.to(dev, torch.float64), ref.to(dev, torch.float64)
        assert ours.shape == ref.shape, (what, ours.shape, ref.shape)
        assert bool(torch.isfinite(ours).all()), f"{what}: non-finite values"
        d = ours - ref
        return (float(d.abs().max() / ref.abs().max().clamp_min(floor)),
                float(d.norm() / ref.norm().clamp_min(floor * ref.numel() ** 0.5)))

    def check(self, ours, ref, tol, kind, case, floor=1e-30, per_face=False):
        """Both norms <= tol.  floor bounds the reference's max (and RMS) from below.  per_face: every face (row of dim 0)
        against its own maximum, and ref may be a function of a face slice returning that slice of the reference."""
        if per_face:
            errs = [self._errors(ours[f:f + 1], ref(slice(f, f + 1)) if callable(ref) else ref[f:f + 1], floor,
                                 f"{case} {kind} face {f}") for f in range(ours.shape[0])]
        else:
            errs = [self._errors(ours, ref, floor, f"{case} {kind}")]
        e, r = max(x[0] for x in errs), max(x[1] for x in errs)
        if per_face:
            face = max(range(len(errs)), key=lambda f: max(errs[f]))
            print(f"{case}: {kind} max-rel {e:.2e} rel-RMS {r:.2e} (bar {tol:.1e}, worst face {face})")
        else:
            print(f"{case}: {kind} max-rel {e:.2e} rel-RMS {r:.2e} (bar {tol:.0e})")
        self.note(kind, e, r, case)
        bad = [f for f, (fe, fr) in enumerate(errs) if not (fe <= tol and fr <= tol)]
        where = f" on faces {bad}" if per_face else ""
        assert not bad, f"{case} {kind}: max-rel {e:.3e} rel-RMS {r:.3e} over the bar {tol:.1e}{where}"

    def note(self, kind, e, r, case):
        """Keep (e, r, case) for report() if e is the largest max-rel of this kind so far (NaN counts as largest)."""
        if kind not in self.worst or not e <= self.worst[kind][0]:
            self.worst[kind] = (e, r, case)

    def report(self):
        if self.worst:
            print("\nlargest observed error per output kind (max-rel, rel-RMS, case):")
            for kind in sorted(self.worst):
                e, r, what = self.worst[kind]
                print(f"  {kind:{self.width}s} {e:.2e}  {r:.2e}  {what}")


# ============================================================================ float64 references (plain torch ops)
def pm(t):
    """NCHW -> pixel-major [B, H, W, C] view."""
    return t.permute(0, 2, 3, 1)


def nchw(t):
    """pixel-major [B, H, W, C] -> NCHW view."""
    return t.permute(0, 3, 1, 2)


def act(v, act_from=None):
    """FusedLeakyReLU's activation sqrt(2) * leaky_relu(v, 0.2); with act_from the branch is taken from act_from > 0
    instead of from v."""
    if act_from is None:
        return F.leaky_relu(v, 0.2) * SQRT2
    return torch.where(act_from > 0, v * SQRT2, v * (0.2 * SQRT2))


def blur_fir(device):
    """The 4 x 4 blur of the up-sampling StyledConvs and of the ToRGB skip, float64."""
    return O.make_fir((1, 3, 3, 1), 4.0, dtype=torch.float64).to(device)


def region_of(label, ncls):
    """Region of every pixel, long: labels >= ncls count as the last region, as the kernels count them."""
    return label.long().clamp(max=ncls - 1)


def _regions(label, ncls):
    """(region, mask [B, 1, H, W]) for every region present in label, or (0, None) without a label map."""
    if label is None:
        yield 0, None
        return
    lab = region_of(label, ncls)
    for r in torch.unique(lab).tolist():
        yield r, (lab == r)[:, None]


def _scaled(w):
    """Equalised learning rate: the raw weight in float64 scaled by 1 / sqrt(fan_in)."""
    return w.double() * (1.0 / math.sqrt(w[0].numel()))


def equal_linear(x, weight, bias, lr_mul=1.0):
    """EqualLinear (the modulation of every StyledConv and ToRGB) in float64: x @ (W lr_mul / sqrt(in))^T + bias lr_mul."""
    return F.linear(x.double(), weight.double() * ((1.0 / math.sqrt(weight.shape[1])) * lr_mul), bias.double() * lr_mul)


def demod(s, w):
    """rsqrt(sum_{i,k} (W[o, i, k] s_i / sqrt(9 Cin))^2 + 1e-8) for s [..., Cin] and the raw weight w [Cout, Cin, 3, 3]
    -> [..., Cout]."""
    return torch.rsqrt(s.double().pow(2) @ _scaled(w).pow(2).sum((2, 3)).t() + 1e-8)


def styled_preact(x, s, w, label, noise, noise_w, bias, up, demodulate, s_demod=None):
    """Pre-activation of StyledConv in float64: sum over the regions r present of [label == r] * d_r * conv(x * s_r, W)
    + noise_w * noise + bias.

    x [B, Cin, H, W]; s [B, R, Cin]; w the raw weight [Cout, Cin, 3, 3] (scaled here by 1/sqrt(9 Cin)); label [B, Ho, Wo]
    or None (R == 1); noise [B | 1, 1, Ho, Wo] or None; bias [Cout] or None.  Up-sampling layers: conv_transpose2d
    (stride 2) then the 4x4 blur with pad (1, 1).  d_r = demod(s_demod_r, w) is computed inside the graph from ``s_demod``
    (default: s); passing a separate leaf there splits the style gradient into its convolution and demodulation parts."""
    x, s = x.double(), s.double()
    ws = _scaled(w)
    d = demod(s if s_demod is None else s_demod, w) if demodulate else None
    out = 0
    for r, sel in _regions(label, s.shape[1]):
        xs = x * s[:, r, :, None, None]
        if up:
            t = O.upfirdn2d(F.conv_transpose2d(xs, ws.transpose(0, 1), stride=2), blur_fir(x.device), pad=(1, 1))
        else:
            t = F.conv2d(xs, ws, padding=1)
        if d is not None:
            t = t * d[:, r, :, None, None]
        out = out + (t if sel is None else t * sel)
    if noise is not None:
        out = out + noise_w.double() * noise.double()
    if bias is not None:
        out = out + bias.double()[None, :, None, None]
    return out


def parity_kernels(ws):
    """[2 (py), 2 (px), Cout, Cin, 3, 3] from the scaled weight ws: output pixel (2m + py, 2n + px) of conv_transpose2d
    (stride 2) + the 4x4 blur with pad (1, 1) is sum_{dy,dx} K[py, px][:, :, dy, dx] x[m + dy - 1, n + dx - 1].  Read off
    the impulse response at input pixel (2, 2) of a 5 x 5 grid: it reaches output pixel (m, n) = (3 - dy, 3 - dx)."""
    cout, cin = ws.shape[:2]
    imp = ws.new_zeros(1, 1, 5, 5)
    imp[0, 0, 2, 2] = 1.0
    resp = O.upfirdn2d(F.conv_transpose2d(imp, ws.reshape(1, cout * cin, 3, 3), stride=2), blur_fir(ws.device), pad=(1, 1))
    resp = resp.view(cout, cin, 5, 2, 5, 2)                       # [o, c, m, py, n, px]
    inner = resp[:, :, 1:4, :, 1:4, :]
    total = float(resp.detach().abs().sum())
    outside = total - float(inner.detach().abs().sum())
    assert abs(outside) <= 1e-12 * total, "support wider than 3 x 3"
    return inner.flip(2, 4).permute(3, 5, 0, 1, 2, 4).contiguous()


def _pixel_conv(x, s, d, lab, ws, weff, up):
    """d * conv(x * s) of a masked layer, each output pixel with the style of its own region: unfold x, scale the patch
    of pixel p by s[lab[p]], one DGEMM with the weight (per output parity when up-sampling: weff), scale by d[lab[p]]."""
    b, cin, h, wd = x.shape
    cout = ws.shape[0]
    n = 2 if up else 1
    cols = F.unfold(x, 3, padding=1).view(b, cin, 9, h * wd)      # patch of every input pixel, (c, tap) order
    rows = torch.arange(b, device=x.device)[:, None]
    out = x.new_empty(b, cout, n * h, n * wd)
    for py in range(n):
        for px in range(n):
            pl = lab[:, py::n, px::n].reshape(b, h * wd)
            mod = cols * s[rows, pl].transpose(1, 2)[:, :, None, :]                # the style of each pixel's region
            k = (weff[py, px] if up else ws).reshape(cout, cin * 9)
            y = (k @ mod.view(b, cin * 9, h * wd)) * d[rows, pl].transpose(1, 2)
            out[:, :, py::n, px::n] = y.view(b, cout, h, wd)
    return out


def styled_conv_per_pixel(x, s, w, label, noise, noise_w, bias, up, act_from=None):
    """StyledConv forward, act(styled_preact(...)) with demodulation, in float64 a chunk of faces at a time.  A masked layer
    takes the per-pixel form (_pixel_conv: one DGEMM for all regions instead of one convolution per region, which the 1024
    generator's 12-region layers at 16 faces need for time and memory); an unmasked one is styled_preact itself.  noise
    [B | 1, 1, Ho, Wo]; act_from [B, Cout, Ho, Wo] or None: the sign of act_from picks the leaky-ReLU branch (act).
    Differentiable."""
    x, s = x.double(), s.double()
    b, cin, h, wd = x.shape
    cout = w.shape[0]
    ho, wo = (2 * h, 2 * wd) if up else (h, wd)
    if label is None:
        face = 8 * 4 * (cin * h * wd + cout * ho * wo)
    else:
        ws, d, lab = _scaled(w), demod(s, w), region_of(label, s.shape[1])
        weff = parity_kernels(ws) if up else None
        face = 8 * (2 * 9 * cin * h * wd + 3 * cout * ho * wo)
    n = max(1, min(b, int(CHUNK_BYTES // face)))
    out = x.new_empty(b, cout, ho, wo)
    for sl in (slice(i, min(i + n, b)) for i in range(0, b, n)):
        nz = noise if noise.shape[0] == 1 else noise[sl]
        if label is None:
            pre = styled_preact(x[sl], s[sl], w, None, nz, noise_w, bias, up, True)
        else:
            pre = _pixel_conv(x[sl], s[sl], d[sl], lab[sl], ws, weff, up) + bias.double()[None, :, None, None]
            pre = pre + noise_w.double() * nz.double()
        out[sl] = act(pre, None if act_from is None else act_from[sl])
    return out


def to_rgb(x, s, w, label, bias, skip):
    """ToRGB in float64: sum_r [label == r] * conv1x1(x * s_r, W / sqrt(Cin)) + bias + upfirdn2d(skip, up 2, pad (2, 1)).
    x [B, Cin, H, W]; s [B, R, Cin]; w the raw weight (any shape holding [3, Cin]); bias 3 values or None; skip
    [B, 3, H/2, W/2] or None.  The style modulates the weight, so no scaled copy of x is made."""
    x, s = x.double(), s.double()
    b, cin, h, wd = x.shape
    ws = _scaled(w.reshape(3, cin))
    out = 0
    for r, sel in _regions(label, s.shape[1]):
        t = (ws * s[:, r, None, :]).matmul(x.reshape(b, cin, h * wd)).view(b, 3, h, wd)
        out = out + (t if sel is None else t * sel)
    if bias is not None:
        out = out + bias.double().reshape(1, 3, 1, 1)
    if skip is not None:
        out = out + O.upfirdn2d(skip.double(), blur_fir(x.device), up=2, pad=(2, 1))
    return out


def style_codes(net, style_vectors):
    """Net3.cal_style_codes in float64 from net's own parameters (start_from_latent_avg, not learn_in_w): LocalMLP j
    (EqualLinear, leaky ReLU 0.01, EqualLinear) maps region j's texture vector to its first codes, latent_avg is added to
    them and its remaining rows follow.  style_vectors [B, ncls, 1280] -> [B, ncls, 18, 512] (as many rows as latent_avg).
    Differentiable."""
    v = style_vectors.double()
    b, ncls, _ = v.shape
    avg = net.latent_avg.double()
    codes = []
    for j in range(ncls):
        l0, l2 = net.MLPs[j].mlp[0], net.MLPs[j].mlp[2]
        h = F.leaky_relu(equal_linear(v[:, j], l0.weight, l0.bias, l0.lr_mul), 0.01)
        codes.append(equal_linear(h, l2.weight, l2.bias, l2.lr_mul).view(b, -1, avg.shape[1]))
    codes = torch.stack(codes, 1)
    k = codes.shape[2]
    return torch.cat([codes + avg[:k], avg[k:].expand(b, ncls, -1, -1)], 2)


class RefChain:
    """The generator forward in float64, one scheduled layer (Generator._schedule) at a time.  seek(i) returns the state
    before layer i (the activation x and the ToRGB skip), recomputing from the start if layer i has been passed;
    step() computes the next layer and returns its output.  Only the current state is held.

    The chain is differentiable in latent (and through it in whatever latent was computed from); callers that want no
    gradient run it under torch.no_grad().  act_from: None, or one tensor per StyledConv in execution order (as noise)
    whose sign picks that layer's leaky-ReLU branch (act), so the chain's gradient is the one of a network whose branches
    are fixed where act_from has them - a smooth function of its inputs."""

    def __init__(self, G, latent, labels, noise, act_from=None):
        from e4s_b200.stylegan2.model import StyledConv
        self.G, self.latent, self.labels, self.noise, self.act_from = G, latent.double(), labels, noise, act_from
        self.sched = G._schedule()
        self.is_conv = [isinstance(m, StyledConv) for m, _, _ in self.sched]
        self.noise_index = [sum(self.is_conv[:i]) for i in range(len(self.sched))]   # StyledConv k takes noise[k]
        self._levels = {}
        self.reset()

    def reset(self):
        self.pos, self.skip = 0, None
        self.x = self.G.input.input.double().repeat(self.latent.shape[0], 1, 1, 1)

    def label_at(self, side):
        """Nearest-resized region labels [B, side, side] (long), as F.interpolate(mask, mode='nearest') picks them."""
        if side not in self._levels:
            lab = F.interpolate(self.labels[:, None].double(), size=(side, side), mode="nearest")
            self._levels[side] = lab[:, 0].long()
        return self._levels[side]

    def style(self, i):
        m, idx, per_region = self.sched[i]
        lat = self.latent[:, :, idx] if per_region else self.latent[:, 0, idx][:, None]
        lin = m.conv.modulation
        s = equal_linear(lat, lin.weight, lin.bias, lin.lr_mul)
        return s, (demod(s, m.conv.weight[0]) if self.is_conv[i] else None)

    def seek(self, i):
        if self.pos > i:
            self.reset()
        while self.pos < i:
            self.step()
        return self.x, self.skip

    def step(self):
        i = self.pos
        m = self.sched[i][0]
        s, _ = self.style(i)
        side = self.x.shape[2]
        if self.is_conv[i]:
            up = m.conv.upsample
            k = self.noise_index[i]
            label = self.label_at(2 * side if up else side) if m.mask_op else None
            out = styled_conv_per_pixel(self.x, s, m.conv.weight[0], label, self.noise[k], m.noise.weight,
                                        m.activate.bias, up, None if self.act_from is None else self.act_from[k])
            self.x = out
        else:
            out = to_rgb(self.x, s, m.conv.weight, self.label_at(side) if m.mask_op else None, m.bias, self.skip)
            self.skip = out
        self.pos += 1
        if self.pos == len(self.sched):
            self.x = None
        return out

    def image(self):
        return self.seek(len(self.sched))[1]


# ============================================================================ inputs
def onehot(label, ncls, dtype):
    """Label map [B, H, W] -> one-hot mask [B, ncls, H, W]."""
    return F.one_hot(label.long(), ncls).permute(0, 3, 1, 2).to(dtype).contiguous()


@functools.lru_cache(maxsize=None)
def _golden_faces():
    gold = golden_io.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_vectors.npz"))
    return tuple(torch.from_numpy(gold[k]) for k in ("mask/source_cls12", "mask/target_cls12"))


def face_labels(b, h, w, roll=False):
    """Face-like 12-region maps [b, h, w] uint8: the committed 512 x 512 parsing masks (classes 7, 10, 11 empty in one or
    both), alternately mirrored, nearest-resized to h x w.  roll: each sample is also shifted by (3 i, -5 i) pixels first,
    so no two samples share a map."""
    faces = _golden_faces()
    labs = [faces[i % 2] if i % 4 < 2 else faces[i % 2].flip(-1) for i in range(b)]
    if roll:
        labs = [torch.roll(lab, shifts=(3 * i, -5 * i), dims=(0, 1)) for i, lab in enumerate(labs)]
    lab = torch.stack(labs)
    idx_y = (torch.arange(h) * lab.shape[1]) // h
    idx_x = (torch.arange(w) * lab.shape[2]) // w
    return lab[:, idx_y][:, :, idx_x].contiguous()


def labels(kind, b, h, w, ncls, g, roll=False):
    """Region maps [b, h, w] uint8 of a kind: iid (drawn from g); face (face_labels); face32 (face, region 3 moved to 31);
    one-pixel (face with class 11 left on exactly one pixel per sample: the first, the last or an inner one)."""
    if kind == "iid":
        return torch.randint(0, ncls, (b, h, w), generator=g, dtype=torch.uint8)
    lab = face_labels(b, h, w, roll)
    if kind == "face32":
        lab[lab == 3] = 31
    elif kind == "one-pixel":
        lab[lab == 11] = 0
        for i in range(b):
            q = (0 if i % 3 == 0 else h * w - 1 if i % 3 == 1 else (37 * i) % (h * w))
            lab[i].view(-1)[q] = 11
    return lab


def row_list(label, ncls, h, w):
    """need / base / count / rows of one sample as the masked transposed convolution's row-list kernel builds them: T'
    pixel (m, n) needs every region of the clipped output window [2m-2, 2m+2] x [2n-2, 2n+2]; rows are numbered in
    (m, n, region) order."""
    need = [[0] * (w + 1) for _ in range(h + 1)]
    base = [[0] * (w + 1) for _ in range(h + 1)]
    rows, total = [], 0
    for m in range(h + 1):
        for n in range(w + 1):
            win = region_of(label[max(2 * m - 2, 0):2 * m + 3, max(2 * n - 2, 0):2 * n + 3], ncls)
            bits = 0
            for r in win.unique().tolist():
                bits |= 1 << r
            need[m][n], base[m][n] = bits, total
            rows += [(m, n, r) for r in range(32) if (bits >> r) & 1]
            total += bin(bits).count("1")
    return need, base, rows


# ============================================================================ the layer table of the 1024 generator
RES, K_LAYERS = 1024, 13
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
