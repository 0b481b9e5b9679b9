"""The up-sampling layers' transposed-convolution GEMMs against float64 at the edges of the gathered-row schedule and of
the row cap (csrc/wgmma_convt.cu): the masked entry e4s_modconv3x3_up_masked_tcr_fwd (row-list kernel, rows_rs_kernel,
region-aware blur pass, folded fallback for the samples over the cap) and the unmasked entry
e4s_modconv3x3_up_tcr_fwd (convt_rs_kernel and blur pass).

Every masked case builds its label maps here and asserts the property that makes it a case - a sample with exactly
(H+1)(W+1), 128 k, 128 k + 1, cap or cap + 1 rows, where the samples over the cap sit in the batch, non-square or odd
sides, labels >= ncls - so that a change of the cap rule or the width rule cannot turn it into an ordinary one.

The masked entry is called through the C ABI with its own need / base / count / rows lists (filled with -1) and NaN-filled
T'c and output buffers: an item no CTA takes, a row the list kernel does not write or a pixel that neither the blur pass
nor the folded kernel writes stays non-finite.  T'c (the raw GEMM output) and the layer output are both compared with
float64: T'c with the stride-2 transposed convolution of x * s[region] of each listed row, the output with
f64ref.styled_conv_per_pixel (f64ref.styled_preact where demodulation, bias or activation is off).

share_layout restates how launch_rows and rows_rs_kernel split a launch's K steps over the persistent CTAs.  It only
selects and labels cases (and names the CTA of an item a failure points at); no kernel result is checked against it."""
import math
import zlib
from bisect import bisect_left, bisect_right
from collections import namedtuple
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err, rel_rms
from f64ref import act, default_kernels, labels, modconv_case, row_counts, row_list, styled_conv_per_pixel  # noqa: F401
from f64ref import styled_preact
from test_synthesis_at_scale import TOL_CONV

DEV = "cuda:0"
TOL = TOL_CONV            # the StyledConv bar of the at-scale synthesis check; T'c is held to it too
M_ROWS, KC = 128, 32      # rows per row block and channels per K step of the gathered-row GEMM (wgmma_conv::M, KC)
ROW_NBITS = 13            # wgmma_conv::row_pack: m << (ROW_NBITS + 5) | n << 5 | region
BLUR_ROWS, BLUR_PIX = 32, 4   # output rows per thread of the unmasked blur pass, output pixels per thread of the masked one
H100_SMS = 132            # H100 SXM; share layouts are computed with the device's own count when there is one

WORST = {}                # entry -> (max-rel, rel-RMS, case) of the largest error seen


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nlargest error against float64 per entry (max-rel, rel-RMS, case):")
        for k in sorted(WORST):
            e, r, case = WORST[k]
            print(f"  {k:28s} {e:.2e}  {r:.2e}  {case}")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else H100_SMS


def _cap(h, w):
    from e4s_b200.kernels import convt_masked_cap
    return convt_masked_cap(h, w)


# ============================================================================ share layout (host model)
Item = namedtuple("Item", "b rb cls sl s n")                  # n K steps from step s of the launch
Cta = namedtuple("Cta", "i lo hi first inside")               # first: index of the first item it takes (or None);
                                                              # inside: index of the item whose steps hold lo (or None)


def rows_ntile(cout, row_blocks, sms, forced=None):
    """pick_ntile_rows: the N-tile width of the gathered-row GEMM; row_blocks counted to the cap (ceil(cap / 128) B)."""
    if forced in (64, 128) and cout % forced == 0:
        return forced
    if cout % 128 == 0 and row_blocks * 4 * (cout // 128) >= 2 * sms:
        return 128
    return 64 if cout % 64 == 0 else 32


def share_layout(counts, cap, cin, cout, nt, sms):
    """launch_rows and rows_rs_kernel's partition: grid = min(items counted to the cap, SMs); the items, in the order sample,
    row block holding rows (none for a sample over the cap), class, slice; each CTA's share [lo, hi) = [total i / grid,
    total (i + 1) / grid) of the launch's K steps, and the items that start inside it."""
    nsl, nchunks = cout // nt, cin // KC
    blocks = [-(-c // M_ROWS) if c <= cap else 0 for c in counts]
    grid = min(-(-cap // M_ROWS) * len(counts) * 4 * nsl, sms)
    items, s = [], 0
    for b, nb in enumerate(blocks):
        for rb in range(nb):
            for k in range(4 * nsl):
                n = (4 >> bin(k // nsl).count("1")) * nchunks
                items.append(Item(b, rb, k // nsl, k % nsl, s, n))
                s += n
    total = s
    assert total == sum(blocks) * 9 * nchunks * nsl
    starts = [it.s for it in items]
    ctas = []
    for i in range(grid):
        lo, hi = total * i // grid, total * (i + 1) // grid
        j = bisect_left(starts, lo)
        first = j if j < len(items) and starts[j] < hi else None
        k = bisect_right(starts, lo) - 1
        inside = k if lo < total and k >= 0 and starts[k] < lo < starts[k] + items[k].n else None
        ctas.append(Cta(i, lo, hi, first, inside))
    return SimpleNamespace(grid=grid, total=total, nt=nt, nsl=nsl, nchunks=nchunks, items=items, ctas=ctas,
                           owner={(it.b, it.rb, it.cls, it.sl): _owner(ctas, it.s) for it in items})


def _owner(ctas, s):
    return [c.i for c in ctas if c.lo <= s < c.hi]


def layout_properties(lay):
    """Which of the schedule's edges the layout reaches."""
    empty = any(c.lo == c.hi for c in lay.ctas)
    in00 = any(c.inside is not None and lay.items[c.inside].cls == 0 for c in lay.ctas)
    in11 = any(c.inside is not None and lay.items[c.inside].cls == 3 for c in lay.ctas)
    within = any(c.lo < c.hi and c.inside is not None and c.hi <= lay.items[c.inside].s + lay.items[c.inside].n
                 for c in lay.ctas)
    return {"empty share": empty, "share begins in a class-(0, 0) chain": in00,
            "share begins in a class-(1, 1) chain": in11, "share inside one item": within}


def describe(lay):
    cls = ("(0, 0)", "(0, 1)", "(1, 0)", "(1, 1)")

    def item(j):
        it = lay.items[j]
        return f"item {j} (sample {it.b}, block {it.rb}, class {cls[it.cls]}, slice {it.sl}, steps {it.s}+{it.n})"
    lines = [f"  grid {lay.grid}, {len(lay.items)} items, {lay.total} K steps, N tile {lay.nt} ({lay.nsl} slices), "
             f"{lay.nchunks} chunks"]
    for c in lay.ctas:
        where = (f"starts at {item(c.first)}" if c.first is not None else "takes no item") + (
            f"; lo inside {item(c.inside)}" if c.inside is not None else "")
        lines.append(f"  CTA {c.i}: [{c.lo}, {c.hi}) {'empty' if c.lo == c.hi else where}")
    return "\n".join(lines)


# ============================================================================ label maps with the counts that make the cases
def _count(lab, ncls):
    return int(row_counts(lab[None], ncls)[0])


def map_with_rows(h, w, ncls, target, seed):
    """A [2H, 2W] label map whose gathered list has exactly `target` rows.  A blob map (one region where the blobs alone
    have more rows) has its first p raster pixels replaced by iid labels, p the largest that stays at or below the target
    (by bisection); then greedy single-pixel edits: of 256 random ones (half on the border, where a pixel reaches fewer
    T' pixels and adds fewer rows) the one that adds the most rows without passing the target, until the count is exact."""
    g = torch.Generator().manual_seed(seed)
    ho, wo = 2 * h, 2 * w
    lab = labels("blobs", 1, ho, wo, ncls, g)[0]
    if _count(lab, ncls) > target:
        lab = torch.zeros_like(lab)
    iid = torch.randint(0, ncls, lab.shape, generator=g, dtype=torch.uint8)

    def prefix(p):
        out = lab.clone().view(-1)
        out[:p] = iid.view(-1)[:p]
        return out.view(ho, wo)
    lo, hi = 0, lab.numel()
    if _count(prefix(hi), ncls) <= target:
        lo = hi
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if _count(prefix(mid), ncls) <= target else (lo, mid)
    lab = prefix(lo)
    c = _count(lab, ncls)
    n = 256
    for _ in range(400):
        if c == target:
            return lab
        ys, xs = torch.randint(0, ho, (n,), generator=g), torch.randint(0, wo, (n,), generator=g)
        side, odd = torch.randint(0, 4, (n,), generator=g), torch.arange(n) % 2 == 1
        ys = torch.where(odd & (side == 0), 0, torch.where(odd & (side == 1), ho - 1, ys))
        xs = torch.where(odd & (side == 2), 0, torch.where(odd & (side == 3), wo - 1, xs))
        trials = lab.expand(n, ho, wo).clone()
        trials[torch.arange(n), ys, xs] = torch.randint(0, ncls, (n,), generator=g, dtype=torch.uint8)
        ct = row_counts(trials, ncls)
        ok = (ct > c) & (ct <= target)
        if bool(ok.any()):
            j = int(torch.where(ok, ct, -1).argmax())
            lab, c = trials[j].clone(), int(ct[j])
    raise AssertionError(f"no map with {target} rows at {h}x{w}, ncls {ncls} (stuck at {c})")


def _target(spec, h, w):
    """Row count a sample spec asks for, or None for a drawn map."""
    cap, region = _cap(h, w), (h + 1) * (w + 1)
    if isinstance(spec, int):
        return spec
    return {"cap": cap, "cap+1": cap + 1, "128k": (cap - 1) // M_ROWS * M_ROWS,
            "128k+1": (cap - 1) // M_ROWS * M_ROWS + 1}.get(spec)


def sample_map(spec, h, w, ncls, seed, i):
    """One sample's [2H, 2W] uint8 map: "region" (one region everywhere: (H+1)(W+1) rows), "blobs", "face" (the committed
    face masks: sample i of a rolled batch), "iid" (over the cap), "clamp" (blobs with the regions of the last and the first pixel relabelled to 255
    and ncls + 5, which count as the last region), or a row count: an int, "cap", "cap+1", "128k" (the largest multiple of 128 below the cap) or "128k+1"
    (a last row block holding one row)."""
    g = torch.Generator().manual_seed(seed)
    ho, wo = 2 * h, 2 * w
    t = _target(spec, h, w)
    if t is not None:
        return map_with_rows(h, w, ncls, t, seed)
    if spec == "region":
        return torch.full((ho, wo), seed % ncls, dtype=torch.uint8)
    if spec == "clamp":
        lab = labels("blobs", 1, ho, wo, ncls, g)[0]
        first, last = int(lab[0, 0]), int(lab[-1, -1])
        lab[lab == last] = 255
        if ncls > 2 and first != last:
            lab[lab == first] = ncls + 5
        return lab
    if spec == "face":
        return labels("face", i + 1, ho, wo, ncls, g, roll=True)[i]
    return labels(spec, 1, ho, wo, ncls, g)[0]


# name, batch, Cin, Cout, input H x W, ncls, one label spec per sample
Case = namedtuple("Case", "name b cin cout h w ncls samples")
MASKED = [
    Case("1x1-one-region-B1", 1, 64, 64, 1, 1, 12, ("region",)),
    Case("1x1-over-then-cap", 2, 32, 32, 1, 1, 12, (16, "cap")),
    Case("5x19-region-128k-128k1-cap", 4, 64, 96, 5, 19, 12, ("region", "128k", "128k+1", "cap")),
    Case("19x5-over-last", 3, 128, 64, 19, 5, 12, ("blobs", "cap", "cap+1")),
    Case("13x7-over-first-cin32", 3, 32, 128, 13, 7, 12, ("cap+1", "128k+1", "blobs")),
    Case("11x9-alternating-cout160", 4, 64, 160, 11, 9, 12, ("iid", "blobs", "iid", "128k")),
    Case("9x9-sparse-cin32-cout32", 4, 32, 32, 9, 9, 12, ("region", "iid", "iid", "iid")),
    Case("9x15-all-over", 3, 64, 64, 9, 15, 12, ("iid", "iid", "cap+1")),
    Case("7x3-all-over-B1", 1, 64, 32, 7, 3, 12, ("iid",)),
    Case("10x13-ncls32-clamped", 2, 64, 64, 10, 13, 32, ("clamp", "clamp")),
    Case("6x11-ncls2-cout256", 3, 64, 256, 6, 11, 2, ("blobs", "clamp", "region")),
    Case("17x29-default-128", 6, 64, 128, 17, 29, 12, ("face",) * 5 + ("cap",)),
    # (H+1)(W+1) > LIST_THREADS: the row-list kernel counts over two 1024-pixel chunks and stops after the one past the cap
    Case("47x21-two-list-chunks", 3, 64, 64, 47, 21, 12, ("cap+1", "128k+1", "cap")),
    Case("128x128-c10-class", 4, 256, 128, 128, 128, 12, ("face",) * 4),
]
BY_NAME = {c.name: c for c in MASKED}
# cases run again at each width E4S_B200_RS_NTILE can force (Cout 128 and 256)
FORCED = [("13x7-over-first-cin32", 64), ("13x7-over-first-cin32", 128), ("6x11-ncls2-cout256", 64),
          ("6x11-ncls2-cout256", 128)]

_MAPS = {}


def case_labels(case):
    """[B, 2H, 2W] uint8 maps of a case (built once)."""
    if case.name not in _MAPS:
        _MAPS[case.name] = torch.stack([sample_map(spec, case.h, case.w, case.ncls, zlib.crc32(f"{case.name}/{i}".encode()), i)
                                        for i, spec in enumerate(case.samples)])
    return _MAPS[case.name].clone()


def case_layout(case, counts, forced=None, sms=None):
    sms = sms or _sms()
    cap = _cap(case.h, case.w)
    nt = rows_ntile(case.cout, -(-cap // M_ROWS) * case.b, sms, forced)
    return share_layout([int(c) for c in counts], cap, case.cin, case.cout, nt, sms)


def _over(spec, h, w):
    t = _target(spec, h, w)
    return spec == "iid" if t is None else t > _cap(h, w)


@pytest.mark.parametrize("case", MASKED, ids=[c.name for c in MASKED])
def test_case_has_its_property(case):
    """Every sample's row count is the one its spec names; drawn maps sit on the side of the cap their spec says."""
    lab = case_labels(case)
    counts = row_counts(lab, case.ncls).tolist()
    cap = _cap(case.h, case.w)
    assert len(case.samples) == case.b and lab.shape == (case.b, 2 * case.h, 2 * case.w)
    for i, spec in enumerate(case.samples):
        t = _target(spec, case.h, case.w)
        if t is not None:
            assert counts[i] == t, (case.name, i, spec, counts[i], t)
        elif spec == "region":
            assert counts[i] == (case.h + 1) * (case.w + 1)
        assert (counts[i] > cap) == _over(spec, case.h, case.w), (case.name, i, spec, counts[i], cap)
        if spec == "128k":
            assert counts[i] % M_ROWS == 0 and counts[i] >= (case.h + 1) * (case.w + 1)
        if spec == "128k+1":
            assert counts[i] % M_ROWS == 1
        if spec == "clamp":
            assert int(lab[i].max()) >= case.ncls
    print(f"{case.name}: cap {cap}, rows {counts}")


def test_case_list_covers_the_boundaries():
    """The cases include every boundary the schedule and the blur passes have, and in the share model every item of every
    case is started by exactly one CTA."""
    def counts(c):
        return row_counts(case_labels(c), c.ncls).tolist()
    props = {c.name: counts(c) for c in MASKED}
    caps = {c.name: _cap(c.h, c.w) for c in MASKED}

    def over(c):
        return [n > caps[c.name] for n in props[c.name]]
    assert any(caps[c.name] in props[c.name] for c in MASKED), "count == cap"
    assert any(caps[c.name] + 1 in props[c.name] for c in MASKED), "count == cap + 1"
    assert any((c.h + 1) * (c.w + 1) in props[c.name] for c in MASKED), "one region"
    assert any(any(n <= caps[c.name] and n % M_ROWS == 0 for n in props[c.name]) for c in MASKED), "128 k"
    assert any(any(n <= caps[c.name] and n % M_ROWS == 1 for n in props[c.name]) for c in MASKED), "128 k + 1"
    assert any(c.b > 1 and all(over(c)) for c in MASKED), "every sample over the cap"
    assert any(c.b == 1 and all(over(c)) for c in MASKED) and any(c.b == 1 and not any(over(c)) for c in MASKED), "B = 1"
    assert any(c.b > 1 and over(c)[0] and not all(over(c)) for c in MASKED), "over the cap first"
    assert any(c.b > 1 and over(c)[-1] and not all(over(c)) for c in MASKED), "over the cap last"
    assert any(c.b > 3 and over(c)[0::2] == [True] * len(over(c)[0::2]) and not any(over(c)[1::2]) for c in MASKED), \
        "alternating"
    assert any(c.h != c.w and c.h > c.w for c in MASKED) and any(c.h != c.w and c.h < c.w for c in MASKED), "non-square"
    assert any((2 * c.w) % BLUR_PIX and (2 * c.h) % BLUR_ROWS for c in MASKED), "odd sides"
    assert any(c.h == c.w == 1 for c in MASKED), "1 x 1"
    assert any((c.b, c.cin, c.cout, c.h) == (4, 256, 128, 128) for c in MASKED), "c10's shape class"
    assert any(c.cin == 32 for c in MASKED), "Cin 32"
    assert {32, 64, 96, 128, 160, 256} <= {c.cout for c in MASKED}, "Cout"
    assert {2, 12, 32} <= {c.ncls for c in MASKED}, "ncls"
    assert any(c.ncls == 32 and int(case_labels(c).max()) >= 32 for c in MASKED), "ncls 32 with clamped labels"

    found = dict.fromkeys(layout_properties(case_layout(MASKED[0], props[MASKED[0].name])), False)
    for c in MASKED:
        for forced in [None] + [nt for name, nt in FORCED if name == c.name]:
            lay = case_layout(c, props[c.name], forced)
            for key, took in lay.owner.items():
                assert len(took) == 1, f"{c.name}: item {key} started by CTAs {took}\n{describe(lay)}"
            for k, v in layout_properties(lay).items():
                found[k] |= v
    assert all(found.values()), found
    assert rows_ntile(128, -(-_cap(17, 29) // M_ROWS) * 6, _sms()) == 128, "17x29-default-128 picks 128 by default"


# ============================================================================ float64 references
def _scaled(w):
    return w.double() / math.sqrt(w[0].numel())


def tprime(x, s, ws):
    """T' of one sample in float64: the stride-2 transposed convolution of x * s (x [Cin, H, W], s [Cin]) on the
    (H + 1) x (W + 1) grid, [H + 1, W + 1, 4 Cout], class (a, c) = T[2m + a, 2n + c] at columns (2a + c) Cout + o, zero
    past 2H, 2W."""
    t = F.pad(F.conv_transpose2d((x * s[:, None, None])[None], ws.transpose(0, 1), stride=2)[0], (0, 1, 0, 1))
    cout, hh, ww = t.shape
    return t.view(cout, hh // 2, 2, ww // 2, 2).permute(1, 3, 2, 4, 0).reshape(hh // 2, ww // 2, 4 * cout)


def _note(entry, e, r, case):
    if entry not in WORST or not e <= WORST[entry][0]:
        WORST[entry] = (e, r, case)


def check_f64(ours, ref, entry, case, tol=TOL, samples=None):
    """Both of conftest.assert_close's norms, every sample (dim 0; numbered by samples) against its own maximum."""
    assert bool(torch.isfinite(ours).all()), f"{case} {entry}: non-finite values"
    for i in range(ours.shape[0]):
        e, r = rel_err(ours[i], ref[i]), rel_rms(ours[i], ref[i])
        what = f"{case} {entry} sample {i if samples is None else samples[i]}"
        print(f"{what}: max-rel {e:.2e} rel-RMS {r:.2e} (bar {tol:.0e})")
        _note(entry, e, r, what)
        assert e <= tol and r <= tol, f"{what}: max-rel {e:.3e} rel-RMS {r:.3e} over {tol:.1e}"


def layer_ref(c, act_on=True, noise=True, demod=True, bias=True):
    """The StyledConv output in float64, NCHW: the per-pixel form with demodulation, bias and activation, else
    styled_preact (the per-region form) with those that are on."""
    x = c.x.permute(0, 3, 1, 2)
    nz, nw = (c.noise, c.nw) if noise else (None, None)
    if demod and bias and act_on and noise:
        return styled_conv_per_pixel(x, c.s, c.w, c.label, nz, nw, c.bias, True)
    pre = styled_preact(x, c.s, c.w, c.label, nz, nw, c.bias if bias else None, True, demod)
    return act(pre) if act_on else pre


# ============================================================================ GPU: the masked entry
def masked_direct(c, act_on=True, noise=True):
    """e4s_modconv3x3_up_masked_tcr_fwd through the C ABI on lists filled with -1 and NaN-filled T'c and output."""
    from e4s_b200 import _lib
    from e4s_b200._lib import check, ptr, stream_ptr
    b, h, w, cin = c.x.shape
    cout, ncls, cap = c.prep.w_convt_hilo.shape[3] // 4, c.s.shape[1], _cap(h, w)
    i32 = dict(device=DEV, dtype=torch.int32)
    r = SimpleNamespace(need=torch.full((b, h + 1, w + 1), -1, **i32), base=torch.full((b, h + 1, w + 1), -1, **i32),
                        count=torch.full((b,), -1, **i32), rows=torch.full((b, cap), -1, **i32),
                        t=torch.full((b, cap, 4 * cout), float("nan"), device=DEV),
                        y=torch.full((b, 2 * h, 2 * w, cout), float("nan"), device=DEV))
    nz, nw = (c.noise, c.nw) if noise else (None, None)
    rc = _lib.load().e4s_modconv3x3_up_masked_tcr_fwd(
        ptr(c.x), ptr(c.prep.w_convt_hilo), ptr(c.prep.w_hilo), ptr(c.prep.fir), ptr(c.s), ptr(c.dm), ptr(c.label),
        ptr(nz), ptr(nw), ptr(c.bias), ptr(r.need), ptr(r.base), ptr(r.count), ptr(r.rows), ptr(r.t), ptr(r.y), b, h, w,
        cin, cout, ncls, cap, nz.shape[0] if noise else 1, int(act_on), stream_ptr())
    check(rc, "e4s_modconv3x3_up_masked_tcr_fwd")
    torch.cuda.synchronize()
    return r


def masked_wrapper(c, act_on=True, noise=True):
    from e4s_b200 import kernels as K
    return K.modconv3x3_up_masked_tcr_fwd(c.x, c.prep.w_convt_hilo, c.prep.w_hilo, c.prep.fir, c.s, c.dm, c.label,
                                          c.noise if noise else None, c.nw if noise else None, c.bias, act_on)


def build_case(case, seed=None, noise_b=None, demod=True, bias=True):
    c = modconv_case(case.b, case.cin, case.cout, case.h, case.w, case.ncls, "blobs", up=True,
                     noise_b=case.b if noise_b is None else noise_b, demod=demod, bias=bias,
                     seed=zlib.crc32(case.name.encode()) if seed is None else seed, device=DEV)
    c.lab_cpu = case_labels(case)
    c.label = c.lab_cpu.to(DEV).contiguous()
    return c


def check_lists_and_tprime(c, r, lay, name):
    """count, need, base and rows against the host row list; T'c written exactly on the listed rows of the samples within
    the cap (nowhere for the others) and equal to the float64 T' of each row's region."""
    b, h, w, _ = c.x.shape
    ncls, cap, cout = c.s.shape[1], _cap(h, w), r.t.shape[2] // 4
    host = row_counts(c.lab_cpu, ncls).tolist()
    count, need, base, rows = (v.cpu().long() for v in (r.count, r.need, r.base, r.rows))
    print(f"{name}: cap {cap}, host rows {host}, device count {count.tolist()}")
    ws = _scaled(c.w).to(DEV)
    x = c.x.permute(0, 3, 1, 2).double()
    for i in range(b):
        if host[i] > cap:
            # an overflowing list stops counting after the 1024-pixel chunk that passes the cap
            assert cap < int(count[i]) <= host[i], (name, i, int(count[i]), host[i])
            assert bool(r.t[i].isnan().all()), f"{name}: T'c of sample {i} (over the cap) written"
            continue
        n = host[i]
        assert int(count[i]) == n, (name, i, int(count[i]), n)
        need_ref, base_ref, rows_ref = row_list(c.lab_cpu[i], ncls, h, w)
        assert torch.equal(need[i] & 0xFFFFFFFF, torch.tensor(need_ref)), f"{name}: need of sample {i}"
        assert torch.equal(base[i], torch.tensor(base_ref)), f"{name}: base of sample {i}"
        packed = torch.tensor([(m << (ROW_NBITS + 5)) | (nn << 5) | g for m, nn, g in rows_ref], dtype=torch.long)
        assert torch.equal(rows[i, :n] & 0xFFFFFFFF, packed), f"{name}: rows of sample {i}"
        assert bool((rows[i, n:] == -1).all()), f"{name}: rows written past the count of sample {i}"
        assert bool(r.t[i, n:].isnan().all()), f"{name}: T'c written past the count of sample {i}"
        bad = (~torch.isfinite(r.t[i, :n])).nonzero()
        if bad.numel():
            row, col = (int(v) for v in bad[0])
            key = (i, row // M_ROWS, col // cout, (col % cout) // lay.nt)
            raise AssertionError(f"{name}: T'c row {row} column {col} of sample {i} not written: item (sample, block, "
                                 f"class, slice) {key}, started by CTAs {lay.owner.get(key)}\n{describe(lay)}")
        mi, ni, gi = (torch.tensor(v, device=DEV) for v in zip(*rows_ref))
        ref = torch.empty(n, 4 * cout, dtype=torch.float64, device=DEV)
        for g in gi.unique().tolist():
            sel = gi == g
            ref[sel] = tprime(x[i], c.s[i, g].double(), ws)[mi[sel], ni[sel]]
        check_f64(r.t[i, :n][None], ref[None], "masked T'c", name, samples=[i])


def run_masked(case, monkeypatch, forced=None):
    if forced is not None:
        monkeypatch.setenv("E4S_B200_RS_NTILE", str(forced))
    c = build_case(case)
    lay = case_layout(case, row_counts(c.lab_cpu, case.ncls).tolist(), forced)
    name = case.name + (f" N tile {forced}" if forced else "")
    print(f"{name}: share layout\n{describe(lay)}")
    r = masked_direct(c)
    check_lists_and_tprime(c, r, lay, name)
    check_f64(r.y.permute(0, 3, 1, 2), layer_ref(c), "masked y", name)
    assert torch.equal(masked_wrapper(c), r.y), f"{name}: the wrapper's output differs from the direct call's"
    return r.y


@pytest.mark.gpu
@pytest.mark.parametrize("case", MASKED, ids=[c.name for c in MASKED])
def test_masked_entry_against_float64(case, monkeypatch):
    run_masked(case, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("name,nt", FORCED, ids=[f"{n}-N{nt}" for n, nt in FORCED])
def test_masked_entry_at_forced_widths(name, nt, monkeypatch):
    """The widths E4S_B200_RS_NTILE forces, against float64 and bit for bit against the default width."""
    y = run_masked(BY_NAME[name], monkeypatch, nt)
    monkeypatch.delenv("E4S_B200_RS_NTILE")
    assert torch.equal(y, masked_wrapper(build_case(BY_NAME[name])))


EPILOGUE = Case("7x13-epilogue", 3, 64, 64, 7, 13, 12, ("blobs", "cap", "iid"))


@pytest.mark.gpu
@pytest.mark.parametrize("noise_b", ["1", "B"])
@pytest.mark.parametrize("demod,bias,act_on", [(True, True, True), (False, False, False), (True, False, True),
                                               (False, True, False)])
def test_masked_epilogue_inputs_against_float64(noise_b, demod, bias, act_on):
    """Per-sample and broadcast noise, no noise, and demodulation, bias and activation each on and off, on a batch with a
    sample at the cap (gathered) and one over it (folded)."""
    c = build_case(EPILOGUE, noise_b=1 if noise_b == "1" else EPILOGUE.b, demod=demod, bias=bias)
    name = f"{EPILOGUE.name} noise {noise_b} demod {demod} bias {bias} act {act_on}"
    for noise in (True, False):
        r = masked_direct(c, act_on, noise)
        check_f64(r.y.permute(0, 3, 1, 2), layer_ref(c, act_on, noise, demod, bias), "masked y", f"{name} noise {noise}")
        assert torch.equal(masked_wrapper(c, act_on, noise), r.y)


# ---------------------------------------------------------------------------- invariances, bit for bit
@pytest.mark.gpu
def test_permuting_the_batch_permutes_the_output():
    """A permutation moves the samples over the cap and every item's start in the launch; each output keeps its bits."""
    case = BY_NAME["11x9-alternating-cout160"]
    c = build_case(case)
    y = masked_wrapper(c)
    perm = torch.tensor([2, 0, 3, 1])
    p = build_case(case)
    p.x, p.s, p.dm, p.label, p.noise = (v[perm.to(DEV)].contiguous() for v in (c.x, c.s, c.dm, c.label, c.noise))
    assert torch.equal(masked_wrapper(p), y[perm.to(DEV)])


@pytest.mark.gpu
def test_sample_alone_equals_sample_among_overflowing_ones():
    """Sample 1 of a batch whose samples 0 and 2 overflow the cap (so all of the launch's items are sample 1's) computed
    alone: the same bits."""
    case = BY_NAME["11x9-alternating-cout160"]
    c = build_case(case)
    three = build_case(case)
    three.x, three.s, three.dm, three.label, three.noise = (v[:3].contiguous() for v in (c.x, c.s, c.dm, c.label, c.noise))
    one = build_case(case)
    one.x, one.s, one.dm, one.label, one.noise = (v[1:2].contiguous() for v in (c.x, c.s, c.dm, c.label, c.noise))
    counts = row_counts(c.lab_cpu[:3], case.ncls).tolist()
    assert counts[0] > _cap(case.h, case.w) and counts[2] > _cap(case.h, case.w) >= counts[1]
    assert torch.equal(masked_wrapper(one)[0], masked_wrapper(three)[1])


@pytest.mark.gpu
def test_64_and_128_channel_tiles_agree_where_the_default_is_128(monkeypatch):
    case = BY_NAME["17x29-default-128"]
    c = build_case(case)
    assert rows_ntile(case.cout, -(-_cap(case.h, case.w) // M_ROWS) * case.b, _sms()) == 128
    y = masked_wrapper(c)
    for nt in ("64", "128"):
        monkeypatch.setenv("E4S_B200_RS_NTILE", nt)
        assert torch.equal(masked_wrapper(c), y), f"N tile {nt}"


# ============================================================================ GPU: the unmasked entry
# batch, Cin, Cout, input H x W: non-square both ways, odd sides (2H not a multiple of BLUR_ROWS, partial pixel tiles),
# 1 x 1, several 32-channel slices
UNMASKED = [(2, 64, 64, 5, 19), (3, 32, 32, 19, 5), (2, 128, 96, 13, 7), (1, 64, 160, 1, 1), (3, 256, 128, 1, 1),
            (2, 64, 256, 23, 9)]


@pytest.mark.gpu
@pytest.mark.parametrize("stream", [False, True], ids=["resident", "streamed"])
@pytest.mark.parametrize("b,cin,cout,h,w", UNMASKED)
def test_unmasked_entry_against_float64(b, cin, cout, h, w, stream, monkeypatch):
    """e4s_modconv3x3_up_tcr_fwd through the C ABI into NaN-filled T' and output buffers: every T' pixel against the
    float64 transposed convolution, the output against float64, the wrapper bit for bit."""
    from e4s_b200 import _lib
    from e4s_b200 import kernels as K
    from e4s_b200._lib import check, ptr, stream_ptr
    if stream:
        monkeypatch.setenv("E4S_B200_RS_STREAM", "1")
    c = modconv_case(b, cin, cout, h, w, 1, None, up=True, noise_b=b, seed=b + cin + cout + h + w, device=DEV)
    t = torch.full((b, h + 1, w + 1, 4 * cout), float("nan"), device=DEV)
    y = torch.full((b, 2 * h, 2 * w, cout), float("nan"), device=DEV)
    rc = _lib.load().e4s_modconv3x3_up_tcr_fwd(ptr(c.x), ptr(c.prep.w_convt_hilo), ptr(c.prep.fir), ptr(c.s), ptr(c.dm),
                                               ptr(c.noise), ptr(c.nw), ptr(c.bias), ptr(t), ptr(y), b, h, w, cin, cout, b,
                                               1, stream_ptr())
    check(rc, "e4s_modconv3x3_up_tcr_fwd")
    torch.cuda.synchronize()
    name = f"unmasked {b}x{cin}->{cout} {h}x{w} {'streamed' if stream else 'resident'}"
    ws, x = _scaled(c.w).to(DEV), c.x.permute(0, 3, 1, 2).double()
    check_f64(t, torch.stack([tprime(x[i], c.s[i, 0].double(), ws) for i in range(b)]), "unmasked T'", name)
    check_f64(y.permute(0, 3, 1, 2), layer_ref(c), "unmasked y", name)
    assert torch.equal(K.modconv3x3_up_tcr_fwd(c.x, c.prep.w_convt_hilo, c.prep.fir, c.s, c.dm, c.noise, c.nw, c.bias, True),
                       y)
