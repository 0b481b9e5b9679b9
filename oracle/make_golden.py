"""Pin the oracle against the reference itself and write tests/golden/*.npz.

Run in the BUILD container only (needs /root/reference):

    python oracle/make_golden.py

The reference's hot path is Python, so it is imported from /root/reference, never copied.  Its
two CUDA-only ops cannot run without a GPU (fused_bias_act.cpp:13 raises), so - exactly as
BASELINE.md section 2/4 describes - they are routed to the reference's OWN CPU spellings:
`upfirdn2d_native` (src/models/stylegan2/op/upfirdn2d.py:150-184, with the `F` import it forgot)
and the CPU branch of GPEN's fused_leaky_relu (src/pretrained/gpen/face_model/op/fused_act.py:96).
`torch.utils.cpp_extension.load` is stubbed so the import does not try to JIT-build CUDA code.

Every case is run through (1) the reference modules and (2) oracle/e4s_oracle.py on the same
seeded tensors; the script asserts they agree (fp32, tolerance below) and stores the REFERENCE
outputs as the golden vectors.  Inputs are regenerated from seeds by the tests, so only outputs
(and a few small inputs) are stored.
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)

from oracle import e4s_oracle as O  # noqa: E402
from oracle import golden_io  # noqa: E402

TOL = 2e-5  # max|ref-oracle| / max|ref|, fp32 CPU on both sides


def import_reference():
    import torch.utils.cpp_extension as cpp
    cpp.load = lambda *a, **k: types.SimpleNamespace()       # no JIT build, no GPU here
    sys.path.insert(0, REF)
    import src.models.stylegan2.model as M                     # noqa
    up_mod = sys.modules["src.models.stylegan2.op.upfirdn2d"]
    act_mod = sys.modules["src.models.stylegan2.op.fused_act"]
    up_mod.F = F                                               # the missing import (SURVEY App. B)

    def upfirdn2d_cpu(input, kernel, up=1, down=1, pad=(0, 0)):
        n, c, h, w = input.shape
        out = up_mod.upfirdn2d_native(input.reshape(-1, h, w, 1), kernel, up, up, down, down,
                                      pad[0], pad[1], pad[0], pad[1])
        return out.view(n, c, out.shape[1], out.shape[2])

    def fused_leaky_relu_cpu(input, bias, negative_slope=0.2, scale=2 ** 0.5):
        # body of src/pretrained/gpen/face_model/op/fused_act.py:96 (reference's own CPU branch)
        return scale * F.leaky_relu(input + bias.view((1, -1) + (1,) * (len(input.shape) - 2)),
                                    negative_slope=negative_slope)

    up_mod.upfirdn2d = upfirdn2d_cpu
    act_mod.fused_leaky_relu = fused_leaky_relu_cpu
    M.upfirdn2d = upfirdn2d_cpu
    M.fused_leaky_relu = fused_leaky_relu_cpu
    return M, upfirdn2d_cpu, fused_leaky_relu_cpu


def rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def check(name, ref, ora):
    e = rel_err(ora, ref)
    print(f"  {name:38s} ref-vs-oracle max-rel {e:.2e}  shape {tuple(ref.shape)}")
    assert e <= TOL, f"oracle disagrees with the reference on {name}: {e}"
    return e


def load_synth(module, salt=0, prefix_filter=None):
    shapes = {k: tuple(v.shape) for k, v in module.state_dict().items()}
    state = O.synthetic_state(shapes, salt)
    module.load_state_dict(state)
    return state


def main():
    os.makedirs(OUT, exist_ok=True)
    torch.manual_seed(0)
    torch.set_grad_enabled(False)
    M, ref_upfirdn2d, ref_flrelu = import_reference()
    gold = {}

    # ---------------------------------------------------------------- upfirdn2d
    print("upfirdn2d")
    fir4 = O.make_fir((1, 3, 3, 1), 4.0)
    fir1 = O.make_fir((1, 3, 3, 1), 1.0)
    cases = [  # (tag, N, C, H, W, fir, up, down, pad)
        ("blur_up", 2, 5, 17, 17, fir4, 1, 1, (1, 1)),       # Blur after stride-2 convT, model.py:206-213
        ("skip_up", 2, 3, 8, 8, fir4, 2, 1, (2, 1)),         # Upsample of RGB skip, model.py:42-47
        ("blur_dn", 1, 4, 16, 16, fir1, 1, 1, (2, 2)),       # Blur before stride-2 conv (D), model.py:215-221
        ("down2", 1, 3, 16, 16, fir1, 1, 2, (1, 1)),         # Downsample, model.py:56-75
        ("ragged", 3, 2, 7, 13, fir4, 2, 1, (2, 1)),         # non-square, odd sizes
        ("crop", 1, 2, 9, 9, fir1, 1, 1, (-1, 0)),           # negative pad = crop (upfirdn2d.py:166-171)
    ]
    g = torch.Generator().manual_seed(10)
    for tag, n, c, h, w, fir, up, down, pad in cases:
        x = torch.randn(n, c, h, w, generator=g)
        r = ref_upfirdn2d(x, fir, up=up, down=down, pad=pad)
        check("upfirdn2d/" + tag, r, O.upfirdn2d(x, fir, up, down, pad))
        gold[f"upfirdn2d/{tag}/x"] = x.numpy()
        gold[f"upfirdn2d/{tag}/y"] = r.numpy()
        gold[f"upfirdn2d/{tag}/cfg"] = np.array([up, down, pad[0], pad[1], float(fir.sum())], dtype=np.float64)
    # asymmetric FIR proves the op is a true convolution (kernel flip, upfirdn2d_kernel.cu:77)
    fir_asym = torch.tensor([[1., 2., 0., -1.], [0.5, 3., 1., 0.], [0., 1., 4., 2.], [-2., 0., 1., 1.]]) / 7
    x = torch.randn(1, 2, 6, 6, generator=g)
    r = ref_upfirdn2d(x, fir_asym, up=2, down=1, pad=(2, 1))
    check("upfirdn2d/asym", r, O.upfirdn2d(x, fir_asym, 2, 1, (2, 1)))
    gold["upfirdn2d/asym/x"], gold["upfirdn2d/asym/y"], gold["upfirdn2d/asym/fir"] = x.numpy(), r.numpy(), fir_asym.numpy()

    # ------------------------------------------------------- fused_leaky_relu
    print("fused_leaky_relu")
    x = torch.randn(2, 6, 5, 7, generator=g)
    b = torch.randn(6, generator=g)
    r = ref_flrelu(x, b)
    check("fused_leaky_relu/fwd", r, O.fused_leaky_relu(x, b))
    gold["flrelu/x"], gold["flrelu/b"], gold["flrelu/y"] = x.numpy(), b.numpy(), r.numpy()
    with torch.enable_grad():
        xg, bg = x.clone().requires_grad_(True), b.clone().requires_grad_(True)
        go = torch.randn(2, 6, 5, 7, generator=g)
        yy = ref_flrelu(xg, bg)
        yy.backward(go)
    gx, gb = O.fused_leaky_relu_backward(go, r)
    check("fused_leaky_relu/grad_x", xg.grad, gx)
    check("fused_leaky_relu/grad_b", bg.grad, gb)
    gold["flrelu/go"], gold["flrelu/gx"], gold["flrelu/gb"] = go.numpy(), xg.grad.numpy(), bg.grad.numpy()

    # ------------------------------------------------ ModulatedConv2d variants
    print("ModulatedConv2d / StyledConv / ToRGB")
    for tag, (cin, cout, k, demod, up, hw) in O.MODCONV_CASES.items():
        m = M.ModulatedConv2d(cin, cout, k, 512, demodulate=demod, upsample=up)
        st = load_synth(m, salt=len(tag))
        x, w = O.modconv_case(tag)
        r = m(x, w)
        o = O.modulated_conv2d(x, w, st["weight"], st["modulation.weight"], st["modulation.bias"], demod, up)
        check("modconv/" + tag, r, o)
        gold[f"modconv/{tag}/y"] = r.numpy()

    for tag, (cin, cout, up, hw) in O.STYLEDCONV_CASES.items():
        m = M.StyledConv(cin, cout, 3, 512, upsample=up, mask_op=True)
        st = load_synth(m, salt=7 + len(tag))
        x, nz, codes, mask = O.styledconv_case(tag)
        r = m(x, codes[:, :, 0], mask, noise=nz)
        o = O.styled_conv(x, codes[:, :, 0], mask, nz, st, "", up, True)
        check("styledconv_masked/" + tag, r, o)
        gold[f"styledconv/{tag}/y"] = r.numpy()
    m = M.ToRGB(24, 512, upsample=True, mask_op=True)
    st = load_synth(m, salt=11)
    x, skip, codes, mask = O.torgb_case()
    r = m(x, codes[:, :, 1], mask, skip)
    check("torgb_masked", r, O.to_rgb(x, codes[:, :, 1], mask, skip, st, "", True))
    gold["torgb/y"] = r.numpy()

    # ------------------------------------------------------------- Generator
    print("Generator")
    for tag, size, K, B, nc, msz, kind in [("g64_k5", 64, 5, 2, 5, 32, "blobs"),
                                           ("g32_k13_iid", 32, 13, 1, 12, 64, "iid"),
                                           ("g256_k13", 256, 13, 1, 12, 512, "blobs")]:
        G = M.Generator(size, 512, 8, split_layer_idx=5, remaining_layer_idx=K).eval()
        st = load_synth(G, salt=size)
        codes, mask, label, noise = O.synthetic_inputs(B, nc, size, msz, seed=size + K, kind=kind)
        img, _, feats = G([codes], None, mask, input_is_latent=True, noise=noise)
        oi, of = O.generator_forward(st, codes, mask, noise, size, K)
        check(f"generator/{tag}/image", img, oi)
        check(f"generator/{tag}/feats", feats, of)
        gold[f"generator/{tag}/image"] = img.numpy()
        gold[f"generator/{tag}/feats_absmean"] = np.array(float(feats.abs().mean()))
        gold[f"generator/{tag}/feats_sub"] = feats[:, ::16, ::2, ::2].numpy()
        if tag == "g32_k13_iid":
            # first-order gradients of a fixed linear functional wrt the latent codes and the noise
            with torch.enable_grad():
                cg = codes.clone().requires_grad_(True)
                R = torch.randn(img.shape, generator=torch.Generator().manual_seed(99))
                gi, _, _ = G([cg], None, mask, input_is_latent=True, noise=noise)
                (gi * R).sum().backward()
                og = codes.clone().requires_grad_(True)
                oi2, _ = O.generator_forward(st, og, mask, noise, size, K)
                (oi2 * R).sum().backward()
            check(f"generator/{tag}/dcodes", cg.grad, og.grad)
            gold[f"generator/{tag}/dcodes"] = cg.grad.numpy()
        del G

    # --------------------------------------------------- Net3: MLPs + encoder
    print("Net3 cal_style_codes / get_style_vectors")
    import src.models.networks as N
    opts = types.SimpleNamespace(fsencoder_type="psp", remaining_layer_idx=13, num_seg_cls=12, out_size=64,
                                 train_G=False, start_from_latent_avg=True, learn_in_w=False)
    net = N.Net3(opts).eval()
    st = load_synth(net, salt=5)
    sv, latent_avg, img, mask = O.net3_case()
    net.latent_avg = latent_avg
    r = net.cal_style_codes(sv)
    check("cal_style_codes", r, O.cal_style_codes(st, sv, net.latent_avg, 13))
    gold["net3/style_codes_sub"] = r[:, :, :, ::8].numpy()
    vec, struct = net.get_style_vectors(img, mask)
    ov, ostruct = O.get_style_vectors(st, img, mask)
    check("get_style_vectors", vec, ov)
    assert struct.shape == ostruct.shape and float(struct.abs().max()) == 0.0
    gold["net3/style_vectors"] = vec.numpy()
    feats, m5 = O.region_mean_case()
    r = net.encoder.get_per_comp_styleCode(feats, m5)
    check("region_mean", r, O.region_mean(feats, m5))
    gold["region_mean/y"] = r.numpy()

    # ------------------------------------------------------ bit-exact mask ops
    print("mask / index ops")
    for missing in ("matplotlib", "matplotlib.pyplot"):      # absent here; torch_utils only plots with it
        sys.modules.setdefault(missing, types.ModuleType(missing))
    from src.utils.torch_utils import labelMap2OneHot
    lab = torch.randint(0, 12, (2, 1, 9, 11), generator=g)
    assert torch.equal(labelMap2OneHot(lab, 12), O.label_to_onehot(lab, 12))
    import src.datasets.dataset as D
    from PIL import Image
    conv = getattr(D, "__celebAHQ_masks_to_faceParser_mask_detailed")
    for who in ("source", "target"):
        raw = np.array(Image.open(f"{REF}/example/input/faceswap/{who}_mask.png"))
        c12 = conv(raw)
        gold[f"mask/{who}_raw19"] = raw.astype(np.uint8)
        gold[f"mask/{who}_cls12"] = c12.astype(np.uint8)
    m = torch.rand(1, 3, 24, 24, generator=g)
    for s in (4, 8, 12, 48, 96):
        assert torch.equal(F.interpolate(m, size=(s, s), mode="nearest"), O.nearest_resize(m, s))

    paths = golden_io.save(os.path.join(OUT, "reference_vectors.npz"), gold)
    print(f"wrote {len(gold)} arrays -> " + ", ".join(f"{os.path.relpath(p, ROOT)} ({os.path.getsize(p) / 1e6:.2f} MB)" for p in paths))


if __name__ == "__main__":
    main()
