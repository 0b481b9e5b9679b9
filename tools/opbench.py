#!/usr/bin/env python
"""Per-kernel micro-benchmarks on one GPU (CUDA events, L2 flushed between iterations).

    python tools/opbench.py [--batch 16] [--out gpurun_out/opbench.json] [--conv simt,tcr]

Reports achieved GB/s (HBM-bound kernels, algorithmic bytes) or TFLOP/s (modulated convs, algorithmic FLOPs)
against MEASURED_PEAKS.json (default: the H100 SXM data sheet).  Layer shapes are the 1024x1024 generator's (SURVEY.md
section 8d table).  Unmasked up-sampling layers are timed twice with --conv tcr: the folded parity kernel and the
transposed-convolution GEMM + blur pass ("tcr-convt"), whose two kernels are also timed apart with torch.profiler.  Masked
up-sampling layers are timed the same way ("tcr-convt-masked": row list, gathered GEMM, region-aware blur pass and the folded
fallback launch), with the source face mask or, with --iid, iid labels.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from e4s_b200 import kernels as K
from e4s_b200.stylegan2.modconv import PreparedConv
from e4s_b200.stylegan2.op import upfirdn2d, fused_leaky_relu

DEV = "cuda:0"


def timeit(fn, iters=5, warmup=2, flush=None):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()                       # > L2-sized write: evicts the previous iteration's lines
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--out", default=os.path.join(ROOT, "gpurun_out", "opbench.json"))
    ap.add_argument("--conv", default="tcr", help="comma list of auto,simt,tcr")
    ap.add_argument("--layers", default="all")
    ap.add_argument("--only-conv", action="store_true", help="skip the HBM-bound kernels")
    ap.add_argument("--only-hbm", action="store_true", help="skip the modulated convolutions")
    ap.add_argument("--once", action="store_true", help="one launch per layer, no warm-up (a single-launch profile, e.g. with torch.profiler)")
    ap.add_argument("--unmasked", action="store_true", help="time the masked layers with a single region (no class passes)")
    ap.add_argument("--iid", action="store_true", help="masked layers: iid labels instead of the face mask")
    args = ap.parse_args()
    B = args.batch
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {"hbm_gbs": 3350.0, "bf16_tflops": 989.0}
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=DEV)
    res = {"batch": B, "peaks": {k: peaks[k] for k in ("hbm_gbs", "bf16_tflops") if k in peaks}, "rows": []}

    def row(name, ms, work, unit):
        ach = work / (ms * 1e-3) / (1e9 if unit == "GB/s" else 1e12)
        peak = peaks["hbm_gbs"] if unit == "GB/s" else peaks["bf16_tflops"]
        r = {"kernel": name, "ms": round(ms, 4), "achieved": round(ach, 2), "unit": unit, "frac": round(ach / peak, 4)}
        res["rows"].append(r)
        print(json.dumps(r), flush=True)

    # ---- upfirdn2d: the blur after the last up-sampling conv (largest call of the model) and friends
    fir = torch.tensor([1., 3., 3., 1.]); fir = (torch.outer(fir, fir) / 64 * 4).to(DEV)
    hbm_rows(args, B, fir, flush, row)
    conv_rows(args, B, fir, flush, row, res)


def hbm_rows(args, B, fir, flush, row):
    if args.only_conv:
        return
    for c, h in [(32, 1025), (64, 513), (128, 257)]:
        x = torch.randn(B, c, h, h, device=DEV)
        ms = timeit(lambda: upfirdn2d(x, fir, pad=(1, 1)), flush=flush)
        row(f"upfirdn2d blur [{B},{c},{h},{h}]->{h - 1}", ms, 4.0 * B * c * (h * h + (h - 1) ** 2), "GB/s")
        del x
    x = torch.randn(B, 3, 512, 512, device=DEV)
    ms = timeit(lambda: upfirdn2d(x, fir, up=2, pad=(2, 1)), flush=flush)
    row(f"upfirdn2d up2 [{B},3,512,512]->1024", ms, 4.0 * B * 3 * (512 * 512 + 1024 * 1024), "GB/s")
    x = torch.randn(B, 32, 1024, 1024, device=DEV)
    bias = torch.randn(32, device=DEV)
    ms = timeit(lambda: fused_leaky_relu(x, bias), flush=flush)
    row(f"fused_leaky_relu [{B},32,1024,1024]", ms, 8.0 * x.numel(), "GB/s")
    del x

    # ---- ToRGB at the top resolution
    for cin, h in [(32, 1024), (64, 512)]:
        w = torch.randn(1, 3, cin, 1, 1, device=DEV)
        prep = PreparedConv().get(w, False, None)
        xpm = torch.randn(B, h, h, cin, device=DEV)
        s = torch.randn(B, 1, cin, device=DEV)
        skip = torch.randn(B, 3, h // 2, h // 2, device=DEV)
        b3 = torch.randn(3, device=DEV)
        ms = timeit(lambda: K.torgb_fwd(xpm, prep.wrgb, s, None, b3, skip, fir), flush=flush)
        row(f"torgb [{B},{h},{h},{cin}]", ms, 4.0 * B * h * h * (cin + 3), "GB/s")
        del xpm, skip



def conv_rows(args, B, fir, flush, row, res):
    if args.only_hbm:
        os.makedirs(os.path.dirname(args.out), exist_ok=True)
        json.dump(res, open(args.out, "w"), indent=1)
        return
    # ---- modulated convs, every 3x3 layer of the 1024 generator: (name, cin, cout, in_res, up, masked)
    layers = [("conv1@4", 512, 512, 4, 0, 1), ("c0^8", 512, 512, 4, 1, 1), ("c1@8", 512, 512, 8, 0, 1), ("c2^16", 512, 512, 8, 1, 1),
              ("c3@16", 512, 512, 16, 0, 1), ("c4^32", 512, 512, 16, 1, 1), ("c5@32", 512, 512, 32, 0, 1), ("c6^64", 512, 512, 32, 1, 1),
              ("c7@64", 512, 512, 64, 0, 1), ("c8^128", 512, 256, 64, 1, 1), ("c9@128", 256, 256, 128, 0, 1),
              ("c10^256", 256, 128, 128, 1, 1), ("c11@256", 128, 128, 256, 0, 1), ("c12^512", 128, 64, 256, 1, 0),
              ("c13@512", 64, 64, 512, 0, 0), ("c14^1024", 64, 32, 512, 1, 0), ("c15@1024", 32, 32, 1024, 0, 0)]
    if args.layers != "all":
        keep = set(args.layers.split(","))
        layers = [l for l in layers if l[0] in keep]
    import numpy as np
    from oracle import golden_io
    gold = golden_io.load(os.path.join(ROOT, "tests", "golden", "reference_vectors.npz"))
    face = torch.from_numpy(gold["mask/source_cls12"]).to(DEV)[None].repeat(B, 1, 1).contiguous()
    blur = fir
    total = {m: 0.0 for m in args.conv.split(",")}
    for name, cin, cout, r, up, masked in layers:
        if args.unmasked:
            masked = 0
        ncls = 12 if masked else 1
        w = torch.randn(1, cout, cin, 3, 3, device=DEV)
        prep = PreparedConv().get(w, bool(up), blur if up else None)
        xpm = torch.randn(B, r, r, cin, device=DEV)
        s = 1.0 + 0.1 * torch.randn(B, ncls, cin, device=DEV)
        ro = 2 * r if up else r
        label = K.label_resize_nearest(face, ro, ro) if masked else None
        if masked and args.iid:
            label = torch.randint(0, ncls, (B, ro, ro), device=DEV, dtype=torch.uint8)
        noise = torch.randn(B, 1, ro, ro, device=DEV)
        nw = torch.tensor([0.1], device=DEV)
        bias = torch.randn(cout, device=DEV)
        dm = K.demod(s, prep.wsq)
        flops = 2.0 * 9 * cin * cout * B * r * r
        for mode in args.conv.split(","):
            if mode in ("auto", "tcr"):             # the tensor-core kernel the generator uses
                if prep.w_hilo is None:
                    continue
                fn = lambda: K.modconv3x3_tcr_fwd(xpm, prep.w_hilo, s, dm, label, noise, nw, bias, bool(up), True)
            else:
                fn = lambda: K.modconv3x3_fwd(xpm, prep.wt, s, dm, label, noise, nw, bias, bool(up), True)
            ms = timeit(fn, iters=1, warmup=0, flush=flush) if args.once else timeit(fn, iters=3, warmup=1, flush=flush)
            total[mode] += ms
            row(f"modconv[{mode}] {name} {cin}->{cout} in{r} up{up} ncls{ncls}", ms, flops, "TFLOP/s")
            if mode in ("auto", "tcr") and up and label is None:     # what StyledConvFn runs for this layer
                fn = lambda: K.modconv3x3_up_tcr_fwd(xpm, prep.w_convt_hilo, prep.fir, s, dm, noise, nw, bias, True)
                ms = timeit(fn, iters=1, warmup=0, flush=flush) if args.once else timeit(fn, iters=3, warmup=1, flush=flush)
                row(f"modconv[tcr-convt] {name} {cin}->{cout} in{r} up{up} ncls{ncls}", ms, flops, "TFLOP/s")
                convt_kernel_rows(fn, flush, row, B, cin, cout, r, flops)
            if mode in ("auto", "tcr") and up and label is not None:
                fn = lambda: K.modconv3x3_up_masked_tcr_fwd(xpm, prep.w_convt_hilo, prep.w_hilo, prep.fir, s, dm, label, noise, nw,
                                                            bias, True)
                ms = timeit(fn, iters=1, warmup=0, flush=flush) if args.once else timeit(fn, iters=3, warmup=1, flush=flush)
                row(f"modconv[tcr-convt-masked] {name} {cin}->{cout} in{r} up{up} ncls{ncls}", ms, flops, "TFLOP/s")
                convt_masked_kernel_rows(fn, flush, row, B, cin, cout, r, flops, label, ncls)
        del xpm, noise
    res["conv_total_ms"] = total
    print(json.dumps({"conv_total_ms": total}))
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    json.dump(res, open(args.out, "w"), indent=1)


def convt_kernel_rows(fn, flush, row, B, cin, cout, r, flops):
    """Device time of the two kernels of e4s_modconv3x3_up_tcr_fwd (torch.profiler, three launches after a warm-up, L2
    flushed before each): the GEMM against its algorithmic FLOPs, the blur pass against the bytes it must move (T' read,
    output and one noise map written / read)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            flush.zero_()
            fn()
        torch.cuda.synchronize()
    # the GEMM runs on the register-operand kernel (a library built before it: on conv3x3_wgmma_kernel)
    us = {"gemm": [], "blur": []}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        if "conv3x3_rs_kernel" in ev.name or "conv3x3_wgmma_kernel" in ev.name:
            us["gemm"].append(ev.device_time_total)
        elif "convt_blur_kernel" in ev.name:
            us["blur"].append(ev.device_time_total)
    if not all(us.values()):
        return
    gemm_ms = sum(us["gemm"]) / len(us["gemm"]) / 1e3
    blur_ms = sum(us["blur"]) / len(us["blur"]) / 1e3
    row(f"  convT GEMM {cin}->{4 * cout} on ({r}+1)^2", gemm_ms, flops, "TFLOP/s")
    blur_bytes = 4.0 * B * ((r + 1) ** 2 * 4 * cout + 4 * r * r * cout + 4 * r * r)
    row(f"  blur pass [{B},{2 * r},{2 * r},{cout}]", blur_ms, blur_bytes, "GB/s")


def convt_masked_kernel_rows(fn, flush, row, B, cin, cout, r, flops, label, ncls):
    """Device time of the four kernels of e4s_modconv3x3_up_masked_tcr_fwd, as convt_kernel_rows: the row list, the gathered
    GEMM against the algorithmic FLOPs of its rows, the blur pass against the bytes it must move, the folded fallback
    launch (idle for samples whose rows fit)."""
    from torch.profiler import ProfilerActivity, profile
    from e4s_b200.kernels import convt_masked_cap
    fn()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            flush.zero_()
            fn()
        torch.cuda.synchronize()
    evs = sorted((ev for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA), key=lambda ev: ev.time_range.start)
    us = {"list": [], "gemm": [], "blur": [], "folded": []}
    wg = 0
    for ev in evs:
        if "convt_row_list_kernel" in ev.name:
            us["list"].append(ev.device_time_total)
        elif "convt_blur_masked_kernel" in ev.name:
            us["blur"].append(ev.device_time_total)
        elif "conv3x3_wgmma_kernel" in ev.name:                 # launch order: gathered GEMM, then the folded fallback
            us["gemm" if wg % 2 == 0 else "folded"].append(ev.device_time_total)
            wg += 1
    if not all(us.values()):
        return
    ms = {k: sum(v) / len(v) / 1e3 for k, v in us.items()}
    # rows the GEMM computed: the same count the row-list kernel makes (5 x 5 output window of each T' pixel)
    lab = label.long().clamp(max=ncls - 1)
    onehot = torch.nn.functional.one_hot(lab, ncls).permute(0, 3, 1, 2).float()
    win = torch.nn.functional.max_pool2d(torch.nn.functional.pad(onehot, (2, 3, 2, 3)), 5, stride=2)   # [B, ncls, r+1, r+1]
    per = win.sum(1).flatten(1).sum(1)                                                     # rows per sample
    ok = per <= convt_masked_cap(r, r)
    rows = float(per[ok].sum())
    row(f"  row list [{B},{r + 1},{r + 1}] rows/px {float(per.mean()) / (r * r):.2f} fallback {int((~ok).sum())}/{B}",
        ms["list"], 1.0 * B * 4 * r * r, "GB/s")
    row(f"  gathered GEMM {cin}->{4 * cout} on {rows:.0f} rows", ms["gemm"], 2.0 * 9 * cin * cout * rows, "TFLOP/s")
    blur_bytes = 4.0 * (rows * 4 * cout + int(ok.sum()) * (4 * r * r * cout + 4 * r * r))
    row(f"  masked blur pass [{B},{2 * r},{2 * r},{cout}]", ms["blur"], blur_bytes, "GB/s")
    row(f"  folded fallback launch", ms["folded"], flops * float((~ok).sum()) / B, "TFLOP/s")


if __name__ == "__main__":
    main()
