#!/usr/bin/env python
"""RGI encoder (Net3.get_style_vectors) on one GPU: whole-call time and per-entry-point kernel times (CUDA events).

    python tools/enc_bench.py [--batch 16] [--out gpurun_out/enc_bench.json]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from bench import build_net, face_label_maps
from e4s_b200 import kernels as K
from e4s_b200.masks import labelMap2OneHot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--out", default=os.path.join(ROOT, "gpurun_out", "enc_bench.json"))
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    net = build_net(1024, 12, dev)
    img = torch.randn(args.batch, 3, 1024, 1024, generator=torch.Generator().manual_seed(3)).to(dev)
    onehot = labelMap2OneHot(face_label_maps(args.batch, 12, "faces", 5).to(dev), 12)
    with torch.no_grad():
        for _ in range(3):
            net.get_style_vectors(img, onehot)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            net.get_style_vectors(img, onehot)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 5
        K.LaunchStats.reset(timing=True)
        net.get_style_vectors(img, onehot)
        torch.cuda.synchronize()
        summ = {k: {"launches": v[0], "ms": round(v[1], 3), "gflop_or_gb": round(v[2] / 1e9, 2)} for k, v in K.LaunchStats.summary().items()}
        # per conv launch: shape and time
        convs = []
        for name, work, a, b in K.LaunchStats.records:
            if name == "e4s_conv3x3_tcr_f32":
                convs.append({"gflop_algorithmic_as_launched": round(work / 1e9, 2), "ms": round(a.elapsed_time(b), 4)})
        K.LaunchStats.reset(False)
    res = {"batch": args.batch, "ms_per_call": ms, "faces_per_sec": args.batch / (ms * 1e-3), "entries": summ, "conv_launches": convs}
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    json.dump(res, open(args.out, "w"), indent=1)
    print(json.dumps({k: res[k] for k in ("batch", "ms_per_call", "faces_per_sec", "entries")}))


if __name__ == "__main__":
    main()
