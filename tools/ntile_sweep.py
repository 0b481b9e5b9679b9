#!/usr/bin/env python
"""N-tile width of the register-operand forward, per layer: 64 against 128 channels per work item.

    python tools/ntile_sweep.py [--batches 16,1,8] [--rounds 3] [--out FILE.json]

Times e4s_modconv3x3_tcr_fwd on the plain 3x3 layers of the 1024x1024 generator that have 128 or more output channels
(masked, the face label map, 12 regions) and on GPEN-BFR-512's 128-channel 512^2 layer (unmasked) with
E4S_B200_RS_NTILE=64 and =128 alternated: CUDA events, L2 flushed before every launch, per round the median of five
launches; reported per width as min-max over the rounds, in ms and algorithmic TFLOP/s (2 * 9 * Cin * Cout * pixels),
one JSON line per layer on stdout and, with --out, all of them in one file.
The card's name, power limit and maximum SM clock are read first and stored with the numbers.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from e4s_b200 import _lib
from e4s_b200 import kernels as K
from e4s_b200.stylegan2.modconv import PreparedConv
from opbench import timeit

DEV = "cuda:0"
# (name, cin, cout, resolution, masked)
LAYERS = [("c1@8", 512, 512, 8, 1), ("c3@16", 512, 512, 16, 1), ("c5@32", 512, 512, 32, 1), ("c7@64", 512, 512, 64, 1),
          ("c9@128", 256, 256, 128, 1), ("c11@256", 128, 128, 256, 1), ("gpen128@512", 128, 128, 512, 0)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, clock = (f.strip() for f in q.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="16,1,8")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--layers", default="all")
    ap.add_argument("--out", default=None, help="also write the card and every row to this JSON file")
    args = ap.parse_args()
    for var in ("E4S_B200_NTILE", "E4S_B200_RS_NTILE"):
        os.environ.pop(var, None)
    res = {"card": card(), "rows": []}
    print(json.dumps(res["card"]), flush=True)
    from oracle import golden_io
    gold = golden_io.load(os.path.join(ROOT, "tests", "golden", "reference_vectors.npz"))
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=DEV)
    keep = None if args.layers == "all" else set(args.layers.split(","))
    for B in (int(b) for b in args.batches.split(",")):
        face = torch.from_numpy(gold["mask/source_cls12"]).to(DEV)[None].repeat(B, 1, 1).contiguous()
        for name, cin, cout, r, masked in LAYERS:
            if keep is not None and name not in keep:
                continue
            ncls = 12 if masked else 1
            prep = PreparedConv().get(torch.randn(1, cout, cin, 3, 3, device=DEV), False, None)
            x = torch.randn(B, r, r, cin, device=DEV)
            s = 1.0 + 0.1 * torch.randn(B, ncls, cin, device=DEV)
            label = K.label_resize_nearest(face, r, r) if masked else None
            noise = torch.randn(B, 1, r, r, device=DEV)
            nw = torch.tensor([0.1], device=DEV)
            bias = torch.randn(cout, device=DEV)
            dm = K.demod(s, prep.wsq)
            fn = lambda: K.modconv3x3_tcr_fwd(x, prep.w_hilo, s, dm, label, noise, nw, bias, False, True)
            auto = ctypes.c_int()
            _lib.check(_lib.load().e4s_modconv3x3_tcr_fwd_plan(B, r, r, cout, ctypes.byref(auto)), "e4s_modconv3x3_tcr_fwd_plan")
            ms = {64: [], 128: []}
            for _ in range(args.rounds):
                for nt in (64, 128):
                    os.environ["E4S_B200_RS_NTILE"] = str(nt)
                    ms[nt].append(timeit(fn, iters=5, warmup=1, flush=flush))
            os.environ.pop("E4S_B200_RS_NTILE")
            tf = 2.0 * 9 * cin * cout * B * r * r / 1e9
            row = {"layer": name, "batch": B, "cin": cin, "cout": cout, "auto": auto.value,
                   "tiles": -(-r // 8) * -(-r // 16) * B,
                   "speedup_min": round(min(a / b for a, b in zip(ms[64], ms[128])), 3)}
            for nt in (64, 128):
                row[f"ms{nt}"] = [round(min(ms[nt]), 4), round(max(ms[nt]), 4)]
                row[f"tflops{nt}"] = [round(tf / max(ms[nt]), 1), round(tf / min(ms[nt]), 1)]
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
            del x, noise
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
