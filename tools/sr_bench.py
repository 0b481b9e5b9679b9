"""RealESRNet x4 throughput on the GPU (needs one; fails without).

    python tools/sr_bench.py [--batch 16] [--iters 5] [--profile out_dir]

Times, with CUDA events after warm-up, 256 x 256 faces -> 1024 x 1024:
  * RRDBNet.forward (the library's kernels) at the batch, with the weights resident in shared memory where they fit (the
    default) and streamed with every channel chunk (E4S_B200_RS_STREAM=1);
  * the oracle's torch formulation of the same network (torch.cat + F.conv2d + F.interpolate) on cuDNN, fp32 and TF32, at
    the batch;
  * the reference's per-image path as RealESRNet.process runs it - uint8 BGR numpy -> tensor -> forward -> .cpu() -> uint8 -
    spelled with the oracle, one image at a time (fp32 cuDNN).
Prints the card, its power limit and max SM clock, faces/s and algorithmic TFLOP/s (1296.9 GFLOP per face: 2 * 9 * Cin *
Cout per output pixel of every convolution); with --profile, a per-kernel breakdown of RRDBNet.forward from torch.profiler in
a separate run.  One JSON line at the end.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import sr_oracle as SO  # noqa: E402


def gflop_per_face(h=256, w=256, nf=32, gc=32, blocks=23):
    """Algorithmic GFLOP of RRDBNet x4 on one h x w image (2 * 9 * Cin * Cout per output pixel)."""
    px, f = h * w, 0.0
    f += px * 3 * nf                                              # conv_first
    f += blocks * 3 * px * (sum((nf + j * gc) * gc for j in range(4)) + (nf + 4 * gc) * nf)
    f += px * nf * nf                                             # conv_body
    f += 4 * px * nf * nf + 16 * px * nf * nf * 2 + 16 * px * nf * 3   # conv_up1 @2x, conv_up2 and conv_hr @4x, conv_last
    return 18.0 * f / 1e9


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--profile", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sr_bench: needs a GPU")
    from e4s_b200.gpen.sr_model.rrdbnet_arch import RRDBNet
    torch.set_grad_enabled(False)
    dev = torch.device("cuda")
    net = RRDBNet(num_in_ch=3, num_out_ch=3, num_feat=32, num_block=23, num_grow_ch=32, scale=4)
    net.load_state_dict(SO.synthetic_state(), strict=True)
    net = net.eval().requires_grad_(False).to(dev)
    b = a.batch
    imgs_u8 = [SO.case_image(256, 256, 100 + i) for i in range(b)]
    x = torch.cat([SO.to_input(i) for i in imgs_u8]).to(dev)
    gf = gflop_per_face()
    res = {"card": card(), "batch": b, "gflop_per_face": gf}

    for tag, stream in (("", None), ("_streamed", "1")):
        if stream:
            os.environ["E4S_B200_RS_STREAM"] = stream
        ms = timed(lambda: net(x), a.iters)
        os.environ.pop("E4S_B200_RS_STREAM", None)
        res[f"forward{tag}_ms"] = ms
        res[f"forward{tag}_faces_per_s"] = b / ms * 1e3
        res[f"forward{tag}_tflops"] = gf * b / ms                 # GFLOP per ms = TFLOP/s

    st = {k: v.to(dev) for k, v in SO.synthetic_state().items()}
    for tf32 in (False, True):
        torch.backends.cudnn.allow_tf32 = tf32
        torch.backends.cuda.matmul.allow_tf32 = tf32
        o_ms = timed(lambda: SO.rrdbnet_forward(st, x), max(2, a.iters // 2))
        key = "cudnn_tf32" if tf32 else "cudnn_fp32"
        res[f"{key}_ms"], res[f"{key}_faces_per_s"], res[f"{key}_tflops"] = o_ms, b / o_ms * 1e3, gf * b / o_ms
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

    pi_ms = timed(lambda: [SO.process(st, i, dev) for i in imgs_u8], 1)
    res["per_image_path_ms"], res["per_image_path_faces_per_s"] = pi_ms, b / pi_ms * 1e3
    res["speedup_vs_cudnn_fp32"] = res["cudnn_fp32_ms"] / res["forward_ms"]

    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(a.profile, exist_ok=True)
        net(x)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            net(x)
            torch.cuda.synchronize()
        table_txt = prof.key_averages().table(sort_by="cuda_time_total", row_limit=15)
        with open(os.path.join(a.profile, "sr_kernels.txt"), "w") as f:
            f.write(table_txt)
        print(table_txt)
    for k, v in res.items():
        print(f"{k}: {v:.3f}" if isinstance(v, float) else f"{k}: {v}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
