"""GPEN ParseNet throughput on the GPU (needs one; fails without).

    python tools/gpen_parse_bench.py [--batch 16] [--iters 5] [--calls 3] [--split] [--profile out_dir]

Times, with CUDA events after warm-up, 512 x 512 faces -> {0, 255} paste masks with the seeded stand-in checkpoint:
  * FaceParse.process_tensor (the library's kernels, no logits written) at the batch, `--calls` timed calls of `--iters`
    iterations each;
  * the oracle's torch formulation of ParseNet.forward (F.pad reflect + F.conv2d + F.batch_norm + F.interpolate) plus the
    argmax and colormap, on cuDNN, fp32 and TF32, at the batch;
  * the reference's per-image path as FaceParse.process runs it - cv2.resize and float64 normalisation on the host, the
    forward, argmax on the device, .cpu() - spelled with the oracle, one image at a time (fp32 cuDNN).
Prints the card, its power limit and max SM clock (read in the same call), ms per batch, faces/s and algorithmic TFLOP/s at
468.1 GFLOP per face (the mask path: every convolution but out_img_conv, 2 * 9 * Cin * Cout per output pixel).  --split: the
device time per library entry point (CUDA events around every launch) in a separate run; --profile: a torch.profiler
per-kernel table in a separate run.  One JSON line at the end.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import gpen_parse_oracle as PO  # noqa: E402

GFLOP_PER_FACE = 468.1


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
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--split", action="store_true")
    ap.add_argument("--profile", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpen_parse_bench: needs a GPU")
    from e4s_b200 import kernels as K
    from e4s_b200.gpen.face_parse.face_parsing import FaceParse
    torch.set_grad_enabled(False)
    dev = torch.device("cuda")
    st_cpu = PO.synthetic_state()
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "weights"))
        torch.save(st_cpu, os.path.join(tmp, "weights", "ParseNet-latest.pth"))
        fp = FaceParse(tmp, device="cuda")
    fp.faceparse.requires_grad_(False)
    b = a.batch
    imgs_u8 = [PO.case_image(512, 512, 100 + i) for i in range(b)]
    x = torch.cat([PO.image_tensor(i) for i in imgs_u8]).to(dev)
    gf = GFLOP_PER_FACE
    res = {"card": card(), "batch": b, "gflop_per_face": gf}

    calls = [timed(lambda: fp.process_tensor(x), a.iters) for _ in range(a.calls)]
    ms = min(calls)
    res["process_tensor_ms_calls"] = calls
    res["process_tensor_ms"], res["process_tensor_faces_per_s"], res["process_tensor_tflops"] = ms, b / ms * 1e3, gf * b / ms

    st = {k: v.to(dev) for k, v in st_cpu.items()}
    for tf32 in (False, True):
        torch.backends.cudnn.allow_tf32 = tf32
        torch.backends.cuda.matmul.allow_tf32 = tf32
        o_ms = timed(lambda: PO.to_mask(PO.parsenet_forward(st, PO.tensor_input(x))[0]), max(2, a.iters // 2))
        key = "cudnn_tf32" if tf32 else "cudnn_fp32"
        res[f"{key}_ms"], res[f"{key}_faces_per_s"], res[f"{key}_tflops"] = o_ms, b / o_ms * 1e3, gf * b / o_ms
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

    def per_image():
        for i in imgs_u8:
            PO.to_mask(PO.parsenet_forward(st, PO.process_input(i).to(dev))[0]).cpu().numpy()

    pi_ms = timed(per_image, 1)
    res["per_image_path_ms"], res["per_image_path_faces_per_s"] = pi_ms, b / pi_ms * 1e3
    res["speedup_vs_cudnn_fp32"] = res["cudnn_fp32_ms"] / ms
    res["speedup_vs_cudnn_tf32"] = res["cudnn_tf32_ms"] / ms

    if a.split:
        fp.process_tensor(x)
        torch.cuda.synchronize()
        K.LaunchStats.reset(timing=True)
        fp.process_tensor(x)
        torch.cuda.synchronize()
        summ = K.LaunchStats.summary()
        K.LaunchStats.reset()
        tot = sum(v[1] for v in summ.values())
        print(f"per entry point, one process_tensor call at B = {b} (events around every launch; total {tot:.2f} ms):")
        for name, (n, t, w) in sorted(summ.items(), key=lambda kv: -kv[1][1]):
            print(f"  {name:32s} {n:3d} launches {t:8.2f} ms  {t / tot:6.1%}  {w / t / 1e9 if t else 0:7.1f} TFLOP/s or TB/s")
        res["split_ms"] = {name: v[1] for name, v in summ.items()}
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(a.profile, exist_ok=True)
        fp.process_tensor(x)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fp.process_tensor(x)
            torch.cuda.synchronize()
        table_txt = prof.key_averages().table(sort_by="cuda_time_total", row_limit=15)
        with open(os.path.join(a.profile, "gpen_parse_kernels.txt"), "w") as f:
            f.write(table_txt)
        print(table_txt)
    for k, v in res.items():
        print(f"{k}: {v:.3f}" if isinstance(v, float) else f"{k}: {v}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
