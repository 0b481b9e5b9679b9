"""Face-parser throughput on the GPU (needs one; fails without).

    python tools/parse_bench.py [--batch 16] [--iters 20] [--profile out_dir]

Times, with CUDA events after warm-up, on 1024 x 1024 images:
  * FaceParser.parse (the library's kernels, labels only) at the batch;
  * the oracle's torch formulation of the same label path (preprocess + BiSeNet first head + argmax + table) on cuDNN,
    fp32 and TF32, at the batch;
  * the reference's per-image path as faceParsing_demo runs it - PIL image -> tensor -> forward -> .cpu() -> numpy table -
    spelled with the oracle's restatement, one image at a time.
Prints the card, its power limit, images/s, the convolutions' algorithmic TFLOP/s (26.77 GFLOP per image on the label
path) and the preprocess / head kernels' GB/s against 3.35 TB/s; with --profile, a per-kernel breakdown of parse() from
torch.profiler in a separate run.  One JSON line at the end.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import parser_oracle as PO  # noqa: E402

GFLOP_LABEL_PATH = 26.77        # per image, 512 x 512 network input (torch.utils.flop_counter on the reference module)
HBM_TBS = 3.35


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
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--profile", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("parse_bench: needs a GPU")
    from PIL import Image
    import torchvision
    from e4s_b200 import kernels as K
    from e4s_b200.face_parsing.face_parsing_demo import FaceParser
    torch.set_grad_enabled(False)
    dev = torch.device("cuda")
    with tempfile.TemporaryDirectory() as tmp:
        ckpt = os.path.join(tmp, "bisenet.pth")
        torch.save(PO.synthetic_state(), ckpt)
        parser = FaceParser(ckpt, device="cuda")
    b = a.batch
    imgs_u8 = [PO.case_image(1024, 100 + i) for i in range(b)]
    images = torch.stack([torch.from_numpy(i).permute(2, 0, 1) for i in imgs_u8]).to(dev).float() / 255
    res = {"card": card(), "batch": b}

    ms = timed(lambda: parser.parse(images), a.iters)
    res["parse_ms"] = ms
    res["parse_images_per_s"] = b / ms * 1e3
    res["parse_conv_tflops"] = GFLOP_LABEL_PATH * b / ms          # GFLOP per ms = TFLOP/s

    # the two streaming kernels on their own
    mean, std, lut, _ = parser._device_consts(dev)
    taps = parser.downsample.taps(dev)
    pre_ms = timed(lambda: K.bicubic_down_norm(images, taps, 2, mean, std), a.iters)
    pre_bytes = 4.0 * (images.numel() + images.numel() / 4)
    res["preprocess_ms"], res["preprocess_GBs"] = pre_ms, pre_bytes / pre_ms * 1e-6
    P = parser.seg._prepared(dev)
    feat = torch.relu(torch.randn(b, 64, 64, 256, device=dev))
    head_ms = timed(lambda: K.parse_head(feat, P["conv_out.cls"], 512, 512, lut=lut), a.iters)
    head_bytes = 4.0 * feat.numel() + b * 512 * 512
    res["head_ms"], res["head_GBs"] = head_ms, head_bytes / head_ms * 1e-6
    res["hbm_TBs_datasheet"] = HBM_TBS

    # the oracle's formulation on cuDNN, fp32 and TF32
    st = {k: v.to(dev) for k, v in PO.synthetic_state().items()}
    oracle = lambda: PO.labels(PO.main_logits(st, PO.preprocess(images, 2)))  # noqa: E731
    for tf32 in (False, True):
        torch.backends.cudnn.allow_tf32 = tf32
        torch.backends.cuda.matmul.allow_tf32 = tf32
        o_ms = timed(oracle, max(2, a.iters // 4))
        res[f"cudnn_{'tf32' if tf32 else 'fp32'}_ms"] = o_ms
        res[f"cudnn_{'tf32' if tf32 else 'fp32'}_images_per_s"] = b / o_ms * 1e3
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

    # the reference's per-image path: PIL -> tensor -> forward -> .cpu() -> numpy table
    pils = [Image.fromarray(i) for i in imgs_u8]
    table = np.asarray(PO.FFHQ19_TO_12, dtype=np.uint8)

    def per_image():
        for p in pils:
            x = torchvision.transforms.ToTensor()(p)[:3].unsqueeze(0).to(dev)
            seg = PO.main_logits(st, PO.preprocess(x, 2)).argmax(1)[0].cpu().numpy().astype(np.uint8)
            table[seg]
    pi_ms = timed(per_image, 2)
    res["per_image_path_ms"] = pi_ms
    res["per_image_path_images_per_s"] = b / pi_ms * 1e3

    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(a.profile, exist_ok=True)
        parser.parse(images)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                parser.parse(images)
            torch.cuda.synchronize()
        table_txt = prof.key_averages().table(sort_by="cuda_time_total", row_limit=25)
        with open(os.path.join(a.profile, "parse_kernels.txt"), "w") as f:
            f.write(table_txt)
        print(table_txt)
    for k, v in res.items():
        print(f"{k}: {v:.3f}" if isinstance(v, float) else f"{k}: {v}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
