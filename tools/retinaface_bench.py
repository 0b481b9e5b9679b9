"""Time GPEN's RetinaFace-R50 detector on the library's kernels at the face swap's shape: 16 seeded 1024 x 1024 images, the
seeded stand-in checkpoint.

    python tools/retinaface_bench.py [--out DIR]

Prints one JSON object (and writes it to DIR/retinaface_bench.json): the card and its power limit (read in the same call),
detect_batch and forward times (CUDA events, three calls after warm-up), algorithmic TFLOP/s (the convolutions' FLOPs from
their shapes, summed over the launches of one forward), the oracle's torch formulation on cuDNN in fp32 and with TF32, the
reference's per-image path (detect() spelled with the oracle: host mean subtraction, per-image forward on cuDNN fp32,
decode, .cpu(), numpy selection and NMS), the per-kernel split of one forward (CUDA events around every launch) and of one
detect_batch call (torch.profiler), each in a separate call, and every 1x1 shape of the network at B = 16 on the pointwise
kernel against the centre tap of the 3x3 kernel (e4s_conv3x3_bias_tcr_f32, tap mask 0x10), alternating.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from e4s_b200 import kernels as K  # noqa: E402
from e4s_b200.encoders.psp_encoders import _conv_planes  # noqa: E402
from oracle import retinaface_oracle as RO  # noqa: E402

B, S = 16, 1024


def timed(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1))
    return min(out), out


def reference_path(st_gpu, imgs_np):
    """RetinaFaceDetection.detect per image as the reference runs it, spelled with the oracle on the GPU (fp32 cuDNN)."""
    out = []
    for img in imgs_np:
        x = np.float32(img)
        h, w = x.shape[:2]
        x -= (104, 117, 123)
        x = torch.from_numpy(x.transpose(2, 0, 1).copy()).unsqueeze(0).cuda()
        loc, conf, landms = RO.forward(st_gpu, x)
        pri = RO.prior_box(h, w).cuda()
        boxes = (RO.decode(loc[0], pri) * torch.tensor([w, h, w, h], dtype=torch.float32, device="cuda")).cpu().numpy()
        scores = conf[0, :, 1].cpu().numpy()
        lm = (RO.decode_landm(landms[0], pri) * torch.tensor([w, h] * 5, dtype=torch.float32, device="cuda")).cpu().numpy()
        out.append(RO.select(boxes, lm, scores))
    return out


def profile(fn):
    """Device time per kernel name over one call of fn (torch.profiler, CUDA activity), largest first."""
    from torch.profiler import ProfilerActivity, profile as prof
    fn()
    torch.cuda.synchronize()
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        fn()
        torch.cuda.synchronize()
    rows = {}
    for ev in p.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        if t > 0:
            rows[ev.key[:90]] = round(t / 1e3, 3)
    return dict(sorted(rows.items(), key=lambda kv: -kv[1])[:25])


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name()


def pointwise_shapes():
    """(cin, cout, out h, out w, stride) of every distinct 1x1 convolution at 1024 x 1024, with its count per forward."""
    shapes = {}
    add = lambda k: shapes.__setitem__(k, shapes.get(k, 0) + 1)  # noqa: E731
    res, cin = S // 4, 64
    for li, (n, width) in enumerate(((3, 64), (4, 128), (6, 256), (3, 512))):
        for i in range(n):
            stride = 2 if (i == 0 and li) else 1
            add((cin, width, res, res, 1))                               # conv1 (at the input grid)
            if i == 0:
                add((cin, 4 * width, res // stride, res // stride, stride))   # downsample
            res //= stride
            add((width, 4 * width, res, res, 1))                         # conv3
            cin = 4 * width
    for c, r in ((512, S // 8), (1024, S // 16), (2048, S // 32)):
        add((c, 256, r, r, 1))                                           # FPN laterals
    for r in (S // 8, S // 16, S // 32):
        add((256, 32, r, r, 1))                                          # heads
    return shapes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from e4s_b200.gpen.face_detect.retinaface_detection import RetinaFaceDetection
    st = RO.synthetic_state()
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "weights"))
        torch.save({"module." + k: v for k, v in st.items()}, os.path.join(tmp, "weights", "RetinaFace-R50.pth"))
        det = RetinaFaceDetection(tmp, device="cuda")
    imgs_np = [RO.case_image(S, S, 100 + i) for i in range(B)]
    imgs = torch.stack([torch.from_numpy(im.transpose(2, 0, 1).copy()) for im in imgs_np]).cuda()
    x = K.retinaface_prep(imgs)
    res = {"card": card(), "batch": B, "size": S}
    with torch.no_grad():
        ms, runs = timed(lambda: det.detect_batch(imgs))
        res["detect_batch_ms"], res["detect_batch_runs"] = ms, runs
        ms, runs = timed(lambda: det.net(x))
        res["forward_ms"], res["forward_runs"] = ms, runs
        K.LaunchStats.reset(timing=True)
        det.net(x)
        torch.cuda.synchronize()
        summ = K.LaunchStats.summary()
        K.LaunchStats.reset()
        conv = ("e4s_conv1x1_tcr_f32", "e4s_conv3x3_zero_tcr_f32", "e4s_parser_stem_f32")
        flops = sum(w for name, (_, _, w) in summ.items() if name in conv)
        res["gflop_per_image"] = flops / B / 1e9
        res["tflops_forward"] = flops / (res["forward_ms"] * 1e-3) / 1e12
        res["tflops_detect_batch"] = flops / (res["detect_batch_ms"] * 1e-3) / 1e12
        res["per_kernel_ms"] = {name: round(ms, 3) for name, (n, ms, _) in sorted(summ.items(), key=lambda kv: -kv[1][1])}
        dets = det.detect_batch(imgs)
        res["detections_per_image"] = dets[2].tolist()
        # the oracle's torch formulation on cuDNN
        st_gpu = {k: v.cuda() for k, v in st.items()}
        for tf32 in (False, True):
            torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
            ms, _ = timed(lambda: RO.forward(st_gpu, x))
            res["cudnn_tf32_ms" if tf32 else "cudnn_fp32_ms"] = ms
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        reference_path(st_gpu, imgs_np[:2])                     # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ref_dets = reference_path(st_gpu, imgs_np)
        res["reference_per_image_path_ms"] = (time.perf_counter() - t0) * 1e3
        res["reference_detections_per_image"] = [len(d) for d, _ in ref_dets]
        res["profiler_detect_batch_ms"] = profile(lambda: det.detect_batch(imgs))
        # pointwise against centre tap, alternating
        table = []
        g = torch.Generator(device="cuda").manual_seed(1)
        for (cin, cout, h, w, stride), count in sorted(pointwise_shapes().items()):
            xi = torch.randn(B, h * stride, w * stride, cin, device="cuda", generator=g)
            wt = torch.randn(cout, cin, device="cuda", generator=g) / cin ** 0.5
            bias = torch.zeros(cout, device="cuda")
            pw, c3 = K.split_bf16(wt), _conv_planes(wt[:, :, None, None]).cuda()
            f_pw = lambda: K.conv1x1_tc(xi, pw, bias, stride=stride, lrelu=0.0)  # noqa: E731
            f_c3 = lambda: K.conv3x3_bias_tc(xi, c3, bias, relu=True, out_stride=stride, tap_mask=0x10)  # noqa: E731
            t_pw, t_c3 = [], []
            for _ in range(3):
                t_pw.append(timed(f_pw, 2)[0])
                t_c3.append(timed(f_c3, 2)[0])
            fl = 2.0 * cin * cout * B * h * w
            table.append({"cin": cin, "cout": cout, "out": f"{h}x{w}", "stride": stride, "count": count,
                          "pointwise_ms": min(t_pw), "centre_tap_ms": min(t_c3), "gflop": fl / 1e9})
        res["pointwise_vs_centre_tap"] = table
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "retinaface_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
