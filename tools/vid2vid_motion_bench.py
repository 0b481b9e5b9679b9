"""Time face-vid2vid's dense-motion network on the library's kernels against the same network on cuDNN.

    python tools/vid2vid_motion_bench.py [--batch 16] [--iters 3] [--out result.json]

Runs the seeded stand-in checkpoint (oracle/vid2vid_motion_oracle.py) on `batch` seeded pairs (the [B, 32, 16, 64, 64]
feature and the keypoints): DenseMotionNetwork.forward with CUDA events after warm-up and its algorithmic TFLOP/s at
238 GFLOP per pair (mask 80.6, decoder.conv 44.4, down0 18.1, the other nine 3x3x3 blocks 94.3, occlusion 0.7); the
oracle's torch formulation of the same batched work on cuDNN in fp32 and TF32; the reference's per-pair sequence (the
oracle on cuDNN in fp32, one pair after another); and per entry of the library (LaunchStats: time and TFLOP/s).  The
card's name, power limit and maximum SM clock are read in the same call.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from e4s_b200 import kernels as K  # noqa: E402
from e4s_b200.face_vid2vid.modules.dense_motion import DenseMotionNetwork  # noqa: E402
from oracle import vid2vid_motion_oracle as O  # noqa: E402

GFLOP_PER_PAIR = 238.1


def _events(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vid2vid_motion_bench: needs a CUDA device")
    torch.set_grad_enabled(False)
    dev = torch.device("cuda")
    st = O.synthetic_state()
    net = DenseMotionNetwork(**O.PARAMS)
    net.load_state_dict(st, strict=True)
    net = net.eval().to(dev)
    stg = {k: v.to(dev) for k, v in st.items()}
    b = a.batch
    feat = O.synthetic_feature(b, 7).to(dev)
    kd, ks = (t.to(dev) for t in O.synthetic_keypoints(b, 8))
    ours = lambda: net(feat, {"value": kd}, {"value": ks})  # noqa: E731
    oracle = lambda: O.forward(stg, feat, kd, ks)  # noqa: E731

    def per_pair():
        for i in range(b):
            O.forward(stg, feat[i:i + 1], kd[i:i + 1], ks[i:i + 1])

    res = {"card": _card(), "batch": b, "gflop_per_pair": GFLOP_PER_PAIR}
    for name, fn, tf32 in (("ours", ours, False), ("cudnn_fp32", oracle, False), ("cudnn_tf32", oracle, True),
                           ("reference_per_pair_fp32", per_pair, False)):
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
        fn()                                                              # warm-up (and algorithm selection)
        torch.cuda.synchronize()
        ms = _events(fn, a.iters)
        res[name] = {"ms": round(ms, 3), "tflops": round(GFLOP_PER_PAIR * b / ms, 1)}      # GFLOP / ms
        print(f"{name:24s} {ms:9.2f} ms  {GFLOP_PER_PAIR * b / ms:6.1f} TFLOP/s", flush=True)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    K.LaunchStats.reset(timing=True)
    ours()
    torch.cuda.synchronize()
    entries = {}
    for name, (n, ms, work) in sorted(K.LaunchStats.summary().items(), key=lambda kv: -kv[1][1]):
        entries[name] = {"launches": n, "ms": round(ms, 3), "tflops": round(work / ms / 1e9, 1)}
        print(f"  {name:34s} {n:3d} launches {ms:9.3f} ms  {work / ms / 1e9:7.1f} TFLOP/s")
    K.LaunchStats.reset()
    res["entries"] = entries
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
