"""Time face-vid2vid's keypoint front end on the library's kernels against the same networks on cuDNN.

    python tools/vid2vid_kp_bench.py [--batch 16] [--iters 10] [--out result.json]
    python tools/vid2vid_kp_bench.py --profile          # torch.profiler of one drive_keypoints call, nothing else

Runs the seeded stand-in checkpoints (oracle/vid2vid_kp_oracle.py) on `batch` seeded 256² (source, driving) pairs:
drive_keypoints with CUDA events after warm-up and its algorithmic TFLOP/s at 69.9 GFLOP per pair (KPDetector 38.69 +
2 x HEEstimator 15.61); KPDetector alone at 38.69 GFLOP per face; the oracle's torch formulation of the same batched
work on cuDNN in fp32 and TF32; the reference's per-pair make_animation sequence (kp_detector(source), he_estimator on
the source, on the driving twice, keypoint_transformation three times) spelled with the oracle on cuDNN (fp32), pair
after pair; per entry of the library (LaunchStats: time and TFLOP/s); and per volumetric layer its time, TFLOP/s and
the useful-row fraction of its tiles.  The card's name, power limit and maximum SM clock are read in the same call.
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
from e4s_b200.face_vid2vid.keypoints import drive_keypoints  # noqa: E402
from e4s_b200.face_vid2vid.modules.keypoint_detector import HEEstimator, KPDetector  # noqa: E402
from oracle import vid2vid_kp_oracle as O  # noqa: E402

GFLOP_PER_FACE = 38.69
GFLOP_PER_PAIR = 69.9
VOL_LAYERS = ("up0", "up1", "up2", "up3", "up4", "kp")


def _events(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _oracle_pairs(kst, hst, src, drv):
    """drive_keypoints' work in the oracle's torch formulation, batched."""
    canon = O.kp_forward(kst, src)["value"]
    he = O.he_forward(hst, torch.cat([src, drv]))
    b = src.shape[0]
    return (O.keypoint_transformation(canon, {k: v[:b] for k, v in he.items()}),
            O.keypoint_transformation(canon, {k: v[b:] for k, v in he.items()}))


def _reference_sequence(kst, hst, src, drv):
    """make_animation's per-pair front end: one pair at a time, the unused *_initial work included."""
    for i in range(src.shape[0]):
        s, d = src[i:i + 1], drv[i:i + 1]
        canon = O.kp_forward(kst, s)["value"]
        he_s, he_d0, he_d = O.he_forward(hst, s), O.he_forward(hst, d), O.he_forward(hst, d)
        for he in (he_s, he_d0, he_d):
            O.keypoint_transformation(canon, he)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vid2vid_kp_bench: needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    det = KPDetector(**O.PARAMS)
    det.load_state_dict(O.synthetic_state(), strict=True)
    det = det.eval().cuda()
    he = HEEstimator(**O.HE_PARAMS)
    he.load_state_dict(O.he_synthetic_state(), strict=True)
    he = he.eval().cuda()
    src, drv = O.synthetic_faces(a.batch, 1).cuda(), O.synthetic_faces(a.batch, 2).cuda()
    res = {"card": card, "pairs": a.batch}
    with torch.no_grad():
        for _ in range(3):
            drive_keypoints(det, he, src, drv)
        torch.cuda.synchronize()
        if a.profile:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                drive_keypoints(det, he, src, drv)
                torch.cuda.synchronize()
            print(card)
            print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=25))
            return
        ms = _events(lambda: drive_keypoints(det, he, src, drv), a.iters)
        res["drive_keypoints_ms"] = round(ms, 3)
        res["drive_keypoints_tflops"] = round(a.batch * GFLOP_PER_PAIR * 1e9 / (ms * 1e-3) / 1e12, 1)
        kp_ms = _events(lambda: det(src), a.iters)
        res["kp_detector_ms"] = round(kp_ms, 3)
        res["kp_detector_tflops"] = round(a.batch * GFLOP_PER_FACE * 1e9 / (kp_ms * 1e-3) / 1e12, 1)
        K.LaunchStats.reset(timing=True)
        drive_keypoints(det, he, src, drv)
        torch.cuda.synchronize()
        res["launches"] = {k: dict(n=n, ms=round(t, 3), tflops=round(w / (t * 1e-3) / 1e12, 1) if t else 0.0)
                           for k, (n, t, w) in K.LaunchStats.summary().items()}
        vol = [(w, e0.elapsed_time(e1)) for name, w, e0, e1 in K.LaunchStats.records if name == "e4s_conv3d_tcr_f32"]
        K.LaunchStats.reset()
        sides = (4, 8, 16, 32, 64, 64)
        res["volumetric_layers"] = [dict(layer=n, slice=f"{s}x{s}", ms=round(t, 3), tflops=round(w / (t * 1e-3) / 1e12, 1),
                                         useful_rows=round(K.conv3d_useful_rows(a.batch, 16, s, s), 3))
                                    for n, s, (w, t) in zip(VOL_LAYERS, sides, vol)]
        kst = {k: v.cuda() for k, v in O.synthetic_state().items()}
        hst = {k: v.cuda() for k, v in O.he_synthetic_state().items()}
        for tf32 in (False, True):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            for _ in range(2):
                _oracle_pairs(kst, hst, src, drv)
            torch.cuda.synchronize()
            ref_ms = _events(lambda: _oracle_pairs(kst, hst, src, drv), max(1, a.iters // 2))
            tag = "tf32" if tf32 else "fp32"
            res[f"cudnn_{tag}_ms"] = round(ref_ms, 3)
            res[f"speedup_vs_cudnn_{tag}"] = round(ref_ms / ms, 2)
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        _reference_sequence(kst, hst, src, drv)
        torch.cuda.synchronize()
        seq_ms = _events(lambda: _reference_sequence(kst, hst, src, drv), 2)
        res["reference_per_pair_sequence_ms"] = round(seq_ms, 3)
        res["speedup_vs_reference_sequence"] = round(seq_ms / ms, 2)
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
