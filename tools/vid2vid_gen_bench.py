"""Time face-vid2vid's SPADE generator and the whole re-enactment on the library's kernels against the same work on cuDNN.

    python tools/vid2vid_gen_bench.py [--batch 16] [--iters 3] [--out result.json]

Runs the seeded stand-in checkpoints (oracle/vid2vid_gen_oracle.py, oracle/vid2vid_kp_oracle.py) on `batch` seeded
(source, driving) pairs: ``reenact`` (drive_keypoints + the generator) and OcclusionAwareSPADEGenerator.forward alone with
CUDA events after warm-up, with algorithmic TFLOP/s from the GFLOP per pair computed below from the layer shapes; the
oracle's batched formulation of the generator on cuDNN in fp32 and TF32; the reference's per-pair sequence (the oracle
on cuDNN in fp32, one pair after another); per entry of the library (LaunchStats: time and TFLOP/s); the NCDHW permute
copy handed to the dense-motion network; and the device's peak allocated memory during one generator pass.  The card's
name, power limit and maximum SM clock are read in the same call.
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
from e4s_b200.face_vid2vid.keypoints import reenact  # noqa: E402
from e4s_b200.face_vid2vid.modules.generator import OcclusionAwareSPADEGenerator  # noqa: E402
from e4s_b200.face_vid2vid.modules.keypoint_detector import HEEstimator, KPDetector  # noqa: E402
from oracle import vid2vid_gen_oracle as O  # noqa: E402
from oracle import vid2vid_kp_oracle as KPO  # noqa: E402
from oracle import vid2vid_motion_oracle as MO  # noqa: E402

DENSE_MOTION_GFLOP = 238.1          # tools/vid2vid_motion_bench.py
KEYPOINT_GFLOP = 70.0               # KPDetector on the source, HEEstimator on the source and the driving face


def conv(k, cin, cout, hw):
    return 2.0 * k * k * cin * cout * hw * hw / 1e9


def generator_gflop() -> dict:
    """GFLOP per pair of the generator's own layers (the dense-motion network apart), by part."""
    parts = {"encoder": conv(3, 3, 64, 256) + conv(3, 64, 128, 256) + conv(3, 128, 256, 128) + conv(1, 256, 512, 64),
             "resblocks_3d": 12 * 2.0 * 27 * 32 * 32 * 16 * 64 * 64 / 1e9,
             "third_fourth": conv(3, 512, 256, 64) + conv(1, 256, 256, 64)}
    dec = conv(3, 256, 512, 64) + 12 * conv(3, 256, 128, 64)                       # fc, G_middle mlp_shared
    dec += 6 * (2 * conv(3, 128, 1024, 64) + 2 * conv(3, 512, 512, 64))          # G_middle gamma / beta, conv_0, conv_1
    for hw, fin, fout in ((128, 512, 256), (256, 256, 64)):
        fmid = min(fin, fout)
        dec += 3 * conv(3, 256, 128, hw)                                           # mlp_shared of norm_0, norm_1, norm_s
        dec += 2 * conv(3, 128, 2 * fin, hw) + conv(3, 128, 2 * fmid, hw)         # gamma / beta of norm_0, norm_s, norm_1
        dec += conv(3, fin, fmid, hw) + conv(3, fmid, fout, hw) + conv(1, fin, fout, hw)
    parts["decoder"] = dec + conv(3, 64, 3, 256)
    return parts


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
        raise SystemExit("vid2vid_gen_bench: needs a CUDA device")
    torch.set_grad_enabled(False)
    dev = torch.device("cuda")
    st = O.synthetic_state()
    gen = OcclusionAwareSPADEGenerator(**O.PARAMS)
    gen.load_state_dict(st, strict=True)
    gen = gen.eval().to(dev)
    kp_detector = KPDetector(**KPO.PARAMS)
    kp_detector.load_state_dict(KPO.synthetic_state(), strict=True)
    he_estimator = HEEstimator(**KPO.HE_PARAMS)
    he_estimator.load_state_dict(KPO.he_synthetic_state(), strict=True)
    kp_detector, he_estimator = kp_detector.eval().to(dev), he_estimator.eval().to(dev)
    stg = {k: v.to(dev) for k, v in st.items()}
    b = a.batch
    src, drv = KPO.synthetic_faces(b, 7).to(dev), KPO.synthetic_faces(b, 8).to(dev)
    kd, ks = (t.to(dev) for t in MO.synthetic_keypoints(b, 9))
    parts = generator_gflop()
    g_gen = sum(parts.values()) + DENSE_MOTION_GFLOP
    g_all = g_gen + KEYPOINT_GFLOP
    ours = lambda: gen(src, {"value": kd}, {"value": ks})  # noqa: E731
    oracle = lambda: O.forward(stg, src, kd, ks)  # noqa: E731

    def per_pair():
        for i in range(b):
            O.forward(stg, src[i:i + 1], kd[i:i + 1], ks[i:i + 1])

    res = {"card": _card(), "batch": b, "gflop_per_pair": {"generator": round(g_gen, 1), "reenact": round(g_all, 1),
                                                           **{k: round(v, 1) for k, v in parts.items()},
                                                           "dense_motion": DENSE_MOTION_GFLOP}}
    print(res["card"], res["gflop_per_pair"], flush=True)
    for name, fn, tf32, gf in (("reenact", lambda: reenact(kp_detector, he_estimator, gen, src, drv), False, g_all),
                               ("generator", ours, False, g_gen), ("generator_cudnn_fp32", oracle, False, g_gen),
                               ("generator_cudnn_tf32", oracle, True, g_gen),
                               ("generator_reference_per_pair_fp32", per_pair, False, g_gen)):
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
        fn()                                                              # warm-up (and algorithm selection)
        torch.cuda.synchronize()
        ms = _events(fn, a.iters)
        res[name] = {"ms": round(ms, 2), "tflops": round(gf * b / ms, 1)}                 # GFLOP / ms
        print(f"{name:36s} {ms:9.2f} ms  {gf * b / ms:6.1f} TFLOP/s", flush=True)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    # the one torch op on an activation: the NCDHW copy of the [B, 64, 64, 16, 32] volume handed to DenseMotionNetwork
    vol = torch.randn(b, 64, 64, 16, 32, device=dev)
    copy = lambda: vol.permute(0, 4, 3, 1, 2).contiguous()  # noqa: E731
    copy()
    ms = _events(copy, 20)
    res["permute_copy"] = {"ms": round(ms, 3), "share_of_generator": round(ms / res["generator"]["ms"], 4)}
    print(f"permute copy {ms:.3f} ms, {100 * ms / res['generator']['ms']:.2f} % of the generator", flush=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ours()
    torch.cuda.synchronize()
    res["generator_peak_gib"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    res["generator_peak_above_inputs_gib"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 2)
    print(f"generator peak allocated {res['generator_peak_gib']} GiB ({res['generator_peak_above_inputs_gib']} GiB above the "
          f"weights and inputs)")
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
