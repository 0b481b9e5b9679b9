"""Pin oracle/vid2vid_kp_oracle.py against the reference's face-vid2vid KPDetector, HEEstimator and pose arithmetic and
write tests/golden/vid2vid_kp_vectors.npz and tests/golden/vid2vid_kp_checkpoint_layout.json.

Run where the reference checkout is (CPU only):

    python oracle/make_golden_vid2vid_kp.py

src/pretrained/face_vid2vid/modules/keypoint_detector.py and driven_demo.py (and what they import) are imported
UNMODIFIED; imageio and skimage, which driven_demo imports for its file handling only, are replaced by empty stand-in
modules first.  The seeded stand-ins load with strict=True.  On seeded faces (quantised to 8 bits, stored as uint8) the
script asserts oracle == reference: the keypoints and the HEEstimator outputs within 2e-5, headpose_pred_to_degree,
get_rotation_matrix and keypoint_transformation to fp32 rounding on the reference's own outputs and on seeded bin logits.
It prints the statistics that show the stand-ins are not degenerate (the top voxel's softmax mass per keypoint, the
keypoints' range, the angles, the BatchNorm running statistics) and asserts them.  The layout JSON holds every
state-dict key and shape of the reference's two modules.
"""
from __future__ import annotations

import json
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden", "vid2vid_kp_vectors.npz")
LAYOUT = os.path.join(ROOT, "tests", "golden", "vid2vid_kp_checkpoint_layout.json")
POSE_TOL = 1e-5
TOL = 2e-5
sys.path.insert(0, ROOT)

from oracle import golden_io  # noqa: E402
from oracle import vid2vid_kp_oracle as O  # noqa: E402


def faces_u8(b, seed):
    return (O.synthetic_faces(b, seed) * 255).round().to(torch.uint8)


def main():
    sys.path.insert(0, REF)
    for name in ("imageio", "skimage", "skimage.transform"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["skimage.transform"].resize = None
    sys.modules["skimage"].img_as_ubyte = None
    from src.pretrained.face_vid2vid.modules.keypoint_detector import KPDetector, HEEstimator
    from src.pretrained.face_vid2vid import driven_demo as DD
    torch.set_grad_enabled(False)
    st, he_st = O.synthetic_state(), O.he_synthetic_state()
    ref = KPDetector(**O.PARAMS).eval()
    ref.load_state_dict(st, strict=True)
    he_ref = HEEstimator(**O.HE_PARAMS).eval()
    he_ref.load_state_dict(he_st, strict=True)

    x8 = faces_u8(1, 2024)                      # source
    d8 = faces_u8(2, 2025)                      # two drivings
    x, d = x8.float() / 255, d8.float() / 255
    want = ref(x)["value"]
    lay = O.kp_layers(st, x)
    err = float((lay["value"] - want).abs().max())
    print(f"KPDetector oracle vs reference: max abs keypoint difference {err:.2e}")
    assert err < TOL, err

    he_in = torch.cat([x, d])
    he_want = he_ref(he_in)
    he_got = O.he_forward(he_st, he_in)
    for k in ("yaw", "pitch", "roll", "t", "exp"):
        e = float((he_got[k] - he_want[k]).abs().max() / he_want[k].abs().max())
        print(f"HEEstimator oracle vs reference {k}: rel {e:.2e}")
        assert e < TOL, (k, e)

    # pose: the reference's functions on its own HEEstimator outputs and on seeded bin logits (clones: the reference
    # unsqueezes he['t'] in place)
    g = torch.Generator().manual_seed(7)
    bins = {k: torch.randn(5, 66, generator=g) * 3 for k in ("yaw", "pitch", "roll")}
    pose_he = dict(bins, t=torch.randn(5, 3, generator=g) * 0.1, exp=torch.randn(5, 45, generator=g) * 0.05)
    pose_kp = torch.rand(5, 15, 3, generator=g) * 2 - 1
    out = {}
    for tag, he, kp in (("net", he_want, want.expand(3, 15, 3)), ("seeded", pose_he, pose_kp)):
        deg = {k: DD.headpose_pred_to_degree(he[k].clone()) for k in ("yaw", "pitch", "roll")}
        rot = DD.get_rotation_matrix(deg["yaw"], deg["pitch"], deg["roll"])
        kpt = DD.keypoint_transformation({"value": kp.clone()}, {k: v.clone() for k, v in he.items()}, False)["value"]
        for k in ("yaw", "pitch", "roll"):
            assert float((O.headpose_pred_to_degree(he[k]) - deg[k]).abs().max()) < POSE_TOL * 100
        assert float((O.get_rotation_matrix(deg["yaw"], deg["pitch"], deg["roll"]) - rot).abs().max()) < POSE_TOL
        assert float((O.keypoint_transformation(kp, he) - kpt).abs().max()) < POSE_TOL
        print(f"pose ({tag}): yaw {deg['yaw'].tolist()}\n  pitch {deg['pitch'].tolist()}\n  roll {deg['roll'].tolist()}")
        out.update({f"{tag}_deg_{k}": v.numpy() for k, v in deg.items()})
        out.update({f"{tag}_rot": rot.numpy(), f"{tag}_kp_transformed": kpt.numpy()})
    out.update({f"seeded_he_{k}": v.numpy() for k, v in pose_he.items()})
    out["seeded_kp"] = pose_kp.numpy()

    b, k = lay["kp"].shape[:2]
    top = torch.softmax(lay["kp"].reshape(b, k, -1) / O.PARAMS["temperature"], 2).amax(2)
    lo, hi = want.amin((0, 1)), want.amax((0, 1))
    var = torch.cat([v for n, v in list(st.items()) + list(he_st.items()) if n.endswith("running_var")])
    mean = torch.cat([v for n, v in list(st.items()) + list(he_st.items()) if n.endswith("running_mean")])
    more = O.he_forward(he_st, O.synthetic_faces(8, 2026))             # the oracle, just pinned to the reference
    net_deg = torch.stack([O.headpose_pred_to_degree(more[k]) for k in ("yaw", "pitch", "roll")])
    spread = float((net_deg.amax(1) - net_deg.amin(1)).min())
    print(f"top voxel mass per keypoint: min {float(top.min()):.4f} max {float(top.max()):.4f} (uniform {1 / 65536:.2e})")
    print(f"keypoints: x [{lo[0]:.3f}, {hi[0]:.3f}] y [{lo[1]:.3f}, {hi[1]:.3f}] z [{lo[2]:.3f}, {hi[2]:.3f}]")
    print(f"angles over eight seeded faces: smallest range {spread:.1f} degrees")
    print(f"BN running mean std {float(mean.std()):.3f}, running var [{float(var.min()):.3f}, {float(var.max()):.3f}]")
    assert float(top.min()) > 100 / 65536                              # every heatmap peaked
    assert float((hi - lo).min()) > 0.4                                # the keypoints spread along every axis
    assert spread > 10                                                 # poses tens of degrees apart
    assert float(mean.std()) > 0.1 and float(var.max() - var.min()) > 0.5

    out.update({"x_u8": x8.numpy(), "driving_u8": d8.numpy(), "value": want.numpy()})
    out.update({f"he_{k}": v.numpy() for k, v in he_want.items()})
    golden_io.save(OUT, out)
    layout = {name: {k: list(v.shape) for k, v in m.state_dict().items()} for name, m in (("kp_detector", ref),
                                                                                          ("he_estimator", he_ref))}
    with open(LAYOUT, "w") as f:
        json.dump(layout, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", OUT, "and", LAYOUT)


if __name__ == "__main__":
    main()
