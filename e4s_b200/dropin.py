"""Point the reference's import paths at this package, so its scripts run unchanged on this package's kernels.

    import e4s_b200.dropin; e4s_b200.dropin.install()      # before `from src.models.networks import Net3`

After `install()`, these reference module names resolve to the mirrors in this package:

    src.models.stylegan2.op            -> e4s_b200.stylegan2.op            (upfirdn2d, fused_act, conv2d_gradfix)
    src.models.stylegan2.model         -> e4s_b200.stylegan2.model         (Generator, StyledConv, ToRGB, ...)
    src.models.encoders.psp_encoders   -> e4s_b200.encoders.psp_encoders   (FSEncoder_PSP)
    src.models.encoders.helpers        -> e4s_b200.encoders.helpers
    src.models.networks                -> e4s_b200.networks                (Net3, LocalMLP)
    src.pretrained.gpen.face_model.gpen_model -> e4s_b200.gpen.gpen_model  (FullGenerator, Generator, ...; inference classes)
    src.models.encoders.model_irse     -> e4s_b200.encoders.model_irse     (Backbone: the ArcFace net of the identity loss)
    src.criteria.lpips.lpips           -> e4s_b200.criteria.lpips          (LPIPS; no download at construction: load weights)
    src.criteria.id_loss               -> e4s_b200.criteria.id_loss        (IDLoss)
    src.criteria.face_parsing.face_parsing_loss -> e4s_b200.criteria.face_parsing   (FaceParsingLoss, unet)
    src.utils.swap_face_mask           -> e4s_b200.masks                   (swap_head_mask_revisit_considerGlass on the GPU)
    src.pretrained.face_parsing{,.model,.resnet,.face_parsing_demo} -> e4s_b200.face_parsing{...}
                                       (BiSeNet, FaceParser, faceParsing_demo, vis_parsing_maps; FaceParser.parse batched;
                                        Resnet18 downloads nothing)
    src.pretrained.gpen.sr_model.{rrdbnet_arch,real_esrnet} -> e4s_b200.gpen.sr_model.{...}
                                       (RRDBNet, RealESRNet: GPEN's x4 super-resolution on the tensor-core kernels)
    src.pretrained.gpen.face_parse.{blocks,parse_model,face_parsing} -> e4s_b200.gpen.face_parse.{...}
                                       (ParseNet, FaceParse: GPEN's face parser on the tensor-core kernels;
                                        FaceParse.process_tensor batched)
    src.pretrained.gpen.face_detect.{retinaface_detection,facemodels.retinaface,facemodels.net}
                                    -> e4s_b200.gpen.face_detect.{...}
                                       (RetinaFaceDetection, RetinaFace: GPEN's RetinaFace-R50 detector on the tensor-core
                                        kernels; RetinaFaceDetection.detect_batch batched)
    src.pretrained.face_vid2vid.modules.keypoint_detector -> e4s_b200.face_vid2vid.modules.keypoint_detector
                                       (KPDetector, HEEstimator: face-vid2vid's keypoint and head-pose networks on the
                                        tensor-core kernels; driven_demo.make_animation runs them unchanged;
                                        e4s_b200.face_vid2vid.keypoints.drive_keypoints is the batched front end)
    src.pretrained.face_vid2vid.modules.dense_motion -> e4s_b200.face_vid2vid.modules.dense_motion
                                       (DenseMotionNetwork: face-vid2vid's dense-motion network on the tensor-core kernels;
                                        the reference's OcclusionAwareSPADEGenerator builds it unchanged)
    src.pretrained.face_vid2vid.modules.generator -> e4s_b200.face_vid2vid.modules.generator
                                       (OcclusionAwareSPADEGenerator: face-vid2vid's SPADE generator on the tensor-core
                                        kernels; driven_demo.load_checkpoints(gen="spade") and make_animation run all three
                                        networks on the library; e4s_b200.face_vid2vid.reenact is the batched form)
    src.utils.torch_utils.labelMap2OneHot is left alone (it already runs on the GPU); e4s_b200.masks has the kernel.

(`src.utils.morphology` is NOT overlaid: e4s_b200.masks.dilation / erosion implement the flat-box case the swap pipeline
uses, not the module's whole grey-scale API; import them explicitly, INTEGRATION.md.)

Everything else of the reference tree (scripts, options, datasets, the other criteria and pretrained/* nets) keeps importing from
the reference checkout, which must be on sys.path as usual.
"""
import importlib
import sys
import types

_MAP = {
    "src.models.stylegan2.op": "e4s_b200.stylegan2.op",
    "src.models.stylegan2.op.upfirdn2d": "e4s_b200.stylegan2.op.upfirdn2d",
    "src.models.stylegan2.op.fused_act": "e4s_b200.stylegan2.op.fused_act",
    "src.models.stylegan2.op.conv2d_gradfix": "e4s_b200.stylegan2.op.conv2d_gradfix",
    "src.models.stylegan2.model": "e4s_b200.stylegan2.model",
    "src.models.encoders.psp_encoders": "e4s_b200.encoders.psp_encoders",
    "src.models.encoders.helpers": "e4s_b200.encoders.helpers",
    "src.models.networks": "e4s_b200.networks",
    "src.pretrained.gpen.face_model.gpen_model": "e4s_b200.gpen.gpen_model",
    "src.models.encoders.model_irse": "e4s_b200.encoders.model_irse",
    "src.criteria.lpips.lpips": "e4s_b200.criteria.lpips",
    "src.criteria.id_loss": "e4s_b200.criteria.id_loss",
    "src.criteria.face_parsing.face_parsing_loss": "e4s_b200.criteria.face_parsing",
    "src.utils.swap_face_mask": "e4s_b200.masks",
    "src.pretrained.face_parsing": "e4s_b200.face_parsing",
    "src.pretrained.face_parsing.resnet": "e4s_b200.face_parsing.resnet",
    "src.pretrained.face_parsing.model": "e4s_b200.face_parsing.model",
    "src.pretrained.face_parsing.face_parsing_demo": "e4s_b200.face_parsing.face_parsing_demo",
    "src.pretrained.gpen.sr_model.rrdbnet_arch": "e4s_b200.gpen.sr_model.rrdbnet_arch",
    "src.pretrained.gpen.sr_model.real_esrnet": "e4s_b200.gpen.sr_model.real_esrnet",
    "src.pretrained.gpen.face_parse.blocks": "e4s_b200.gpen.face_parse.blocks",
    "src.pretrained.gpen.face_parse.parse_model": "e4s_b200.gpen.face_parse.parse_model",
    "src.pretrained.gpen.face_parse.face_parsing": "e4s_b200.gpen.face_parse.face_parsing",
    "src.pretrained.gpen.face_detect.retinaface_detection": "e4s_b200.gpen.face_detect.retinaface_detection",
    "src.pretrained.gpen.face_detect.facemodels.retinaface": "e4s_b200.gpen.face_detect.facemodels.retinaface",
    "src.pretrained.gpen.face_detect.facemodels.net": "e4s_b200.gpen.face_detect.facemodels.net",
    "src.pretrained.face_vid2vid.modules.keypoint_detector": "e4s_b200.face_vid2vid.modules.keypoint_detector",
    "src.pretrained.face_vid2vid.modules.dense_motion": "e4s_b200.face_vid2vid.modules.dense_motion",
    "src.pretrained.face_vid2vid.modules.generator": "e4s_b200.face_vid2vid.modules.generator",
}


def install() -> None:
    for parent in ("src", "src.models", "src.models.stylegan2", "src.models.encoders", "src.utils", "src.pretrained",
                   "src.pretrained.gpen", "src.pretrained.gpen.face_model", "src.pretrained.gpen.sr_model",
                   "src.pretrained.gpen.face_parse", "src.pretrained.gpen.face_detect",
                   "src.pretrained.gpen.face_detect.facemodels", "src.pretrained.face_vid2vid",
                   "src.pretrained.face_vid2vid.modules", "src.criteria",
                   "src.criteria.lpips",
                   "src.criteria.face_parsing"):
        if parent not in sys.modules:
            try:
                importlib.import_module(parent)          # the reference checkout, if it is on sys.path
            except Exception:
                sys.modules[parent] = types.ModuleType(parent)
                sys.modules[parent].__path__ = []        # namespace stand-in
    for ref_name, ours in _MAP.items():
        sys.modules[ref_name] = importlib.import_module(ours)
        parent, _, leaf = ref_name.rpartition(".")
        if parent in sys.modules:
            setattr(sys.modules[parent], leaf, sys.modules[ref_name])
