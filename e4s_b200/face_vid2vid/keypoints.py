"""Head pose to driven 3D keypoints, as face-vid2vid's driven_demo.py computes them (headpose_pred_to_degree,
get_rotation_matrix, keypoint_transformation), and the batched front end of the re-enactment, ``drive_keypoints``.

The pose arithmetic is a handful of tiny elementwise torch ops on the keypoints' device (no kernel of its own), with the
reference's semantics: degrees = sum(softmax(bins) * i) * 3 - 99; radians = degrees / 180 * 3.14 (3.14, not pi);
R = pitch @ yaw @ roll; keypoints = R kp + t + exp.  Sums and 3x3 products are spelled as elementwise adds in a fixed
order, so a pair's result does not depend on the batch.  Unlike the reference, keypoint_transformation does not
unsqueeze he['t'] in place.
"""
import torch
import torch.nn.functional as F

NUM_BINS = 66


def _tree_sum(x: torch.Tensor) -> torch.Tensor:
    """Sum over the last dimension by halving (zero-padded to a power of two): elementwise adds only, so each row's sum
    order is fixed and does not depend on how many rows there are (torch's reductions choose their split by size)."""
    n = 1 << (x.shape[-1] - 1).bit_length()
    x = F.pad(x, (0, n - x.shape[-1]))
    while x.shape[-1] > 1:
        h = x.shape[-1] // 2
        x = x[..., :h] + x[..., h:]
    return x[..., 0]


def _matmul3(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """[..., 3, 3] @ [..., 3, N] as elementwise products and adds in a fixed order (batch-invariant, unlike batched GEMM)."""
    return a[..., :, 0:1] * b[..., 0:1, :] + a[..., :, 1:2] * b[..., 1:2, :] + a[..., :, 2:3] * b[..., 2:3, :]


def headpose_pred_to_degree(pred: torch.Tensor) -> torch.Tensor:
    """[B, 66] bin logits -> [B] degrees: sum(softmax(pred) * i) * 3 - 99."""
    e = torch.exp(pred - pred.amax(dim=1, keepdim=True))
    p = e / _tree_sum(e).unsqueeze(1)
    idx = torch.arange(NUM_BINS, dtype=torch.float32, device=pred.device)
    return _tree_sum(p * idx) * 3 - 99


def get_rotation_matrix(yaw: torch.Tensor, pitch: torch.Tensor, roll: torch.Tensor) -> torch.Tensor:
    """Degrees [B] each -> [B, 3, 3] = pitch_mat (about x) @ yaw_mat (about y) @ roll_mat (about z)."""
    def mat(rows):
        return torch.stack([torch.stack(r, 1) for r in rows], 1)

    p, y, r = (a / 180 * 3.14 for a in (pitch, yaw, roll))
    one, zero = torch.ones_like(p), torch.zeros_like(p)
    pitch_mat = mat([(one, zero, zero), (zero, torch.cos(p), -torch.sin(p)), (zero, torch.sin(p), torch.cos(p))])
    yaw_mat = mat([(torch.cos(y), zero, torch.sin(y)), (zero, one, zero), (-torch.sin(y), zero, torch.cos(y))])
    roll_mat = mat([(torch.cos(r), -torch.sin(r), zero), (torch.sin(r), torch.cos(r), zero), (zero, zero, one)])
    return _matmul3(_matmul3(pitch_mat, yaw_mat), roll_mat)


def keypoint_transformation(kp_canonical: dict, he: dict, estimate_jacobian: bool = False, free_view: bool = False, yaw=0,
                            pitch=0, roll=0) -> dict:
    """Canonical keypoints {'value': [B, K, 3]} and an HEEstimator output -> {'value': [B, K, 3], 'jacobian': None}.
    The jacobian and free_view raise NotImplementedError.  he is not modified."""
    if estimate_jacobian or free_view:
        raise NotImplementedError("e4s_b200 keypoint_transformation: the jacobian and free_view are not implemented")
    kp = kp_canonical['value']
    rot = get_rotation_matrix(headpose_pred_to_degree(he['yaw']), headpose_pred_to_degree(he['pitch']),
                              headpose_pred_to_degree(he['roll']))
    kp_rotated = _matmul3(rot, kp.transpose(1, 2)).transpose(1, 2)          # R kp of every keypoint
    t = he['t'].unsqueeze(1).repeat(1, kp.shape[1], 1)
    exp = he['exp'].reshape(he['exp'].shape[0], -1, 3)
    return {'value': kp_rotated + t + exp, 'jacobian': None}


def drive_keypoints(kp_detector, he_estimator, source: torch.Tensor, driving: torch.Tensor) -> dict:
    """The keypoints face-vid2vid's generator is driven by, for B (source, driving) pairs at once: CUDA [B, 3, 256, 256] in
    [0, 1] each -> {'kp_source', 'kp_driving': [B, 15, 3], 'kp_canonical': {'value': [B, 15, 3]}, 'he_source',
    'he_driving': HEEstimator outputs}.  One KPDetector pass over the sources and one HEEstimator pass over the 2B sources
    and drivings; the reference's unused *_initial work is skipped.  No host synchronisation (CUDA-graph capturable).
    Either module may be wrapped in a one-device DataParallel.  Call under torch.no_grad()."""
    if source.shape != driving.shape or source.device != driving.device:
        raise ValueError(f"drive_keypoints: source {tuple(source.shape)} on {source.device} and driving "
                         f"{tuple(driving.shape)} on {driving.device} must match")
    b = source.shape[0]
    kp_canonical = kp_detector(source)
    he = he_estimator(torch.cat([source, driving]))
    he_source = {k: v[:b] for k, v in he.items()}
    he_driving = {k: v[b:] for k, v in he.items()}
    return {'kp_canonical': kp_canonical, 'he_source': he_source, 'he_driving': he_driving,
            'kp_source': keypoint_transformation(kp_canonical, he_source)['value'],
            'kp_driving': keypoint_transformation(kp_canonical, he_driving)['value']}


def reenact(kp_detector, he_estimator, generator, source: torch.Tensor, driving: torch.Tensor) -> torch.Tensor:
    """B (source, driving) pairs of CUDA [B, 3, 256, 256] faces in [0, 1] -> the re-enacted faces [B, 3, 256, 256]: each
    source driven into its driving face's pose and expression.  One ``drive_keypoints`` call and one pass of the SPADE
    generator (face-vid2vid's OcclusionAwareSPADEGenerator), the batched form of driven_demo's make_animation loop.  No
    host synchronisation (CUDA-graph capturable).  Any module may be wrapped in a one-device DataParallel.  Call under
    torch.no_grad()."""
    kp = drive_keypoints(kp_detector, he_estimator, source, driving)
    return generator(source, {'value': kp['kp_driving']}, {'value': kp['kp_source']})['prediction']
