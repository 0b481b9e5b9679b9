"""face-vid2vid (src/pretrained/face_vid2vid) on the library's kernels: the keypoint front end of the re-enactment
(KPDetector, HEEstimator, the pose-to-keypoint arithmetic and the batched drive_keypoints), the generator's
DenseMotionNetwork and the OcclusionAwareSPADEGenerator itself, with keypoints.reenact the batched re-enactment."""
