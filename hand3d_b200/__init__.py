"""hand3d_b200 -- H100-native (sm_90a) forward pass of ColorHandPose3D behind the reference's Python API.

    from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork
    from hand3d_b200.utils.general import detect_keypoints, trafo_coords

(the repo root also carries `nets/` and `utils/` shims so the reference's own import lines work unchanged).
"""
__version__ = "0.1.0"
