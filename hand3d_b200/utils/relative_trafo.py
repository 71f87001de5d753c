"""H100-native mirror of utils/relative_trafo.py.

bone_rel_trafo_inv (reference :243-295) assembles bone-relative coordinates (length, angle_x, angle_y per bone
of the 21-node kinematic chain) back into xyz coordinates; it is on the forward path of the PosePriorNetwork 'local'
variants (nets/PosePriorNetwork.py:75) and differentiable, as training_lifting.py:70-73 applies it to the prediction.
bone_rel_trafo (:184-240, the forward direction) builds the 'local' training target and carries no gradient.
"""
from __future__ import annotations

from .. import autograd, runtime

kinematic_chain_dict = {0: 'root', 4: 'root', 3: 4, 2: 3, 1: 2, 8: 'root', 7: 8, 6: 7, 5: 6, 12: 'root', 11: 12, 10: 11, 9: 10,
                        16: 'root', 15: 16, 14: 15, 13: 14, 20: 'root', 19: 20, 18: 19, 17: 18}
kinematic_chain_list = [0, 4, 3, 2, 1, 8, 7, 6, 5, 12, 11, 10, 9, 16, 15, 14, 13, 20, 19, 18, 17]


def bone_rel_trafo_inv(coords_rel):
    """coords_rel: [B,21,3] (or [21,3]) torch CUDA tensor -> xyz [B,21,3]."""
    assert coords_rel.dim() in (2, 3), "Has to be a batch of coords."
    return autograd.bone_rel_trafo_inv(coords_rel)


def bone_rel_trafo(coords_xyz):
    """coords_xyz: [B,21,3] (or [21,3]) torch CUDA tensor -> (length, angle_x, angle_y) [B,21,3], with the reference's own atan2
    (:27-46, atan(y / (x + 1e-8)) plus quadrant corrections)."""
    assert coords_xyz.dim() in (2, 3), "Has to be a batch of coords."
    return runtime.default_context().bone_rel_trafo(coords_xyz.detach())
