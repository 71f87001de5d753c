"""H100-native mirror of utils/relative_trafo.py's inference-time entry point.

bone_rel_trafo_inv (reference :243-295) assembles bone-relative coordinates (length, angle_x, angle_y per bone
of the 21-node kinematic chain) back into xyz coordinates; it is the only function of that module on the forward
path (PosePriorNetwork 'local' variants, nets/PosePriorNetwork.py:75).  bone_rel_trafo (the forward direction)
only builds training targets and is out of scope.
"""
from __future__ import annotations

from .. import runtime

kinematic_chain_dict = {0: 'root', 4: 'root', 3: 4, 2: 3, 1: 2, 8: 'root', 7: 8, 6: 7, 5: 6, 12: 'root', 11: 12, 10: 11, 9: 10,
                        16: 'root', 15: 16, 14: 15, 13: 14, 20: 'root', 19: 20, 18: 19, 17: 18}
kinematic_chain_list = [0, 4, 3, 2, 1, 8, 7, 6, 5, 12, 11, 10, 9, 16, 15, 14, 13, 20, 19, 18, 17]


def bone_rel_trafo_inv(coords_rel):
    """coords_rel: [B,21,3] (or [21,3]) torch CUDA tensor -> xyz [B,21,3]."""
    assert coords_rel.dim() in (2, 3), "Has to be a batch of coords."
    return runtime.default_context().bone_rel_trafo_inv(coords_rel)
