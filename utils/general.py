"""Import shim: `from utils.general import detect_keypoints, trafo_coords, ...` (run.py:27, eval2d.py:36)."""
from hand3d_b200.utils.general import *  # noqa: F401,F403
from hand3d_b200.utils.general import (DeviceEvalUtil, EvalUtil, NetworkOps, calc_auc, calc_center_bb, crop_image_from_xy, detect_keypoints,  # noqa: F401
                                       find_max_location, single_obj_scoremap, trafo_coords, variable_scope)
