#!/usr/bin/env python
"""Forward demo in the shape of the reference's run.py (run.py:29-92), without TensorFlow or matplotlib.

The net / util call lines are the reference's; only the placeholder / session lines are replaced by torch CUDA
tensors.  With no arguments it runs on seeded synthetic 240x320 images and seeded random-init weights (the released
weight pickles and sample images are not redistributable / not available offline); pass image files and --weights
<pickles...> to run the real thing.  --save-dir DIR writes run.py's four-panel figure of each image as a PNG (Pillow), drawn on the
device by hand3d_b200.draw.run_figure.

    python examples/run_demo.py [img.png ...] [--weights w1.pickle w2.pickle] [--save-dir out]
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork      # run.py:26
from utils.general import detect_keypoints, trafo_coords            # run.py:27


def load_images(paths):
    if not paths:
        from hand3d_b200.weights import synthetic_images
        return [("synthetic#%d" % i, im[0]) for i, im in enumerate(np.split(synthetic_images(3, 240, 320, seed=5), 3))]
    import cv2
    out = []
    for p in paths:
        raw = cv2.cvtColor(cv2.imread(p), cv2.COLOR_BGR2RGB)
        raw = cv2.resize(raw, (320, 240), interpolation=cv2.INTER_LINEAR)          # scipy.misc.imresize(image_raw, (240, 320))
        out.append((p, (raw.astype('float') / 255.0 - 0.5).astype(np.float32)))   # run.py:59
    return out


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument("images", nargs="*")
    ap.add_argument("--weights", nargs="*", default=None)
    ap.add_argument("--save-dir", default=None, help="write run.py's figure of each image there as <name>.png")
    args = ap.parse_args()
    if args.save_dir:
        from PIL import Image
        from hand3d_b200.draw import run_figure
        os.makedirs(args.save_dir, exist_ok=True)

    # network input (run.py:39-41): NHWC float32 on the GPU instead of tf.placeholder
    image_tf = torch.empty((1, 240, 320, 3), dtype=torch.float32, device="cuda")
    hand_side_tf = torch.tensor([[1.0, 0.0]], device="cuda")  # left hand (true for all samples provided)
    evaluation = True

    # build network + initialize (run.py:44-53)
    net = ColorHandPose3DNetwork()
    if args.weights:
        net.init(None, weight_files=args.weights)
    else:
        from hand3d_b200.weights import synthetic_weights
        net.init(None, weights=synthetic_weights(0))

    for name, image_v in load_images(args.images):
        image_tf.copy_(torch.from_numpy(image_v[None]))
        outs = net.inference(image_tf, hand_side_tf, evaluation)
        hand_scoremap_v, image_crop_v, scale_v, center_v, keypoints_scoremap_v, keypoint_coord3d_v = [t.cpu().numpy() for t in outs]
        if args.save_dir:     # run.py:76-92, the figure as one uint8 image (the 240x320 image back in bytes: run.py's image_raw)
            image_raw = torch.from_numpy(np.clip(np.rint((image_v + 0.5) * 255.0), 0, 255).astype(np.uint8)).cuda()
            result = dict(zip(("hand_scoremap", "image_crop", "scale_crop", "center", "keypoints_scoremap", "keypoint_coord3d"), outs))
            result["keypoints_uv"] = detect_keypoints(outs[4])
            fig = run_figure(image_raw, result)["grid"].cpu().numpy()
            Image.fromarray(fig).save(os.path.join(args.save_dir, os.path.basename(name).replace("#", "_").split(".")[0] + ".png"))

        hand_scoremap_v = np.squeeze(hand_scoremap_v)
        keypoints_scoremap_v = np.squeeze(keypoints_scoremap_v)
        keypoint_coord3d_v = np.squeeze(keypoint_coord3d_v)

        # post processing (run.py:72-74)
        coord_hw_crop = detect_keypoints(np.squeeze(keypoints_scoremap_v))
        coord_hw = trafo_coords(coord_hw_crop, center_v, scale_v, 256)

        print("%s: hand pixels %d, crop center (%.1f, %.1f) scale %.3f" % (
            name, int((np.argmax(hand_scoremap_v, 2) == 1).sum()), center_v[0, 0], center_v[0, 1], scale_v[0, 0]))
        print("  wrist (row, col) in the image: (%.1f, %.1f); 3D wrist %s; index-finger tip 3D %s" % (
            coord_hw[0, 0], coord_hw[0, 1], np.round(keypoint_coord3d_v[0], 3), np.round(keypoint_coord3d_v[8], 3)))
