"""run.py over a stream of camera frames: every frame is resized to 240x320 on the device exactly as scipy.misc.imresize did
(run.py:57-59), then goes through ColorHandPose3DNetwork.inference; key-points come back in frame pixels.

    python examples/run_frames_demo.py                      # seeded synthetic 1080p frames, synthetic weights
    python examples/run_frames_demo.py --video clip.mp4     # decoded with OpenCV; its BGR frames go in as they are
    python examples/run_frames_demo.py --raw-video clip.nv12 --pixel-format nv12 --height 1080 --width 1920
                                                            # concatenated raw frames, as ffmpeg -f rawvideo -pix_fmt nv12 (or
                                                            # yuv420p -> i420, yuyv422 -> yuyv) writes them
    python examples/run_frames_demo.py --weights weights/   # the reference's pickled weights
    python examples/run_frames_demo.py --track --draw-dir out   # also writes the frames of the first batch with the skeleton and
                                                                # the crop square drawn on the device (PNG, Pillow)
    python examples/run_frames_demo.py --source video:main.mp4 --source raw:side.nv12:nv12:720x1280 \
        --source synthetic:yuyv:480x640 --track --detect slots  # a camera rig: one batch slot per source, each with its own size
                                                                # and pixel format, served by one FrameRunner
"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def synthetic_batches(n_batches, B, H, W, seed):
    rng = np.random.default_rng(seed)
    for _ in range(n_batches):
        yield rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)


def video_batches(path, B, max_batches):
    import cv2
    cap = cv2.VideoCapture(path)
    batch = []
    n = 0
    while n < max_batches:
        ok, bgr = cap.read()
        if not ok:
            break
        batch.append(bgr)                   # FrameRunner(pixel_format="bgr") converts on the device
        if len(batch) == B:
            yield np.stack(batch)
            batch, n = [], n + 1
    cap.release()


def raw_video_batches(path, pixel_format, B, H, W, max_batches):
    """Concatenated raw frames of frame_shape(pixel_format, H, W), read through a memory map (a trailing partial batch is dropped)."""
    from hand3d_b200.frames import frame_shape
    shape = frame_shape(pixel_format, H, W)
    frame_bytes = int(np.prod(shape))
    n = os.path.getsize(path) // frame_bytes
    if n == 0:
        return
    frames = np.memmap(path, dtype=np.uint8, mode="r", shape=(n,) + shape)
    for i in range(min(max_batches, n // B)):
        yield np.ascontiguousarray(frames[i * B:(i + 1) * B])


def source(spec, n_frames, seed):
    """--source SPEC -> (pixel_format, (H, W), iterator of frames): video:PATH (decoded with OpenCV, BGR), raw:PATH:FMT:HxW
    (concatenated raw frames) or synthetic:FMT:HxW (seeded random bytes of that layout)."""
    kind, _, rest = spec.partition(":")
    if kind == "video":
        import cv2
        cap = cv2.VideoCapture(rest)
        hw = (int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT)), int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)))
        cap.release()
        return "bgr", hw, (b[0] for b in video_batches(rest, 1, n_frames))
    path, fmt, size = rest.rsplit(":", 2) if kind == "raw" else (None,) + tuple(rest.split(":", 1))
    if kind not in ("raw", "synthetic") or "x" not in size:
        raise SystemExit("--source %r: expected video:PATH, raw:PATH:FMT:HxW or synthetic:FMT:HxW" % spec)
    hw = tuple(int(v) for v in size.split("x"))
    if kind == "raw":
        return fmt, hw, (b[0] for b in raw_video_batches(path, fmt, 1, hw[0], hw[1], n_frames))
    from hand3d_b200.frames import frame_shape
    shape = frame_shape(fmt, *hw)
    rng = np.random.default_rng(seed)
    return fmt, hw, (rng.integers(0, 256, shape, dtype=np.uint8) for _ in range(n_frames))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--video", default=None, help="video file (cv2 decodes it); default: synthetic frames")
    ap.add_argument("--raw-video", default=None, help="file of concatenated raw frames (ffmpeg -f rawvideo); needs --pixel-format, "
                                                     "--height and --width")
    ap.add_argument("--pixel-format", default=None, choices=["nv12", "i420", "yuyv"], help="with --raw-video: the frames' layout")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--batches", type=int, default=10)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--weights", default=None, help="directory of the reference's pickles (default: synthetic weights)")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--track", action="store_true", help="follow the hand from frame to frame; HandSegNet only to (re-)acquire it")
    ap.add_argument("--redetect-every", type=int, default=None, help="with --track: also detect on every N-th batch")
    ap.add_argument("--min-score", type=float, default=None, help="with --track: a slot whose key-point score is lower is lost")
    ap.add_argument("--detect", default="batch", choices=["batch", "slots"],
                    help="with --track: re-detect the whole batch when a slot is lost (batch), or only the lost slots, chosen on the "
                         "device one step after the loss (slots)")
    ap.add_argument("--draw-dir", default=None, help="draw the skeleton and the crop square into the frames on the device and write "
                                                     "them there as PNG files")
    ap.add_argument("--draw-batches", type=int, default=1, help="with --draw-dir: how many batches to write")
    ap.add_argument("--source", action="append", default=None,
                    help="a camera of a rig, repeated once per batch slot: video:PATH, raw:PATH:FMT:HxW or synthetic:FMT:HxW (FMT one of "
                         "rgb, bgr, nv12, i420, yuyv); --batches steps of one frame per camera, --batch is ignored")
    args = ap.parse_args()

    from hand3d_b200 import runtime, weights as Wt
    from hand3d_b200.frames import FrameRunner
    from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork

    net = ColorHandPose3DNetwork()
    if args.weights:
        net.init(None, weight_files=[os.path.join(args.weights, f) for f in ("handsegnet-rhd.pickle",
                                                                          "posenet3d-rhd-stb-slr-finetuned.pickle")])
    else:
        net.init(None, weights=Wt.synthetic_weights(0))
    ctx = runtime.default_context()

    pixel_format = "rgb"
    if args.source:
        cams = [source(spec, args.batches, args.seed + i) for i, spec in enumerate(args.source)]
        pixel_format, hw = [c[0] for c in cams], [c[1] for c in cams]
        args.batch = len(cams)
        batches = (list(frames) for frames in zip(*[c[2] for c in cams]))
    elif args.raw_video:
        if args.pixel_format is None:
            ap.error("--raw-video needs --pixel-format")
        hw = (args.height, args.width)
        pixel_format = args.pixel_format
        batches = raw_video_batches(args.raw_video, pixel_format, args.batch, hw[0], hw[1], args.batches)
    elif args.video:
        import cv2
        cap = cv2.VideoCapture(args.video)
        hw = (int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT)), int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)))
        cap.release()
        pixel_format = "bgr"
        batches = video_batches(args.video, args.batch, args.batches)
    else:
        hw = (args.height, args.width)
        batches = synthetic_batches(args.batches, args.batch, hw[0], hw[1], args.seed)

    runner = FrameRunner(ctx, args.batch, hw, track=args.track, redetect_every=args.redetect_every, min_score=args.min_score,
                         detect=args.detect, draw=args.draw_dir is not None, pixel_format=pixel_format)
    if args.draw_dir:
        from PIL import Image
        os.makedirs(args.draw_dir, exist_ok=True)
    t0 = time.perf_counter()
    n = 0
    for i, r in enumerate(runner.stream(batches)):
        n += args.batch
        kp = r["keypoints_frame"][0]
        track = ""
        if args.track:
            detected = r["track_detected"][0] if args.detect == "slots" else r["detected"]
            track = " [%s, score %.4g%s]" % ("detect" if detected else "track", r["track_score"][0],
                                             ", lost" if r["track_lost"][0] else "")
        if args.draw_dir and i < args.draw_batches:
            for b, frame in enumerate(r["frame_drawn"]):
                Image.fromarray(frame).save(os.path.join(args.draw_dir, "batch%03d_frame%02d.png" % (i, b)))
        H, W = hw[0] if args.source else hw
        print("batch %d: frame 0 key-points (row, col) in %dx%d pixels: wrist %s, index tip %s%s" % (i, H, W, np.round(kp[0], 1),
                                                                                                 np.round(kp[8], 1), track))
    dt = time.perf_counter() - t0
    print("%d frames in %.3f s: %.1f frames/s" % (n, dt, n / dt if dt > 0 else 0.0))


if __name__ == "__main__":
    main()
