"""Camera frames in: run.py's front door (run.py:57-59) on the device.

    image_raw = scipy.misc.imresize(image_raw, (240, 320))          # Pillow's 8-bit BILINEAR resample
    image_v = np.expand_dims((image_raw.astype('float') / 255.0) - 0.5, 0)

imresize() is that first line, bit for bit, for uint8 RGB frames of 1..4096 pixels a side (scipy.misc.imresize is gone from current
scipy); to_network_input() fuses both lines into one kernel; frame_coords() maps coordinates of the 240x320 image back to frame
pixels; FrameRunner serves a stream of equal-size frames through the resize and the whole pipeline as one CUDA graph per buffer.

to_network_input, to_rgb and FrameRunner also take camera frames as they come from decoders and capture devices (pixel_format "bgr",
"nv12", "i420" or "yuyv"; frame_shape gives each one's tensor layout): the conversion to RGB is OpenCV's cvtColor rule, on the device,
fused into the resize (DESIGN.md section 4.18).
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib, runtime
from . import draw as _draw
from .runtime import frame_shape
from .utils.general import trafo_coords

NETWORK_SIZE = (240, 320)   # run.py:58


def _ctx_for(t):
    return runtime.default_context(t.device if isinstance(t, torch.Tensor) and t.is_cuda else None)


def _batched(frames, pixel_format="rgb"):
    """CUDA uint8 one frame or a batch of frames in pixel_format ([H,W,3] or [B,H,W,3] for RGB) -> (the batch, squeezed)."""
    if not isinstance(frames, torch.Tensor):
        raise TypeError("frames must be a torch.Tensor or a numpy array")
    if not frames.is_cuda:
        raise RuntimeError("frames must be a CUDA tensor here (numpy arrays are accepted by imresize)")
    if frames.dim() == (2 if pixel_format in ("nv12", "i420") else 3):
        return frames.unsqueeze(0), True
    return frames, False


def _out_size(size, H, W):
    """scipy.misc.imresize's size argument: an int is a percentage, a float a fraction, a tuple (h, w[, ...])."""
    if isinstance(size, (bool, np.bool_)):
        raise TypeError("size must be an int, a float or a tuple (h, w)")
    if isinstance(size, (int, np.signedinteger)):
        w, h = (np.array((W, H)) * (size / 100.0)).astype(int)
        return int(h), int(w)
    if isinstance(size, (float, np.floating)):
        w, h = (np.array((W, H)) * size).astype(int)
        return int(h), int(w)
    return int(size[0]), int(size[1])


def imresize(arr, size, interp="bilinear", mode=None):
    """scipy.misc.imresize(arr, size) for uint8 RGB frames (its default interp='bilinear', mode=None), computed on the device.

    arr: numpy uint8 [H,W,3] -> numpy uint8 [h,w,3]; or a CUDA uint8 tensor [H,W,3] / [B,H,W,3] -> a CUDA tensor of the same rank.
    Equal, byte for byte, to Pillow's Image.resize((w, h), BILINEAR), which scipy called (see DESIGN.md section 4.12)."""
    if interp != "bilinear":
        raise ValueError("imresize: only interp='bilinear' (run.py's) is implemented, got %r" % (interp,))
    if mode is not None:
        raise ValueError("imresize: only mode=None (uint8 RGB in, RGB out) is implemented, got %r" % (mode,))
    if isinstance(arr, np.ndarray):
        if arr.dtype != np.uint8:
            raise TypeError("imresize: frames must be uint8 (scipy would have rescaled %s data with bytescale), got %s" % (arr.dtype, arr.dtype))
        if arr.ndim != 3 or arr.shape[2] != 3:
            raise ValueError("imresize: a numpy frame must be [H,W,3] RGB, got %s" % (arr.shape,))
        ctx = runtime.default_context()
        h, w = _out_size(size, arr.shape[0], arr.shape[1])
        t = torch.from_numpy(np.ascontiguousarray(arr)).to(ctx.device).unsqueeze(0)
        return ctx.resize_frames(t, h, w, normalize=False)[0].cpu().numpy()
    frames, squeeze = _batched(arr)
    h, w = _out_size(size, frames.shape[1], frames.shape[2])
    out = _ctx_for(frames).resize_frames(frames, h, w, normalize=False)
    return out[0] if squeeze else out


def to_network_input(frames, size=NETWORK_SIZE, out=None, pixel_format="rgb"):
    """run.py:58-59 in one kernel: CUDA uint8 frames [B,H,W,3] (or [H,W,3]) -> float32 [B,h,w,3] = float64(imresize(frame, size))
    / 255.0 - 0.5 rounded to float32, the pipeline's input.  With `out` (float32 [B,h,w,3]) it writes there and allocates nothing, so a
    call of an already seen size can be captured into a CUDA graph.  frames in another pixel_format ("bgr", "nv12", "i420", "yuyv";
    one frame or a batch of frame_shape(pixel_format, H, W)) are converted to RGB inside the same kernel."""
    frames, squeeze = _batched(frames, pixel_format)
    r = _ctx_for(frames).resize_frames(frames, size[0], size[1], normalize=True, out=None if out is None else (out.unsqueeze(0) if squeeze else out),
                                       pixel_format=pixel_format)
    return r[0] if squeeze else r


def to_rgb(frames, pixel_format, out=None):
    """CUDA uint8 frames in pixel_format (one frame or a batch of frame_shape(pixel_format, H, W)) -> uint8 RGB [B,H,W,3] (or [H,W,3])
    at full size, by OpenCV's cvtColor rule (include/hand3d_b200.h); with `out` it writes there and allocates nothing."""
    frames, squeeze = _batched(frames, pixel_format)
    r = _ctx_for(frames).convert_frames(frames, pixel_format, out=None if out is None else (out.unsqueeze(0) if squeeze else out))
    return r[0] if squeeze else r


def _per_slot_hw(frame_hw):
    """True for a per-slot frame_hw ([B,2] tensor or array, or a list of (H, W) pairs), False for one (H, W)."""
    if isinstance(frame_hw, (torch.Tensor, np.ndarray)):
        return frame_hw.ndim == 2
    return len(frame_hw) > 0 and not isinstance(frame_hw[0], (int, float, np.integer, np.floating))


def frame_coords(keypoints_hw, frame_hw, size=NETWORK_SIZE):
    """Coordinates (row, col) in the size image (trafo_coords' output) -> frame pixels, with Pillow's pixel-centre convention:
    (c + 0.5) * Hf / h - 0.5 for rows, the same with Wf / w for columns, in float64 on the device.  A CUDA tensor gives a CUDA float64
    tensor (no host synchronisation, capturable); numpy gives numpy.

    frame_hw is one (H, W) for every row, or per slot (a camera rig): a [B,2] tensor or a list of B (H, W) pairs, row b of
    keypoints_hw [B,...,2] mapped with its own size by the same float64 formula.  A CUDA [B,2] tensor keeps the call free of host
    synchronisation (and capturable)."""
    if isinstance(keypoints_hw, np.ndarray):
        dev = runtime.default_context().device
        return frame_coords(torch.from_numpy(np.asarray(keypoints_hw, np.float64)).to(dev), frame_hw, size).cpu().numpy()
    c = keypoints_hw.to(torch.float64)
    if _per_slot_hw(frame_hw):
        hw = torch.as_tensor(np.asarray(frame_hw, np.float64) if not isinstance(frame_hw, torch.Tensor) else frame_hw)
        hw = hw.to(device=c.device, dtype=torch.float64)
        if tuple(hw.shape) != (c.shape[0], 2):
            raise ValueError("frame_coords: a per-slot frame_hw must be [%d,2], got %s" % (c.shape[0], tuple(hw.shape)))
        hw = hw.reshape((c.shape[0],) + (1,) * (c.dim() - 2) + (2,))
        h = torch.full_like(c[..., 0], float(size[0]))
        w = torch.full_like(c[..., 1], float(size[1]))
        rows = (c[..., 0] + 0.5) * hw[..., 0] / h - 0.5
        cols = (c[..., 1] + 0.5) * hw[..., 1] / w - 0.5
        return torch.stack([rows, cols], -1)
    # divide by a tensor: torch turns a division by a Python scalar into a multiplication by its reciprocal, which is not IEEE division
    h = torch.full_like(c[..., 0], float(size[0]))
    w = torch.full_like(c[..., 1], float(size[1]))
    rows = (c[..., 0] + 0.5) * float(frame_hw[0]) / h - 0.5
    cols = (c[..., 1] + 0.5) * float(frame_hw[1]) / w - 0.5
    return torch.stack([rows, cols], -1)


def rig_layout(pixel_formats, frame_hw, size=NETWORK_SIZE):
    """The plan of a camera rig as the C library builds it (h3d_frame_rig_query; no device needed): (table, coef), int32 numpy arrays
    laid out as include/hand3d_b200.h describes (slot records, the format order, the launch records; the normalisation table and each
    distinct size's coefficient tables).  Raises ValueError with the library's message (naming the slot) for a rig it refuses."""
    import ctypes as C
    lib = _lib.load()
    B = len(frame_hw)
    if len(pixel_formats) != B:
        raise ValueError("a rig of %d sizes needs %d pixel formats, got %d" % (B, B, len(pixel_formats)))
    fmts = (C.c_int * max(B, 1))(*[_lib.PIXEL_FORMATS.get(f, -1) if isinstance(f, str) else int(f) for f in pixel_formats])
    hw = (C.c_int * max(2 * B, 1))(*[int(v) for p in frame_hw for v in p])
    tw, cw = C.c_int64(0), C.c_int64(0)
    if lib.h3d_frame_rig_query(B, fmts, hw, int(size[0]), int(size[1]), None, C.byref(tw), None, C.byref(cw)) != _lib.OK:
        raise ValueError(_lib.last_error())
    table, coef = np.zeros(tw.value, np.int32), np.zeros(cw.value, np.int32)
    _lib.check(lib.h3d_frame_rig_query(B, fmts, hw, int(size[0]), int(size[1]), table.ctypes.data_as(C.c_void_p), C.byref(tw),
                                       coef.ctypes.data_as(C.c_void_p), C.byref(cw)), "h3d_frame_rig_query")
    return table, coef


def redetect_schedule(B, every):
    """The staggered re-detection of FrameRunner(track=True, detect="slots", redetect_every=every): int32 [every, B], row p = the force
    mask of the steps t with t % every == p; slot b is forced where (t + b) % every == 0, so each step forces about B / every slots."""
    t = np.arange(int(every))[:, None]
    b = np.arange(int(B))[None, :]
    return ((t + b) % int(every) == 0).astype(np.int32)


class FrameRunner:
    """Serves a stream of equal-size uint8 RGB frames through run.py's resize and ColorHandPose3DNetwork.inference.

    Each step is h3d_resize_frames (fused normalisation) followed by Context.pipeline on fixed buffers, captured as one CUDA graph
    per input buffer (two buffers, used alternately).  ctx must have its weights loaded.

    submit(frames, hand_side=None) enqueues one batch and returns its result tensors on the device:
      keypoints_frame [B,21,2] float64 (row, col) key-points in frame pixels, keypoints_uv [B,21,2] int32 (256x256 crop),
      keypoint_coord3d [B,21,3], center [B,2] and scale_crop [B,1] (float32).
    Those tensors belong to buffer (call index mod 2): the replay of the call after next overwrites them, in stream order on the
    current stream; read them (or copy them) before that call.
      - Host frames (numpy or CPU torch, [B,H,W,3] uint8, or pixel_format's shape) are copied into a pinned staging buffer and uploaded on a copy stream, so
        the upload of one batch overlaps the replay of the previous one.  A staging buffer is refilled only after its previous upload
        has finished (an event wait for the upload two calls back).
      - CUDA frames are copied into the graph's input buffer on the current stream; nothing synchronises the host.
    hand_side [B,2] (run.py's constant [[1, 0]] when None) goes with each batch.

    stream(batches) is the overlapped loop: it submits batch i + 1 before it reads back batch i, and yields the host results of
    every batch in order (numpy dicts owned by the caller).

    track=True follows the hand from batch to batch instead of detecting it in every frame (Context.track_step, DESIGN.md section
    4.14): each batch slot is one camera stream, and a track step crops frame t where the key-points of frame t - 1 put the hand,
    without HandSegNet.  It captures a detect graph and a track graph per input buffer around one TrackState, which the graphs
    update in stream order, so no step waits on the host for its crop.  Step t detects when t == 0, when redetect_every is set and
    t % redetect_every == 0, or when any slot was lost at step t - 2 (min_score: the lowest trusted score; None = no score test).
    The choice is made on the host from step t - 2's lost flags: stream() has them already; submit() waits for step t - 2 to finish.
    So a slot lost at step t is re-acquired by a detect step at t + 2 at the latest.  The results gain detected (bool, the step's
    kind), track_score [B] float32 and track_lost [B] bool.

    track=True with detect="slots" re-detects per slot instead (Context.track_step_slots, DESIGN.md section 4.15): one graph per input
    buffer runs HandSegNet on the slots the previous step lost, chosen on the device, and tracks the others.  The host reads nothing
    back and submit() never waits on an earlier step, so a slot lost at step t is re-detected at step t + 1.  redetect_every = N forces
    slot b at the steps t with (t + b) % N == 0, so that the re-detections are spread over the N steps; the step's force mask is copied
    from a device table of the N phases before the replay.  The results gain track_detected [B] bool (the slots the step re-detected),
    track_score and track_lost; detected is not given.  detect="batch" (the default) is the policy above; detect="slots" without
    track=True is refused.

    draw=True ends each captured step by drawing into the step's own input buffer, which the resize has consumed by then (no copy):
    the crop square in white, then plot_hand's skeleton at keypoints_frame (as float32), both with draw_linewidth (None = max(1,
    Hf / 240), so that lines look as they would on the 240-row network image; draw.py, DESIGN.md section 4.16).  In track mode a
    slot whose state is lost after the step is not drawn (valid = state lost == 0, on the device).  The results gain frame_drawn
    [B,Hf,Wf,3] uint8: that buffer, valid until the call after next like the other results.  stream(batches, drawn_every=N) reads
    it back for every N-th batch only (0: never).

    pixel_format ("rgb", "bgr", "nv12", "i420" or "yuyv") is the layout of the submitted frames: the input buffers and the pinned
    staging take frame_shape(pixel_format, *frame_hw), so a host upload carries the format's bytes (half of RGB's for 4:2:0), and the
    captured resize converts to RGB as it reads.  frame_hw stays the picture's (H, W).  With draw=True and a format other than "rgb",
    the captured step first converts the frames into an RGB frame buffer (h3d_convert_frames) and draws there; frame_drawn is that
    buffer, [B,Hf,Wf,3] RGB as for "rgb".

    A camera rig (DESIGN.md section 4.19): frame_hw may be a list of B (H, W) sizes and pixel_format a list of B formats, one per
    slot.  When all slots agree, the runner is exactly the single-size runner above (frame_hw and pixel_format become the common
    value; the same kernels and graphs), but it still takes and gives what a rig does: a list of B frames per submit(), frame_drawn
    as a list of B [H,W,3] views and draw_linewidth as a list.  Any single-size runner also takes such a list.  Otherwise each slot gets its own input buffers, and the captured step resizes them with h3d_resize_frames_rig (one kernel
    per format present) into the one [B,240,320,3] network batch; from there on everything is as above.  submit() then takes a list
    of B frames (numpy, CPU torch or CUDA torch, each frame_shape(fmt_b, H_b, W_b) or (1,) + that), stream() an iterable of such lists
    or of (list, hand_side) pairs.  Host frames of a list are uploaded through pinned staging on the copy stream as above; its CUDA
    frames are copied on the current stream after that upload.  keypoints_frame is in each slot's own frame pixels; with draw=True, frame_drawn is a list of B uint8
    RGB tensors [H_b,W_b,3], and draw_linewidth=None means max(1, H_b / 240) per slot."""

    RESULT_KEYS = ("keypoints_frame", "keypoints_uv", "keypoint_coord3d", "center", "scale_crop")
    TRACK_KEYS = ("track_score", "track_lost")
    SLOTS_KEYS = ("track_score", "track_lost", "track_detected")

    def __init__(self, ctx, batch, frame_hw, size=NETWORK_SIZE, outputs="keypoints", track=False, redetect_every=None, min_score=None,
                 track_margin=1.5, detect="batch", draw=False, draw_linewidth=None, pixel_format="rgb"):
        self.ctx, self.B = ctx, int(batch)
        self.size = (int(size[0]), int(size[1]))
        hws, fmts = self._rig_slots(frame_hw, pixel_format)
        self.rig = len(set(hws)) > 1 or len(set(fmts)) > 1      # else exactly the single-size runner
        # built through the rig interface (a list of sizes or of formats): frame_drawn and draw_linewidth are per-slot lists even when
        # the slots agree, so that code written for a rig keeps working when its cameras match
        self.per_slot = _per_slot_hw(frame_hw) or not isinstance(pixel_format, str)
        self._slot_formats, self._slot_hw = fmts, hws
        self.frame_hw, self.pixel_format = (hws, fmts) if self.rig else (hws[0], fmts[0])
        pixel_format = self.pixel_format
        self.track = bool(track)
        if detect not in ("batch", "slots"):
            raise ValueError("FrameRunner: detect must be 'batch' or 'slots', got %r" % (detect,))
        if detect == "slots" and not self.track:
            raise ValueError("FrameRunner: detect='slots' re-detects tracked slots; it needs track=True")
        self.slots = detect == "slots"
        if redetect_every is not None and int(redetect_every) < 1:
            raise ValueError("FrameRunner: redetect_every must be None or >= 1, got %r" % (redetect_every,))
        self.redetect_every = None if redetect_every is None else int(redetect_every)
        self.min_score, self.track_margin = min_score, float(track_margin)
        dev = ctx.device
        self.draw = bool(draw)
        if self.draw:
            self._draw_colors = np.concatenate([np.repeat(_draw.WHITE[None], 4, 0), _draw.PALETTE])
        h, w = self.size
        if self.rig:
            self._init_rig_buffers(draw_linewidth, dev)
        else:
            self._frame_shape = frame_shape(pixel_format, *self.frame_hw)
            self._slot_shapes = [self._frame_shape] * self.B
            Hf, Wf = self.frame_hw
            self._linewidth = max(1.0, Hf / 240.0) if draw_linewidth is None else float(draw_linewidth)
            self.draw_linewidth = [self._linewidth] * self.B if self.per_slot else self._linewidth
            self._frames = [torch.zeros((self.B,) + self._frame_shape, dtype=torch.uint8, device=dev) for _ in range(2)]
            # the frames drawn into: the input buffers themselves for RGB, else an RGB conversion of them made by the step
            self._drawn = self._frames if pixel_format == "rgb" or not self.draw else \
                [torch.zeros((self.B, Hf, Wf, 3), dtype=torch.uint8, device=dev) for _ in range(2)]
            self._stage = [None, None]      # pinned host copies of frames, created on the first host submission
        self._default_hs = torch.tensor([[1.0, 0.0]], dtype=torch.float32).expand(self.B, 2).contiguous().to(dev)
        self._hs = [self._default_hs.clone() for _ in range(2)]
        self._image = [torch.empty((self.B, h, w, 3), dtype=torch.float32, device=dev) for _ in range(2)]
        self._stage_hs = [torch.empty((self.B, 2), dtype=torch.float32).pin_memory() for _ in range(2)]
        self._copy = torch.cuda.Stream(device=dev)
        self._d2h = torch.cuda.Stream(device=dev)
        self._uploaded = [torch.cuda.Event() for _ in range(2)]
        self._consumed = [torch.cuda.Event() for _ in range(2)]
        self._d2h_done = [torch.cuda.Event() for _ in range(2)]
        self._host = [None, None]
        self._host_keys = [(), ()]          # the results the latest read-back of each buffer copied
        self._i = 0
        ctx.ensure_workspace(self.B, h, w)

        self._force, self._force_table = None, None
        if self.slots and self.redetect_every is not None:
            self._force_table = torch.from_numpy(redetect_schedule(self.B, self.redetect_every)).to(dev)   # [N, B]: phase t % N
            self._force = [torch.zeros(self.B, dtype=torch.int32, device=dev) for _ in range(2)]
        if self.track:
            self._state = runtime.TrackState(self.B, dev)
            self._lost_host = [torch.zeros(self.B, dtype=torch.bool).pin_memory() for _ in range(2)]   # step t's lost flags
            self._lost_ready = [torch.cuda.Event() for _ in range(2)]
            self._detected = [True, True]
        if self.rig:
            ctx.frame_rig_plan(self.pixel_format, self.frame_hw, h, w)
            self._capture(lambda k, detect: self._rig_body(k, detect, outputs), dev)
            return

        def body(k, detect=True):
            ctx.resize_frames(self._frames[k], h, w, normalize=True, out=self._image[k], pixel_format=pixel_format)
            r = self._network_step(k, detect, outputs)
            r["keypoints_frame"] = frame_coords(trafo_coords(r["keypoints_uv"], r["center"], r["scale_crop"], 256), self.frame_hw, self.size)
            if self.draw:
                seg = torch.cat([_draw.crop_box_segments(r["center"], r["scale_crop"], self.frame_hw, self.size),
                                 _draw.hand_segments(r["keypoints_frame"].to(torch.float32))], 1).contiguous()
                valid = (self._state.lost == 0).to(torch.int32) if self.track else None
                if self._drawn is not self._frames:
                    ctx.convert_frames(self._frames[k], pixel_format, out=self._drawn[k])
                r["frame_drawn"] = ctx.draw_segments(self._drawn[k], seg, self._draw_colors, self._linewidth, valid)
            return r

        self._capture(body, dev)

    def _rig_slots(self, frame_hw, pixel_format):
        """(sizes, formats), one per slot, from one or B of each."""
        if _per_slot_hw(frame_hw):
            hws = [(int(p[0]), int(p[1])) for p in np.asarray(frame_hw).tolist()] if isinstance(frame_hw, (torch.Tensor, np.ndarray)) \
                else [(int(p[0]), int(p[1])) for p in frame_hw]
            if len(hws) != self.B:
                raise ValueError("FrameRunner: frame_hw must be one (H, W) or %d of them, one per slot, got %d" % (self.B, len(hws)))
        else:
            hws = [(int(frame_hw[0]), int(frame_hw[1]))] * self.B
        if isinstance(pixel_format, str):
            fmts = [pixel_format] * self.B
        else:
            fmts = list(pixel_format)
            if len(fmts) != self.B:
                raise ValueError("FrameRunner: pixel_format must be one format or %d of them, one per slot, got %d" % (self.B, len(fmts)))
        if len(set(hws)) == 1 and len(set(fmts)) == 1:
            frame_shape(fmts[0], *hws[0])           # one camera geometry: refused as the single-size runner refuses it
        for b, (f, hw) in enumerate(zip(fmts, hws)):
            try:
                frame_shape(f, *hw)
            except ValueError as e:
                raise ValueError("FrameRunner: slot %d: %s" % (b, e)) from None
        return hws, fmts

    def _init_rig_buffers(self, draw_linewidth, dev):
        """A rig's per-slot input buffers, drawing targets, sizes on the device and staging."""
        self.draw_linewidth = [max(1.0, H / 240.0) if draw_linewidth is None else float(draw_linewidth) for H, _ in self.frame_hw]
        self._frame_shape = [frame_shape(f, *hw) for f, hw in zip(self.pixel_format, self.frame_hw)]
        self._slot_shapes = self._frame_shape
        self._frames = [[torch.zeros(shp, dtype=torch.uint8, device=dev) for shp in self._frame_shape] for _ in range(2)]
        # the frames drawn into: an RGB slot's input buffer itself, else an RGB conversion of it made by the step
        self._drawn = [[fr if f == "rgb" or not self.draw else torch.zeros(hw + (3,), dtype=torch.uint8, device=dev)
                        for fr, f, hw in zip(self._frames[k], self.pixel_format, self.frame_hw)] for k in range(2)]
        self._hw_dev = torch.tensor(self.frame_hw, dtype=torch.float64, device=dev)    # [B,2]: keypoints_frame's per-slot sizes
        self._stage = [[None] * self.B for _ in range(2)]   # pinned host copies of each camera's frame, made on its first host submission

    def _rig_body(self, k, detect, outputs):
        ctx = self.ctx
        ctx.resize_frames_rig(self._frames[k], self.size[0], self.size[1], normalize=True, out=self._image[k], pixel_formats=self.pixel_format)
        r = self._network_step(k, detect, outputs)
        r["keypoints_frame"] = frame_coords(trafo_coords(r["keypoints_uv"], r["center"], r["scale_crop"], 256), self._hw_dev, self.size)
        if self.draw:
            # one conversion per non-RGB slot and one drawing per slot, inside the graph: the slots' images differ in size
            seg = torch.cat([_draw.crop_box_segments(r["center"], r["scale_crop"], self._hw_dev, self.size),
                             _draw.hand_segments(r["keypoints_frame"].to(torch.float32))], 1).contiguous()
            valid = (self._state.lost == 0).to(torch.int32) if self.track else None
            drawn = []
            for b, f in enumerate(self.pixel_format):
                img = self._drawn[k][b]
                if img is not self._frames[k][b]:
                    ctx.convert_frames(self._frames[k][b].unsqueeze(0), f, out=img.unsqueeze(0))
                ctx.draw_segments(img.unsqueeze(0), seg[b:b + 1], self._draw_colors, self.draw_linewidth[b],
                                  None if valid is None else valid[b:b + 1])
                drawn.append(img)
            r["frame_drawn"] = drawn
        return r

    def _network_step(self, k, detect, outputs):
        """The step after the resize, on the network batch self._image[k]: the pipeline, or a track step of either policy."""
        ctx = self.ctx
        if self.slots:
            r = ctx.track_step_slots(self._image[k], self._hs[k], self._state, None if self._force is None else self._force[k],
                                     margin=self.track_margin, min_score=self.min_score, outputs=outputs)
            r["track_score"] = self._state.score.clone()
            r["track_lost"] = self._state.lost != 0
        elif self.track:
            r = ctx.track_step(self._image[k], self._hs[k], self._state, detect, margin=self.track_margin, min_score=self.min_score,
                               outputs=outputs)
            r["track_score"] = self._state.score.clone()
            r["track_lost"] = self._state.lost != 0
        else:
            r = ctx.pipeline(self._image[k], self._hs[k], True, outputs=outputs)
        return r

    def _capture(self, body, dev):
        """Warms body(k, detect) up outside capture, then captures one graph per input buffer and step kind."""
        ctx = self.ctx
        kinds = (True, False) if self.track and not self.slots else (True,)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):       # warm-up outside capture: builds the resize and stage plans, packs weights
            for k in range(2):
                for detect in kinds:
                    body(k, detect)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize(dev)
        self._graphs, self._results = [], []   # [buffer][kind]: kind 0 = detect, 1 = track
        for k in range(2):
            gs, rs = [], []
            for detect in kinds:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    r = body(k, detect)
                ctx._graphs_captured = getattr(ctx, "_graphs_captured", 0) + 1   # the graphs bake in workspace pointers
                gs.append(g)
                rs.append(r)
            self._graphs.append(gs)
            self._results.append(rs)
        if self.track:
            self._state.reset()             # forget the warm-up's steps
            torch.cuda.synchronize(dev)

    def _slot_stage(self, k, b, shape):
        """The pinned staging of slot b of buffer k: a rig's own per camera, else slot b of the batch's staging."""
        if self.rig:
            if self._stage[k][b] is None:
                self._stage[k][b] = torch.empty(shape, dtype=torch.uint8).pin_memory()
            return self._stage[k][b]
        if self._stage[k] is None:
            self._stage[k] = torch.empty((self.B,) + tuple(shape), dtype=torch.uint8).pin_memory()
        return self._stage[k][b]

    def _upload_slots(self, frames, hand_side, k, cur):
        """Fills buffer k's inputs from a list of B frames, one per slot (a rig's, or a single-size runner's).  Host frames go through
        the pinned staging and the copy stream, under the single-size runner's event rules; CUDA frames are copied device to device
        on the current stream, after that upload, so that they are read in the caller's stream order."""
        if not isinstance(frames, (list, tuple)) or len(frames) != self.B:
            raise ValueError("FrameRunner: a rig of %d cameras takes a list of %d frames, got %s" %
                             (self.B, self.B, len(frames) if isinstance(frames, (list, tuple)) else type(frames).__name__))
        srcs, on_dev = [], []
        for b, f in enumerate(frames):
            shp = self._slot_shapes[b]
            if isinstance(f, np.ndarray):
                f = torch.from_numpy(np.ascontiguousarray(f))
            if not isinstance(f, torch.Tensor) or f.dtype != torch.uint8:
                raise TypeError("FrameRunner: slot %d: frames must be uint8 (numpy, CPU torch or CUDA torch)" % b)
            if f.is_cuda and not f.is_contiguous():
                raise TypeError("FrameRunner: slot %d: frames must be contiguous uint8" % b)
            if tuple(f.shape) not in (shp, (1,) + shp):
                raise ValueError("FrameRunner: slot %d: a %s %dx%d frame must be %s or %s, got %s" %
                                 ((b, self._slot_formats[b]) + self._slot_hw[b] + (shp, (1,) + shp, tuple(f.shape))))
            srcs.append(f.reshape(shp))
            on_dev.append(f.is_cuda)
        hs = None if hand_side is None else torch.as_tensor(hand_side, dtype=torch.float32)
        if not all(on_dev):
            self._uploaded[k].synchronize()         # the upload that last read these staging buffers (two calls back) has finished
            for b, (src, d) in enumerate(zip(srcs, on_dev)):
                if not d:
                    self._slot_stage(k, b, src.shape).copy_(src)
            self._stage_hs[k].copy_(torch.as_tensor(np.asarray([[1.0, 0.0]] * self.B, np.float32)) if hs is None else
                                    hs.cpu().reshape(self.B, 2))
            with torch.cuda.stream(self._copy):
                self._copy.wait_event(self._consumed[k])      # the replay that last read these input buffers has finished
                if self.draw:
                    self._copy.wait_event(self._d2h_done[k])  # and stream()'s read-back of frame_drawn, which may be these buffers
                for b, d in enumerate(on_dev):
                    if not d:
                        self._frames[k][b].copy_(self._slot_stage(k, b, srcs[b].shape), non_blocking=True)
                self._hs[k].copy_(self._stage_hs[k], non_blocking=True)
                self._uploaded[k].record(self._copy)
            cur.wait_event(self._uploaded[k])
        elif hs is None:
            self._hs[k].copy_(self._default_hs)
        else:
            self._hs[k].copy_(hs.to(self.ctx.device).reshape(self.B, 2))
        for b, d in enumerate(on_dev):              # CUDA frames (all, or the device part of a mixed list) on the current stream
            if d:
                self._frames[k][b].copy_(srcs[b])

    def _detect_now(self, t):
        """The host's detect / track choice for step t (deterministic: t, redetect_every and step t - 2's lost flags)."""
        if t == 0 or (self.redetect_every is not None and t % self.redetect_every == 0):
            return True
        if t < 2:
            return False
        k = t & 1                                   # step t - 2 used the same buffer
        self._lost_ready[k].synchronize()
        return bool(self._lost_host[k].any())

    def _check_frames(self, frames):
        shape = (self.B,) + self._frame_shape
        if tuple(frames.shape) != shape:
            raise ValueError("FrameRunner: frames must be %s, got %s" % (shape, tuple(frames.shape)))

    def submit(self, frames, hand_side=None):
        """Enqueues one batch; returns its device result tensors (see the class notes), and in track mode also detected (bool)."""
        t = self._i
        k = t & 1
        detect = self._detect_now(t) if self.track and not self.slots else True
        self._i += 1
        cur = torch.cuda.current_stream(self.ctx.device)
        cur.wait_event(self._d2h_done[k])           # stream() may still be reading this buffer's previous results
        if self.rig or isinstance(frames, (list, tuple)):
            self._upload_slots(frames, hand_side, k, cur)
        elif isinstance(frames, torch.Tensor) and frames.is_cuda:
            if frames.dtype != torch.uint8 or not frames.is_contiguous():
                raise TypeError("FrameRunner: frames must be contiguous uint8")
            self._check_frames(frames)
            self._frames[k].copy_(frames)
            if hand_side is None:
                self._hs[k].copy_(self._default_hs)
            else:
                self._hs[k].copy_(torch.as_tensor(hand_side, dtype=torch.float32).to(self.ctx.device).reshape(self.B, 2))
        else:
            src = torch.from_numpy(np.ascontiguousarray(frames)) if isinstance(frames, np.ndarray) else frames
            if not isinstance(src, torch.Tensor) or src.dtype != torch.uint8:
                raise TypeError("FrameRunner: frames must be uint8 (numpy, CPU torch or CUDA torch)")
            self._check_frames(src)
            if self._stage[k] is None:
                self._stage[k] = torch.empty(src.shape, dtype=torch.uint8).pin_memory()
            self._uploaded[k].synchronize()         # the upload that last read this staging buffer (two calls back) has finished
            self._stage[k].copy_(src)
            self._stage_hs[k].copy_(torch.as_tensor(np.asarray([[1.0, 0.0]] * self.B if hand_side is None else hand_side, np.float32)).reshape(self.B, 2))
            with torch.cuda.stream(self._copy):
                self._copy.wait_event(self._consumed[k])      # the replay that last read this input buffer has finished
                if self.draw:
                    self._copy.wait_event(self._d2h_done[k])  # and stream()'s read-back of frame_drawn, which is this buffer
                self._frames[k].copy_(self._stage[k], non_blocking=True)
                self._hs[k].copy_(self._stage_hs[k], non_blocking=True)
                self._uploaded[k].record(self._copy)
            cur.wait_event(self._uploaded[k])
        kind = 0 if detect else 1
        if self._force_table is not None:           # this step's phase of the staggered schedule (device to device, no host wait)
            self._force[k].copy_(self._force_table[t % self.redetect_every])
        self._graphs[k][kind].replay()
        self._consumed[k].record(cur)
        res = {n: self._results[k][kind][n] for n in self.RESULT_KEYS}
        if self.draw:
            fd = self._results[k][kind]["frame_drawn"]
            res["frame_drawn"] = list(fd.unbind(0)) if self.per_slot and not self.rig else fd   # one [H,W,3] view per slot
        if self.slots:
            res.update({n: self._results[k][kind][n] for n in self.SLOTS_KEYS})
        elif self.track:
            res.update({n: self._results[k][kind][n] for n in self.TRACK_KEYS})
            self._lost_host[k].copy_(res["track_lost"], non_blocking=True)   # read by step t + 2's choice
            self._lost_ready[k].record(cur)
            self._detected[k] = detect
            res["detected"] = detect
        return res

    def stream(self, batches, drawn_every=1):
        """batches: iterable of frames, or of (frames, hand_side) -> yields one numpy dict per batch, in order.

        With draw=True, frame_drawn is read back for batches i with i % drawn_every == 0 only (drawn_every = 0: never), so that a
        stream that wants key-points and an occasional picture does not copy every drawn frame to the host."""
        drawn_every = int(drawn_every)
        if drawn_every < 0:
            raise ValueError("FrameRunner.stream: drawn_every must be >= 0, got %d" % drawn_every)
        pending = None
        for i, item in enumerate(batches):
            if self.per_slot:               # a list of frames, or a (list, hand_side) pair
                pair = isinstance(item, tuple) and len(item) == 2 and isinstance(item[0], (list, tuple))
                frames, hs = item if pair else (item, None)
            else:
                frames, hs = item if isinstance(item, tuple) else (item, None)
            res = self.submit(frames, hs)
            res.pop("detected", None)       # a host value: _collect adds it
            if "frame_drawn" in res and (drawn_every == 0 or i % drawn_every):
                del res["frame_drawn"]
            k = (self._i - 1) & 1
            if self._host[k] is None:
                self._host[k] = {}
            for n, t in res.items():        # pinned host copies, created on the first read-back of each result
                if n not in self._host[k]:
                    self._host[k][n] = [torch.empty(x.shape, dtype=x.dtype).pin_memory() for x in t] if isinstance(t, list) else \
                        torch.empty(t.shape, dtype=t.dtype).pin_memory()
            self._host_keys[k] = tuple(res)
            with torch.cuda.stream(self._d2h):
                self._d2h.wait_event(self._consumed[k])
                for n, t in res.items():
                    if isinstance(t, list):     # a rig's frame_drawn: one image per camera
                        for dst, src in zip(self._host[k][n], t):
                            dst.copy_(src, non_blocking=True)
                    else:
                        self._host[k][n].copy_(t, non_blocking=True)
                self._d2h_done[k].record(self._d2h)
            if pending is not None:
                yield self._collect(pending)
            pending = k
        if pending is not None:
            yield self._collect(pending)

    def _collect(self, k):
        self._d2h_done[k].synchronize()             # the read-back the caller asked for
        out = {n: [x.numpy().copy() for x in self._host[k][n]] if isinstance(self._host[k][n], list) else self._host[k][n].numpy().copy()
               for n in self._host_keys[k]}
        if self.track and not self.slots:
            out["detected"] = self._detected[k]
        return out
