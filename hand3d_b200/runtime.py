"""Host-side runtime over the C ABI: one Context per CUDA device (weights, workspace, precision).

Mirrors the role the default TF graph + tf.Session play in the reference (nets/ColorHandPose3DNetwork.py:34-59):
`default_context()` is what `ColorHandPose3DNetwork.init()` loads the pickled variables into and what the
static `inference_detection()` / `NetworkOps` helpers look their variables up in.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import PRECISIONS, VARIANTS


def _ptr(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _chk_f32(t, name, ndim=None):
    if not isinstance(t, torch.Tensor):
        raise TypeError("%s must be a torch.Tensor" % name)
    if not t.is_cuda:
        raise RuntimeError("%s must live on a CUDA device (hand3d_b200 has no CPU path)" % name)
    if t.dtype != torch.float32:
        raise TypeError("%s must be float32" % name)
    if ndim is not None and t.dim() != ndim:
        raise ValueError("%s must be %d-D, got %s" % (name, ndim, tuple(t.shape)))
    return t.contiguous()


def frame_shape(pixel_format, H, W):
    """The tensor shape of one H x W frame in pixel_format (include/hand3d_b200.h's table): rgb / bgr (H, W, 3), nv12 / i420
    (H * 3 / 2, W) with H and W even, yuyv (H, W, 2) with W even."""
    if pixel_format not in _lib.PIXEL_FORMATS:
        raise ValueError("pixel_format must be one of %s, got %r" % (sorted(_lib.PIXEL_FORMATS), pixel_format))
    H, W = int(H), int(W)
    if pixel_format in ("nv12", "i420"):
        if H % 2 or W % 2:
            raise ValueError("%s frames must have an even height and width, got %dx%d" % (pixel_format, H, W))
        return (H * 3 // 2, W)
    if pixel_format == "yuyv":
        if W % 2:
            raise ValueError("yuyv frames must have an even width, got %d" % W)
        return (H, W, 2)
    return (H, W, 3)


def _frames_bhw(frames, pixel_format):
    """A CUDA uint8 batch of frames in pixel_format -> (B, H, W) of its pictures; the sizes themselves are checked by the C entry."""
    if pixel_format not in _lib.PIXEL_FORMATS:
        raise ValueError("pixel_format must be one of %s, got %r" % (sorted(_lib.PIXEL_FORMATS), pixel_format))
    if not isinstance(frames, torch.Tensor):
        raise TypeError("frames must be a torch.Tensor")
    if not frames.is_cuda:
        raise RuntimeError("frames must live on a CUDA device (hand3d_b200 has no CPU path)")
    if frames.dtype != torch.uint8:
        raise TypeError("frames must be uint8, got %s" % frames.dtype)
    shp = tuple(frames.shape)
    if pixel_format in ("nv12", "i420"):
        if len(shp) != 3 or shp[1] % 3:
            raise ValueError("%s frames must be [B,H*3/2,W], got %s" % (pixel_format, shp))
        B, H, W = shp[0], shp[1] * 2 // 3, shp[2]
    elif pixel_format == "yuyv":
        if len(shp) != 4 or shp[3] != 2:
            raise ValueError("yuyv frames must be [B,H,W,2], got %s" % (shp,))
        B, H, W = shp[:3]
    else:
        if len(shp) != 4 or shp[3] != 3:
            raise ValueError("frames must be [B,H,W,3] %s, got %s" % (pixel_format.upper(), shp))
        B, H, W = shp[:3]
    if not frames.is_contiguous():
        raise ValueError("frames must be contiguous")
    return B, H, W


def _chk_params(params, B):
    if params is None:
        return None
    params = _chk_f32(params, "params", 2)
    if tuple(params.shape) != (B, _lib.AUG_PARAMS):
        raise ValueError("params must be [%d, %d], got %s" % (B, _lib.AUG_PARAMS, tuple(params.shape)))
    return params


class Context:
    def __init__(self, device=None, precision="bf16x3"):
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise RuntimeError("hand3d_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        h = C.c_void_p()
        _lib.check(self.lib.h3d_create(C.byref(h), self.device.index), "h3d_create")
        self.h = h
        self._ws = None
        self._ws_key = (0, 0, 0)
        self.weights = {}
        self.dropout_seed = None     # set_dropout()
        self._dropout_on = False     # the C-level switch, turned per call by _dropout_mode()
        self._draw = None
        self.set_precision(precision)

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.lib.h3d_destroy(self.h)
                self.h = None
        except Exception:
            pass

    # ---- configuration -------------------------------------------------------------------
    def _no_live_graphs(self, what):
        # captured graphs bake in plan-owned device pointers (packed operands, workspace views): rebuilding the plans under a
        # live graph would make its replay touch freed memory
        if getattr(self, "_graphs_captured", 0):
            raise RuntimeError("%s rebuilds the stage plans, which captured CUDA graphs still point into; drop the graphs and call "
                               "release_graphs() first" % what)

    def set_precision(self, precision):
        p = PRECISIONS[precision] if isinstance(precision, str) else int(precision)
        if p != getattr(self, "precision", None):
            self._no_live_graphs("set_precision()")
        _lib.check(self.lib.h3d_set_precision(self.h, p), "h3d_set_precision")
        self.precision = p

    def set_tuning(self, key, value):
        """Kernel-selection switch (process-wide, see include/hand3d_b200.h: h3d_set_tuning); drops this context's plans."""
        self._no_live_graphs("set_tuning()")
        _lib.check(self.lib.h3d_set_tuning(self.h, key.encode(), int(value)), "h3d_set_tuning(%s)" % key)

    # ---- dropout (evaluation=False in the lifting stage; include/hand3d_b200.h: H3D_DROPOUT_*) ---------------------------
    def set_dropout(self, seed):
        """Seeds the context's dropout generator and sets its draw counter to 0; None turns dropout off again.  Only calls that ask for
        dropout apply it (evaluation=False, or dropout=True here); every other call computes what it computes without a seed."""
        if seed is None:
            self._dropout_mode(False)
            self.dropout_seed = None
            return
        seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        _lib.check(self.lib.h3d_set_dropout(self.h, 1, C.c_uint64(seed)), "h3d_set_dropout")
        self._dropout_on = True
        self.dropout_seed = seed
        self._draw_counter().zero_()          # the same seed again restarts its stream as well

    def _dropout_mode(self, on):
        if on and self.dropout_seed is None:
            raise NotImplementedError("evaluation=False applies dropout, which needs a seeded generator: call set_dropout(seed) on the "
                                      "context (runtime.default_context()) first")
        if bool(on) != self._dropout_on:
            _lib.check(self.lib.h3d_set_dropout(self.h, int(bool(on)), C.c_uint64(self.dropout_seed or 0)), "h3d_set_dropout")
            self._dropout_on = bool(on)

    def _draw_counter(self):
        """The int64 [1] draw counter in the context's device memory (an alias, not a copy)."""
        if self._draw is None:
            p = C.c_void_p()
            _lib.check(self.lib.h3d_dropout_draw(self.h, C.byref(p)), "h3d_dropout_draw")

            class _Counter:
                __cuda_array_interface__ = {"shape": (1,), "typestr": "<i8", "data": (p.value, False), "version": 2}
            self._draw = torch.as_tensor(_Counter(), device=self.device)
        return self._draw

    def dropout_state(self):
        """A device copy (int64 [1]) of the draw counter, enqueued on the current stream: pass it to load_dropout_state() to replay
        the same masks."""
        return self._draw_counter().clone()

    def load_dropout_state(self, state):
        """Sets the draw counter from dropout_state()'s tensor or an int."""
        d = self._draw_counter()
        if torch.is_tensor(state):
            d.copy_(state.reshape(1))
        else:
            d.fill_(int(state))

    def dropout_forward(self, x, keep_prob, layer):
        """TF 1.3 dropout of x [rows, ...] fp32 at the current draw (row = index along dim 0) -> (y, keep uint8), without advancing."""
        x = _chk_f32(x, "x")
        if x.dim() < 1 or x.numel() == 0:
            raise ValueError("dropout needs a non-empty tensor")
        self._dropout_mode(True)
        y = torch.empty_like(x)
        keep = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
        _lib.check(self.lib.h3d_dropout_forward(self.h, _ptr(x), x.shape[0], x.numel() // x.shape[0], float(keep_prob), int(layer), _ptr(y),
                                                _ptr(keep), _stream()), "h3d_dropout_forward")
        return y, keep

    def dropout_backward(self, dy, keep, keep_prob):
        """dx = (dy * keep) / keep_prob."""
        dy = _chk_f32(dy, "dy")
        if keep.dtype != torch.uint8 or keep.shape != dy.shape or keep.device != dy.device:
            raise ValueError("keep must be a uint8 tensor shaped like dy on its device")
        self._dropout_mode(True)
        dx = torch.empty_like(dy)
        _lib.check(self.lib.h3d_dropout_backward(self.h, _ptr(dy), _ptr(keep.contiguous()), dy.shape[0], dy.numel() // dy.shape[0],
                                                 float(keep_prob), _ptr(dx), _stream()), "h3d_dropout_backward")
        return dx

    def dropout_advance(self):
        """Adds 1 to the draw counter on the device."""
        self._dropout_mode(True)
        _lib.check(self.lib.h3d_dropout_advance(self.h, _stream()), "h3d_dropout_advance")

    @property
    def launch_count(self):
        return int(self.lib.h3d_launch_count(self.h))

    def check_errors(self):
        """Raises if a kernel reported a device-side timeout (bounded barrier wait, missing gather peer); see h3d_check_errors."""
        code = C.c_int(0)
        _lib.check(self.lib.h3d_check_errors(self.h, C.byref(code)), "device-side error word = %d" % code.value)

    def profile_begin(self):
        _lib.check(self.lib.h3d_profile_begin(self.h), "h3d_profile_begin")

    def profile_end(self):
        ms = (C.c_double * 4)(); fl = (C.c_int64 * 4)(); nl = (C.c_int64 * 4)()
        _lib.check(self.lib.h3d_profile_end(self.h, ms, fl, nl), "h3d_profile_end")
        names = ("tc_conv", "direct_conv", "fc", "other")
        return {n: {"ms": ms[i], "flops": int(fl[i]), "launches": int(nl[i])} for i, n in enumerate(names)}

    def load_weights(self, weight_dict):
        for name, arr in weight_dict.items():
            a = np.ascontiguousarray(arr, dtype=np.float32)
            shape = (C.c_int64 * a.ndim)(*a.shape)
            rc = self.lib.h3d_load_weight(self.h, name.encode(), a.ctypes.data_as(C.c_void_p), shape, a.ndim)
            if rc == _lib.EWEIGHTS:
                raise ValueError(_lib.last_error())
            _lib.check(rc, "h3d_load_weight(%s)" % name)
            self.weights[name] = a
            self.__dict__.get("_dev_w", {}).pop(name, None)    # the operator-level device copy follows the reload
            scope = name.split("/")[0]
            var = self.__dict__.get("_variables", {}).get(scope)
            if var is not None and name in var and tuple(var[name].shape) != a.shape:
                del self._variables[scope]    # fc_xyz changed between 512 x 63 and 30 x 63 (fc_bottleneck): new Parameters next time
                var = None
            if var is not None and name in var:   # so do the trainable variables: in place, so an optimiser over them stays valid
                with torch.no_grad():
                    var[name].copy_(torch.from_numpy(a))

    def scope_ready(self, scope):
        return bool(self.lib.h3d_scope_ready(self.h, scope.encode()))

    def dev_weight(self, name):
        """fp32 device copy of a loaded variable (for the operator-level NetworkOps mirror)."""
        cache = self.__dict__.setdefault("_dev_w", {})
        if name not in cache:
            if name not in self.weights:
                raise ValueError("variable %s was not loaded" % name)
            cache[name] = torch.from_numpy(self.weights[name]).to(self.device)
        return cache[name]

    def ensure_workspace(self, B, H, W):
        kB, kH, kW = max(B, self._ws_key[0]), max(H, self._ws_key[1]), max(W, self._ws_key[2])
        if (kB, kH, kW) == self._ws_key and self._ws is not None:
            return
        if getattr(self, "_graphs_captured", 0):
            raise RuntimeError("the workspace cannot grow (to B=%d, %dx%d) after capture_pipeline(): captured CUDA graphs hold its "
                               "pointers; call release_graphs() first or size it up front with ensure_workspace()" % (kB, kH, kW))
        need = int(self.lib.h3d_workspace_bytes(self.h, kB, kH, kW))
        if need < 0:
            _lib.check(need, "h3d_workspace_bytes")
        torch.cuda.synchronize(self.device)
        self._ws = None
        self._ws = torch.empty(need + 1024, dtype=torch.uint8, device=self.device)
        base = (self._ws.data_ptr() + 1023) // 1024 * 1024
        _lib.check(self.lib.h3d_set_workspace(self.h, C.c_void_p(base), need), "h3d_set_workspace")
        self._ws_key = (kB, kH, kW)

    def fill_scratch(self, byte):
        """Fills the workspace and the operator scratch with one byte value on the current stream (h3d_fill_scratch): no result may
        depend on what they held before a call.  For tests; the scratch grows on demand, so size it with one call first."""
        _lib.check(self.lib.h3d_fill_scratch(self.h, int(byte), _stream()), "h3d_fill_scratch")

    # ---- stages ----------------------------------------------------------------------------
    def handsegnet(self, image):
        image = _chk_f32(image, "image", 4)
        B, H, W, _ = image.shape
        self.ensure_workspace(B, H, W)
        out = torch.empty((B, H, W, 2), dtype=torch.float32, device=image.device)
        _lib.check(self.lib.h3d_handsegnet_forward(self.h, _ptr(image), B, H, W, _ptr(out), _stream()), "h3d_handsegnet_forward")
        return out

    def posenet(self, image_crop):
        image_crop = _chk_f32(image_crop, "image_crop", 4)
        B, H, W, _ = image_crop.shape
        self.ensure_workspace(B, H if H > 256 else 8, W if W > 256 else 8)   # crops up to 256x256 fit every layout
        outs = [torch.empty((B, H // 8, W // 8, 21), dtype=torch.float32, device=image_crop.device) for _ in range(3)]
        _lib.check(self.lib.h3d_posenet_forward(self.h, _ptr(image_crop), B, H, W, _ptr(outs[0]), _ptr(outs[1]), _ptr(outs[2]),
                                                _stream()), "h3d_posenet_forward")
        return outs

    def pose2d(self, image_crop, outputs="all"):
        """inference_pose2d + x8 up-sampling + detect_keypoints (eval2d_gt_cropped.py:45-50,78).  Returns dict with
        keypoints_scoremap [B,H,W,21] (None with outputs="keypoints" and crops <= 256x256) and keypoints_uv [B,21,2] int32."""
        image_crop = _chk_f32(image_crop, "image_crop", 4)
        B, H, W, _ = image_crop.shape
        self.ensure_workspace(B, H if H > 256 else 8, W if W > 256 else 8)
        big = outputs == "all" or H > 256 or W > 256
        sm = torch.empty((B, H, W, 21), dtype=torch.float32, device=image_crop.device) if big else None
        uv = torch.empty((B, 21, 2), dtype=torch.int32, device=image_crop.device)
        _lib.check(self.lib.h3d_pose2d_forward(self.h, _ptr(image_crop), B, H, W, _ptr(sm), _ptr(uv), _stream()), "h3d_pose2d_forward")
        return {"keypoints_scoremap": sm, "keypoints_uv": uv}

    def lifting(self, scoremap32, hand_side, variant="proposed", dropout=False):
        """PosePrior (+ ViewpointNet): [B,32,32,21], [B,2] -> (out, can, R).  dropout=True (evaluation=False) applies the four dropout
        layers at the current draw and advances it; it needs set_dropout()."""
        scoremap32 = _chk_f32(scoremap32, "scoremap", 4)
        hand_side = _chk_f32(hand_side, "hand_side", 2)
        B = scoremap32.shape[0]
        if tuple(scoremap32.shape[1:]) != (32, 32, 21):
            raise ValueError("lifting expects a [B,32,32,21] score map, got %s" % (tuple(scoremap32.shape),))
        self.ensure_workspace(B, 8, 8)
        dev = scoremap32.device
        out = torch.empty((B, 21, 3), dtype=torch.float32, device=dev)
        can = torch.empty((B, 21, 3), dtype=torch.float32, device=dev)
        v = VARIANTS[variant]
        rot = torch.empty((B, 3, 3), dtype=torch.float32, device=dev) if variant == "proposed" else None
        self._dropout_mode(dropout)
        _lib.check(self.lib.h3d_lifting_forward(self.h, _ptr(scoremap32), _ptr(hand_side), B, v, _ptr(out), _ptr(can), _ptr(rot),
                                                _stream()), "h3d_lifting_forward")
        return out, can, rot

    def pipeline(self, image, hand_side=None, with_pose3d=True, force_center=None, force_scale=None, want_mask=False,
                 outputs="all", dropout=False):
        """ColorHandPose3DNetwork.inference / inference2d + detect_keypoints.  outputs="all" materialises the
        reference's large tensors; outputs="keypoints" keeps them in the workspace (serving mode).  dropout=True: the lifting as in
        lifting(dropout=True)."""
        image = _chk_f32(image, "image", 4)
        B, H, W, _ = image.shape
        dev = image.device
        if with_pose3d:
            hand_side = _chk_f32(hand_side, "hand_side", 2)
        self.ensure_workspace(B, H, W)
        f32 = dict(dtype=torch.float32, device=dev)
        big = outputs == "all"
        r = {
            "hand_scoremap": torch.empty((B, H, W, 2), **f32) if big else None,
            "image_crop": torch.empty((B, 256, 256, 3), **f32) if big else None,
            "scale_crop": torch.empty((B, 1), **f32),
            "center": torch.empty((B, 2), **f32),
            "keypoints_scoremap": torch.empty((B, 256, 256, 21), **f32) if big else None,
            "keypoint_coord3d": torch.empty((B, 21, 3), **f32) if with_pose3d else None,
            "keypoints_uv": torch.empty((B, 21, 2), dtype=torch.int32, device=dev),
            "hand_mask": torch.empty((B, H, W), dtype=torch.uint8, device=dev) if want_mask else None,
        }
        fc = _chk_f32(force_center, "force_center") if force_center is not None else None
        fs = _chk_f32(force_scale, "force_scale") if force_scale is not None else None
        self._dropout_mode(dropout)
        _lib.check(self.lib.h3d_pipeline_forward(
            self.h, _ptr(image), _ptr(hand_side if with_pose3d else None), B, H, W, int(bool(with_pose3d)), _ptr(fc), _ptr(fs),
            _ptr(r["hand_scoremap"]), _ptr(r["image_crop"]), _ptr(r["scale_crop"]), _ptr(r["center"]),
            _ptr(r["keypoints_scoremap"]), _ptr(r["keypoint_coord3d"]), _ptr(r["keypoints_uv"]), _ptr(r["hand_mask"]),
            _stream()), "h3d_pipeline_forward")
        return r

    def capture_pipeline(self, image, hand_side=None, with_pose3d=True, outputs="keypoints"):
        """Captures one pipeline() call on fixed input tensors into a CUDA graph (the forward pass has no host
        synchronisation, no allocation and only fixed workspace pointers, so ~90 launches replay as one).
        Returns (replay, results): refill `image` / `hand_side` in place, call replay(), read `results`."""
        image = _chk_f32(image, "image", 4)
        self.ensure_workspace(*image.shape[:3])
        side = torch.cuda.Stream(device=image.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):                       # warm-up outside capture: builds plans, packs weights
            self.pipeline(image, hand_side, with_pose3d, outputs=outputs)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize(image.device)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            results = self.pipeline(image, hand_side, with_pose3d, outputs=outputs)
        self._graphs_captured = getattr(self, "_graphs_captured", 0) + 1    # the graph bakes in workspace pointers: no growth from now on
        return graph.replay, results

    def release_graphs(self):
        """Declares every graph returned by capture_pipeline() dead (the caller must drop them); the workspace may grow again."""
        self._graphs_captured = 0

    def track_step(self, image, hand_side, state, detect, margin=1.5, min_score=None, outputs="all", with_pose3d=True, dropout=False):
        """One step of a tracked stream per batch slot (h3d_track_step, DESIGN.md section 4.14).  detect=True runs pipeline() (no
        forced crop); detect=False crops at state.center / state.scale and skips HandSegNet and the mask post-processing.  Either way
        the step then updates `state` (a TrackState of the same batch) from its key-points: the next crop, the score and the lost
        flag.  min_score None turns the score test off.  Returns image_crop, scale_crop, center (the crop this step used),
        keypoints_scoremap, keypoint_coord3d and keypoints_uv as pipeline() does; outputs="keypoints" leaves the large ones in the
        workspace.  dropout=True: the lifting as in lifting(dropout=True).  Enqueue-only: a call on fixed tensors can be captured into a
        CUDA graph."""
        image = _chk_f32(image, "image", 4)
        B, H, W, _ = image.shape
        dev = image.device
        if with_pose3d:
            hand_side = _chk_f32(hand_side, "hand_side", 2)
        if not isinstance(state, TrackState) or state.B != B or state.buffer.device != dev:
            raise ValueError("state must be a TrackState of batch %d on %s" % (B, dev))
        self.ensure_workspace(B, H, W)
        f32 = dict(dtype=torch.float32, device=dev)
        big = outputs == "all"
        r = {
            "image_crop": torch.empty((B, 256, 256, 3), **f32) if big else None,
            "scale_crop": torch.empty((B, 1), **f32),
            "center": torch.empty((B, 2), **f32),
            "keypoints_scoremap": torch.empty((B, 256, 256, 21), **f32) if big else None,
            "keypoint_coord3d": torch.empty((B, 21, 3), **f32) if with_pose3d else None,
            "keypoints_uv": torch.empty((B, 21, 2), dtype=torch.int32, device=dev),
        }
        self._dropout_mode(dropout)
        _lib.check(self.lib.h3d_track_step(
            self.h, _ptr(image), _ptr(hand_side if with_pose3d else None), B, H, W, int(bool(with_pose3d)), int(bool(detect)),
            float(margin), float("nan") if min_score is None else float(min_score), _ptr(state.buffer),
            _ptr(r["image_crop"]), _ptr(r["scale_crop"]), _ptr(r["center"]), _ptr(r["keypoints_scoremap"]),
            _ptr(r["keypoint_coord3d"]), _ptr(r["keypoints_uv"]), _stream()), "h3d_track_step")
        return r

    def track_step_slots(self, image, hand_side, state, force=None, margin=1.5, min_score=None, outputs="all", with_pose3d=True,
                         dropout=False):
        """A track step that re-detects only the slots that need it (h3d_track_step_slots, DESIGN.md section 4.15): slot b runs
        HandSegNet and the mask post-processing when state.lost[b] (from the previous step) or force[b] (optional CUDA int32 or bool [B])
        is set, and is cropped from the state otherwise.  The choice is made on the device: nothing is read back.  Returns track_step's
        keys plus track_detected [B] bool (the slots this step re-detected).  Enqueue-only after the first call for a shape: a call on
        fixed tensors can be captured into a CUDA graph."""
        image = _chk_f32(image, "image", 4)
        B, H, W, _ = image.shape
        dev = image.device
        if with_pose3d:
            hand_side = _chk_f32(hand_side, "hand_side", 2)
        if not isinstance(state, TrackState) or state.B != B or state.buffer.device != dev:
            raise ValueError("state must be a TrackState of batch %d on %s" % (B, dev))
        if force is not None:
            if not isinstance(force, torch.Tensor) or not force.is_cuda or force.device != dev or force.numel() != B:
                raise ValueError("force must be a CUDA tensor of %d elements on %s" % (B, dev))
            if force.dtype != torch.int32:
                force = force.to(torch.int32)
            force = force.contiguous()
        self.ensure_workspace(B, H, W)
        f32 = dict(dtype=torch.float32, device=dev)
        big = outputs == "all"
        r = {
            "image_crop": torch.empty((B, 256, 256, 3), **f32) if big else None,
            "scale_crop": torch.empty((B, 1), **f32),
            "center": torch.empty((B, 2), **f32),
            "keypoints_scoremap": torch.empty((B, 256, 256, 21), **f32) if big else None,
            "keypoint_coord3d": torch.empty((B, 21, 3), **f32) if with_pose3d else None,
            "keypoints_uv": torch.empty((B, 21, 2), dtype=torch.int32, device=dev),
        }
        detected = torch.empty(B, dtype=torch.int32, device=dev)
        self._dropout_mode(dropout)
        _lib.check(self.lib.h3d_track_step_slots(
            self.h, _ptr(image), _ptr(hand_side if with_pose3d else None), B, H, W, int(bool(with_pose3d)),
            float(margin), float("nan") if min_score is None else float(min_score), _ptr(state.buffer), _ptr(force), _ptr(detected),
            _ptr(r["image_crop"]), _ptr(r["scale_crop"]), _ptr(r["center"]), _ptr(r["keypoints_scoremap"]),
            _ptr(r["keypoint_coord3d"]), _ptr(r["keypoints_uv"]), _stream()), "h3d_track_step_slots")
        r["track_detected"] = detected != 0
        return r

    def track_update(self, scoremap32, keypoints_uv, center, scale_crop, state, margin=1.5, min_score=None):
        """track_step's update alone (h3d_track_update): scoremap32 [B,32,32,21], keypoints_uv [B,21,2] int32, center [B,2] and
        scale_crop [B] or [B,1] of the crop the key-points were found in -> `state` (a TrackState of batch B)."""
        scoremap32 = _chk_f32(scoremap32, "scoremap32", 4)
        B = scoremap32.shape[0]
        if tuple(scoremap32.shape[1:]) != (32, 32, 21):
            raise ValueError("track_update expects a [B,32,32,21] score map, got %s" % (tuple(scoremap32.shape),))
        center = _chk_f32(center, "center").reshape(B, 2)
        scale_crop = _chk_f32(scale_crop, "scale_crop").reshape(B)
        if keypoints_uv.dtype != torch.int32 or tuple(keypoints_uv.shape) != (B, 21, 2) or not keypoints_uv.is_cuda:
            raise ValueError("keypoints_uv must be a CUDA int32 [%d,21,2] tensor" % B)
        if not isinstance(state, TrackState) or state.B != B:
            raise ValueError("state must be a TrackState of batch %d" % B)
        _lib.check(self.lib.h3d_track_update(self.h, _ptr(scoremap32), _ptr(keypoints_uv.contiguous()), _ptr(center), _ptr(scale_crop),
                                             B, float(margin), float("nan") if min_score is None else float(min_score),
                                             _ptr(state.buffer), _stream()), "h3d_track_update")

    # ---- operators ---------------------------------------------------------------------------
    def conv2d(self, x, w, b, stride=1, leaky=False):
        x = _chk_f32(x, "x", 4); w = _chk_f32(w, "w", 4); b = _chk_f32(b, "b", 1)
        B, H, W, Cin = x.shape
        k, _, _, Cout = w.shape
        y = torch.empty((B, -(-H // stride), -(-W // stride), Cout), dtype=torch.float32, device=x.device)
        _lib.check(self.lib.h3d_conv2d_f32(self.h, _ptr(x), _ptr(w), _ptr(b), _ptr(y), B, H, W, Cin, Cout, k, stride, int(leaky),
                                           _stream()), "h3d_conv2d_f32")
        return y

    def conv2d_tc(self, x, w_host, b_host, leaky=False, precision="bf16x3", stride=1):
        """Host-weight convenience form (packs, uploads and frees the weights around the call)."""
        x = _chk_f32(x, "x", 4)
        w = np.ascontiguousarray(w_host, np.float32); b = np.ascontiguousarray(b_host, np.float32)
        B, H, W, Cin = x.shape
        k, _, _, Cout = w.shape
        if stride not in (1, 2) or (stride == 2 and (H % 2 or W % 2 or k < 3)):
            raise ValueError("conv2d_tc: stride must be 1, or 2 with even H and W and a kernel size >= 3")
        y = torch.empty((B, H // stride, W // stride, Cout), dtype=torch.float32, device=x.device)
        _lib.check(self.lib.h3d_conv2d_tc_strided(self.h, _ptr(x), w.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), _ptr(y),
                                                  B, H, W, Cin, Cout, k, stride, int(leaky), PRECISIONS[precision], _stream()),
                   "h3d_conv2d_tc_strided")
        return y

    def pack_conv(self, w_host, b_host, precision="bf16x3"):
        """Packs HWIO weights once for conv2d_tc_packed (the enqueue-only tensor-core operator)."""
        w = np.ascontiguousarray(w_host, np.float32); b = np.ascontiguousarray(b_host, np.float32)
        k, _, Cin, Cout = w.shape
        h = C.c_void_p()
        _lib.check(self.lib.h3d_pack_conv_weights(self.h, w.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), k, Cin, Cout,
                                                  PRECISIONS[precision], C.byref(h)), "h3d_pack_conv_weights")
        return PackedConv(self, h, k, Cin, Cout)

    def conv2d_tc_packed(self, x, packed, leaky=False, stride=1):
        x = _chk_f32(x, "x", 4)
        B, H, W, Cin = x.shape
        if Cin != packed.Cin:
            raise ValueError("conv2d_tc_packed: input has %d channels, weights expect %d" % (Cin, packed.Cin))
        y = torch.empty((B, H // stride, W // stride, packed.Cout), dtype=torch.float32, device=x.device)
        _lib.check(self.lib.h3d_conv2d_tc_packed(self.h, _ptr(x), packed.h, _ptr(y), B, H, W, stride, int(leaky), _stream()),
                   "h3d_conv2d_tc_packed")
        return y

    def conv2d_tc_dev(self, x, w, b, stride=1, leaky=False, precision="bf16x3"):
        """Tensor-core convolution with DEVICE weights (w HWIO [k,k,Cin,Cout], b [Cout]): packed on the GPU every call, enqueue-only;
        bit-identical to pack_conv + conv2d_tc_packed for the same weights."""
        x = _chk_f32(x, "x", 4); w = _chk_f32(w, "w", 4); b = _chk_f32(b, "b", 1)
        B, H, W, Cin = x.shape
        k, _, wc, Cout = w.shape
        if wc != Cin or b.shape[0] != Cout:
            raise ValueError("conv2d_tc_dev: x %s, w %s and b %s do not match" % (tuple(x.shape), tuple(w.shape), tuple(b.shape)))
        y = torch.empty((B, H // stride, W // stride, Cout), dtype=torch.float32, device=x.device)
        _lib.check(self.lib.h3d_conv2d_tc_dev(self.h, _ptr(x), _ptr(w), _ptr(b), _ptr(y), B, H, W, Cin, Cout, k, stride, int(leaky),
                                              PRECISIONS[precision], _stream()), "h3d_conv2d_tc_dev")
        return y

    # plane canaries of conv_layer: NaN bit patterns in every format, which no layer output of finite operands takes
    CANARY16, CANARY8, CANARY32 = 0x7FA5, 0x7F, 0x7FC0A5A5

    def conv_layer(self, x, w_host, b_host, precision, route=0, pool=0, leaky=True, perm=None, planes=True, Cy_total=None, cy_off=0,
                   yf=False, Cyf_total=None, cyf_off=0, out=None):
        """One network layer as the stage entries build it (h3d_conv2d_layer_planes): x fp32 [B,H,W,Cx] on the device, host weights
        HWIO [k,k,Cin,Cout].  Returns {"hi", "lo", "l8", "h8", "yf"}: the raw planes (uint16 / uint8 [B,Ho,Wo,Cy_total], all four
        whatever the precision, so a test can see which ones were written) and the fp32 output [B,Ho,Wo,Cyf_total], each None when not
        requested.  Buffers come from `out` (a dict of the same keys) or are filled with the CANARY* patterns."""
        x = _chk_f32(x, "x", 4)
        w = np.ascontiguousarray(w_host, np.float32); b = np.ascontiguousarray(b_host, np.float32)
        B, H, W, Cx = x.shape
        k, _, Cin, Cout = w.shape
        Ho, Wo = (H // 2, W // 2) if pool else (H, W)
        Cout_pad = -(-Cout // 64) * 64
        out = dict(out or {})
        dev = x.device

        def buf(key, C, dtype, fill):
            if out.get(key) is None:
                t = torch.empty((B, Ho, Wo, C), dtype=dtype, device=dev)
                t.view(torch.int32 if dtype == torch.float32 else dtype).fill_(fill)
                out[key] = t
            return out[key]
        if planes:
            Cy_total = Cout_pad if Cy_total is None else Cy_total
            for key in ("hi", "lo"):
                buf(key, Cy_total, torch.int16, self.CANARY16)
            for key in ("l8", "h8"):
                buf(key, Cy_total, torch.uint8, self.CANARY8)
        else:
            Cy_total = 0
            for key in ("hi", "lo", "l8", "h8"):
                out[key] = None
        if yf:
            Cyf_total = Cout if Cyf_total is None else Cyf_total
            buf("yf", Cyf_total, torch.float32, self.CANARY32)
        else:
            Cyf_total, out["yf"] = 0, None
        p = None
        if perm is not None:
            p = np.ascontiguousarray(perm, np.int32)
            if p.shape != (-(-Cin // 64) * 64,):
                raise ValueError("conv_layer: perm must have align_up(Cin, 64) = %d entries, got %s" % (-(-Cin // 64) * 64, p.shape))
        _lib.check(self.lib.h3d_conv2d_layer_planes(
            self.h, _ptr(x), B, H, W, Cx, w.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), k, Cin, Cout,
            None if p is None else p.ctypes.data_as(C.c_void_p), int(pool), int(bool(leaky)), PRECISIONS[precision], int(route),
            _ptr(out["hi"]), _ptr(out["lo"]), _ptr(out["l8"]), _ptr(out["h8"]), int(Cy_total), int(cy_off), _ptr(out["yf"]),
            int(Cyf_total), int(cyf_off), _stream()), "h3d_conv2d_layer_planes")
        return out

    def conv2d_tc_backward(self, x, y, dy, w, stride=1, leaky=False, precision="bf16x3", need_dx=True, need_dw=True, need_db=True):
        """Gradients (dx, dw, db) of y = act(conv_SAME(x, w, stride) + b); outputs not needed come back as None.  y (the forward
        output) is read only with leaky, x only for dw, w only for dx."""
        dy = _chk_f32(dy, "dy", 4)
        w = _chk_f32(w, "w", 4)
        k, _, Cin, Cout = w.shape
        B, Ho, Wo, _ = dy.shape
        H, W = Ho * stride, Wo * stride
        if need_dw:
            x = _chk_f32(x, "x", 4)
            if tuple(x.shape) != (B, H, W, Cin):
                raise ValueError("conv2d_tc_backward: x %s does not match dy %s / w %s" % (tuple(x.shape), tuple(dy.shape), tuple(w.shape)))
        if leaky:
            y = _chk_f32(y, "y", 4)
        f32 = dict(dtype=torch.float32, device=dy.device)
        dx = torch.empty((B, H, W, Cin), **f32) if need_dx else None
        dw = torch.empty((k, k, Cin, Cout), **f32) if need_dw else None
        db = torch.empty((Cout,), **f32) if need_db else None
        _lib.check(self.lib.h3d_conv2d_tc_backward(
            self.h, _ptr(x if need_dw else None), _ptr(y if leaky else None), _ptr(dy), _ptr(w if need_dx else None), _ptr(dx), _ptr(dw),
            _ptr(db), B, H, W, Cin, Cout, k, stride, int(leaky), PRECISIONS[precision], _stream()), "h3d_conv2d_tc_backward")
        return dx, dw, db

    def leaky_relu(self, x):
        x = _chk_f32(x, "x")
        y = torch.empty_like(x)
        _lib.check(self.lib.h3d_leaky_relu_f32(self.h, _ptr(x), _ptr(y), x.numel(), _stream()), "h3d_leaky_relu_f32")
        return y

    def calc_center_bb(self, mask):
        """mask [B,H,W] float32 -> (center [B,2], bb [B,2,2], crop_size [B,1]) (utils/general.py:271-328)."""
        mask = _chk_f32(mask, "binary_class_mask", 3)
        B, H, W = mask.shape
        dev = mask.device
        center = torch.empty((B, 2), dtype=torch.float32, device=dev)
        bb = torch.empty((B, 2, 2), dtype=torch.float32, device=dev)
        size = torch.empty((B, 1), dtype=torch.float32, device=dev)
        _lib.check(self.lib.h3d_calc_center_bb(self.h, _ptr(mask), B, H, W, _ptr(center), _ptr(bb), _ptr(size), _stream()), "h3d_calc_center_bb")
        return center, bb, size

    def flip_right_hand(self, coords_xyz, cond_right):
        coords_xyz = _chk_f32(coords_xyz, "coords_xyz_canonical", 3)
        B = coords_xyz.shape[0]
        cond = cond_right.reshape(B).to(torch.uint8).contiguous()
        out = torch.empty_like(coords_xyz)
        _lib.check(self.lib.h3d_flip_right_hand(self.h, _ptr(coords_xyz), _ptr(cond), B, _ptr(out), _stream()), "h3d_flip_right_hand")
        return out

    def pack_records(self, coord3d, keypoints_uv, center, scale_crop):
        """[B,108] float32 records (coord3d | key-points bit-cast | center | scale_crop), one kernel."""
        B = coord3d.shape[0]
        out = torch.empty((B, 108), dtype=torch.float32, device=coord3d.device)
        _lib.check(self.lib.h3d_pack_records(self.h, _ptr(coord3d.contiguous()), _ptr(keypoints_uv.contiguous()), _ptr(center.contiguous()),
                                             _ptr(scale_crop.contiguous()), B, _ptr(out), _stream()), "h3d_pack_records")
        return out

    def max_pool(self, x):
        x = _chk_f32(x, "x", 4)
        B, H, W, Cc = x.shape
        y = torch.empty((B, H // 2, W // 2, Cc), dtype=torch.float32, device=x.device)
        _lib.check(self.lib.h3d_maxpool2x2_f32(self.h, _ptr(x), _ptr(y), B, H, W, Cc, _stream()), "h3d_maxpool2x2_f32")
        return y

    def max_pool_backward(self, x, dy):
        """Gradient of max_pool: x [B,H,W,C] (forward input), dy [B,H/2,W/2,C] -> dx [B,H,W,C] (first maximum of each window)."""
        x = _chk_f32(x, "x", 4); dy = _chk_f32(dy, "dy", 4)
        B, H, W, Cc = x.shape
        if tuple(dy.shape) != (B, H // 2, W // 2, Cc):
            raise ValueError("max_pool_backward: dy %s does not match x %s" % (tuple(dy.shape), tuple(x.shape)))
        dx = torch.empty_like(x)
        _lib.check(self.lib.h3d_maxpool2x2_backward_f32(self.h, _ptr(x), _ptr(dy), _ptr(dx), B, H, W, Cc, _stream()),
                   "h3d_maxpool2x2_backward_f32")
        return dx

    def fully_connected(self, x, w, b, leaky=False):
        x = _chk_f32(x, "x", 2); w = _chk_f32(w, "w", 2); b = _chk_f32(b, "b", 1)
        y = torch.empty((x.shape[0], w.shape[1]), dtype=torch.float32, device=x.device)
        _lib.check(self.lib.h3d_fully_connected_f32(self.h, _ptr(x), _ptr(w), _ptr(b), _ptr(y), x.shape[0], w.shape[0], w.shape[1],
                                                    int(leaky), _stream()), "h3d_fully_connected_f32")
        return y

    def resize_bilinear(self, x, out_h, out_w):
        x = _chk_f32(x, "x", 4)
        B, H, W, Cc = x.shape
        y = torch.empty((B, out_h, out_w, Cc), dtype=torch.float32, device=x.device)
        _lib.check(self.lib.h3d_resize_bilinear_tf1(self.h, _ptr(x), _ptr(y), B, H, W, Cc, out_h, out_w, _stream()),
                   "h3d_resize_bilinear_tf1")
        return y

    def resize_frames(self, frames, out_h, out_w, normalize, out=None, pixel_format="rgb"):
        """run.py:57-59 on the device: frames uint8 CUDA (contiguous; [B,H,W,3] RGB, or pixel_format's layout, see frame_shape) ->
        [B,out_h,out_w,3], uint8 scipy.misc.imresize bytes (Pillow BILINEAR) of the RGB frames or, with normalize, float32 u / 255.0 - 0.5
        computed in double.  Other formats are converted to RGB inside the kernel first (OpenCV's cvtColor rule,
        include/hand3d_b200.h).  The first call with a new format and size builds its plan (not under graph capture); later calls only
        enqueue one kernel."""
        B, H, W = _frames_bhw(frames, pixel_format)
        dt = torch.float32 if normalize else torch.uint8
        if out is None:
            out = torch.empty((B, int(out_h), int(out_w), 3), dtype=dt, device=frames.device)
        elif out.dtype != dt or tuple(out.shape) != (B, int(out_h), int(out_w), 3) or not out.is_contiguous() or out.device != frames.device:
            raise ValueError("out must be a contiguous %s tensor [%d,%d,%d,3] on the frames' device" % (dt, B, out_h, out_w))
        _lib.check(self.lib.h3d_resize_frames_fmt(self.h, _ptr(frames), _lib.PIXEL_FORMATS[pixel_format], B, H, W, int(out_h), int(out_w),
                                                  int(bool(normalize)), _ptr(out), _stream()), "h3d_resize_frames_fmt")
        return out

    def _rig_args(self, B, pixel_formats, frame_hw, out_h, out_w):
        if len(pixel_formats) != B or len(frame_hw) != B:
            raise ValueError("a rig of %d slots needs %d pixel formats and %d sizes, got %d and %d" % (B, B, B, len(pixel_formats), len(frame_hw)))
        for b, f in enumerate(pixel_formats):
            if f not in _lib.PIXEL_FORMATS:
                raise ValueError("slot %d: pixel_format must be one of %s, got %r" % (b, sorted(_lib.PIXEL_FORMATS), f))
        fmts = (C.c_int * B)(*[_lib.PIXEL_FORMATS[f] for f in pixel_formats])
        hw = (C.c_int * (2 * B))(*[int(v) for s in frame_hw for v in s])
        return fmts, hw

    def frame_rig_plan(self, pixel_formats, frame_hw, out_h, out_w):
        """h3d_frame_rig_plan: builds the plan of a rig (slot b in pixel_formats[b] at frame_hw[b]) for resize_frames_rig, outside
        graph capture, so that a later captured call only enqueues."""
        B = len(frame_hw)
        fmts, hw = self._rig_args(B, pixel_formats, frame_hw, out_h, out_w)
        _lib.check(self.lib.h3d_frame_rig_plan(self.h, B, fmts, hw, int(out_h), int(out_w), _stream()), "h3d_frame_rig_plan")

    def resize_frames_rig(self, frames, out_h, out_w, normalize, out=None, pixel_formats=None):
        """resize_frames for a camera rig: frames is a list of B CUDA uint8 frames, one per slot, each of its own size and pixel format
        (pixel_formats[b], "rgb" when None; one frame of frame_shape(fmt, H, W), with or without a leading 1) -> [B,out_h,out_w,3], slot b
        bit for bit resize_frames of frame b alone.  One kernel per pixel format present; the first call of a new rig builds its plan
        (not under graph capture)."""
        B = len(frames)
        pixel_formats = ["rgb"] * B if pixel_formats is None else list(pixel_formats)
        if len(pixel_formats) != B:
            raise ValueError("a rig of %d frames needs %d pixel formats, got %d" % (B, B, len(pixel_formats)))
        hw, dev = [], None
        for b, (f, fmt) in enumerate(zip(frames, pixel_formats)):
            if fmt not in _lib.PIXEL_FORMATS:
                raise ValueError("slot %d: pixel_format must be one of %s, got %r" % (b, sorted(_lib.PIXEL_FORMATS), fmt))
            if isinstance(f, torch.Tensor) and f.dim() == len(frame_shape(fmt, 2, 2)):
                f = f.unsqueeze(0)
            try:
                n, H, W = _frames_bhw(f, fmt)
            except (TypeError, ValueError, RuntimeError) as e:
                raise type(e)("slot %d: %s" % (b, e)) from None
            if n != 1:
                raise ValueError("slot %d: one frame per slot, got a batch of %d" % (b, n))
            if dev is not None and f.device != dev:
                raise ValueError("slot %d: the frames must be on one device" % b)
            dev = f.device
            hw.append((H, W))
        fmts, hwa = self._rig_args(B, pixel_formats, hw, out_h, out_w)
        dt = torch.float32 if normalize else torch.uint8
        if out is None:
            out = torch.empty((B, int(out_h), int(out_w), 3), dtype=dt, device=dev)
        elif out.dtype != dt or tuple(out.shape) != (B, int(out_h), int(out_w), 3) or not out.is_contiguous() or out.device != dev:
            raise ValueError("out must be a contiguous %s tensor [%d,%d,%d,3] on the frames' device" % (dt, B, out_h, out_w))
        ptrs = (C.c_void_p * B)(*[f.data_ptr() for f in frames])
        _lib.check(self.lib.h3d_resize_frames_rig(self.h, ptrs, B, fmts, hwa, int(out_h), int(out_w), int(bool(normalize)), _ptr(out),
                                                  _stream()), "h3d_resize_frames_rig")
        return out

    def convert_frames(self, frames, pixel_format, out=None):
        """h3d_convert_frames: frames uint8 CUDA in pixel_format's layout -> uint8 RGB [B,H,W,3] at full size (OpenCV's cvtColor
        rule).  With `out` (contiguous uint8 [B,H,W,3]) it writes there and allocates nothing, so it can be captured."""
        B, H, W = _frames_bhw(frames, pixel_format)
        if out is None:
            out = torch.empty((B, H, W, 3), dtype=torch.uint8, device=frames.device)
        elif out.dtype != torch.uint8 or tuple(out.shape) != (B, H, W, 3) or not out.is_contiguous() or out.device != frames.device:
            raise ValueError("out must be a contiguous uint8 tensor [%d,%d,%d,3] on the frames' device" % (B, H, W))
        _lib.check(self.lib.h3d_convert_frames(self.h, _ptr(frames), _lib.PIXEL_FORMATS[pixel_format], B, H, W, _ptr(out), _stream()),
                   "h3d_convert_frames")
        return out

    def draw_segments(self, images, segments, colors, linewidth=1.0, valid=None):
        """h3d_draw_segments: anti-aliased segments drawn into images (CUDA uint8 [B,H,W,3], contiguous) in place, which it returns.
        segments CUDA float32 [B,S,4] (r0, c0, r1, c1) in pixels; colors [S,3] in 0..255 (host values, carried by a captured graph);
        valid CUDA int32 [B] or None (an image with valid[b] == 0 is left alone).  Enqueues one kernel and nothing else, so it can
        be captured into a CUDA graph."""
        if not isinstance(images, torch.Tensor) or not images.is_cuda:
            raise RuntimeError("images must be a CUDA tensor (hand3d_b200 has no CPU path)")
        if images.dtype != torch.uint8 or images.dim() != 4 or images.shape[3] != 3 or not images.is_contiguous():
            raise ValueError("images must be contiguous uint8 [B,H,W,3], got %s %s" % (images.dtype, tuple(images.shape)))
        B, H, W, _ = images.shape
        segments = _chk_f32(segments, "segments", 3)
        if segments.shape[0] != B or segments.shape[2] != 4 or segments.device != images.device:
            raise ValueError("segments must be [%d,S,4] on the images' device, got %s" % (B, tuple(segments.shape)))
        S = segments.shape[1]
        cols = np.ascontiguousarray(colors, dtype=np.float32)
        if cols.shape != (S, 3):
            raise ValueError("colors must be [%d,3], got %s" % (S, cols.shape))
        if valid is not None:
            if not isinstance(valid, torch.Tensor) or valid.dtype != torch.int32 or tuple(valid.shape) != (B,) or valid.device != images.device:
                raise ValueError("valid must be an int32 tensor [%d] on the images' device" % B)
            valid = valid.contiguous()
        _lib.check(self.lib.h3d_draw_segments(self.h, _ptr(images), B, H, W, _ptr(segments), S, cols.ctypes.data_as(C.c_void_p),
                                              _ptr(valid), C.c_float(linewidth), _stream()), "h3d_draw_segments")
        return images

    # ---- training (h3d_resize_bilinear_tf1_backward, the two losses, Adam) ----------------------
    def variables(self, scope):
        """Ordered {reference variable name: torch.nn.Parameter} of "HandSegNet", "PoseNet2D", "PosePrior" (with fc_bottleneck when
        the loaded fc_xyz is 30 x 63) or "ViewpointNet" (layer order of the reference graph, weights before biases): fp32 device copies of the host arrays load_weights keeps, created once per context and then shared by
        every train=True graph, so an optimiser over them trains the network in place.

        The inference path (train=False, pipeline(), the stage entries) keeps the weights last loaded, not these Parameters: call
        commit_variables(scope) to make it use the trained values.  A later load_weights of the scope writes the loaded values into
        the same Parameters in place, so an optimiser built over them keeps working (its m / v slots are not reset)."""
        from . import arch
        layers = {"HandSegNet": arch.HANDSEGNET, "PoseNet2D": arch.POSENET2D, "PosePrior": list(arch.POSEPRIOR),
                  "ViewpointNet": arch.VIEWPOINT}
        if scope not in layers:
            raise ValueError("variables(): scope must be 'HandSegNet', 'PoseNet2D', 'PosePrior' or 'ViewpointNet', got %r" % (scope,))
        xyz = self.weights.get("PosePrior/fc_xyz/weights")
        if scope == "PosePrior" and xyz is not None and xyz.shape[0] == 30:      # the 'bottleneck' variant: 512 -> 30 -> 63
            layers["PosePrior"].insert(8, arch.POSEPRIOR_BOTTLENECK)
        cache = self.__dict__.setdefault("_variables", {})
        if scope not in cache:
            names = ["%s/%s/%s" % (scope, l[0], what) for l in layers[scope] for what in ("weights", "biases")]
            missing = [n for n in names if n not in self.weights]
            if missing:
                raise ValueError("variables(%r): the scope was not loaded (%d of %d variables missing, e.g. %s); call "
                                 "ColorHandPose3DNetwork().init() first" % (scope, len(missing), len(names), missing[0]))
            cache[scope] = {n: torch.nn.Parameter(torch.from_numpy(self.weights[n].copy()).to(self.device)) for n in names}
        return cache[scope]

    def commit_variables(self, scope):
        """Loads the current values of variables(scope) as the inference weights of the scope (as load_weights does with a pickle),
        so that train=False graphs, pipeline() and the stage entries use the trained network.  Reads the Parameters on the host."""
        self.load_weights({n: p.detach().cpu().numpy() for n, p in self.variables(scope).items()})

    def resize_bilinear_backward(self, dy, H, W):
        """Gradient of resize_bilinear(x [B,H,W,C], out_h, out_w): dy [B,out_h,out_w,C] -> dx [B,H,W,C]."""
        dy = _chk_f32(dy, "dy", 4)
        B, oh, ow, Cc = dy.shape
        dx = torch.empty((B, int(H), int(W), Cc), dtype=torch.float32, device=dy.device)
        _lib.check(self.lib.h3d_resize_bilinear_tf1_backward(self.h, _ptr(dy), _ptr(dx), B, int(H), int(W), Cc, oh, ow, _stream()),
                   "h3d_resize_bilinear_tf1_backward")
        return dx

    def _scoremap_args(self, pred, target, vis):
        pred = _chk_f32(pred, "pred", 4); target = _chk_f32(target, "target", 4)
        B, H, W, K = pred.shape
        if K != 21 or tuple(target.shape) != tuple(pred.shape):
            raise ValueError("scoremap loss: pred and target must both be [B,H,W,21], got %s and %s" % (tuple(pred.shape), tuple(target.shape)))
        vis = _chk_f32(vis.to(torch.float32).reshape(B, 21), "vis")
        return pred, target, vis, B, H, W

    def scoremap_loss(self, pred, target, vis):
        """training_posenet.py:61 for one map -> (loss, a 0-d device tensor; rms [B,21])."""
        pred, target, vis, B, H, W = self._scoremap_args(pred, target, vis)
        loss = torch.empty((), dtype=torch.float32, device=pred.device)
        rms = torch.empty((B, 21), dtype=torch.float32, device=pred.device)
        _lib.check(self.lib.h3d_scoremap_loss_forward(self.h, _ptr(pred), _ptr(target), _ptr(vis), B, H, W, _ptr(loss), _ptr(rms), _stream()),
                   "h3d_scoremap_loss_forward")
        return loss, rms

    def scoremap_loss_backward(self, pred, target, vis, rms, grad_loss=None):
        """dL/dpred for the incoming gradient grad_loss (a device scalar, None = 1)."""
        pred, target, vis, B, H, W = self._scoremap_args(pred, target, vis)
        rms = _chk_f32(rms, "rms", 2)
        g = _chk_f32(grad_loss.reshape(()), "grad_loss") if grad_loss is not None else None
        dpred = torch.empty_like(pred)
        _lib.check(self.lib.h3d_scoremap_loss_backward(self.h, _ptr(pred), _ptr(target), _ptr(vis), _ptr(rms), _ptr(g), B, H, W, _ptr(dpred),
                                                       _stream()), "h3d_scoremap_loss_backward")
        return dpred

    def _xent_args(self, logits, labels):
        logits = _chk_f32(logits, "logits"); labels = _chk_f32(labels, "labels")
        if logits.shape[-1] != 2 or tuple(labels.shape) != tuple(logits.shape):
            raise ValueError("softmax_xent: logits and labels must both be [..., 2], got %s and %s" % (tuple(logits.shape), tuple(labels.shape)))
        return logits, labels, logits.numel() // 2

    def softmax_xent(self, logits, labels):
        """training_handsegnet.py:60: mean softmax cross-entropy of [..., 2] logits and labels -> 0-d device tensor."""
        logits, labels, rows = self._xent_args(logits, labels)
        loss = torch.empty((), dtype=torch.float32, device=logits.device)
        _lib.check(self.lib.h3d_softmax_xent_forward(self.h, _ptr(logits), _ptr(labels), rows, _ptr(loss), _stream()), "h3d_softmax_xent_forward")
        return loss

    def softmax_xent_backward(self, logits, labels, grad_loss=None):
        logits, labels, rows = self._xent_args(logits, labels)
        g = _chk_f32(grad_loss.reshape(()), "grad_loss") if grad_loss is not None else None
        d = torch.empty_like(logits)
        _lib.check(self.lib.h3d_softmax_xent_backward(self.h, _ptr(logits), _ptr(labels), _ptr(g), rows, _ptr(d), _stream()),
                   "h3d_softmax_xent_backward")
        return d

    def adam_state_set(self, state, lr, beta1_power, beta2_power):
        _lib.check(self.lib.h3d_adam_state_set(self.h, _ptr(state), C.c_float(lr), C.c_float(beta1_power), C.c_float(beta2_power), _stream()),
                   "h3d_adam_state_set")

    def adam_set_lr(self, state, lr):
        _lib.check(self.lib.h3d_adam_set_lr(self.h, _ptr(state), C.c_float(lr), _stream()), "h3d_adam_set_lr")

    def adam_step(self, table, n, state, beta1, beta2, epsilon):
        """table: int64 device tensor [n, 5] of h3d_adam_tensor rows (param, grad, m, v pointers, numel)."""
        _lib.check(self.lib.h3d_adam_step(self.h, _ptr(table), int(n), _ptr(state), C.c_float(beta1), C.c_float(beta2), C.c_float(epsilon),
                                          _stream()), "h3d_adam_step")

    def avg_pool8(self, x):
        x = _chk_f32(x, "x", 4)
        B, H, W, Cc = x.shape
        y = torch.empty((B, H // 8, W // 8, Cc), dtype=torch.float32, device=x.device)
        _lib.check(self.lib.h3d_avgpool8(self.h, _ptr(x), _ptr(y), B, H, W, Cc, _stream()), "h3d_avgpool8")
        return y

    def seg_postprocess(self, logits):
        logits = _chk_f32(logits, "scoremap", 4)
        B, H, W, Cc = logits.shape
        if Cc != 2:
            raise ValueError("single_obj_scoremap kernel expects 2 classes (background, hand)")
        dev = logits.device
        mask = torch.empty((B, H, W), dtype=torch.uint8, device=dev)
        loc = torch.empty((B, 2), dtype=torch.int32, device=dev)
        center = torch.empty((B, 2), dtype=torch.float32, device=dev)
        size = torch.empty((B, 1), dtype=torch.float32, device=dev)
        scale = torch.empty((B, 1), dtype=torch.float32, device=dev)
        _lib.check(self.lib.h3d_seg_postprocess(self.h, _ptr(logits), B, H, W, _ptr(mask), _ptr(loc), _ptr(center), _ptr(size),
                                                _ptr(scale), _stream()), "h3d_seg_postprocess")
        return {"hand_mask": mask, "max_loc": loc, "center": center, "crop_size": size, "scale_crop": scale}

    def crop_image_from_xy(self, image, center, crop_size, scale):
        image = _chk_f32(image, "image", 4)
        B, H, W, Cc = image.shape
        center = _chk_f32(center.to(torch.float32).reshape(B, 2), "crop_location")
        scale = _chk_f32(scale.to(torch.float32).reshape(-1).expand(B).contiguous(), "scale")
        out = torch.empty((B, crop_size, crop_size, Cc), dtype=torch.float32, device=image.device)
        _lib.check(self.lib.h3d_crop_image_from_xy(self.h, _ptr(image), _ptr(center), _ptr(scale), _ptr(out), B, H, W, Cc,
                                                   int(crop_size), _stream()), "h3d_crop_image_from_xy")
        return out

    def detect_keypoints(self, scoremaps):
        scoremaps = _chk_f32(scoremaps, "scoremaps", 4)
        B, H, W, Cc = scoremaps.shape
        uv = torch.empty((B, Cc, 2), dtype=torch.int32, device=scoremaps.device)
        _lib.check(self.lib.h3d_detect_keypoints(self.h, _ptr(scoremaps), B, H, W, Cc, _ptr(uv), _stream()), "h3d_detect_keypoints")
        return uv

    def upsample_detect_keypoints(self, scoremaps, out_h, out_w):
        """Fused tf.image.resize_images + detect_keypoints for 21-channel maps -> (maps [B,out_h,out_w,21], uv [B,21,2] int32)."""
        scoremaps = _chk_f32(scoremaps, "scoremaps", 4)
        B, H, W, Cc = scoremaps.shape
        if Cc != 21:
            raise ValueError("upsample_detect_keypoints expects 21 key-point channels")
        up = torch.empty((B, out_h, out_w, 21), dtype=torch.float32, device=scoremaps.device)
        uv = torch.empty((B, 21, 2), dtype=torch.int32, device=scoremaps.device)
        _lib.check(self.lib.h3d_upsample_detect_keypoints(self.h, _ptr(scoremaps), B, H, W, int(out_h), int(out_w), _ptr(up), _ptr(uv), _stream()),
                   "h3d_upsample_detect_keypoints")
        return up, uv

    def decode_records(self, records, dataset="rhd", step=1, want_aux=True):
        """records: uint8 CUDA tensor [B, record_bytes] -> dict(image fp32 NHWC, header, mask, visibility)."""
        if records.dtype != torch.uint8 or not records.is_cuda or records.dim() != 2:
            raise TypeError("records must be a 2-D uint8 CUDA tensor")
        records = records.contiguous()
        ds, image, header, mask, vis = self._decode_outputs(records, dataset, records.shape[0], step, want_aux)
        _lib.check(self.lib.h3d_decode_records(self.h, ds, _ptr(records), records.shape[0], step, _ptr(header), _ptr(image), _ptr(mask),
                                               _ptr(vis), _stream()), "h3d_decode_records")
        return {"image": image, "header": header, "mask": mask, "visibility": vis}

    @staticmethod
    def _decode_outputs(records, dataset, B, step, want_aux):
        ds = {"rhd": 0, "stb": 1}[dataset]
        rb, H, W, hdr = (410520, 320, 320, 219) if ds == 0 else (922104, 480, 640, 126)
        if records.shape[1] != rb:
            raise ValueError("%s records are %d bytes, got %d" % (dataset, rb, records.shape[1]))
        dev = records.device
        image = torch.empty((B, H // step, W // step, 3), dtype=torch.float32, device=dev)
        header = torch.empty((B, hdr), dtype=torch.float32, device=dev) if want_aux else None
        mask = torch.empty((B, H, W), dtype=torch.uint8, device=dev) if (want_aux and ds == 0) else None
        vis = torch.empty((B, 42), dtype=torch.uint8, device=dev) if (want_aux and ds == 0) else None
        return ds, image, header, mask, vis

    def decode_records_gather(self, file, serials, dataset="rhd", step=1, want_aux=True):
        """decode_records of records gathered on the device: file uint8 CUDA [n_records, record_bytes] (a resident dataset file),
        serials int64 CUDA [B] (stream positions >= 0) -> the items of record serials[b] mod n_records, bit for bit as decode_records
        computes them from those records.  Only enqueues work: capturable into a CUDA graph."""
        if file.dtype != torch.uint8 or not file.is_cuda or file.dim() != 2 or not file.is_contiguous():
            raise TypeError("file must be a contiguous 2-D uint8 CUDA tensor of whole records")
        if serials.dtype != torch.int64 or serials.device != file.device or serials.dim() != 1 or not serials.is_contiguous():
            raise TypeError("serials must be a contiguous 1-D int64 tensor on the file's device")
        B = serials.shape[0]
        ds, image, header, mask, vis = self._decode_outputs(file, dataset, B, step, want_aux)
        _lib.check(self.lib.h3d_decode_records_gather(self.h, ds, _ptr(file), file.shape[0], _ptr(serials), B, step, _ptr(header), _ptr(image),
                                                      _ptr(mask), _ptr(vis), _stream()), "h3d_decode_records_gather")
        return {"image": image, "header": header, "mask": mask, "visibility": vis}

    def reader_next_serials(self, state, B, seed, shuffle):
        """The next B stream positions of a reader queue whose state lives on the device (int64 [_lib.READER_STATE_WORDS], advanced in
        place) -> int64 CUDA [B].  With shuffle, the same stream as BinaryDbReader's host queue for the same seed."""
        if state.dtype != torch.int64 or not state.is_cuda or state.numel() != _lib.READER_STATE_WORDS or not state.is_contiguous():
            raise TypeError("state must be a contiguous int64 CUDA tensor of %d words" % _lib.READER_STATE_WORDS)
        out = torch.empty((int(B),), dtype=torch.int64, device=state.device)
        _lib.check(self.lib.h3d_reader_next_serials(self.h, _ptr(state), int(B), C.c_uint64(int(seed) & (2 ** 64 - 1)), int(bool(shuffle)),
                                                    _ptr(out), _stream()), "h3d_reader_next_serials")
        return out

    def rhd_reader_items(self, header, hand_parts, visibility, use_wrist_coord=True, hand_crop=False, crop_size=256):
        """Derived items of BinaryDbReader.get() (evaluation mode) from the outputs of decode_records(..., "rhd")."""
        B = header.shape[0]
        dev = header.device
        f = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)      # noqa: E731
        r = {"keypoint_xyz21": f(B, 21, 3), "keypoint_uv21": f(B, 21, 2), "keypoint_vis21": torch.empty((B, 21), dtype=torch.uint8, device=dev),
             "hand_side": f(B, 2), "keypoint_scale": f(B), "keypoint_xyz21_normed": f(B, 21, 3), "cam_mat": f(B, 3, 3),
             "crop_center": f(B, 2) if hand_crop else None, "crop_scale": f(B) if hand_crop else None}
        _lib.check(self.lib.h3d_rhd_reader_items(
            self.h, _ptr(header.contiguous()), _ptr(hand_parts.contiguous()), _ptr(visibility.contiguous()), B, int(bool(use_wrist_coord)),
            int(bool(hand_crop)), int(crop_size), _ptr(r["keypoint_xyz21"]), _ptr(r["keypoint_uv21"]), _ptr(r["keypoint_vis21"]),
            _ptr(r["hand_side"]), _ptr(r["keypoint_scale"]), _ptr(r["keypoint_xyz21_normed"]), _ptr(r["crop_center"]), _ptr(r["crop_scale"]),
            _ptr(r["cam_mat"]), _stream()), "h3d_rhd_reader_items")
        return r

    def stb_reader_items(self, header, use_wrist_coord=True):
        B = header.shape[0]
        dev = header.device
        f = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)      # noqa: E731
        r = {"keypoint_xyz21": f(B, 21, 3), "keypoint_uv21": f(B, 21, 2), "keypoint_vis21": torch.empty((B, 21), dtype=torch.uint8, device=dev),
             "keypoint_scale": f(B), "keypoint_xyz21_normed": f(B, 21, 3)}
        _lib.check(self.lib.h3d_stb_reader_items(self.h, _ptr(header.contiguous()), B, int(bool(use_wrist_coord)), _ptr(r["keypoint_xyz21"]),
                                                 _ptr(r["keypoint_uv21"]), _ptr(r["keypoint_vis21"]), _ptr(r["keypoint_scale"]),
                                                 _ptr(r["keypoint_xyz21_normed"]), _stream()), "h3d_stb_reader_items")
        return r

    def gaussian_scoremap(self, coords_hw, output_size, sigma, valid=None):
        """create_multiple_gaussian_map, batched: coords_hw [B,N,2] (row, col), valid [B,N] -> [B,H,W,N]."""
        coords_hw = _chk_f32(coords_hw, "coords_hw", 3)
        B, N, _ = coords_hw.shape
        H, W = int(output_size[0]), int(output_size[1])
        v = valid.to(torch.uint8).contiguous() if valid is not None else None
        out = torch.empty((B, H, W, N), dtype=torch.float32, device=coords_hw.device)
        _lib.check(self.lib.h3d_gaussian_scoremap(self.h, _ptr(coords_hw), _ptr(v), B, N, H, W, C.c_float(float(sigma)), _ptr(out), _stream()),
                   "h3d_gaussian_scoremap")
        return out

    def reader_aug_params(self, serials, seed, flags):
        """Per-sample random parameters of the RHD reader's training augmentation: serials int64 [B] (enqueue positions) ->
        params [B, _lib.AUG_PARAMS] fp32, a pure function of (seed, serial) for each flag in `flags` (the _lib.AUG_* bits)."""
        serials = serials.to(device=self.device, dtype=torch.int64).contiguous()
        B = serials.shape[0]
        params = torch.empty((B, _lib.AUG_PARAMS), dtype=torch.float32, device=self.device)
        _lib.check(self.lib.h3d_reader_aug_params(self.h, _ptr(serials), B, C.c_uint64(int(seed) & (2 ** 64 - 1)), int(flags), _ptr(params),
                                                  _stream()), "h3d_reader_aug_params")
        return params

    def augment_image(self, image, params, flags, hand_parts=None, window=256):
        """tf.image.random_hue and / or the random_crop window in one pass: image [B,H,W,3] -> image [B,h,w,3]; with
        _lib.AUG_RANDOM_CROP in flags also the hand_parts [B,h,w] and hand_mask [B,h,w,2] int32 windows of hand_parts u8 [B,H,W]."""
        image = _chk_f32(image, "image", 4)
        B, H, W, _ = image.shape
        crop = bool(flags & _lib.AUG_RANDOM_CROP)
        oh, ow = (window, window) if crop else (H, W)
        dev = image.device
        out = torch.empty((B, oh, ow, 3), dtype=torch.float32, device=dev)
        parts = mask = None
        if crop and hand_parts is not None:
            hand_parts = hand_parts.to(torch.uint8).contiguous()
            parts = torch.empty((B, oh, ow), dtype=torch.int32, device=dev)
            mask = torch.empty((B, oh, ow, 2), dtype=torch.int32, device=dev)
        p = _chk_params(params, B)
        _lib.check(self.lib.h3d_augment_image(self.h, _ptr(image), _ptr(hand_parts if parts is not None else None), _ptr(p), B, H, W,
                                              int(flags), int(window), _ptr(out), _ptr(parts), _ptr(mask), _stream()), "h3d_augment_image")
        return out, parts, mask

    def rhd_reader_items_aug(self, header, hand_parts, visibility, params, flags, use_wrist_coord=True, hand_crop=False, crop_size=256):
        """rhd_reader_items with the coordinate / crop noises of `flags` read from params; also returns keypoint_uv [B,42,2]."""
        B = header.shape[0]
        dev = header.device
        f = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)      # noqa: E731
        r = {"keypoint_uv": f(B, 42, 2), "keypoint_xyz21": f(B, 21, 3), "keypoint_uv21": f(B, 21, 2),
             "keypoint_vis21": torch.empty((B, 21), dtype=torch.uint8, device=dev), "hand_side": f(B, 2), "keypoint_scale": f(B),
             "keypoint_xyz21_normed": f(B, 21, 3), "cam_mat": f(B, 3, 3), "crop_center": f(B, 2) if hand_crop else None,
             "crop_scale": f(B) if hand_crop else None}
        p = _chk_params(params, B)
        _lib.check(self.lib.h3d_rhd_reader_items_aug(
            self.h, _ptr(header.contiguous()), _ptr(hand_parts.contiguous()), _ptr(visibility.contiguous()), B, int(bool(use_wrist_coord)),
            int(bool(hand_crop)), int(crop_size), _ptr(p), int(flags), _ptr(r["keypoint_uv"]), _ptr(r["keypoint_xyz21"]), _ptr(r["keypoint_uv21"]),
            _ptr(r["keypoint_vis21"]), _ptr(r["hand_side"]), _ptr(r["keypoint_scale"]), _ptr(r["keypoint_xyz21_normed"]), _ptr(r["crop_center"]),
            _ptr(r["crop_scale"]), _ptr(r["cam_mat"]), _stream()), "h3d_rhd_reader_items_aug")
        return r

    def gaussian_scoremap_dropout(self, coords_hw, output_size, sigma, valid, keep, keep_prob=0.8):
        """gaussian_scoremap followed by TF 1.3 dropout with per-(sample, key-point) keep bits and the reader's * keep_prob.
        keep: fp32 [B, >= N] rows (a column slice of the augmentation parameters is fine: its row stride is used)."""
        coords_hw = _chk_f32(coords_hw, "coords_hw", 3)
        B, N, _ = coords_hw.shape
        H, W = int(output_size[0]), int(output_size[1])
        if keep.dtype != torch.float32 or keep.dim() != 2 or keep.shape[0] != B or keep.shape[1] < N or keep.stride(1) != 1:
            raise ValueError("keep must be fp32 [B, >= N] with unit column stride")
        v = valid.to(torch.uint8).contiguous() if valid is not None else None
        out = torch.empty((B, H, W, N), dtype=torch.float32, device=coords_hw.device)
        _lib.check(self.lib.h3d_gaussian_scoremap_dropout(self.h, _ptr(coords_hw), _ptr(v), _ptr(keep), int(keep.stride(0)), C.c_float(float(keep_prob)),
                                                          B, N, H, W, C.c_float(float(sigma)), _ptr(out), _stream()), "h3d_gaussian_scoremap_dropout")
        return out

    def canonical_trafo(self, coords_xyz, cond_right=None):
        """-> (coords_can [B,21,3], rot_mat [B,3,3], rot_mat_inv [B,3,3]) (utils/canonical_trafo.py:97-162)."""
        coords_xyz = _chk_f32(coords_xyz.reshape(-1, 21, 3), "coords_xyz", 3)
        B = coords_xyz.shape[0]
        dev = coords_xyz.device
        cr = cond_right.reshape(B).to(torch.uint8).contiguous() if cond_right is not None else None
        can = torch.empty((B, 21, 3), dtype=torch.float32, device=dev)
        rot = torch.empty((B, 3, 3), dtype=torch.float32, device=dev)
        inv = torch.empty((B, 3, 3), dtype=torch.float32, device=dev)
        _lib.check(self.lib.h3d_canonical_trafo(self.h, _ptr(coords_xyz), _ptr(cr), B, _ptr(can), _ptr(rot), _ptr(inv), _stream()), "h3d_canonical_trafo")
        return can, rot, inv

    def eval_keypoint_dist(self, gt, vis, pred):
        gt = _chk_f32(gt, "keypoint_gt"); pred = _chk_f32(pred, "keypoint_pred")
        D = gt.shape[-1]
        n = gt.numel() // D
        vis = vis.to(torch.uint8).contiguous()
        dist = torch.empty(gt.shape[:-1], dtype=torch.float32, device=gt.device)
        _lib.check(self.lib.h3d_eval_keypoint_dist(self.h, _ptr(gt), _ptr(vis), _ptr(pred), n, D, _ptr(dist), _stream()),
                   "h3d_eval_keypoint_dist")
        return dist

    def eval_feed(self, store, num_kp, num_samples, gt, vis, pred):
        """h3d_eval_feed: appends the distances of gt / pred [n, K, D] (float32 or float64, the store's dtype) where vis [n, K] (uint8,
        nonzero = visible) to the store (a uint8 CUDA tensor of h3d_eval_store_bytes bytes).  Enqueue-only and capturable."""
        dtype = {torch.float32: _lib.EVAL_FLOAT32, torch.float64: _lib.EVAL_FLOAT64}.get(gt.dtype)
        if dtype is None or pred.dtype != gt.dtype:
            raise TypeError("gt and pred must both be float32 or both float64, got %s and %s" % (gt.dtype, pred.dtype))
        if vis.dtype != torch.uint8:
            raise TypeError("vis must be uint8, got %s" % vis.dtype)
        for t, name in ((store, "store"), (gt, "gt"), (vis, "vis"), (pred, "pred")):
            if not t.is_cuda or not t.is_contiguous():
                raise ValueError("%s must be a contiguous CUDA tensor" % name)
        if gt.dim() != 3 or tuple(pred.shape) != tuple(gt.shape) or tuple(vis.shape) != tuple(gt.shape[:2]) or gt.shape[1] != num_kp:
            raise ValueError("gt / pred must be [n, %d, D] and vis [n, %d], got %s, %s and %s"
                             % (num_kp, num_kp, tuple(gt.shape), tuple(pred.shape), tuple(vis.shape)))
        n, _, D = gt.shape
        _lib.check(self.lib.h3d_eval_feed(self.h, _ptr(store), int(num_kp), int(num_samples), dtype, _ptr(gt), _ptr(vis), _ptr(pred), int(n),
                                          int(D), _stream()), "h3d_eval_feed")

    def eval_stats(self, store, num_kp, num_samples, dtype, thresholds):
        """h3d_eval_stats: -> int64 [K, EVAL_STAT_COUNTS + T] on the device, per key-point n_k, the mean and median (float64 bit patterns)
        and the threshold counts; thresholds is a float64 CUDA tensor [T]."""
        code = {torch.float32: _lib.EVAL_FLOAT32, torch.float64: _lib.EVAL_FLOAT64}[dtype]
        if thresholds.dtype != torch.float64 or not thresholds.is_cuda or thresholds.dim() != 1 or not thresholds.is_contiguous():
            raise TypeError("thresholds must be a contiguous float64 CUDA tensor [T]")
        T = thresholds.shape[0]
        out = torch.empty((int(num_kp), _lib.EVAL_STAT_COUNTS + T), dtype=torch.int64, device=store.device)
        _lib.check(self.lib.h3d_eval_stats(self.h, _ptr(store), int(num_kp), int(num_samples), code, _ptr(thresholds), int(T), _ptr(out),
                                           _stream()), "h3d_eval_stats")
        return out

    def bone_rel_trafo_inv(self, coords_rel):
        coords_rel = _chk_f32(coords_rel, "coords_rel")
        if coords_rel.dim() == 2:
            coords_rel = coords_rel.unsqueeze(0)
        B = coords_rel.shape[0]
        out = torch.empty((B, 21, 3), dtype=torch.float32, device=coords_rel.device)
        _lib.check(self.lib.h3d_bone_rel_trafo_inv(self.h, _ptr(coords_rel), _ptr(out), B, _stream()), "h3d_bone_rel_trafo_inv")
        return out

    def rotate_canonical(self, coord_can, uxyz, hand_side):
        coord_can = _chk_f32(coord_can, "coord_can", 3); uxyz = _chk_f32(uxyz, "uxyz", 2); hand_side = _chk_f32(hand_side, "hand_side", 2)
        B = coord_can.shape[0]
        rot = torch.empty((B, 3, 3), dtype=torch.float32, device=coord_can.device)
        out = torch.empty((B, 21, 3), dtype=torch.float32, device=coord_can.device)
        _lib.check(self.lib.h3d_rotate_canonical(self.h, _ptr(coord_can), _ptr(uxyz), _ptr(hand_side), B, _ptr(rot), _ptr(out),
                                                 _stream()), "h3d_rotate_canonical")
        return rot, out

    # ---- lifting training (h3d_rotate_canonical_backward, h3d_bone_rel_trafo*, h3d_mse_loss_*) --------------------------------
    def rotate_canonical_backward(self, coord_can, uxyz, hand_side, d_out=None, d_rot=None):
        """Gradient of rotate_canonical -> (d_can [B,21,3], d_uxyz [B,3]); d_out [B,21,3] and d_rot [B,3,3] may be None (= 0)."""
        coord_can = _chk_f32(coord_can, "coord_can", 3); uxyz = _chk_f32(uxyz, "uxyz", 2); hand_side = _chk_f32(hand_side, "hand_side", 2)
        B = coord_can.shape[0]
        if tuple(coord_can.shape) != (B, 21, 3) or tuple(uxyz.shape) != (B, 3) or tuple(hand_side.shape) != (B, 2):
            raise ValueError("rotate_canonical_backward: expects can [B,21,3], uxyz [B,3], hand_side [B,2], got %s, %s, %s"
                             % (tuple(coord_can.shape), tuple(uxyz.shape), tuple(hand_side.shape)))
        d_out = _chk_f32(d_out.reshape(B, 21, 3), "d_out") if d_out is not None else None
        d_rot = _chk_f32(d_rot.reshape(B, 3, 3), "d_rot") if d_rot is not None else None
        d_can = torch.empty((B, 21, 3), dtype=torch.float32, device=coord_can.device)
        d_u = torch.empty((B, 3), dtype=torch.float32, device=coord_can.device)
        _lib.check(self.lib.h3d_rotate_canonical_backward(self.h, _ptr(coord_can), _ptr(uxyz), _ptr(hand_side), _ptr(d_out), _ptr(d_rot), B,
                                                          _ptr(d_can), _ptr(d_u), _stream()), "h3d_rotate_canonical_backward")
        return d_can, d_u

    def _rel_arg(self, t, name):
        t = _chk_f32(t, name)
        if t.dim() == 2:
            t = t.unsqueeze(0)
        if t.dim() != 3 or tuple(t.shape[1:]) != (21, 3):
            raise ValueError("%s must be [B,21,3] (or [21,3]), got %s" % (name, tuple(t.shape)))
        return t

    def bone_rel_trafo_inv_backward(self, coords_rel, d_xyz):
        """Gradient of bone_rel_trafo_inv: coords_rel (its input), d_xyz [B,21,3] -> d_rel [B,21,3]."""
        coords_rel = self._rel_arg(coords_rel, "coords_rel")
        d_xyz = self._rel_arg(d_xyz, "d_xyz")
        if d_xyz.shape != coords_rel.shape:
            raise ValueError("bone_rel_trafo_inv_backward: d_xyz %s does not match coords_rel %s" % (tuple(d_xyz.shape), tuple(coords_rel.shape)))
        d_rel = torch.empty_like(coords_rel)
        _lib.check(self.lib.h3d_bone_rel_trafo_inv_backward(self.h, _ptr(coords_rel), _ptr(d_xyz), _ptr(d_rel), coords_rel.shape[0], _stream()),
                   "h3d_bone_rel_trafo_inv_backward")
        return d_rel

    def bone_rel_trafo(self, coords_xyz):
        """utils/relative_trafo.py:184-240: xyz [B,21,3] -> (length, angle_x, angle_y) [B,21,3]."""
        coords_xyz = self._rel_arg(coords_xyz, "coords_xyz")
        rel = torch.empty_like(coords_xyz)
        _lib.check(self.lib.h3d_bone_rel_trafo(self.h, _ptr(coords_xyz), _ptr(rel), coords_xyz.shape[0], _stream()), "h3d_bone_rel_trafo")
        return rel

    def _mse_args(self, pred, target):
        pred = _chk_f32(pred, "pred"); target = _chk_f32(target, "target")
        if tuple(pred.shape) != tuple(target.shape) or pred.numel() == 0:
            raise ValueError("mse_loss: pred and target must have one non-empty shape, got %s and %s" % (tuple(pred.shape), tuple(target.shape)))
        return pred, target

    def mse_loss(self, pred, target):
        """reduce_mean(square(pred - target)) -> 0-d device tensor."""
        pred, target = self._mse_args(pred, target)
        loss = torch.empty((), dtype=torch.float32, device=pred.device)
        _lib.check(self.lib.h3d_mse_loss_forward(self.h, _ptr(pred), _ptr(target), pred.numel(), _ptr(loss), _stream()), "h3d_mse_loss_forward")
        return loss

    def mse_loss_backward(self, pred, target, grad_loss=None):
        pred, target = self._mse_args(pred, target)
        g = _chk_f32(grad_loss.reshape(()), "grad_loss") if grad_loss is not None else None
        d = torch.empty_like(pred)
        _lib.check(self.lib.h3d_mse_loss_backward(self.h, _ptr(pred), _ptr(target), _ptr(g), pred.numel(), _ptr(d), _stream()),
                   "h3d_mse_loss_backward")
        return d


class PackedConv:
    """Handle of h3d_pack_conv_weights (freed with the object; the free waits for kernels still reading the planes)."""
    def __init__(self, ctx, h, k, Cin, Cout):
        self.ctx, self.h, self.k, self.Cin, self.Cout = ctx, h, k, Cin, Cout

    def __del__(self):
        try:
            if self.h and getattr(self.ctx, "h", None):
                self.ctx.lib.h3d_free_packed_conv(self.ctx.h, self.h)
            self.h = None
        except Exception:
            pass


class TrackState:
    """The device state of B tracked streams (include/hand3d_b200.h, H3D_TRACK_*): one float32 buffer of h3d_track_state_bytes(B)
    bytes and views of it: center [B,2] and scale [B] (the crop the next track step uses), score [B] float32 and lost [B] int32.
    A new state holds the reference's fall-back crop (centre (160, 160), crop size 100 at its margin 1.25) in every slot, a NaN
    score and lost = 1: nothing has been found yet.  reset() restores that."""

    def __init__(self, B, device=None):
        self.B = int(B)
        words = int(_lib.load().h3d_track_state_bytes(self.B))
        if words < 0:
            _lib.check(words, "h3d_track_state_bytes")
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.buffer = torch.empty(words // 4, dtype=torch.float32, device=dev)
        B = self.B
        self.center = self.buffer[_lib.TRACK_CENTER * B:(_lib.TRACK_CENTER + 2) * B].view(B, 2)
        self.scale = self.buffer[_lib.TRACK_SCALE * B:(_lib.TRACK_SCALE + 1) * B]
        self.score = self.buffer[_lib.TRACK_SCORE * B:(_lib.TRACK_SCORE + 1) * B]
        self.lost = self.buffer[_lib.TRACK_LOST * B:(_lib.TRACK_LOST + 1) * B].view(torch.int32)
        self.reset()

    def reset(self):
        self.center.fill_(160.0)
        self.scale.fill_(float(np.float32(256.0) / (np.float32(100.0) * np.float32(1.25))))
        self.score.fill_(float("nan"))
        self.lost.fill_(1)


def conv2d_tc_geometry(B, H, W, Cout, pool=0, precision="bf16x3"):
    """(TW, TH, TB, BN) the tensor-core convolution runs this layer on (h3d_conv2d_tc_geometry; pool 2 = stride 2).  Needs no device."""
    out = (C.c_int * 4)()
    _lib.check(_lib.load().h3d_conv2d_tc_geometry(B, H, W, Cout, int(pool), PRECISIONS[precision], out), "h3d_conv2d_tc_geometry")
    return tuple(out)


def conv2d_wgrad_geometry(B, H, W, ksize, Cin, Cout):
    """(TW, TH, TB, BN, num_tiles, splits) of the weight-gradient kernel (h3d_conv2d_wgrad_geometry).  Needs no device."""
    out = (C.c_int * 6)()
    _lib.check(_lib.load().h3d_conv2d_wgrad_geometry(B, H, W, ksize, Cin, Cout, out), "h3d_conv2d_wgrad_geometry")
    return tuple(out)


def conv2d_f32_geometry(B, H, W, Cin, Cout, ksize, stride=1, Cin_total=None, cin_off=0, Cout_total=None, cout_off=0, yf=True,
                        planes=None, Cs_total=None, cs_off=0, x_aligned=True, splitk_scratch_floats=_lib.CONV_SPLITK_SCRATCH_FLOATS):
    """(kernel, (grid x, y, z), ksplit, k_per_split) of the CUDA-core convolution (h3d_conv2d_f32_geometry): kernel is one of
    "c3_tc", "c3_ffma", "vec", "scalar"; planes a tensor-core precision or None.  Needs no device."""
    out = (C.c_int * 6)()
    _lib.check(_lib.load().h3d_conv2d_f32_geometry(
        B, H, W, Cin, Cin if Cin_total is None else Cin_total, cin_off, Cout, Cout if Cout_total is None else Cout_total, cout_off,
        int(bool(yf)), PRECISIONS[planes or "fp32_ffma"], Cout if Cs_total is None else Cs_total, cs_off, ksize, stride, int(bool(x_aligned)),
        int(splitk_scratch_floats), out), "h3d_conv2d_f32_geometry")
    return _lib.DIRECT_KERNELS[out[0]], tuple(out[1:4]), out[4], out[5]


def fully_connected_f32_geometry(B, in_features, out_features):
    """(ksplit, k_per_split, (grid x, y, z)) of the fp32 fully connected layer (h3d_fully_connected_f32_geometry).  Needs no device."""
    out = (C.c_int * 5)()
    _lib.check(_lib.load().h3d_fully_connected_f32_geometry(B, in_features, out_features, out), "h3d_fully_connected_f32_geometry")
    return out[0], out[1], tuple(out[2:5])


_default = {}


def default_context(device=None) -> Context:
    idx = torch.cuda.current_device() if device is None else torch.device(device).index or 0
    if idx not in _default:
        _default[idx] = Context(idx)
    return _default[idx]


def reset_default_context():
    _default.clear()
