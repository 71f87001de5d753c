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
        # captured graphs bake in plan-owned device pointers (tile-ticket / completion counters, packed operands): rebuilding the
        # plans under a live graph would make its replay touch freed memory
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
            var = self.__dict__.get("_variables", {}).get(name.split("/")[0])
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

    def lifting(self, scoremap32, hand_side, variant="proposed"):
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
        _lib.check(self.lib.h3d_lifting_forward(self.h, _ptr(scoremap32), _ptr(hand_side), B, v, _ptr(out), _ptr(can), _ptr(rot),
                                                _stream()), "h3d_lifting_forward")
        return out, can, rot

    def pipeline(self, image, hand_side=None, with_pose3d=True, force_center=None, force_scale=None, want_mask=False,
                 outputs="all"):
        """ColorHandPose3DNetwork.inference / inference2d + detect_keypoints.  outputs="all" materialises the
        reference's large tensors; outputs="keypoints" keeps them in the workspace (serving mode)."""
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

    # ---- training (h3d_resize_bilinear_tf1_backward, the two losses, Adam) ----------------------
    def variables(self, scope):
        """Ordered {reference variable name: torch.nn.Parameter} of "HandSegNet" or "PoseNet2D" (layer order of the reference graph,
        weights before biases): fp32 device copies of the host arrays load_weights keeps, created once per context and then shared by
        every train=True graph, so an optimiser over them trains the network in place.

        The inference path (train=False, pipeline(), the stage entries) keeps the weights last loaded, not these Parameters: call
        commit_variables(scope) to make it use the trained values.  A later load_weights of the scope writes the loaded values into
        the same Parameters in place, so an optimiser built over them keeps working (its m / v slots are not reset)."""
        from . import arch
        layers = {"HandSegNet": arch.HANDSEGNET, "PoseNet2D": arch.POSENET2D}
        if scope not in layers:
            raise ValueError("variables(): scope must be 'HandSegNet' or 'PoseNet2D', got %r" % (scope,))
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
        B = records.shape[0]
        ds = {"rhd": 0, "stb": 1}[dataset]
        rb, H, W, hdr = (410520, 320, 320, 219) if ds == 0 else (922104, 480, 640, 126)
        if records.shape[1] != rb:
            raise ValueError("%s records are %d bytes, got %d" % (dataset, rb, records.shape[1]))
        dev = records.device
        image = torch.empty((B, H // step, W // step, 3), dtype=torch.float32, device=dev)
        header = torch.empty((B, hdr), dtype=torch.float32, device=dev) if want_aux else None
        mask = torch.empty((B, H, W), dtype=torch.uint8, device=dev) if (want_aux and ds == 0) else None
        vis = torch.empty((B, 42), dtype=torch.uint8, device=dev) if (want_aux and ds == 0) else None
        _lib.check(self.lib.h3d_decode_records(self.h, ds, _ptr(records), B, step, _ptr(header), _ptr(image), _ptr(mask), _ptr(vis),
                                               _stream()), "h3d_decode_records")
        return {"image": image, "header": header, "mask": mask, "visibility": vis}

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


_default = {}


def default_context(device=None) -> Context:
    idx = torch.cuda.current_device() if device is None else torch.device(device).index or 0
    if idx not in _default:
        _default[idx] = Context(idx)
    return _default[idx]


def reset_default_context():
    _default.clear()
