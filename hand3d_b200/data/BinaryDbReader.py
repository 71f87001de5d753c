"""BinaryDbReader / BinaryDbReaderSTB -- H100-native mirrors of the reference's dataset readers (data/BinaryDbReader.py:21-412,
data/BinaryDbReaderSTB.py:21-330): same constructor arguments, `num_samples`, and `get()` returning the same dictionary keys, but
eager: every get() call uploads the next `batch_size` fixed-length records as bytes and produces the raw and derived items on the GPU
(h3d_decode_records, h3d_rhd_reader_items / h3d_stb_reader_items, h3d_crop_image_from_xy, h3d_gaussian_scoremap,
h3d_canonical_trafo).

The RHD reader also runs in training mode, as training_handsegnet.py, training_posenet.py and training_lifting.py build it:
`shuffle=True` and the seven augmentation flags (hue_aug, coord_uv_noise, crop_center_noise, crop_scale_noise, crop_offset_noise,
scoremap_dropout, random_crop_to_size) in the reference's order (data/BinaryDbReader.py:160-401).  TF's random streams cannot be
reproduced, so the draws are the project's own: every random value is a pure function of (seed, serial, value), where `serial` is
the sample's position in the enqueue stream (record = serial mod records in the file), computed on the device with Philox4x64-10
(h3d_reader_aug_params; layouts in include/hand3d_b200.h).  The deterministic transforms given those draws follow the reference
exactly.  `seed=None` draws a seed from OS entropy; `reader.seed` replays a run.  `shuffle=True` is the steady state of
shuffle_batch_join(capacity=100, min_after_dequeue=50): a buffer of the next 100 stream positions, each dequeue taking a uniformly
random slot that the stream then refills -- a windowed shuffle, not a permutation of the file.  A flag that is off is skipped, so
with all flags off the items are bit-identical to the evaluation path.  STB keeps refusing augmentation and shuffling: no training
script reads it.

`device_resident=True` (both readers) uploads the file's whole records to the device once, through a bounded pinned staging buffer,
and keeps the queue state there too: get() then runs the queue (h3d_reader_next_serials), the fused gather + decode
(h3d_decode_records_gather) and the same item, augmentation and score-map kernels as the host path, with no host tensor, no
host-to-device copy and no synchronisation, so a whole training iteration can be captured into one CUDA graph.  It costs
`reader.device_bytes` of device memory (16.9 GB for rhd_training.bin) and the upload; the default keeps the file on the host.  The
items are bit-identical to the host reader's for the same seed.  `state_dict()` / `load_state_dict()` carry the stream position (queue
slots, next position, dequeue count) and move between the two modes.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from .. import _lib, runtime
from .records import RHD_RECORD_BYTES, STB_RECORD_BYTES

_AUG = ("random_crop_to_size", "hue_aug", "coord_uv_noise", "crop_center_noise", "crop_scale_noise", "crop_offset_noise", "scoremap_dropout")
_AUG_BITS = {"coord_uv_noise": _lib.AUG_COORD_UV_NOISE, "crop_center_noise": _lib.AUG_CROP_CENTER_NOISE, "crop_scale_noise": _lib.AUG_CROP_SCALE_NOISE,
             "crop_offset_noise": _lib.AUG_CROP_OFFSET_NOISE, "hue_aug": _lib.AUG_HUE, "random_crop_to_size": _lib.AUG_RANDOM_CROP,
             "scoremap_dropout": _lib.AUG_SCOREMAP_DROPOUT}
_ITEM_NOISE = _lib.AUG_COORD_UV_NOISE | _lib.AUG_CROP_CENTER_NOISE | _lib.AUG_CROP_SCALE_NOISE | _lib.AUG_CROP_OFFSET_NOISE


class _RecordFile:
    def __init__(self, path, record_bytes, num_samples):
        assert os.path.exists(path), "Could not find the binary data file!"
        self.mm = np.memmap(path, dtype=np.uint8, mode="r")
        self.record_bytes = record_bytes
        self.available = self.mm.size // record_bytes
        self.num_samples = min(num_samples, self.available) if self.available else num_samples
        self.pos = 0

    def gather(self, serials):
        """The records at stream positions `serials`, uploaded: the TF queue cycles through the file, so record = serial mod count."""
        n, rb = max(1, self.available), self.record_bytes
        rec = np.stack([np.asarray(self.mm[(s % n) * rb:(s % n + 1) * rb]) for s in serials])
        dev = runtime.default_context().device
        return torch.from_numpy(rec).pin_memory().to(dev, non_blocking=True)

    def next_batch(self, n):
        serials = range(self.pos, self.pos + n)
        self.pos += n
        return self.gather(serials)


def _refuse_short_file(path, record_bytes):
    if os.path.exists(path) and os.path.getsize(path) < record_bytes:
        raise ValueError("device_resident: %s holds %d bytes, less than one %d-byte record" % (path, os.path.getsize(path), record_bytes))


class _ResidentFile:
    """The `available` whole records of a _RecordFile as one uint8 device tensor [available, record_bytes], uploaded once through a
    pinned staging buffer of at most STAGING_BYTES (two halves, so reading the file overlaps the copies): the file is never pinned."""
    STAGING_BYTES = 64 << 20

    def __init__(self, rf, device):
        n, rb = rf.available, rf.record_bytes
        self.records = torch.empty((n, rb), dtype=torch.uint8, device=device)
        per = max(1, self.STAGING_BYTES // 2 // rb)              # whole records per half
        stage = [torch.empty((per, rb), dtype=torch.uint8, pin_memory=True) for _ in range(2)]
        done = [None, None]
        stream = torch.cuda.current_stream(device)
        for k, r0 in enumerate(range(0, n, per)):
            m, h = min(per, n - r0), k % 2
            if done[h] is not None:
                done[h].synchronize()                             # the copy out of this half has finished
            stage[h].numpy()[:m] = np.asarray(rf.mm[r0 * rb:(r0 + m) * rb]).reshape(m, rb)
            self.records[r0:r0 + m].copy_(stage[h][:m], non_blocking=True)
            done[h] = torch.cuda.Event()
            done[h].record(stream)
        stream.synchronize()

    @property
    def nbytes(self):
        return self.records.numel()


def _stream_state(shuffle, count, nxt, slots):
    return {"shuffle": bool(shuffle), "count": int(count), "next": int(nxt), "slots": [int(s) for s in slots] if shuffle else None}


def _check_stream_state(state, shuffle):
    if bool(state["shuffle"]) != bool(shuffle):
        raise ValueError("state_dict of a %s reader cannot resume a %s one" % (("shuffled", "in-order")[not state["shuffle"]],
                                                                            ("shuffled", "in-order")[not shuffle]))
    if shuffle and len(state["slots"]) != _lib.READER_QUEUE_CAPACITY:
        raise ValueError("the queue holds %d slots" % _lib.READER_QUEUE_CAPACITY)
    if not 0 <= int(state["count"]) < 2 ** 63 or not 0 <= int(state["next"]) < 2 ** 63:
        raise ValueError("stream positions must lie in [0, 2**63)")


class _DeviceStream:
    """The queue state of a resident reader, int64 [READER_STATE_WORDS] on the device (layout with H3D_READER_STATE_* in
    include/hand3d_b200.h), advanced in place by h3d_reader_next_serials, so that a captured get() keeps reading on replay."""

    def __init__(self, seed, shuffle, device):
        self.seed, self.shuffle = seed, bool(shuffle)
        self.state = torch.zeros(_lib.READER_STATE_WORDS, dtype=torch.int64, device=device)
        cap = _lib.READER_QUEUE_CAPACITY
        self.load_state_dict(_stream_state(shuffle, 0, cap if shuffle else 0, range(cap)))

    def take(self, n):
        return runtime.default_context(self.state.device).reader_next_serials(self.state, n, self.seed, self.shuffle)

    def state_dict(self):
        w = self.state.tolist()
        return _stream_state(self.shuffle, w[_lib.READER_STATE_COUNT], w[_lib.READER_STATE_NEXT],
                             w[_lib.READER_STATE_SLOTS:_lib.READER_STATE_SLOTS + _lib.READER_QUEUE_CAPACITY])

    def load_state_dict(self, state):
        _check_stream_state(state, self.shuffle)
        w = np.zeros(_lib.READER_STATE_WORDS, np.int64)
        w[_lib.READER_STATE_COUNT], w[_lib.READER_STATE_NEXT] = int(state["count"]), int(state["next"])
        if self.shuffle:
            w[_lib.READER_STATE_SLOTS:_lib.READER_STATE_SLOTS + _lib.READER_QUEUE_CAPACITY] = state["slots"]
        self.state.copy_(torch.from_numpy(w))                     # in place: a captured get() reads this buffer


class _ShuffleQueue:
    """tf.train.shuffle_batch_join(capacity=100, min_after_dequeue=50) over the in-order record stream, in its steady state: the
    buffer holds the next CAPACITY stream positions; each dequeue takes slot (w mod CAPACITY) and the stream refills it.  The words w
    come from Philox4x64-10 keyed (seed, H3D_AUG_STREAM_SHUFFLE), one per dequeue in order (numpy.random.Philox, counter from 0),
    so the sequence of serials depends on the seed only, not on how it is cut into batches."""
    CAPACITY = 100

    def __init__(self, seed):
        self._seed = seed
        self._bits = np.random.Philox(key=np.array([seed, _lib.AUG_STREAM_SHUFFLE], np.uint64))
        self._slots = list(range(self.CAPACITY))
        self._next = self.CAPACITY
        self._count = 0

    def take(self, n):
        out = []
        for w in self._bits.random_raw(n):
            k = int(w) % self.CAPACITY
            out.append(self._slots[k])
            self._slots[k] = self._next
            self._next += 1
        self._count += n
        return out

    def state_dict(self):
        return _stream_state(True, self._count, self._next, self._slots)

    def load_state_dict(self, state):
        _check_stream_state(state, True)
        count = int(state["count"])
        # numpy.random.Philox bumps its counter before it fills its 4-word buffer: after `count` words the counter is count // 4 with
        # an empty buffer, advanced by the count % 4 words already used of the next block
        bits = np.random.Philox(key=np.array([self._seed, _lib.AUG_STREAM_SHUFFLE], np.uint64))
        st = bits.state
        st["state"]["counter"] = np.array([count // 4, 0, 0, 0], np.uint64)
        st["buffer_pos"] = 4
        bits.state = st
        bits.random_raw(count % 4)
        self._bits, self._count = bits, count
        self._slots, self._next = [int(s) for s in state["slots"]], int(state["next"])


class BinaryDbReader(object):
    """ Reads data from a binary dataset created by create_binary_db.py (RHD). """
    def __init__(self, mode=None, batch_size=1, shuffle=True, use_wrist_coord=True, sigma=25.0, hand_crop=False, random_crop_to_size=False,
                 scale_to_size=False, hue_aug=False, coord_uv_noise=False, crop_center_noise=False, crop_scale_noise=False,
                 crop_offset_noise=False, scoremap_dropout=False, path_to_db=None, seed=None, device_resident=False):
        if mode == 'training':
            path, n = './data/bin/rhd_training.bin', 41258
        elif mode == 'evaluation':
            path, n = './data/bin/rhd_evaluation.bin', 2728
        else:
            assert 0, "Unknown dataset mode."
        if device_resident:
            _refuse_short_file(path_to_db or path, RHD_RECORD_BYTES)
        flags = 0
        for name in _AUG:
            if locals()[name]:
                flags |= _AUG_BITS[name]
        if scale_to_size:                  # random_crop_to_size is the elif branch after scale_to_size (:369-392)
            flags &= ~_lib.AUG_RANDOM_CROP
        if seed is None:                   # like TF's unseeded random ops; reader.seed replays the run
            seed = int.from_bytes(os.urandom(8), "little")
        if not 0 <= int(seed) < 2 ** 64:
            raise ValueError("seed must be in [0, 2**64)")
        self._file = _RecordFile(path_to_db or path, RHD_RECORD_BYTES, n)
        self.path_to_db = path_to_db or path
        self.num_samples = self._file.num_samples
        self.batch_size, self.sigma, self.shuffle, self.use_wrist_coord = batch_size, sigma, shuffle, use_wrist_coord
        self.scale_to_size, self.scale_target_size, self.hand_crop = scale_to_size, (240, 320), hand_crop
        self.image_size, self.crop_size, self.num_kp = (320, 320), 256, 42
        self.random_crop_size = 256
        self.seed = int(seed)
        self._flags = flags
        self._queue = _ShuffleQueue(self.seed) if shuffle else None
        self._next_serial = 0
        self._resident = self._stream = None
        if device_resident:
            dev = runtime.default_context().device
            self._resident = _ResidentFile(self._file, dev)
            self._stream = _DeviceStream(self.seed, shuffle, dev)

    @property
    def device_bytes(self):
        """Device memory held by the resident records (0 on the host path)."""
        return self._resident.nbytes if self._resident is not None else 0

    def state_dict(self):
        """The stream position: {'shuffle', 'count' (dequeues so far), 'next' (next position to enqueue), 'slots' (queue, or None)}.
        Readers built with the same seed read the same stream, so a state moves between host and resident readers."""
        if self._stream is not None:
            return self._stream.state_dict()
        if self._queue is not None:
            return self._queue.state_dict()
        return _stream_state(False, self._next_serial, self._next_serial, ())

    def load_state_dict(self, state):
        """Resumes the stream at `state` (from state_dict()); the resident reader writes its device state in place."""
        if self._stream is not None:
            self._stream.load_state_dict(state)
        elif self._queue is not None:
            self._queue.load_state_dict(state)
        else:
            _check_stream_state(state, False)
            self._next_serial = int(state["next"])

    def get(self):
        """ Next batch as a dict of CUDA tensors with the reference's keys (data/BinaryDbReader.py:100-411). """
        B = self.batch_size
        if self._stream is not None:
            serials = self._stream.take(B)
        elif self._queue is not None:
            serials = self._queue.take(B)
        else:
            serials = list(range(self._next_serial, self._next_serial + B))
            self._next_serial += B
        return self._get(serials)

    def _get(self, serials, params=None):
        """The samples at enqueue positions `serials` (a list, or an int64 device tensor on the resident path); `params`
        [B, H3D_AUG_PARAMS] replaces the drawn augmentation parameters."""
        ctx = runtime.default_context()
        B = len(serials)
        flags = self._flags
        if torch.is_tensor(serials):
            raw = ctx.decode_records_gather(self._resident.records, serials, "rhd", 1)
        else:
            raw = ctx.decode_records(self._file.gather(serials), "rhd", 1)
        if flags and params is None:
            params = ctx.reader_aug_params(serials if torch.is_tensor(serials) else torch.tensor(list(serials), dtype=torch.int64),
                                           self.seed, flags)
        if flags & _lib.AUG_RANDOM_CROP:   # :382-392: only the three windows are kept, so nothing else is computed
            img, parts, mask = ctx.augment_image(raw["image"], params, flags & (_lib.AUG_HUE | _lib.AUG_RANDOM_CROP), raw["mask"],
                                                 self.random_crop_size)
            return {"image": img, "hand_parts": parts, "hand_mask": mask}
        h = raw["header"]
        if flags:
            it = ctx.rhd_reader_items_aug(h, raw["mask"], raw["visibility"], params, flags & _ITEM_NOISE, self.use_wrist_coord, self.hand_crop,
                                          self.crop_size)
        else:
            it = ctx.rhd_reader_items(h, raw["mask"], raw["visibility"], self.use_wrist_coord, self.hand_crop, self.crop_size)
        image = raw["image"]
        if flags & _lib.AUG_HUE:           # :183-184, before image_crop is cut from it
            image = ctx.augment_image(image, params, _lib.AUG_HUE)[0]
        xyz = h[:, :126].reshape(B, 42, 3)
        uv = h[:, 126:210].reshape(B, 42, 2).to(torch.int32).to(torch.float32)
        vis = raw["visibility"].to(torch.bool)
        if not self.use_wrist_coord:       # the 42-key-point views with the palm substituted (:139-162,195-200)
            xyz = torch.cat([0.5 * (xyz[:, 0:1] + xyz[:, 12:13]), xyz[:, 1:21], 0.5 * (xyz[:, 21:22] + xyz[:, 33:34]), xyz[:, 22:]], 1)
            uv = torch.cat([0.5 * (uv[:, 0:1] + uv[:, 12:13]), uv[:, 1:21], 0.5 * (uv[:, 21:22] + uv[:, 33:34]), uv[:, 22:]], 1)
            vis = torch.cat([vis[:, 0:1] | vis[:, 12:13], vis[:, 1:21], vis[:, 21:22] | vis[:, 33:34], vis[:, 22:]], 1)
        if flags:
            uv = it["keypoint_uv"]         # palm-substituted on the device, + coord_uv_noise (:160-164)
        parts = raw["mask"].to(torch.int32)
        hand = parts > 1
        d = {"keypoint_xyz": xyz, "keypoint_uv": uv, "cam_mat": it["cam_mat"], "image": image, "hand_parts": parts,
             "hand_mask": torch.stack([~hand, hand], 3).to(torch.int32), "keypoint_vis": vis, "hand_side": it["hand_side"],
             "keypoint_xyz21": it["keypoint_xyz21"], "keypoint_scale": it["keypoint_scale"], "keypoint_xyz21_normed": it["keypoint_xyz21_normed"],
             "keypoint_vis21": it["keypoint_vis21"].to(torch.bool), "keypoint_uv21": it["keypoint_uv21"]}
        right = it["hand_side"][:, 1] > 0.5
        can, _, rot_inv = ctx.canonical_trafo(it["keypoint_xyz21_normed"], right)
        d["keypoint_xyz21_can"], d["rot_mat"] = can, rot_inv
        d["keypoint_xyz21_local"] = ctx.bone_rel_trafo(it["keypoint_xyz21_normed"])      # :245-247, the 'local' lifting target
        size = self.image_size
        if self.hand_crop:
            d["crop_scale"] = it["crop_scale"]
            d["image_crop"] = ctx.crop_image_from_xy(image, it["crop_center"], self.crop_size, it["crop_scale"])
            size = (self.crop_size, self.crop_size)
        hw21 = torch.stack([it["keypoint_uv21"][..., 1], it["keypoint_uv21"][..., 0]], -1).contiguous()
        if flags & _lib.AUG_SCOREMAP_DROPOUT:      # :362-365
            d["scoremap"] = ctx.gaussian_scoremap_dropout(hw21, size, self.sigma, it["keypoint_vis21"],
                                                          params[:, _lib.AUG_KEEP:_lib.AUG_KEEP + 21], 0.8)
        else:
            d["scoremap"] = ctx.gaussian_scoremap(hw21, size, self.sigma, it["keypoint_vis21"])
        if self.scale_to_size:             # :368-381: everything else is dropped
            s = self.image_size
            image = ctx.resize_bilinear(image, *self.scale_target_size)
            sc = (self.scale_target_size[0] / float(s[0]), self.scale_target_size[1] / float(s[1]))
            uv21 = torch.stack([d["keypoint_uv21"][..., 0] * sc[1], d["keypoint_uv21"][..., 1] * sc[0]], -1)
            d = {"image": image, "keypoint_uv21": uv21, "keypoint_vis21": d["keypoint_vis21"]}
        return d


class BinaryDbReaderSTB(object):
    """ Reads data from the STB binary dataset (data/BinaryDbReaderSTB.py). """
    def __init__(self, mode=None, batch_size=1, shuffle=True, use_wrist_coord=True, sigma=25.0, hand_crop=False, random_crop_to_size=False,
                 hue_aug=False, coord_uv_noise=False, crop_center_noise=False, crop_scale_noise=False, crop_offset_noise=False,
                 scoremap_dropout=False, path_to_db=None, with_scoremap=False, device_resident=False):
        if mode == 'training':
            path, n = './data/stb/stb_train_shuffled.bin', 30000
        elif mode == 'evaluation':
            path, n = './data/stb/stb_eval.bin', 6000
        else:
            assert 0, "Unknown dataset mode."
        for name in _AUG:                  # no training script reads STB; its coord_uv_noise (:158-160) cannot build a graph either
            if locals().get(name):
                raise NotImplementedError("BinaryDbReaderSTB serves the evaluation driver: %s is training-time augmentation" % name)
        if shuffle or hand_crop:
            raise NotImplementedError("shuffle / hand_crop on STB are training-time options; the evaluation driver (eval_full.py:45) uses neither")
        if device_resident:
            _refuse_short_file(path_to_db or path, STB_RECORD_BYTES)
        self._file = _RecordFile(path_to_db or path, STB_RECORD_BYTES, n)
        self.path_to_db = path_to_db or path
        self.num_samples = self._file.num_samples
        self.batch_size, self.sigma, self.use_wrist_coord, self.with_scoremap = batch_size, sigma, use_wrist_coord, with_scoremap
        self.image_size, self.crop_size, self.num_kp = (480, 640), 256, 21
        self._resident = self._stream = None
        if device_resident:
            dev = runtime.default_context().device
            self._resident = _ResidentFile(self._file, dev)
            self._stream = _DeviceStream(0, False, dev)
            self._consts = self._constants(dev)      # made once: get() creates no tensor from host data

    @staticmethod
    def _constants(dev):
        return (torch.tensor([[822.79041, 0.0, 318.47345], [0.0, 822.79041, 250.31296], [0.0, 0.0, 1.0]], device=dev),
                torch.tensor([1.0, 0.0], device=dev))

    @property
    def device_bytes(self):
        """Device memory held by the resident records (0 on the host path)."""
        return self._resident.nbytes if self._resident is not None else 0

    def state_dict(self):
        """The stream position, as BinaryDbReader.state_dict() (in order: 'slots' is None and 'count' == 'next')."""
        if self._stream is not None:
            return self._stream.state_dict()
        return _stream_state(False, self._file.pos, self._file.pos, ())

    def load_state_dict(self, state):
        if self._stream is not None:
            self._stream.load_state_dict(state)
        else:
            _check_stream_state(state, False)
            self._file.pos = int(state["next"])

    def get(self):
        ctx = runtime.default_context()
        B = self.batch_size
        if self._stream is not None:
            raw = ctx.decode_records_gather(self._resident.records, self._stream.take(B), "stb", 1, want_aux=True)
            cam_mat, hand_side = self._consts
        else:
            raw = ctx.decode_records(self._file.next_batch(B), "stb", 1, want_aux=True)
            cam_mat, hand_side = self._constants(raw["image"].device)
        it = ctx.stb_reader_items(raw["header"], self.use_wrist_coord)
        d = {"keypoint_xyz21": it["keypoint_xyz21"], "keypoint_vis21": it["keypoint_vis21"].to(torch.bool), "keypoint_uv21": it["keypoint_uv21"],
             "image": raw["image"], "keypoint_scale": it["keypoint_scale"], "keypoint_xyz21_normed": it["keypoint_xyz21_normed"],
             "cam_mat": cam_mat.expand(B, 3, 3), "hand_side": hand_side.expand(B, 2).contiguous()}
        can, _, rot_inv = ctx.canonical_trafo(it["keypoint_xyz21_normed"], None)
        d["keypoint_xyz21_can"], d["rot_mat"] = can, rot_inv
        d["keypoint_xyz21_local"] = ctx.bone_rel_trafo(it["keypoint_xyz21_normed"])      # :199-202
        if self.with_scoremap:             # 480 x 640 x 21 targets (26 MB per sample): training only, off by default
            hw21 = torch.stack([it["keypoint_uv21"][..., 1], it["keypoint_uv21"][..., 0]], -1).contiguous()
            d["scoremap"] = ctx.gaussian_scoremap(hw21, self.image_size, self.sigma, it["keypoint_vis21"])
        return d
