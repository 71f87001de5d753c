"""Golden vectors of the RHD reader's TRAINING mode, produced by running the reference's UNMODIFIED reader class
(data/BinaryDbReader.py with utils/ underneath, imported from a checkout of lmb-freiburg/hand3d ($H3D_REFERENCE)) over the eager TF
stand-in (oracle/tf1_eager.py) on the seeded synthetic records (tests/golden/synth_records.py).

TF's random streams cannot be reproduced, so this script SCRIPTS the reader's random ops: each returns the draws of
tests/reader_train_oracle.py for the serial being read (the same parameters the device generator computes).  What the vectors pin is
everything the reference source decides around the draws: where each noise enters (coord_uv_noise on all 42 key-points before the
21-subset, crop_center_noise before the crop size, crop_scale_noise on the clamped scale, crop_offset_noise after it), that image_crop
is cut from the hue-shifted image, the dropout's noise shape and rescale, random_crop_to_size as the elif after scale_to_size and the
keys each configuration returns.  The scripted ops, set on the stand-in module in this process only:
    truncated_normal   -> the parameters' noise for (shape, stddev) = ([42, 2], 2.5), ([2], 20), ([2], 10)
    random_uniform     -> the crop-scale factor for ([1], 1.0, 1.2)
    image.random_hue   -> reader_train_oracle.adjust_hue(image, delta) for max_delta 0.1
    random_crop        -> the window at the parameters' offsets for size [256, 256, 5]
    nn.dropout         -> keep_prob 0.8, noise_shape [1, 1, 21]: (x / 0.8) * keep bits; keep_prob 1 keeps the stand-in's assertion
    train.shuffle_batch_join -> capacity 100, min_after_dequeue 50 asserted; one sample (the queue is restated by the oracle)

    H3D_REFERENCE=<checkout of lmb-freiburg/hand3d> python tests/golden/make_golden_reference_reader_train.py
Large tensors are stored as an 8x sub-sampled copy plus float64 sum / sum of squares, as in golden_reference_reader.npz.
"""
import io
import os
import sys
import tempfile
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "golden_reference_reader_train.npz")
sys.path.insert(0, HERE)
import make_golden_reference_reader as MG  # noqa: E402
import synth_records as SR  # noqa: E402

SEED = 20171003
SERIALS = [0, 1, 2, 3]
# the reader arguments of training_handsegnet.py:37-39, training_posenet.py:37-39, training_lifting.py:44-46, and every flag at once
CONFIGS = {
    "handsegnet": dict(shuffle=True, hue_aug=True, random_crop_to_size=True),
    "posenet": dict(shuffle=True, use_wrist_coord=False, hand_crop=True, coord_uv_noise=True, crop_center_noise=True),
    "lifting": dict(shuffle=True, hand_crop=True, use_wrist_coord=False, coord_uv_noise=True, crop_center_noise=True, crop_offset_noise=True,
                    crop_scale_noise=True),
    "all": dict(shuffle=True, hand_crop=True, use_wrist_coord=False, hue_aug=True, coord_uv_noise=True, crop_center_noise=True,
                crop_scale_noise=True, crop_offset_noise=True, scoremap_dropout=True),
}


def script(tf, A, cur):
    """Binds the random ops of the stand-in to the oracle's draws for cur["params"]."""
    f32 = np.float32
    plain_dropout = tf.nn.dropout

    def truncated_normal(shape, mean=0.0, stddev=1.0, **k):
        p = cur["params"]
        assert float(mean) == 0.0
        sl = {(42, 2, 2.5): slice(A.UV_NOISE, A.UV_NOISE + 84), (2, 20.0): slice(A.CENTER_NOISE, A.CENTER_NOISE + 2),
              (2, 10.0): slice(A.OFFSET_NOISE, A.OFFSET_NOISE + 2)}[tuple(shape) + (float(stddev),)]
        cur["calls"].append("truncated_normal%s/%g" % (list(shape), stddev))
        return tf._w(p[sl].reshape(shape).copy())

    def random_uniform(shape, minval=0, maxval=None, dtype=np.float32, **k):
        assert list(shape) == [1] and float(minval) == 1.0 and float(maxval) == 1.2, (shape, minval, maxval)
        cur["calls"].append("random_uniform")
        return tf._w(cur["params"][A.SCALE:A.SCALE + 1].copy())

    def random_hue(image, max_delta, **k):
        assert max_delta == 0.1
        cur["calls"].append("random_hue")
        return tf._w(A.adjust_hue(np.asarray(image), cur["params"][A.HUE_DELTA]))

    def random_crop(value, size, **k):
        value = np.asarray(value)
        assert list(size) == [256, 256, value.shape[2]] and value.shape[:2] == (320, 320)
        oy, ox = int(cur["params"][A.WINDOW]), int(cur["params"][A.WINDOW + 1])
        cur["calls"].append("random_crop")
        return tf._w(value[oy:oy + 256, ox:ox + 256].copy())

    def dropout(x, keep_prob, noise_shape=None, **k):
        if keep_prob == 1.0:
            return plain_dropout(x, keep_prob, noise_shape=noise_shape, **k)
        assert f32(keep_prob) == f32(0.8) and list(noise_shape) == [1, 1, 21]
        cur["calls"].append("dropout")
        kp = f32(keep_prob)
        return tf._w((np.asarray(x, f32) / kp) * cur["params"][A.KEEP:A.KEEP + 21].reshape(1, 1, 21))

    def shuffle_batch_join(tensors_list, batch_size, capacity=None, min_after_dequeue=None, enqueue_many=False, **k):
        assert capacity == 100 and min_after_dequeue == 50 and not enqueue_many
        cur["calls"].append("shuffle_batch_join")
        return tf._batch_join(tensors_list, batch_size)

    # TF tensors are immutable: `crop_center += noise` (:279, :312) rebinds the name.  The stand-in's ndarray would add in place and,
    # since crop_center is a view of keypoint_uv21[12], move that key-point too; so augmented assignment makes a new array here.
    for op, fn in (("__iadd__", np.add), ("__isub__", np.subtract), ("__imul__", np.multiply), ("__itruediv__", np.true_divide)):
        setattr(tf.Tensor, op, lambda self, other, fn=fn: fn(self, other))
    tf.truncated_normal, tf.random_uniform, tf.random_crop = truncated_normal, random_uniform, random_crop
    tf.image.random_hue = random_hue
    tf.nn.dropout = dropout
    tf.train.shuffle_batch_join = shuffle_batch_join


def main():
    tf, rhd, _ = MG.setup_imports()
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import reader_train_oracle as A
    cur = {"params": None, "calls": []}
    script(tf, A, cur)
    out = {"seed": np.array(SEED, np.uint64), "serials": np.array(SERIALS, np.int64)}
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            os.makedirs("data/bin")
            recs = SR.rhd_records(4)
            with open("data/bin/rhd_training.bin", "wb") as f:
                f.write(b"".join(recs))
            for name, kw in CONFIGS.items():
                flags = A.flags_of(**kw)
                params = A.aug_params(SEED, SERIALS, flags)
                tf.reset_readers()
                for i, serial in enumerate(SERIALS):
                    assert serial % len(recs) == i            # the stand-in's reader hands the records out in order
                    cur["params"], cur["calls"] = params[i], []
                    MG.pack("%s/%d" % (name, i), rhd.BinaryDbReader(mode="training", batch_size=1, **kw).get(), out)
                    out["%s/%d/params" % (name, i)] = params[i]
                    out["%s/%d/calls" % (name, i)] = np.array(cur["calls"])
        finally:
            os.chdir(cwd)
    with zipfile.ZipFile(OUT, "w", compression=zipfile.ZIP_LZMA) as z:
        for k, v in sorted(out.items()):
            b = io.BytesIO()
            np.save(b, np.asarray(v))
            z.writestr(k + ".npy", b.getvalue())
    print("wrote %s: %d arrays, %.1f KB" % (OUT, len(out), os.path.getsize(OUT) / 1024))


if __name__ == "__main__":
    main()
