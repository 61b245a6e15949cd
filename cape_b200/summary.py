"""TensorBoard event files without TensorFlow: what the reference's `tf.summary.FileWriter` writes during `fit`
(lib/models.py:868,907-922), the scalars and weight histograms of its `op_summary`.

Format (tensorflow/core/util/event.proto, core/framework/summary.proto, core/lib/io/record_writer, restated from their
published description): a file `events.out.tfevents.<10-digit unix time>.<hostname>` of TFRecords -- u64 length, masked
CRC32C of the length, the serialised `Event`, masked CRC32C of it.  The first event carries `file_version:
"brain.Event:2"`; every other one `{wall_time, step, summary}` with `Summary.Value{tag, simple_value}` or
`{tag, histo: HistogramProto}`.  The protobuf and CRC helpers are tf_checkpoint's.

Histograms follow TF-1.13's `HistogramSummary` op (core/lib/histogram): fixed bucket limits growing by 10% from 1e-12
to 1e20 (`bucket_limits`), counted on the GPU by `cape_histogram` (CapeNetwork.weight_histograms), encoded with every
run of empty buckets collapsed into one entry (`EncodeToProto(preserve_zero_buckets=false)`).
"""
import glob
import os
import socket
import struct
import time

import numpy as np

from .tf_checkpoint import _field, _put_varint, crc32c, mask_crc

# Tags of op_summary's scalars, in the reference's order.  TF-1's tf.summary.scalar opens a uniquified name scope inside
# the enclosing tf.name_scope blocks: `loss/reconstruction_loss` and `loss/latent_loss` were opened already by the
# `with tf.name_scope(...)` blocks of loss() (lib/models.py:356,370), so those two take `_1`; the averages sit in
# `loss/averages` (:407), the learning rates in `training` (:421,443-444).  The edge loss is not summarised.
SCALAR_TAGS = ("loss/reconstruction_loss_1", "loss/latent_loss_1", "loss/fc_regularization_g", "loss/fc_regularization_d",
               "loss/gan_loss_generator", "loss/gan_loss_discriminator", "loss/averages/loss_g",
               "loss/averages/loss_d", "training/lr_g", "training/lr_d")
VALIDATION_TAG = "validation/loss"                         # added by fit (lib/models.py:920)
# the moving averages of the loss totals: tf.train.ExponentialMovingAverage(0.9) (lib/models.py:408)
LOSS_AVERAGE_DECAY = 0.9
# the generator's regularised dense kernels (tf.layers.dense with kernel_regularizer, lib/models.py:378)
FC_REGULARISED = ("generator/encoder/fc_mean/dense/kernel", "generator/encoder/fc_var/dense/kernel",
                  "generator/decoder/fc1/dense/kernel")


def is_histogrammed(name):
    """_weight_variable / _bias_variable (lib/models.py:217-227) histogram every `.../weights` and `.../bias` they
    create: the graph-conv, 1x1 and graph-linear weights, the brelu biases and `outputs/bias`.  Dense layers
    (tf.layers.dense: `.../dense/kernel`, `.../dense/bias`) and GroupNorm's gamma / beta are not theirs."""
    return (name.endswith("/weights") or name.endswith("/bias")) and "/dense/" not in name


def histogram_names(specs):
    """The histogrammed variables of a parameter inventory (params.param_specs), in its order."""
    return [n for n in specs if is_histogrammed(n)]


def bucket_limits():
    """TF-1's default histogram bucket limits (histogram.cc, InitDefaultBucketsInner), as float64: 1e-12 growing by
    10% while below 1e20, then DBL_MAX; the same negated in reverse order in front, 0.0 in the middle."""
    pos = []
    v = 1.0e-12
    while v < 1.0e20:
        pos.append(v)
        v *= 1.1
    pos.append(np.finfo(np.float64).max)
    return np.array([-x for x in reversed(pos)] + [0.0] + pos, np.float64)


def encode_histogram(stats, counts, limits):
    """HistogramProto bytes: stats = (min, max, num, sum, sum_squares); counts[b] the number of values in bucket b
    (limits[b-1] <= x < limits[b]).  Each run of empty buckets becomes one entry carrying the run's last limit."""
    counts = np.asarray(counts)
    out_lim, out_cnt = [], []
    i, n = 0, len(counts)
    while i < n:
        end, c = limits[i], counts[i]
        i += 1
        if c <= 0:
            while i < n and counts[i] <= 0:
                end, c = limits[i], counts[i]
                i += 1
        out_lim.append(end)
        out_cnt.append(c)
    packed = lambda a: _put_varint(8 * len(a)) + np.asarray(a, "<f8").tobytes()
    mn, mx, num, s, sq = (float(x) for x in stats)
    return (_field(1, 1, struct.pack("<d", mn)) + _field(2, 1, struct.pack("<d", mx)) +
            _field(3, 1, struct.pack("<d", num)) + _field(4, 1, struct.pack("<d", s)) +
            _field(5, 1, struct.pack("<d", sq)) + _field(6, 2, packed(out_lim)) + _field(7, 2, packed(out_cnt)))


def _record(data):
    n = struct.pack("<Q", len(data))
    return n + struct.pack("<I", mask_crc(crc32c(n))) + data + struct.pack("<I", mask_crc(crc32c(data)))


def _event(wall_time, step=None, file_version=None, values=()):
    out = _field(1, 1, struct.pack("<d", wall_time))
    if step is not None:
        out += _field(2, 0, _put_varint(int(step)))
    if file_version is not None:
        fv = file_version.encode()
        out += _field(3, 2, _put_varint(len(fv)) + fv)
    if values:
        summ = b"".join(_field(1, 2, _put_varint(len(v)) + v) for v in values)
        out += _field(5, 2, _put_varint(len(summ)) + summ)
    return out


def _value(tag, simple_value=None, histo=None):
    t = tag.encode()
    out = _field(1, 2, _put_varint(len(t)) + t)
    if histo is not None:
        return out + _field(5, 2, _put_varint(len(histo)) + histo)
    return out + _field(2, 5, struct.pack("<f", np.float32(simple_value)))


def event_files(logdir):
    return sorted(glob.glob(os.path.join(glob.escape(logdir), "events.out.tfevents.*")))


def remove_event_files(logdir):
    """The event files directly in `logdir` (nothing else in it, nothing below it)."""
    for f in event_files(logdir):
        if os.path.isfile(f):
            os.remove(f)


class EventWriter(object):
    """One new event file in `logdir` (created if missing), flushed after every event."""

    def __init__(self, logdir):
        os.makedirs(logdir, exist_ok=True)
        now = time.time()
        self.path = os.path.join(logdir, "events.out.tfevents.%010d.%s" % (int(now), socket.gethostname()))
        self._f = open(self.path, "ab")
        self._write(_event(now, file_version="brain.Event:2"))

    def _write(self, event):
        self._f.write(_record(event))
        self._f.flush()

    def add(self, step, scalars=(), histograms=()):
        """scalars: [(tag, value)], stored as float32; histograms: [(tag, HistogramProto bytes)]."""
        values = [_value(t, simple_value=v) for t, v in scalars] + [_value(t, histo=h) for t, h in histograms]
        self._write(_event(time.time(), step=step, values=values))

    def close(self):
        if self._f is not None:
            self._f.close()
            self._f = None
