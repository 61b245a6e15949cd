"""Host transcriptions the summary tests compare against.

- `TFHistogram`: TF-1.13's `tensorflow::histogram::Histogram` (core/lib/histogram/histogram.cc) line by line in Python
  floats (doubles): the default bucket limits, `Add`, `EncodeToProto(preserve_zero_buckets=false)`.
- `loss_average`: the float32 recurrence of `tf.train.ExponentialMovingAverage(0.9)` over the reference's loss totals
  (lib/models.py:393-414), one update per optimiser application.
- `read_events`: an event-file reader written apart from cape_b200.summary (own CRC32C, own framing).
"""
import bisect
import struct
import sys

import numpy as np

DBL_MAX = sys.float_info.max


class TFHistogram(object):
    def __init__(self):
        buckets, neg = [], []
        v = 1.0e-12
        while v < 1.0e20:
            buckets.append(v)
            neg.append(-v)
            v *= 1.1
        buckets.append(DBL_MAX)
        neg.append(-DBL_MAX)
        neg.reverse()
        self.limits = neg + [0.0] + buckets
        self.min, self.max = self.limits[-1], -self.limits[-1]
        self.num = self.sum = self.sum_squares = 0.0
        self.buckets = [0.0] * len(self.limits)

    def add(self, value):
        value = float(value)
        b = bisect.bisect_right(self.limits, value)          # std::upper_bound
        self.buckets[b] += 1.0
        if self.min > value:
            self.min = value
        if self.max < value:
            self.max = value
        self.num += 1
        self.sum += value
        self.sum_squares += value * value

    def encode(self):
        """(min, max, num, sum, sum_squares, bucket_limit, bucket) of EncodeToProto(preserve_zero_buckets=false)."""
        lim, cnt = collapse(self.limits, self.buckets)
        return self.min, self.max, self.num, self.sum, self.sum_squares, lim, cnt


def collapse(limits, buckets):
    """EncodeToProto's loop: each run of empty buckets becomes one entry with the run's last limit."""
    lim, cnt = [], []
    i = 0
    while i < len(buckets):
        end, count = limits[i], float(buckets[i])
        i += 1
        if count <= 0.0:
            while i < len(buckets) and buckets[i] <= 0.0:
                end, count = limits[i], float(buckets[i])
                i += 1
        lim.append(float(end))
        cnt.append(count)
    return lim, cnt


def histogram(values):
    """TFHistogram's result for many values, vectorised: (min, max, num, sum (math.fsum), sum_squares (math.fsum),
    counts per bucket).  min / max are the first occurrence of the extreme value, as Add's strict compares keep it
    (it decides the sign of a zero)."""
    import math
    x = np.asarray(values, np.float32).reshape(-1).astype(np.float64)
    lim = np.array(TFHistogram().limits)
    counts = np.bincount(np.searchsorted(lim, x, side="right"), minlength=len(lim))
    mn, mx = x[np.argmax(x == x.min())], x[np.argmax(x == x.max())]
    return float(mn), float(mx), float(x.size), math.fsum(x), math.fsum(x * x), counts


def tf_histogram(values):
    h = TFHistogram()
    for v in np.asarray(values, np.float32).reshape(-1):
        h.add(v)
    return h


def loss_totals(losses, fc_sumsq, cfg):
    """(loss_g, loss_d) in float32, op by op (lib/models.py:393-397); losses = the step's loss buffer."""
    f = np.float32
    L = [f(x) for x in losses]
    r = f(cfg["regularization"])
    reg_g = r * (r * (f(fc_sumsq) * f(0.5)))
    g = L[3] * f(cfg["lambda_gan"])
    g = g + L[0] * f(cfg["lambda_recon"])
    g = g + f(0.0)
    g = g + L[1] * f(cfg["lambda_edge"])
    g = g + L[2] * f(cfg["lambda_latent"])
    g = g + reg_g
    d = (L[4] + L[5]) * f(cfg["lambda_gan"]) + f(0.0)
    return f(g), f(d)


def loss_average(applications, cfg, decay=0.9):
    """The shadows (loss_g, loss_d) after the given applications [(losses, fc_sumsq)], from 0:
    s -= (s - v) * (1 - decay), every operation in float32 (assign_moving_average, zero_debias off)."""
    f = np.float32
    k = f(1.0) - f(decay)
    s = [f(0.0), f(0.0)]
    for losses, fc in applications:
        for i, v in enumerate(loss_totals(losses, fc, cfg)):
            s[i] = s[i] - (s[i] - v) * k
    return s


# ---- event files --------------------------------------------------------------------------------------------------
def _crc32c(data):
    crc = 0xFFFFFFFF
    for b in data:
        crc ^= b
        for _ in range(8):
            crc = (crc >> 1) ^ (0x82F63B78 & -(crc & 1))
    return crc ^ 0xFFFFFFFF


def _masked(data):
    c = _crc32c(data)
    return (((c >> 15) | (c << 17)) + 0xA282EAD8) & 0xFFFFFFFF


def read_records(path):
    """The data of every TFRecord of a file, with both checksums verified."""
    out = []
    raw = open(path, "rb").read()
    pos = 0
    while pos < len(raw):
        hdr = raw[pos:pos + 8]
        (n,) = struct.unpack("<Q", hdr)
        (lcrc,) = struct.unpack("<I", raw[pos + 8:pos + 12])
        assert lcrc == _masked(hdr), "length checksum"
        data = raw[pos + 12:pos + 12 + n]
        (dcrc,) = struct.unpack("<I", raw[pos + 12 + n:pos + 16 + n])
        assert dcrc == _masked(data), "data checksum"
        out.append(data)
        pos += 16 + n
    return out


def _f64(b):
    return struct.unpack("<d", b)[0]


def _packed_f64(b):
    return list(np.frombuffer(b, "<f8").astype(np.float64))


def read_events(path):
    """[dict(wall_time, step, file_version, scalars {tag: float32}, histograms {tag: dict})] of an event file."""
    from cape_b200.tf_checkpoint import _parse_proto
    events = []
    for rec in read_records(path):
        p = _parse_proto(rec)
        ev = dict(wall_time=_f64(p[1][0]), step=p.get(2, [0])[0], file_version=p[3][0].decode() if 3 in p else None,
                  scalars={}, histograms={}, tags=[])
        for summ in p.get(5, []):
            for v in _parse_proto(summ).get(1, []):
                vp = _parse_proto(v)
                tag = vp[1][0].decode()
                ev["tags"].append(tag)
                if 2 in vp:
                    ev["scalars"][tag] = np.frombuffer(vp[2][0], "<f4")[0]
                if 5 in vp:
                    hp = _parse_proto(vp[5][0])
                    ev["histograms"][tag] = dict(
                        min=_f64(hp[1][0]), max=_f64(hp[2][0]), num=_f64(hp[3][0]), sum=_f64(hp[4][0]),
                        sum_squares=_f64(hp[5][0]), bucket_limit=_packed_f64(hp[6][0]), bucket=_packed_f64(hp[7][0]))
        events.append(ev)
    return events
