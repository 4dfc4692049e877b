"""Training and synthesis summaries: TensorBoard event files as TF 1.2's ``tf.summary.FileWriter`` writes them, without
TensorFlow (reference: train.py:41,64-75,92-103, test.py:33,59-69, models/tacotron.py:129,139,152,162-164,181).

File and record format, restated from TensorFlow's ``core/util/events_writer`` and ``core/lib/io/record_writer``:
  ``<logdir>/events.out.tfevents.<%010d seconds>.<hostname>``; every record is
  ``uint64 length | masked crc32c(length) | Event | masked crc32c(Event)`` (little-endian; the CRC-32C and its masking are
  tf_checkpoint's); the first event carries ``file_version = "brain.Event:2"``.
  Event{1 wall_time double, 2 step int64, 3 file_version string, 5 summary}, Summary{1 repeated Value},
  Value{1 tag, 2 simple_value float, 4 image, 5 histo, 6 audio}, HistogramProto{1 min, 2 max, 3 num, 4 sum,
  5 sum_squares, 6 bucket_limit (packed double), 7 bucket (packed double)}, Image{1 height, 2 width, 3 colorspace,
  4 encoded_image_string}, Audio{1 sample_rate float, 2 num_channels, 3 length_frames, 4 encoded_audio_string,
  5 content_type}.  Fields holding their proto3 default are omitted, as the C++ serialiser does.

Histograms are TF 1.2's ``histogram::Histogram`` over the default bucket table (``histogram_limits``), binned on the GPU by
``kernels.histogram`` and encoded as ``EncodeToProto(preserve_zero_buckets=false)``: a run of empty buckets collapses into
one entry carrying the run's last limit and count 0.

Restated without a TensorFlow or matplotlib to pin against (the tests pin the restatement):
  - tags: ``clean_tag`` and the name-scope uniquification of TF 1.2's ``summary.py`` / ``Graph.unique_name``;
  - audio: TF's ``EncodeAudioAsS16LEWav``, ``clamp(roundf(x * 32768), -32768, 32767)`` as 16-bit PCM;
  - image: the heat map of ``imshow(alignments, cmap='hot')`` (rows = decoder steps from the top, columns = encoder
    positions, linear min..max normalisation, matplotlib's 256-entry ``hot`` map from its published segment data),
    enlarged by an integer nearest-neighbour factor until the longer side is at least 480 px.  The figure around it (axes,
    labels, the 640x480 canvas) is not reproduced.
Deviation: a NaN or Inf in a histogrammed tensor makes the reference's step fail (``InvalidArgument: Nan in summary
histogram``); here that histogram is skipped with one logged line and training continues.
"""
from __future__ import annotations

import os
import re
import socket
import struct
import time
import zlib

import numpy as np

from .tf_checkpoint import _field, _put_varint, crc32c, mask_crc

HISTOGRAM_TAGS = ("encoder/pre_net_out", "decoder/seq2seq_output", "post-process/output")     # tacotron.py:129,139,152
SCALAR_TAGS = ("seq2seq_loss", "output_loss", "loss", "cap_grads/global_gradient_norm")       # :162-164, :181
GUIDED_ATTENTION_TAG = "guided_attention_loss"         # (new) Config.guided_attention > 0: the guided attention loss


# ---------------------------------------------------------------------------------------------------------------------
# TF's default histogram buckets and its tag rules
# ---------------------------------------------------------------------------------------------------------------------
def histogram_limits():
    """float64 [1551]: histogram::InitDefaultBuckets -- v = 1e-12; while v < 1e20: push v; v *= 1.1 (repeated
    multiplication), then DBL_MAX; the mirrored negatives first and 0.0 between"""
    pos = []
    v = 1.0e-12
    while v < 1.0e20:
        pos.append(v)
        v *= 1.1
    pos.append(np.finfo(np.float64).max)
    pos = np.array(pos, dtype=np.float64)
    return np.concatenate([-pos[::-1], [0.0], pos])


_INVALID_TAG_CHARACTERS = re.compile(r"[^-/\w.]")


def clean_tag(name):
    """TF 1.2 summary.py _clean_tag: characters outside [-/\\w.] become '_', leading '/' are stripped"""
    return _INVALID_TAG_CHARACTERS.sub("_", name).lstrip("/")


class NameScopes:
    """the names ``tf.name_scope`` hands out in one graph (Graph.unique_name): a name used before gets _1, _2, ..."""

    def __init__(self):
        self._used = {}

    def unique(self, name):
        i = self._used.get(name, 0)
        self._used[name] = i + 1
        if i == 0:
            return name
        base = name
        while name in self._used:
            name = f"{base}_{i}"
            i += 1
        self._used[name] = 1
        return name


# ---------------------------------------------------------------------------------------------------------------------
# protobuf encoding
# ---------------------------------------------------------------------------------------------------------------------
def _len_field(num, payload):
    return _field(num, 2, _put_varint(len(payload)) + payload)


def _double_field(num, v):
    b = struct.pack("<d", v)
    return b"" if b == b"\x00" * 8 else _field(num, 1, b)


def _float_field(num, v):
    b = struct.pack("<f", v)
    return b"" if b == b"\x00" * 4 else _field(num, 5, b)


def _int_field(num, v):
    return b"" if v == 0 else _field(num, 0, _put_varint(int(v) & ((1 << 64) - 1)))


def histogram_proto(counts, limits, mn, mx, total, s, sq):
    """HistogramProto bytes as Histogram::EncodeToProto(preserve_zero_buckets=false) writes them"""
    counts = np.asarray(counts, dtype=np.float64)
    # an entry for every nonzero bucket and for the last bucket of every run of empty ones
    empty = counts <= 0
    keep = ~empty
    keep[:-1] |= empty[:-1] & ~empty[1:]
    keep[-1] = True
    bl, bc = np.asarray(limits, dtype=np.float64)[keep], counts[keep]
    return (_double_field(1, mn) + _double_field(2, mx) + _double_field(3, total) + _double_field(4, s) + _double_field(5, sq)
            + _len_field(6, bl.astype("<f8").tobytes()) + _len_field(7, bc.astype("<f8").tobytes()))


def scalar_value(tag, v):
    return _len_field(1, tag.encode("utf-8")) + _float_field(2, float(np.float32(v)))


def histo_value(tag, hproto):
    return _len_field(1, tag.encode("utf-8")) + _len_field(5, hproto)


def audio_value(tag, wave, sr):
    """Summary.Value with Audio{sample_rate, 1 channel, length_frames, 16-bit PCM WAV, "audio/wav"}"""
    wave = np.asarray(wave, dtype=np.float32).reshape(-1)
    msg = (_float_field(1, float(sr)) + _int_field(2, 1) + _int_field(3, len(wave)) + _len_field(4, wav_bytes(wave, sr))
           + _len_field(5, b"audio/wav"))
    return _len_field(1, tag.encode("utf-8")) + _len_field(6, msg)


def image_value(tag, rgba):
    """Summary.Value with Image{height, width, colorspace 4 (RGBA), PNG}"""
    h, w, _ = rgba.shape
    msg = _int_field(1, h) + _int_field(2, w) + _int_field(3, 4) + _len_field(4, png_bytes(rgba))
    return _len_field(1, tag.encode("utf-8")) + _len_field(4, msg)


# ---------------------------------------------------------------------------------------------------------------------
# WAV and PNG encoders
# ---------------------------------------------------------------------------------------------------------------------
def wav_samples(wave):
    """int16 samples of EncodeAudioAsS16LEWav: clamp(roundf(x * 32768), -32768, 32767), roundf = half away from zero"""
    y = (np.asarray(wave, dtype=np.float32) * np.float32(32768.0)).astype(np.float64)
    y = np.sign(y) * np.floor(np.abs(y) + 0.5)
    return np.clip(y, -32768, 32767).astype("<i2")


def wav_bytes(wave, sr):
    data = wav_samples(wave).tobytes()
    fmt = struct.pack("<HHIIHH", 1, 1, int(sr), int(sr) * 2, 2, 16)
    return (b"RIFF" + struct.pack("<I", 36 + len(data)) + b"WAVE" + b"fmt " + struct.pack("<I", 16) + fmt + b"data"
            + struct.pack("<I", len(data)) + data)


def png_bytes(rgba):
    """8-bit RGBA PNG, one IDAT, filter type 0 on every row"""
    rgba = np.ascontiguousarray(rgba, dtype=np.uint8)
    h, w, c = rgba.shape
    assert c == 4
    raw = np.concatenate([np.zeros((h, 1), dtype=np.uint8), rgba.reshape(h, w * 4)], axis=1).tobytes()

    def chunk(kind, data):
        return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data) & 0xffffffff)
    return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 6, 0, 0, 0)) + chunk(b"IDAT", zlib.compress(raw))
            + chunk(b"IEND", b""))


# matplotlib's `hot` (_cm.py _hot_data): (x, y0, y1) per channel
_HOT = {"red": ((0.0, 0.0416, 0.0416), (0.365079, 1.0, 1.0), (1.0, 1.0, 1.0)),
        "green": ((0.0, 0.0, 0.0), (0.365079, 0.0, 0.0), (0.746032, 1.0, 1.0), (1.0, 1.0, 1.0)),
        "blue": ((0.0, 0.0, 0.0), (0.746032, 0.0, 0.0), (1.0, 1.0, 1.0))}


def _segment_lut(seg, N=256):
    """colors._create_lookup_table: linear interpolation of the segment data at x = i/(N-1)"""
    a = np.asarray(seg, dtype=np.float64)
    x, y0, y1 = a[:, 0] * (N - 1), a[:, 1], a[:, 2]
    xind = np.arange(N, dtype=np.float64)
    ind = np.searchsorted(x, xind)[1:-1]
    dist = (xind[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
    lut = np.concatenate([[y1[0]], dist * (y0[ind] - y1[ind - 1]) + y1[ind - 1], [y0[-1]]])
    return np.clip(lut, 0.0, 1.0)


HOT_LUT = (np.stack([_segment_lut(_HOT[c]) for c in ("red", "green", "blue")] + [np.ones(256)], axis=1) * 255).astype(np.uint8)


def attention_rgba(alignment, min_side=480):
    """uint8 [H*f, W*f, 4]: alignment [decoder steps, encoder positions] normalised to its min..max, coloured with `hot`,
    enlarged by the smallest integer f that makes the longer side at least min_side"""
    a = np.asarray(alignment, dtype=np.float32)
    lo, hi = a.min(), a.max()
    v = (a - lo) / (hi - lo) if hi > lo else np.zeros_like(a)
    idx = (v * np.float32(256)).astype(np.int64)
    idx = np.clip(idx, 0, 255)
    img = HOT_LUT[idx]
    f = max(1, -(-min_side // max(a.shape)))
    return np.repeat(np.repeat(img, f, axis=0), f, axis=1)


# ---------------------------------------------------------------------------------------------------------------------
# the event file
# ---------------------------------------------------------------------------------------------------------------------
def _event(wall_time, step=0, summary_values=None, file_version=None):
    msg = _double_field(1, wall_time) + _int_field(2, step)
    if file_version is not None:
        msg += _len_field(3, file_version.encode("utf-8"))
    if summary_values is not None:
        msg += _len_field(5, b"".join(_len_field(1, v) for v in summary_values))
    return msg


def _record(data):
    n = struct.pack("<Q", len(data))
    return n + struct.pack("<I", mask_crc(crc32c(n))) + data + struct.pack("<I", mask_crc(crc32c(data)))


class EventWriter:
    """``<logdir>/events.out.tfevents.<seconds>.<hostname>``; ``add(step, values)`` appends one Event whose Summary holds
    the encoded Summary.Values"""

    def __init__(self, logdir):
        os.makedirs(logdir, exist_ok=True)
        now = time.time()
        self.path = os.path.join(logdir, "events.out.tfevents.%010d.%s" % (int(now), socket.gethostname()))
        self._f = open(self.path, "wb")
        self._f.write(_record(_event(now, file_version="brain.Event:2")))

    def add(self, step, values):
        self._f.write(_record(_event(time.time(), step, values)))

    def flush(self):
        self._f.flush()

    def close(self):
        if not self._f.closed:
            self._f.close()


def histogram_values(res, limits, log=print):
    """Summary.Values of the rows of ``res`` (kernels.histogram results, int64 [3, nlim + 5] on the host) under
    HISTOGRAM_TAGS; a histogram of a tensor with NaN / Inf is skipped and logged"""
    nlim = len(limits)
    out = []
    for tag, r in zip(HISTOGRAM_TAGS, res):
        if r[nlim] > 0:
            log(f"Nan in summary histogram for: {tag}")
            continue
        counts = r[:nlim]
        mn, mx, s, sq = r[nlim + 1:nlim + 5].view(np.float64)
        out.append(histo_value(tag, histogram_proto(counts, limits, mn, mx, float(counts.sum()), s, sq)))
    return out


class TrainSummaries:
    """The reference's per-step ``model.merged`` on the training stream, without a host sync of its own.

    ``enqueue`` (after the step's update, before its one host sync) bins the three histogrammed tensors with
    ``kernels.histogram`` and queues copies of their results and of the four scalars into pinned buffers; ``collect``
    (after the sync) takes them; ``write_pending`` encodes them -- the driver calls it once the NEXT step is enqueued, so the
    encoding and the CRCs run while the GPU computes.  guided_attention=True adds the scalar GUIDED_ATTENTION_TAG, the
    fourth loss ``enqueue`` then takes."""

    def __init__(self, logdir, device, log=print, guided_attention=False):
        import torch
        self.writer = EventWriter(logdir)
        self.limits = histogram_limits()
        self.limits_d = torch.from_numpy(self.limits).to(device)
        self.res = torch.empty((len(HISTOGRAM_TAGS), len(self.limits) + 5), dtype=torch.int64, device=device)
        self.res_h = torch.empty(self.res.shape, dtype=torch.int64, pin_memory=True)
        self.guided_attention = bool(guided_attention)
        self.scal_h = torch.empty(len(SCALAR_TAGS) + self.guided_attention, dtype=torch.float32, pin_memory=True)
        self.log = log
        self._queued = None
        self._pending = []

    def enqueue(self, step, tensors, losses, grad_sumsq):
        """tensors: the pre-net output, seq2seq_output and output; losses: device [loss, seq2seq loss, output loss] (and the
        guided attention loss fourth, when the summaries were built with guided_attention=True)"""
        from . import kernels as K
        if len(losses) != 3 + self.guided_attention:
            raise ValueError(f"TrainSummaries.enqueue: {len(losses)} losses, expected {3 + self.guided_attention}")
        for i, t in enumerate(tensors):
            K.histogram(self.res[i], t, self.limits_d)
        self.res_h.copy_(self.res, non_blocking=True)
        self.scal_h[:3].copy_(losses[:3], non_blocking=True)
        self.scal_h[3:4].copy_(grad_sumsq.reshape(1), non_blocking=True)
        if self.guided_attention:
            self.scal_h[4:].copy_(losses[3:], non_blocking=True)
        self._queued = step

    def collect(self):
        if self._queued is not None:
            self._pending.append((self._queued, self.res_h.numpy().copy(), self.scal_h.numpy().copy()))
            self._queued = None

    def write_pending(self):
        for step, res, scal in self._pending:
            vals = histogram_values(res, self.limits, self.log)
            norm = np.sqrt(np.float32(scal[3]))                              # tf.global_norm, before clipping
            vals += [scalar_value(t, v) for t, v in zip(SCALAR_TAGS, (scal[1], scal[2], scal[0], norm))]
            if self.guided_attention:
                vals.append(scalar_value(GUIDED_ATTENTION_TAG, scal[4]))
            self.writer.add(step, vals)
        self._pending = []

    def save_step(self, step, ideal, sample, alignment, sr):
        """train.py:92-103: the two clips and the attention image of a save step; everything logged so far is flushed"""
        self.write_pending()
        self.writer.add(step, [audio_value(f"ideal_{step}/audio/0", ideal, sr), audio_value(f"sample_{step}/audio/0", sample, sr),
                               image_value(f"attention_{step}/image/0", attention_rgba(alignment))])
        self.writer.flush()

    def close(self):
        self.collect()
        self.write_pending()
        self.writer.close()
