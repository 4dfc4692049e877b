"""TEST INFRASTRUCTURE ONLY -- float64 numpy statements of taco_speech_bounds and taco_join_segments
(include/taco_b200.h), and of the sample range long-form synthesis keeps of each chunk."""
from __future__ import annotations

import numpy as np

from tests import trim_oracle as TO

HOP = 300


def speech_bounds(spec, r, scale=None, shift=None, top_db=60.0):
    """bounds [B, 3] int64: {first voiced frame, last voiced frame + 1, trim_oracle.speech_frames}, voiced = e >= max e -
    top_db ln10/10 in gl_init's frame space; {0, n, n} when any e is not finite"""
    T = np.asarray(spec).shape[1]
    blk, n = 4 * r, 4 * r * (T // 4)
    e = TO.log_power(spec, r, scale, shift)
    out = np.empty((len(e), 3), dtype=np.int64)
    for b, eb in enumerate(e):
        if not np.all(np.isfinite(eb)):
            out[b] = (0, n, n)
            continue
        v = np.flatnonzero(eb >= eb.max() - top_db * TO.LN10_OVER_10)
        out[b] = (v[0], v[-1] + 1, blk * min(max(-(-(v[-1] + 1) // blk), -(-5 // blk)), T // 4))
    return out


def speech_span_like(B, T, r, starts, ends, seed=0, scale=None, shift=None):
    """trim_oracle.speech_like with speech over frames [starts[b], ends[b]) only: the frames before starts[b] hold the
    padding value too"""
    spec = TO.speech_like(B, T, r, ends, seed=seed, scale=scale, shift=shift)
    blk = 4 * r
    for b in range(B):
        for f in range(starts[b]):
            t, c = 4 * (f // blk) + f % 4, (f % blk) // 4
            cols = slice(c * 1025, (c + 1) * 1025)
            pad = np.full(1025, TO.PAD_LOG)
            spec[b, t, cols] = pad if scale is None else (pad - shift[cols]) / scale[cols]
    return spec


def fade(length, fade_len):
    """w [length] float64: min(1, c(i), c(length-1-i)), c(j) = 0.5 - 0.5 cos(pi (j + 0.5) / fade_len) for j < fade_len"""
    def c(j):
        return np.where(j < fade_len, 0.5 - 0.5 * np.cos(np.pi * (j + 0.5) / fade_len), 1.0)
    i = np.arange(length, dtype=np.float64)
    return np.minimum(1.0, np.minimum(c(i), c(length - 1 - i)))


def join_segments(out, src, seg, fade_len):
    """out (float64, modified) [d + i] = src[a + i] * fade(len)[i] for every row {a, d, len} of seg"""
    src = np.asarray(src, dtype=np.float64)
    for a, d, n in np.asarray(seg, dtype=np.int64).reshape(-1, 3).tolist():
        out[d:d + n] = src[a:a + n] * fade(n, fade_len)
    return out


def kept_samples(f0, f1, frames, hop=HOP):
    """[max(hop (f0 - 1), 0), min(hop f1, L)), L = hop (frames - 1) the length of the chunk's Griffin-Lim output"""
    return max(hop * (f0 - 1), 0), min(hop * f1, hop * (frames - 1))
