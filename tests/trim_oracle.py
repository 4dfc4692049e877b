"""TEST INFRASTRUCTURE ONLY -- float64 numpy statement of where an utterance's speech ends (taco_speech_frames,
include/taco_b200.h), and the synthetic spectrograms the trim tests and scripts/trim_time.py use."""
from __future__ import annotations

import numpy as np

LN10_OVER_10 = np.log(10.0) / 10.0
PAD_LOG = np.log(1e-8)                  # log(|X| + 1e-8) of a zero-padded frame (features.cu feature_spec)


def frame_space(spec_b, r):
    """spec_b [T, F*r] -> v [n, F] in gl_init's frame order: frame 4r*q + 4c + l = decoder step 4q + l, column block c"""
    T, W = spec_b.shape
    F, nb = W // r, T // 4
    return spec_b[:nb * 4].reshape(nb, 4, r, F).transpose(0, 2, 1, 3).reshape(nb * 4 * r, F)


def log_power(spec, r, scale=None, shift=None):
    """e [B, n] = log sum_k exp(2 v[f, k]) in float64, max-shifted; non-finite where the kernel's is"""
    spec = np.asarray(spec, dtype=np.float64)
    out = []
    with np.errstate(all="ignore"):
        for sb in spec:
            if scale is not None:
                sb = sb * np.asarray(scale, np.float64) + np.asarray(shift, np.float64)
            x = 2.0 * frame_space(sb, r)
            m = np.max(x, axis=1, keepdims=True)
            out.append(m[:, 0] + np.log(np.sum(np.exp(x - m), axis=1)))
    return np.stack(out)


def speech_frames(spec, r, scale=None, shift=None, top_db=60.0):
    """frames [B] int64: 4r * clamp(ceil((f*+1)/4r), ceil(5/4r), T/4), f* the last frame with e >= max e - top_db ln10/10;
    n = 4r*(T/4) when any e is not finite"""
    T = np.asarray(spec).shape[1]
    blk, n = 4 * r, 4 * r * (T // 4)
    e = log_power(spec, r, scale, shift)
    out = np.empty(len(e), dtype=np.int64)
    for b, eb in enumerate(e):
        if not np.all(np.isfinite(eb)):
            out[b] = n
            continue
        last = int(np.flatnonzero(eb >= eb.max() - top_db * LN10_OVER_10)[-1])
        out[b] = blk * min(max(-(-(last + 1) // blk), -(-5 // blk)), T // 4)
    return out


def margin_db(spec, r, scale=None, shift=None, top_db=60.0):
    """smallest distance, in dB, of a finite utterance's frame powers from its threshold"""
    e = log_power(spec, r, scale, shift)
    gaps = [np.abs(eb - (eb.max() - top_db * LN10_OVER_10)).min() / LN10_OVER_10 for eb in e if np.all(np.isfinite(eb))]
    return min(gaps) if gaps else np.inf


def speech_like(B, T, r, ends, seed=0, scale=None, shift=None):
    """spec float32 [B, T, 1025*r] whose frames [0, ends[b]) are a smooth speech-like log magnitude (powers within
    ~10 dB of each other) and whose later frames hold the padding value log(1e-8) -- normalised by (scale, shift)
    when given, as the model's output is -- so every tail frame lies more than 100 dB below the speech."""
    rng = np.random.RandomState(seed)
    n = 4 * r * (T // 4)
    k = np.linspace(0, 1, 1025)[None, :]
    out = np.empty((B, T, 1025 * r), dtype=np.float32)
    for b in range(B):
        t = np.linspace(0, 1, n)[:, None]
        logmag = -3.0 * k + 0.8 * np.sin(2 * np.pi * (3 * t + 8 * k + rng.rand())) + 0.5 * rng.rand(n, 1) - 1.0
        logmag[ends[b]:] = PAD_LOG
        s = np.zeros((T, 1025 * r))
        nb = T // 4
        s[:nb * 4] = logmag.reshape(nb, r, 4, 1025).transpose(0, 2, 1, 3).reshape(nb * 4, r * 1025)
        s[nb * 4:] = PAD_LOG
        if scale is not None:
            s = (s - shift) / scale
        out[b] = s
    return out
