"""TEST INFRASTRUCTURE ONLY -- torch-CPU restatement of taco_speech_frames and of the packed Griffin-Lim entry points
(csrc/audio.cu); the docstrings are the specification of the CUDA kernels.  The padded kernels and the FFTs are those of
tests/mirror_kernels.py, re-exported so that this module is a whole `K` for audio.invert_speech."""
from __future__ import annotations

import math

import torch

from tests.mirror_kernels import gl_frame, gl_init, gl_ola, gl_phase, irfft2048, rfft2048  # noqa: F401


def speech_frames(frames, spec, r, scale=None, shift=None, top_db=60.0):
    """frames int32 [B] of spec [B, T, F*r] in spec's dtype: in gl_init's frame space (n = 4r*(T/4) frames,
    v[f, k] = spec[b, t(f), c(f)*F + k]*scale + shift), e[f] = m + log sum_k exp(2v - m) with m = max_k 2v;
    E = max e; f* = the last f with e[f] >= E - top_db*ln(10)/10; frames[b] = 4r*clamp(ceil((f*+1)/4r), ceil(5/4r), T/4),
    or n when any e[f] is not finite."""
    B, T, W = spec.shape
    F, blk = W // r, 4 * r
    n = blk * (T // 4)
    f = torch.arange(n)
    q, rem = f // blk, f % blk
    t = 4 * q + rem % 4
    cols = (rem // 4)[:, None] * F + torch.arange(F)[None, :]
    v = spec[:, t[:, None], cols]                                             # [B, n, F]
    if scale is not None:
        v = v * scale[cols] + shift[cols]
    x = 2.0 * v
    m = torch.nan_to_num(x, nan=-math.inf, posinf=math.inf, neginf=-math.inf).amax(dim=2, keepdim=True)         # NaN does not take part in the max ...
    e = m[..., 0] + torch.log(torch.exp(x - m).sum(dim=2))                   # ... but makes the sum NaN
    for b in range(B):
        eb = e[b]
        if not bool(torch.isfinite(eb).all()):
            frames[b] = n
            continue
        last = int(torch.nonzero(eb >= eb.max() - top_db * (math.log(10.0) / 10.0)).max())
        frames[b] = blk * min(max(-(-(last + 1) // blk), -(-5 // blk)), T // 4)


def _rows(off, b):
    return int(off[b]), int(off[b + 1])


def gl_init_packed(full, mag, spec, phase_u, off, r, max_frames, scale=None, shift=None):
    """rows off[b]:off[b+1] of full / mag [N, F] = gl_init of utterance b alone (spec[b:b+1], phase_u's same rows)"""
    for b in range(off.numel() - 1):
        lo, hi = _rows(off, b)
        m = torch.empty((1, hi - lo, mag.shape[1]), dtype=mag.dtype)
        fu = torch.empty((1, hi - lo, mag.shape[1]), dtype=full.dtype)
        gl_init(fu, m, spec[b:b + 1], phase_u[lo:hi][None], r, scale, shift)
        mag[lo:hi], full[lo:hi] = m[0], fu[0]


def gl_ola_packed(y, fr, off, max_frames, hop, win_length):
    """y[hop*(off[b]-b) : + hop*(n_b-1)] = gl_ola of frames fr[off[b]:off[b+1]] alone"""
    for b in range(off.numel() - 1):
        lo, hi = _rows(off, b)
        yb = torch.empty((1, hop * (hi - lo - 1)), dtype=y.dtype)
        gl_ola(yb, fr[lo:hi][None], hop, win_length)
        y[hop * (lo - b):hop * (hi - b - 1)] = yb[0]


def gl_frame_packed(frw, y, off, max_frames, hop, win_length):
    """frw[off[b]:off[b+1]] = gl_frame of utterance b's samples y[hop*(off[b]-b) : + hop*(n_b-1)] alone"""
    for b in range(off.numel() - 1):
        lo, hi = _rows(off, b)
        fb = torch.empty((1, hi - lo, frw.shape[1]), dtype=frw.dtype)
        gl_frame(fb, y[hop * (lo - b):hop * (hi - b - 1)][None], hop, win_length)
        frw[lo:hi] = fb[0]
