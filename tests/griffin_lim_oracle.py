"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY.  float64 statements of the two opt-in synthesis options of
tacotron_b200.audio: fast Griffin-Lim (momentum) on oracle/audio_oracle's stft / istft, de-emphasis with
scipy.signal.lfilter, and the voiced test signal the convergence claims are checked on."""
from __future__ import annotations

import numpy as np
from scipy.signal import lfilter

from oracle import audio_oracle as A
from oracle.tf12 import reshape_frames

PRE_EMPHASIS = 0.97


def fast_griffinlim(magnitude, angles0, n_iter=50, momentum=0.0):
    """librosa >= 0.7's griffinlim loop with audio_oracle.griffinlim's zero-phase convention (angle(0) = 0):
    a = rebuilt - beta*rebuilt_prev, beta = momentum/(1+momentum), rebuilt_prev = 0 before the first iteration.
    momentum = 0 is audio_oracle.griffinlim, operation for operation."""
    beta = momentum / (1.0 + momentum)
    mag = np.abs(magnitude).astype(np.complex128)
    angles = angles0.astype(np.complex128)
    prev = None
    for _ in range(n_iter):
        rebuilt = A.stft(A.istft(mag * angles))
        a = rebuilt if beta == 0 or prev is None else rebuilt - beta * prev
        angles = np.exp(1j * np.angle(a))
        prev = rebuilt
    return A.istft(mag * angles)


def invert_spectrogram(spec, r, angles0, n_iter=50, momentum=0.0):
    """audio_oracle.invert_spectrogram with fast Griffin-Lim"""
    s = reshape_frames(spec, r, forward=False)
    return fast_griffinlim(np.exp(s.T), angles0, n_iter=n_iter, momentum=momentum)


def phase_momentum(mag, rebuilt, prev, beta):
    """taco_gl_phase_momentum in float64: mag * d/|d|, d = rebuilt - beta*prev, mag + 0i where d == 0"""
    d = rebuilt.astype(np.complex128) - beta * prev.astype(np.complex128)
    a = np.abs(d)
    out = mag.astype(np.complex128)
    nz = a > 0
    out[nz] = mag[nz] * d[nz] / a[nz]
    return out


def de_emphasis(x, start, coef=PRE_EMPHASIS):
    """y[i] = x[i] + coef*y[i-1] per segment [start[s], start[s+1]), zero state before each; samples outside every
    segment are left as they are"""
    y = np.array(x, dtype=np.float64)
    for a, b in zip(start[:-1], start[1:]):
        if b > a:
            y[a:b] = lfilter([1.0], [1.0, -coef], y[a:b])
    return y


def pre_emphasis(x, coef=PRE_EMPHASIS):
    """preprocessing's y[n] = x[n] - coef*x[n-1] (y[0] = x[0]), in float64"""
    x = np.asarray(x, dtype=np.float64)
    return np.append(x[0], x[1:] - coef * x[:-1])


def voiced_signal(r, sr=16000, seconds=3.0, seed=0):
    """The voiced, speech-like test signal -> (clean, y, u): clean the signal before pre-emphasis, y = pre_emphasis(clean)
    (what the model learns the spectrogram of), u uniform [0, 1) initial phases [1025, frames] for Griffin-Lim
    (angles0 = exp(2 pi i u)).
      - f0 = 120 + 40 sin(2 pi 0.7 t); harmonics k = 1..39 below Nyquist, weighted by Gaussian formants at 500, 1500 and
        2500 Hz (widths 300, 400, 500 Hz, weights 1, 0.5, 0.2);
      - voiced where sin(2 pi 1.5 t) > -0.3; plus 0.01 N(0, 1) noise; the whole scaled to a peak of 0.5, a recording's
        level (a global gain changes no convergence figure, and makes the peaks of a de-emphasised output meaningful);
        then pre-emphasis with 0.97;
      - cut to hop*(frames-1) samples, frames the largest multiple of 4r the 3 s hold, so the STFT has a frame count the
        decoder's layout can carry; the initial phases are uniform from the same generator (seed)."""
    rng = np.random.default_rng(seed)
    n = int(round(seconds * sr))
    frames = 1 + n // A.HOP_LENGTH
    frames -= frames % (4 * r)
    n = A.HOP_LENGTH * (frames - 1)
    t = np.arange(n) / sr
    f0 = 120.0 + 40.0 * np.sin(2 * np.pi * 0.7 * t)
    phase = 2 * np.pi * np.cumsum(f0) / sr
    x = np.zeros(n)
    for k in range(1, 40):
        fk = k * f0
        w = sum(g * np.exp(-0.5 * ((fk - fc) / bw) ** 2) for fc, bw, g in ((500, 300, 1.0), (1500, 400, 0.5), (2500, 500, 0.2)))
        x += np.where(fk < sr / 2, w * np.sin(k * phase), 0.0)
    x *= np.sin(2 * np.pi * 1.5 * t) > -0.3
    clean = x + 0.01 * rng.standard_normal(n)
    clean *= 0.5 / np.abs(clean).max()
    u = rng.random((A.N_FFT // 2 + 1, frames))
    return clean, pre_emphasis(clean), u


def spectral_convergence(y, mag):
    """|| |STFT(y)| - mag ||_F / ||mag||_F"""
    return np.linalg.norm(np.abs(A.stft(y)) - mag) / np.linalg.norm(mag)
