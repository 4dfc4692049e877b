"""TEST INFRASTRUCTURE ONLY -- tests/mirror_kernels.py plus torch-CPU restatements of the feature-extraction entry points
(taco_trim_bounds, taco_feature_frames, taco_feature_spec; csrc/features.cu).  This module is the kernel namespace `K` that
tacotron_b200/audio.py::process_audio_batch runs over on CPU; the docstrings are the specification of the CUDA kernels of
the same names."""
from __future__ import annotations

import numpy as np
import torch

from tests.mirror_kernels import *            # noqa: F401,F403  (rfft2048 and the rest of the namespace, unchanged)
from tests.mirror_kernels import _hann_padded
from tacotron_b200.audio import reshape_frames


def trim_bounds(bounds, y, offsets, frame_length, hop, top_db):
    """bounds[b] = librosa.effects.trim's span of y[offsets[b]:offsets[b+1]]: frame f < 1 + len//hop of the signal
    reflect-padded by frame_length//2 has energy e_f = mean of its squares (fp64); non-silent frames have
    10 log10(max(1e-10, e_f)) - 10 log10(max(1e-10, max e)) > -top_db; bounds = [first*hop, min(len, (last+1)*hop)),
    [0, 0) if none."""
    off = offsets.tolist()
    for b in range(len(off) - 1):
        x = y[off[b]:off[b + 1]].double().numpy()
        xp = np.pad(x, frame_length // 2, mode="reflect")
        nf = 1 + len(x) // hop
        e = np.array([np.mean(xp[f * hop:f * hop + frame_length] ** 2) for f in range(nf)])
        db = 10.0 * np.log10(np.maximum(1e-10, e)) - 10.0 * np.log10(max(1e-10, e.max()))
        nz = np.flatnonzero(db > -top_db)
        bounds[b] = torch.tensor([nz[0] * hop, min(len(x), (nz[-1] + 1) * hop)] if nz.size else [0, 0], dtype=bounds.dtype)


def feature_frames(frw, y, start, length, max_len, hop, win_length, preemph):
    """frw[b, t, j] = w[j] * e_pad[t*hop + j]: w_b = y[start[b]:start[b]+length[b]] zero-padded to max_len, pre-emphasised
    in float32 (e[0] = w[0], e[i] = f32(w[i] - f32(preemph*w[i-1]))), reflect-padded by n_fft//2; hann window."""
    B, n, n_fft = frw.shape
    win = _hann_padded(win_length, n_fft, frw.dtype)
    for b in range(B):
        s, L = int(start[b]), int(length[b])
        w = torch.zeros(max_len, dtype=torch.float32)
        w[:L] = y[s:s + L]
        e = w.clone()
        e[1:] = w[1:] - w[:-1] * torch.tensor(preemph, dtype=torch.float32)
        ep = torch.nn.functional.pad(e.to(frw.dtype)[None, None], (n_fft // 2, n_fft // 2), mode="reflect")[0, 0]
        for t in range(n):
            frw[b, t] = ep[t * hop:t * hop + n_fft] * win


def feature_spec(stft_out, mel_out, X, basis, lo, hi, r):
    """stft = log(|X| + 1e-8), mel = log(|basis[:, lo:hi] . X| + 1e-8) (the complex spectrum, melspectrogram(S=stft)),
    each in the reshape_frames(forward=True) layout [B, 4*(n//4r), F*r], cast to the output dtype."""
    B = X.shape[0]
    rdt = torch.float64 if X.dtype == torch.complex128 else torch.float32
    Wm = torch.zeros(basis.shape, dtype=rdt)
    for m in range(basis.shape[0]):
        Wm[m, lo[m]:hi[m]] = basis[m, lo[m]:hi[m]].to(rdt)
    for b in range(B):
        Xb = X[b].t()                                                            # [F, n]
        s = torch.log(Xb.abs() + 1e-8)
        m = torch.log((Wm.to(X.dtype) @ Xb).abs() + 1e-8)
        stft_out[b] = reshape_frames(s, r, forward=True).to(stft_out.dtype)
        mel_out[b] = reshape_frames(m, r, forward=True).to(mel_out.dtype)
