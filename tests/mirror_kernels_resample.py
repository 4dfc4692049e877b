"""TEST INFRASTRUCTURE ONLY -- tests/mirror_kernels_features.py plus a torch-CPU restatement of taco_resample
(csrc/resample.cu) with the entry point's arguments.  This module is the kernel namespace `K` that
tacotron_b200/audio.py::process_audio_batch(rates=...) and resample_batch run over on CPU; the docstring is the
specification of the CUDA kernel."""
from __future__ import annotations

import torch

from tests.mirror_kernels_features import *   # noqa: F401,F403  (trim_bounds, feature_frames, feature_spec, rfft2048, ...)

TABLE = 512


def resample(out, y, in_off, out_off, win_delta, step, ratio, treg):
    """out[out_off[b] : out_off[b+1]] = resampy's kaiser_best loop over y[in_off[b] : in_off[b+1]] (n_in samples) for
    t < n_out = int(n_in*ratio), zeros after.  scale = min(1, ratio); at t: n = int(treg[t]), frac = scale*(treg[t]-n),
    idx = frac*512, off = int(idx), eta = idx-off; left taps i < min(n+1, (nwin-off)//step) add
    (win[off+i*step] + eta*delta[off+i*step]) * x[n-i]; then frac = scale-frac and the right taps
    k < min(n_in-n-1, (nwin-off)//step) add the same with x[n+1+k].  Weights and products float64, the running sum
    rounded to float32 after every add, left wing first.  Vectorised over t; each output's taps stay in order."""
    win, delta = win_delta[:, 0], win_delta[:, 1]
    nwin = win_delta.shape[0]
    scale = min(1.0, ratio)
    io, oo = in_off.tolist(), out_off.tolist()
    for b in range(len(io) - 1):
        n_in, n_fix = io[b + 1] - io[b], oo[b + 1] - oo[b]
        n_out = int(n_in * ratio)
        x = y[io[b]:io[b + 1]].double()
        tr = treg[:n_out].double()
        n = tr.to(torch.int64)
        frac = scale * (tr - n.double())
        acc = torch.zeros(n_out, dtype=torch.float32)

        def wing(frac, limit, src):
            nonlocal acc
            idx = frac * TABLE
            off = idx.to(torch.int64)
            eta = idx - off.double()
            count = torch.minimum(limit, torch.div(nwin - off, step, rounding_mode="floor"))
            for i in range(int(count.max()) if n_out else 0):
                m = i < count
                o = torch.where(m, off + i * step, torch.zeros_like(off))
                w = win[o] + eta * delta[o]
                s = (acc.double() + w * x[torch.where(m, src(i), torch.zeros_like(n))]).float()
                acc = torch.where(m, s, acc)

        wing(frac, n + 1, lambda i: n - i)
        wing(scale - frac, n_in - n - 1, lambda i: n + 1 + i)
        out[oo[b]:oo[b] + n_out] = acc
        out[oo[b] + n_out:oo[b + 1]] = 0.0
