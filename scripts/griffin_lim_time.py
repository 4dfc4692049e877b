"""Cost and convergence of fast Griffin-Lim (momentum) and the cost of de-emphasis on the GPU.

    python scripts/griffin_lim_time.py [--rounds 8] [--out griffin_lim_time.json]

  per_iteration  GriffinLimGraph at the synthesis batch shape (B = 32, T = 180, r = 2) and the C5 shape (B = 1, T = 100,
                 r = 5): plain against momentum 0.99, each graph captured for 50 iterations and for 0, so the difference
                 over 50 is the time of one iteration;
  convergence    whole inversions (audio.invert_spectrogram, eager) of a batch of 32 copies of the voiced test signal
                 (tests/griffin_lim_oracle.py voiced_signal, r = 2) with the spectral convergence each reaches: plain 50,
                 momentum 0.99 at 25, 32 and 50 iterations;
  de_emphasis    the kernel on 32 x 108000 samples (one segment per row) and on one 10-minute line at 16 kHz, and the
                 peak of the de-emphasised inversions of the test signal against its clean peak (0.5).
Timed with CUDA events, the variants alternated in blocks (the order reversed every other round); medians and min / max
over rounds.  The card's name, power limit and max SM clock are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import audio_oracle as A  # noqa: E402
from tacotron_b200 import audio  # noqa: E402
from tests import griffin_lim_oracle as G  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def alternate(arms, rounds, reps):
    for fn in arms.values():                                   # warm-up: module loads, allocator
        fn()
    t = {k: [] for k in arms}
    for i in range(rounds):
        for k in (list(arms) if i % 2 == 0 else list(arms)[::-1]):
            t[k].append(timed(arms[k], reps))
    return {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))} for k, v in t.items()}


def per_iteration(name, B, T, r, rounds):
    g = torch.Generator().manual_seed(0)
    spec = (torch.randn(B, T, 1025 * r, generator=g) * 0.5).cuda()
    arms = {}
    for m in (0.0, 0.99):
        for n_iter in (0, 50):
            glg = audio.GriffinLimGraph(B, T, r, n_iter=n_iter, momentum=m)
            arms[f"m{m}_it{n_iter}"] = (lambda glg=glg: glg(spec))
    t = alternate(arms, rounds, 5)
    n = 4 * r * (T // 4)
    res = {"shape": name, "B": B, "T": T, "r": r, "frames": B * n, "graphs_ms": t}
    for m in (0.0, 0.99):
        res[f"iteration_ms_m{m}"] = (t[f"m{m}_it50"]["median"] - t[f"m{m}_it0"]["median"]) / 50
    res["momentum_extra_per_iteration_ms"] = res["iteration_ms_m0.99"] - res["iteration_ms_m0.0"]
    res["momentum_extra_read_MB"] = B * n * 1025 * 8 / 1e6              # the previous iterate, read once per iteration
    return res


def convergence(rounds):
    B, r = 32, 2
    _, y0, u = G.voiced_signal(r)
    mag = np.abs(A.stft(y0))
    spec1 = audio.reshape_frames(torch.from_numpy(np.log(np.maximum(mag, 1e-30))).float(), r, forward=True)[None]
    spec = spec1.expand(B, -1, -1).contiguous().cuda()
    pu = torch.from_numpy(u.T.copy()).float()[None].expand(B, -1, -1).contiguous().cuda()
    variants = {"plain_50": (50, 0.0), "momentum_25": (25, 0.99), "momentum_32": (32, 0.99), "momentum_50": (50, 0.99)}
    arms = {k: (lambda n=n, m=m: audio.invert_spectrogram(spec, r, n_iter=n, phase_u=pu, momentum=m))
            for k, (n, m) in variants.items()}
    t = alternate(arms, rounds, 2)
    res = {"B": B, "r": r, "frames_per_utterance": mag.shape[1]}
    for k, (n, m) in variants.items():
        y = audio.invert_spectrogram(spec, r, n_iter=n, phase_u=pu, momentum=m)
        de = audio.de_emphasis(y.clone())
        torch.cuda.synchronize()
        res[k] = {"n_iter": n, "momentum": m, "ms": t[k],
                  "spectral_convergence": float(G.spectral_convergence(y[0].cpu().double().numpy(), mag)),
                  "peak": float(y[0].abs().max()), "peak_de_emphasised": float(de[0].abs().max())}
    return res


def de_emphasis(rounds):
    rows = torch.randn(32, 108000, device="cuda") * 0.1
    line = torch.randn(16000 * 600, device="cuda") * 0.1
    start_rows = np.arange(33, dtype=np.int64) * 108000
    start_line = np.array([0, line.numel()], dtype=np.int64)
    # (the buffers are filtered again and again in place and grow toward inf: the kernel's time does not depend on the values)
    t = alternate({"rows_32x108000": lambda: audio.de_emphasis(rows, start_rows),
                   "line_10min": lambda: audio.de_emphasis(line, start_line)}, rounds, 20)
    return {"ms": t, "bytes_MB": {"rows_32x108000": 32 * 108000 * 8 / 1e6, "line_10min": line.numel() * 8 / 1e6}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("griffin_lim_time.py needs a CUDA device")
    out = {"card": card(),
           "per_iteration": [per_iteration("synthesis", 32, 180, 2, a.rounds), per_iteration("C5", 1, 100, 5, a.rounds)],
           "convergence": convergence(a.rounds), "de_emphasis": de_emphasis(a.rounds)}
    print(json.dumps(out, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
