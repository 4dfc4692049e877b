"""Preprocessing cost on the GPU: a seeded in-memory corpus of 16 kHz utterances (lengths up to 108000 samples).

    python scripts/preprocess_time.py [--n 512] [--chunk 64] [--out preprocess_time.json]

Reports, for one chunk, each kernel's time (CUDA events, median over repeats) and the bytes it has to move (from shapes:
each operand read or written once), then PCM in host memory -> float16 arrays in pinned host memory per utterance
(process_audio_batch + D2H over the whole corpus, chunked as the driver does, disk excluded), the float64 oracle on the CPU
per utterance for scale, and the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tacotron_b200 import audio, kernels as K  # noqa: E402


def corpus(n, seed=0):
    rng = np.random.RandomState(seed)
    out = []
    for L in rng.randint(20000, 108001, size=n):
        head, tail = rng.randint(0, 4000), rng.randint(0, 4000)
        t = np.arange(L - head - tail) / 16000.0
        body = 0.2 * rng.randn(len(t)) * (0.6 + 0.4 * np.sin(2 * np.pi * 3 * t)) + 0.3 * np.sin(2 * np.pi * 220 * t)
        out.append(np.concatenate([rng.randn(head) * 3e-5, body, rng.randn(tail) * 3e-5]).astype(np.float32))
    return out


def event_time(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--chunk", type=int, default=64)
    ap.add_argument("--r", type=int, default=2)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    waves = corpus(a.n)
    r, B = a.r, a.chunk
    # ---- one chunk, kernel by kernel ----
    chunk = waves[:B]
    lens = np.array([len(w) for w in chunk], dtype=np.int64)
    offsets = np.concatenate([[0], np.cumsum(lens)])
    y = torch.from_numpy(np.concatenate(chunk)).cuda()
    off = torch.from_numpy(offsets).cuda()
    bounds = torch.empty(B, 2, dtype=torch.int32, device="cuda")
    K.trim_bounds(bounds, y, off, audio.TRIM_FRAME, audio.TRIM_HOP, audio.TRIM_TOP_DB)
    b = bounds.cpu().numpy().astype(np.int64)
    kl = np.minimum(b[:, 1] - b[:, 0], audio.maximum_audio_length)
    start = torch.from_numpy(offsets[:-1] + b[:, 0]).cuda()
    length = torch.from_numpy(kl.astype(np.int32)).cuda()
    n = audio.STFT_FRAMES
    T = audio.feature_frames_per_utterance(r)
    frw = torch.empty(B, n, audio.n_fft, device="cuda")
    X = torch.empty(B, n, audio.F_BINS, dtype=torch.complex64, device="cuda")
    stft = torch.empty(B, T, audio.F_BINS * r, dtype=torch.float16, device="cuda")
    mel = torch.empty(B, T, audio.N_MELS * r, dtype=torch.float16, device="cuda")
    basis, lo, hi = (torch.from_numpy(v).cuda() for v in audio.mel_basis())
    frames_b = B * n * audio.n_fft * 4
    spec_b = B * n * audio.F_BINS * 8
    kern = {
        "trim_bounds": (lambda: K.trim_bounds(bounds, y, off, audio.TRIM_FRAME, audio.TRIM_HOP, audio.TRIM_TOP_DB),
                        int(lens.sum()) * 4 + B * 8),
        "feature_frames": (lambda: K.feature_frames(frw, y, start, length, audio.maximum_audio_length, audio.hop_length,
                                                    audio.win_length, audio.PRE_EMPHASIS), int(kl.sum()) * 4 + frames_b),
        "rfft2048": (lambda: K.rfft2048(X, frw), frames_b + spec_b),
        "feature_spec": (lambda: K.feature_spec(stft, mel, X, basis, lo, hi, r),
                         spec_b + basis.numel() * 4 + (stft.numel() + mel.numel()) * 2),
    }
    res = {"card": card, "chunk": B, "r": r, "corpus_utterances": a.n, "kernels": {}}
    for name, (fn, nbytes) in kern.items():
        ms = event_time(fn, a.reps)
        res["kernels"][name] = {"ms": round(ms, 4), "MB": round(nbytes / 1e6, 2), "GB_per_s": round(nbytes / ms / 1e6, 1)}
    # ---- PCM in host memory -> float16 arrays in pinned host memory, whole corpus ----
    def run_corpus():
        kept = 0
        for i in range(0, len(waves), B):
            m, s, keep = audio.process_audio_batch(waves[i:i + B], r)
            mh = torch.empty(m.shape, dtype=m.dtype, pin_memory=True)
            sh = torch.empty(s.shape, dtype=s.dtype, pin_memory=True)
            mh.copy_(m, non_blocking=True); sh.copy_(s, non_blocking=True)
            kept += int(keep.sum())
        torch.cuda.synchronize()
        return kept
    run_corpus()                                                   # warm-up: module loads, allocator, mel basis upload
    times = []
    for _ in range(3):
        t0 = time.perf_counter()
        kept = run_corpus()
        times.append(time.perf_counter() - t0)
    res["end_to_end"] = {"utterances": a.n, "kept": kept, "s_median": round(float(np.median(times)), 4),
                         "ms_per_utterance": round(float(np.median(times)) * 1e3 / a.n, 4),
                         "output_MB_per_utterance": round((T * (audio.F_BINS + audio.N_MELS) * r * 2) / 1e6, 3)}
    # ---- the float64 oracle on the CPU, for scale ----
    from tests import feature_oracle as FO
    t0 = time.perf_counter()
    for w in waves[:4]:
        FO.features(w, r)
    res["cpu_oracle_ms_per_utterance"] = round((time.perf_counter() - t0) * 1e3 / 4, 1)
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
