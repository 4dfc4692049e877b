"""Resampling cost on the GPU: seeded in-memory corpora of speech-like utterances at 48 and 44.1 kHz.

    python scripts/resample_time.py [--n 256] [--chunk 64] [--out resample_time.json]

Reports taco_resample's time for one chunk at 48 -> 24 kHz and 44.1 -> 16 kHz (CUDA events, median over repeats) with
the taps it computes (from the lengths: left and right wing of every output sample), then PCM in host memory -> float16
arrays in pinned host memory per utterance (process_audio_batch + D2H over the whole corpus, chunked as the driver does,
disk excluded) for the same utterances with and without resampling (the latter fed the resampled waveforms at the target
rate), and the card's name, power limit and max SM clock read in the same run.
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


def corpus(n, sr, seed=0):
    """utterances of 1.25-4.5 s (at most 108000 samples at 24 kHz after resampling), quiet lead-in and tail"""
    rng = np.random.RandomState(seed)
    out = []
    for L in rng.randint(int(1.25 * sr), int(4.5 * sr) + 1, size=n):
        head, tail = rng.randint(0, sr // 4), rng.randint(0, sr // 4)
        t = np.arange(L - head - tail) / sr
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


def taps(lens, sr_orig, sr_new):
    """taps resampy's loop computes for these lengths (left + right wing of every output sample)"""
    ratio = float(sr_new) / sr_orig
    scale = min(1.0, ratio)
    step = int(scale * 512)
    total = 0
    for n_in in lens:
        n_out = audio.resample_lengths(n_in, sr_orig, sr_new)[0]
        tr = audio.resample_register(ratio, n_out)
        n = tr.astype(np.int64)
        frac = scale * (tr - n)
        for f, lim in ((frac, n + 1), (scale - frac, n_in - n - 1)):
            off = (f * 512).astype(np.int64)
            total += int(np.minimum(lim, (32769 - off) // step).sum())
    return total


def one_chunk(waves, sr_orig, sr_new, reps):
    lens = [len(w) for w in waves]
    ratio = float(sr_new) / sr_orig
    sizes = [audio.resample_lengths(n, sr_orig, sr_new) for n in lens]
    in_off = torch.tensor(np.concatenate([[0], np.cumsum(lens)])).cuda()
    out_off = torch.tensor(np.concatenate([[0], np.cumsum([s[1] for s in sizes])])).cuda()
    y = torch.from_numpy(np.concatenate(waves)).cuda()
    wd, step = audio.resample_filter(sr_orig, sr_new)
    wd = torch.from_numpy(wd.copy()).cuda()
    n_out = max(s[0] for s in sizes)
    treg = torch.from_numpy(audio.resample_register(ratio, n_out)).cuda()
    out = torch.empty(int(out_off[-1]), device="cuda")
    ms = event_time(lambda: K.resample(out, y, in_off, out_off, wd, step, ratio, treg), reps)
    t = taps(lens, sr_orig, sr_new)
    return {"ms": round(ms, 4), "input_samples": int(sum(lens)), "output_samples": int(out.numel()),
            "taps_G": round(t / 1e9, 3), "Gtaps_per_s": round(t / ms / 1e6, 1)}


def end_to_end(waves, rates, sr, r, B):
    def run():
        for i in range(0, len(waves), B):
            m, s, keep = audio.process_audio_batch(waves[i:i + B], r, rates=None if rates is None else rates[i:i + B], sr=sr)
            mh = torch.empty(m.shape, dtype=m.dtype, pin_memory=True)
            sh = torch.empty(s.shape, dtype=s.dtype, pin_memory=True)
            mh.copy_(m, non_blocking=True); sh.copy_(s, non_blocking=True)
        torch.cuda.synchronize()
    run()                                                          # warm-up: module loads, allocator, tables, registers
    times = []
    for _ in range(3):
        t0 = time.perf_counter()
        run()
        times.append(time.perf_counter() - t0)
    return round(float(np.median(times)) * 1e3 / len(waves), 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--chunk", type=int, default=64)
    ap.add_argument("--r", type=int, default=2)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    res = {"card": card, "chunk": a.chunk, "r": a.r, "kernel": {}, "ms_per_utterance": {}}
    c48, c441 = corpus(a.n, 48000, seed=1), corpus(a.n, 44100, seed=2)
    res["kernel"]["48000->24000"] = one_chunk(c48[:a.chunk], 48000, 24000, a.reps)
    res["kernel"]["44100->16000"] = one_chunk(c441[:a.chunk], 44100, 16000, a.reps)
    for name, waves, q, sr in (("48000->24000", c48, 48000, 24000), ("44100->16000", c441, 44100, 16000)):
        at_sr = audio.resample_batch(waves, [q] * len(waves), sr)
        res["ms_per_utterance"][name] = {"with_resampling": end_to_end(waves, [q] * len(waves), sr, a.r, a.chunk),
                                         "already_at_target_rate": end_to_end(at_sr, None, sr, a.r, a.chunk)}
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
