"""Cost of the synthesis tail trim on the GPU: Griffin-Lim (50 iterations) over every padded frame against the end of
speech plus Griffin-Lim over the kept frames only.

    python scripts/trim_time.py [--rounds 8] [--reps 3] [--out trim_time.json]

Two shapes: C2's synthesis batch (B = 32, r = 2, T = 180, so n = 360 frames) with speech lengths spread evenly over
15-100 % of n, and C5 (B = 1, r = 5, T = 100, n = 500) with 40 % speech.  The spectrograms are synthetic
(tests/trim_oracle.py speech_like): a smooth speech-like log magnitude, then the normalised log(1e-8) padding value of
the training targets.  Timed with CUDA events, alternated in blocks of --reps calls per arm and round:
  padded   audio.invert_spectrogram, 50 iterations over all B*n frames;
  trimmed  audio.speech_frames + audio.invert_speech, 50 iterations over the kept frames (includes the one host read of
           frames);
  frames   the speech_frames kernels alone.
Medians and min / max over rounds.  The card's name, power limit and max SM clock are read in the same run.
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

from tacotron_b200 import audio  # noqa: E402
from tests import trim_oracle as TO  # noqa: E402

N_ITER = 50


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


def shape(name, B, T, r, lo, hi, rounds, reps):
    n = 4 * r * (T // 4)
    ends = [int(round(n * x)) for x in np.linspace(lo, hi, B)]
    rng = np.random.RandomState(0)
    std = (rng.rand(1025 * r) * 0.5 + 1.5).astype(np.float32)
    mean = (rng.randn(1025 * r) * 0.5 - 6).astype(np.float32)
    spec = torch.from_numpy(TO.speech_like(B, T, r, ends, seed=1, scale=std, shift=mean)).cuda()
    mean_d, std_d = torch.from_numpy(mean).cuda(), torch.from_numpy(std).cuda()
    want = TO.speech_frames(spec.cpu().numpy(), r, std, mean)

    def padded():
        audio.invert_spectrogram(spec, r, n_iter=N_ITER, stft_mean=mean_d, stft_std=std_d)

    def trimmed():
        fr = audio.speech_frames(spec, r, stft_mean=mean_d, stft_std=std_d)
        audio.invert_speech(spec, r, fr, n_iter=N_ITER, stft_mean=mean_d, stft_std=std_d)

    def frames():
        audio.speech_frames(spec, r, stft_mean=mean_d, stft_std=std_d)

    got = audio.speech_frames(spec, r, stft_mean=mean_d, stft_std=std_d).cpu().numpy()
    assert got.tolist() == want.tolist(), (got, want)
    arms = {"padded": padded, "trimmed": trimmed, "frames": frames}
    for fn in arms.values():                                   # warm-up: module loads, allocator
        fn()
    t = {k: [] for k in arms}
    for i in range(rounds):
        order = list(arms) if i % 2 == 0 else list(arms)[::-1]
        for k in order:
            t[k].append(timed(arms[k], reps if k != "frames" else 20 * reps))
    kept = int(got.sum())
    res = {"shape": name, "B": B, "T": T, "r": r, "n": n, "frames_kept": kept, "frames_padded": B * n,
           "kept_fraction": kept / (B * n), "speech_frames_read_MB": B * T * 1025 * r * 4 / 1e6}
    for k, v in t.items():
        res[k + "_ms"] = {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
    res["trimmed_over_padded"] = res["trimmed_ms"]["median"] / res["padded_ms"]["median"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("trim_time.py needs a CUDA device")
    out = {"card": card(), "n_iter": N_ITER, "results": [
        shape("C2", 32, 180, 2, 0.15, 1.0, a.rounds, a.reps),
        shape("C5", 1, 100, 5, 0.4, 0.4, a.rounds, a.reps)]}
    print(json.dumps(out, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
