"""Cost of long-form synthesis on the GPU.

    python scripts/longform_time.py [--rounds 8] [--reps 20] [--out longform_time.json]

1. The two kernels at the synthesis shape (B = 32, r = 2, T = 180, so n = 360 frames) on tests/trim_oracle.py
   speech_like spectrograms with speech over frames [3 + b, 0.15..1.0 n): taco_speech_bounds (next to
   taco_speech_frames, which it extends) and taco_join_segments over the kept samples of the 32 Griffin-Lim outputs.
   CUDA events around --reps calls, medians and min / max over --rounds.
2. One ~1500-character paragraph end to end: ``test.test(long_form=True)`` on the paragraph as one line, against
   ``test.test(trim_tail=True)`` on its sentences as separate lines.  The model is an untrained Tacotron (random
   weights, r = 2, written to a temporary directory with its meta.pkl): no trained checkpoint is available, so the
   chunks an untrained model voices up to their last frame are split again, and the rounds that costs are printed with
   the times.  Wall clock per run (the drivers read results to the host), median and min / max over --rounds, the two
   arms alternated; files are written to the temporary directory.
The card's name, power limit and max SM clock are read in the same run.
"""
import argparse
import json
import os
import pickle
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tacotron_b200 import audio, kernels as K  # noqa: E402
from tests import trim_oracle as TO  # noqa: E402

PARAGRAPH = (
    "The old lighthouse stood at the edge of the cliff, its white paint peeling in long strips. For years nobody had "
    "climbed the narrow stairs to the lamp room; the keeper had left when the ships stopped coming. One autumn morning "
    "a girl from the village found the door open. She went up slowly, counting the steps, listening to the wind. At the "
    "top she saw the great lens, dusty but unbroken, and beyond it the grey sea stretching to the horizon. She wiped a "
    "small circle clean with her sleeve. The light that came through it was bright and strange! Was it the sun, or "
    "something older? She did not know. She sat there until the tide turned, watching the gulls and the slow clouds. "
    "When she came down, the village seemed smaller, and the sea much larger than before. She told nobody about the "
    "lens, but every evening after that she walked to the cliff and looked at the dark tower against the sky. In "
    "winter the storms came, and the waves climbed the rocks; still the tower stood. In spring she brought a brush, a "
    "bucket and a bottle of oil. Nobody asked where she was going. The work took all summer - the rust, the glass, the "
    "stubborn brass of the old mechanism. On the last night of August she lit the lamp, and far out on the water a "
    "fishing boat turned its bow toward the shore. The men on board saw the beam sweep across the waves, once, twice, "
    "and then again, steady as a heartbeat. They did not know who had lit it, and they did not ask; they only steered "
    "for home, and the light went with them.")


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


def stats(v):
    return {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}


def kernels(rounds, reps):
    B, T, r = 32, 180, 2
    n = 4 * r * (T // 4)
    ends = [int(round(n * x)) for x in np.linspace(0.15, 1.0, B)]
    g = np.random.RandomState(0)
    std = (g.rand(1025 * r) * 0.5 + 1.5).astype(np.float32)
    mean = (g.randn(1025 * r) * 0.5 - 6).astype(np.float32)
    spec = TO.speech_like(B, T, r, ends, seed=1, scale=std, shift=mean)
    for b in range(B):                                          # leading padding: speech starts at frame 3 + b
        tmp = TO.speech_like(1, T, r, [0], seed=1, scale=std, shift=mean)[0]
        for f in range(3 + b):
            t, c = 4 * (f // (4 * r)) + f % 4, (f % (4 * r)) // 4
            spec[b, t, c * 1025:(c + 1) * 1025] = tmp[t, c * 1025:(c + 1) * 1025]
    sd, md, kd = (torch.from_numpy(x).cuda() for x in (spec, mean, std))
    bounds = audio.speech_bounds(sd, r, stft_mean=md, stft_std=kd).cpu().numpy()
    y, start = audio.invert_speech_packed(sd, r, bounds[:, 2], n_iter=0, stft_mean=md, stft_std=kd)
    seg, pos = [], 0
    for b in range(B):
        a, e = audio.kept_samples(*bounds[b])
        seg.append((int(start[b]) + a, pos, e - a))
        pos += e - a + 4000
    seg = np.array(seg, dtype=np.int64)
    out = torch.zeros(pos, device="cuda")
    seg_d = torch.from_numpy(seg).cuda()
    fade = int(round(16000 * audio.JOIN_FADE_S))
    lib = K.L.lib()
    arms = {
        "speech_bounds": lambda: audio.speech_bounds(sd, r, stft_mean=md, stft_std=kd),
        "speech_frames": lambda: audio.speech_frames(sd, r, stft_mean=md, stft_std=kd),
        # the launch alone (kernels.join_segments adds the host check and the upload of seg)
        "join_segments_launch": lambda: lib.taco_join_segments(K._p(out), out.numel(), K._p(y), K._p(seg_d), B,
                                                               int(seg[:, 2].max()), fade, K._st()),
        "join_speech": lambda: audio.join_speech(out, y, seg, 16000),
    }
    for fn in arms.values():
        fn()
    t = {k: [] for k in arms}
    for i in range(rounds):
        for k in (list(arms) if i % 2 == 0 else list(arms)[::-1]):
            t[k].append(timed(arms[k], reps))
    return {"B": B, "T": T, "r": r, "n": n, "kept_samples": int(seg[:, 2].sum()),
            **{k + "_ms": stats(v) for k, v in t.items()}}


def end_to_end(rounds):
    from tacotron_b200 import checkpoint, test as synth
    from tacotron_b200.models.tacotron import Config, Tacotron
    chars = sorted(set("abcdefghijklmnopqrstuvwxyz.,;:!?'- "))
    vocab = {i + 1: ch for i, ch in enumerate(chars)}
    vocab[0] = "_"
    sentences = []
    cur = ""
    for w in PARAGRAPH.lower().split(" "):
        cur = (cur + " " + w).strip()
        if cur[-1] in ".!?":
            sentences.append(cur)
            cur = ""
    if cur:
        sentences.append(cur)
    old = os.getcwd()
    with tempfile.TemporaryDirectory() as d:
        os.chdir(d)
        try:
            os.makedirs("data/lf")
            with open("data/lf/meta.pkl", "wb") as f:
                pickle.dump({"r": 2, "vocab": vocab}, f)
            torch.manual_seed(0)
            cfg = Config()
            cfg.r, cfg.vocab_size = 2, len(vocab)
            cfg.max_decode_iter = audio.maximum_audio_length // (cfg.r * audio.hop_length)
            m = Tacotron(cfg, None, train=False)
            checkpoint.save(m, "weights/lf/tacotron", np.zeros(2050, np.float16), np.ones(2050, np.float32))
            del m
            logs = []

            def run(long_form):
                c = Config()
                c.data_path, c.save_path = "data/lf/", "lf/tacotron"
                logs.clear()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if long_form:
                    synth.test(Tacotron, c, [PARAGRAPH.lower() + "\n"], log=logs.append, long_form=True)
                else:
                    synth.test(Tacotron, c, [s + "\n" for s in sentences], log=logs.append, trim_tail=True)
                torch.cuda.synchronize()
                return (time.perf_counter() - t0) * 1e3
            run(True), run(False)                                   # warm-up
            t = {"long_form": [], "sentences_trim_tail": []}
            for i in range(rounds):
                for k in (list(t) if i % 2 == 0 else list(t)[::-1]):
                    t[k].append(run(k == "long_form"))
            run(True)
            chunks = open("log/lf/tacotron/test/0_chunks.txt").read().splitlines()
            warnings = sum("warning" in x for x in logs)
        finally:
            os.chdir(old)
    return {"paragraph_chars": len(PARAGRAPH), "sentences": len(sentences), "final_chunks": len(chunks),
            "unsplittable_warnings": warnings, **{k + "_ms": stats(v) for k, v in t.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--e2e-rounds", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("longform_time.py needs a CUDA device")
    out = {"card": card(), "kernels": kernels(a.rounds, a.reps), "end_to_end": end_to_end(a.e2e_rounds)}
    print(json.dumps(out, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
