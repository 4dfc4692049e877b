"""Cost of the training summaries on the GPU, at the benchmark's training shape (C2: B=32, char 128, 200 decoder steps,
r=5; seeded synthetic batch).

    python scripts/summary_time.py [--steps 10] [--rounds 4] [--reps 50] [--out summary_time.json]

Reports taco_histogram's time on each of the three histogrammed tensors (CUDA events, median over repeats) with the bytes
it reads and the rate, then the training step with and without summaries, alternated in blocks of --steps steps on the
same model: the loop of train.train (one host sync per step, the float of the loss; with summaries: one tensor of the
three losses, the histograms and the pinned copies enqueued after the step, the previous step's records encoded and
written before the sync).  Host wall clock per step, mean of each block.  The card's name, power limit and max SM clock
are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tacotron_b200 import Config, Tacotron, kernels as K, summary as S  # noqa: E402

B, TX, T, R = 32, 128, 200, 5


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


def block(m, inputs, steps, summaries, host):
    """mean host wall-clock ms per step of `steps` steps of train.train's loop; adds to host["enqueue"] the host time until
    the step's work is enqueued (train_step, and with summaries the histograms and copies) and to host["encode"] the time
    of write_pending"""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        ta = time.perf_counter()
        loss_t = m.train_step(inputs, lr=1e-4).reshape(1).clone()
        if summaries is not None:
            loss_t = torch.stack([m.loss, m.seq2seq_loss, m.output_loss])
            summaries.enqueue(m.global_step, (m.saved["enc/prenet/l2"], m.seq2seq_output, m.output), loss_t, m.grad_sumsq)
            tb = time.perf_counter()
            summaries.write_pending()
            host["encode"] += time.perf_counter() - tb
        host["enqueue"] += time.perf_counter() - ta
        float(loss_t[0])
        if summaries is not None:
            summaries.collect()
    if summaries is not None:
        summaries.write_pending()
    return (time.perf_counter() - t0) * 1e3 / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    m = Tacotron(Config(r=R, vocab_size=64), None, train=True, seed=1)
    g = torch.Generator().manual_seed(100)
    inputs = {"text": torch.randint(1, 64, (B, TX), generator=g, dtype=torch.int32).cuda(),
              "text_length": torch.full((B,), TX, dtype=torch.int32).cuda(),
              "mel": torch.randn(B, T, 80 * R, generator=g).half().float().cuda(),
              "stft": torch.randn(B, T, 1025 * R, generator=g).half().float().cuda()}
    m.train_step(inputs, lr=1e-4)
    torch.cuda.synchronize()
    res = {"card": card, "shape": f"C2 training: B={B}, char {TX}, {T} decoder steps, r={R}", "kernel": {}}
    lim = torch.from_numpy(S.histogram_limits()).cuda()
    out = torch.empty(len(lim) + 5, dtype=torch.int64, device="cuda")
    total = 0.0
    for tag, t in zip(S.HISTOGRAM_TAGS, (m.saved["enc/prenet/l2"], m.seq2seq_output, m.output)):
        ms = event_time(lambda: K.histogram(out, t, lim), a.reps)
        total += ms
        res["kernel"][tag] = {"elements": t.numel(), "MB": round(t.numel() * 4 / 1e6, 2), "ms": round(ms, 4),
                              "GB_per_s": round(t.numel() * 4 / ms / 1e6, 1)}
    res["kernel"]["three_histograms_ms"] = round(total, 4)
    with tempfile.TemporaryDirectory() as d:
        summ = S.TrainSummaries(d, torch.device("cuda"))
        h_off, h_on = {"enqueue": 0.0, "encode": 0.0}, {"enqueue": 0.0, "encode": 0.0}
        block(m, inputs, 3, None, dict(h_off))
        block(m, inputs, 3, summ, dict(h_on))                      # warm-up of both loops
        off, on = [], []
        for _ in range(a.rounds):
            off.append(block(m, inputs, a.steps, None, h_off))
            on.append(block(m, inputs, a.steps, summ, h_on))
        summ.close()
        res["event_file_bytes_per_step"] = round(os.path.getsize(summ.writer.path) / ((a.rounds * a.steps) + 3))
    res["step_ms"] = {"without_summaries": [round(x, 2) for x in off], "with_summaries": [round(x, 2) for x in on],
                      "median_without": round(float(np.median(off)), 2), "median_with": round(float(np.median(on)), 2)}
    res["step_ms"]["difference_pct"] = round(100 * (np.median(on) - np.median(off)) / np.median(off), 2)
    n = a.rounds * a.steps
    res["host_ms_per_step"] = {"enqueue_without": round(h_off["enqueue"] * 1e3 / n, 2),
                               "enqueue_with_incl_encode": round(h_on["enqueue"] * 1e3 / n, 2),
                               "encode": round(h_on["encode"] * 1e3 / n, 2)}
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
