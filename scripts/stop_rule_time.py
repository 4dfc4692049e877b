"""Cost and savings of the end-of-text stop rule (Config.stop_at_end) on the GPU, at two inference shapes (fp32x3, CUDA
graphs, as bench.py runs them):

  * synth: the synthesis driver's batch, B = 32, Tx = 140 (data_input.MAX_TEXT_LEN), T = max_decode_iter = 180, r = 2;
  * c5:    one utterance, B = 1, Tx = 140, T = 100, r = 5.

For each shape and setting, the decoder section (CUDA events around it) and the whole synthesis (Tacotron.inference
and 50 Griffin-Lim iterations over the frames the setting keeps, host clock around work that ends in a device
synchronise), alternated in blocks in one process, medians:

  * off:        no stop rule (invert_spectrogram over every frame);
  * never:      the rule on, hold 4, stop_at = Tx: it never fires (the overhead of the rule itself);
  * fire_25/50/75: stop_at = 0, so every row ends after exactly `hold` steps, hold = 25 / 50 / 75 % of T (the random
                weights cannot be made to reach the end of a text; this places the stop instead).

The card's name, power limit and max SM clock are printed before and after.

    python scripts/stop_rule_time.py [--blocks N] [--per-block N] [--out FILE]

Prints one JSON object; nothing is written unless --out is given."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = {"synth": (32, 140, 180, 2), "c5": (1, 140, 100, 5)}     # B, Tx, T, r


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def settings(T, Tx):
    """name -> (hold or None, stop_at value)"""
    s = {"off": (None, 0), "never": (4, Tx)}
    for pct in (25, 50, 75):
        s[f"fire_{pct}"] = (max(1, T * pct // 100), 0)
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=4)
    ap.add_argument("--per-block", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    sys.path.insert(0, HERE)
    import torch
    from tacotron_b200 import Config, Tacotron, audio
    from tacotron_b200.models import ops
    if not torch.cuda.is_available():
        sys.exit("stop_rule_time.py needs a CUDA device")
    res = {"card": card(), "shapes": {k: dict(zip(("B", "Tx", "T", "r"), v)) for k, v in SHAPES.items()}}
    real_positions = ops.stop_positions
    models, inputs = {}, {}
    for shape, (B, TX, T, R) in SHAPES.items():
        g = torch.Generator().manual_seed(0)
        tl = torch.randint(TX // 2, TX + 1, (B,), generator=g, dtype=torch.int32)
        text = torch.randint(1, 64, (B, TX), generator=g, dtype=torch.int32) * (torch.arange(TX)[None, :] < tl[:, None]).to(torch.int32)
        inputs[shape] = {"text": text.cuda(), "text_length": tl.cuda()}
        for name, (hold, at) in settings(T, TX).items():
            m = Tacotron(Config(r=R, vocab_size=64, max_decode_iter=T, cuda_graph=True, stop_at_end=hold), None,
                         train=False, seed=1)
            models[(shape, name)] = (m, at)

    def call(shape, name):
        """(decoder section ms, synthesis ms, kept steps) of one inference + Griffin-Lim"""
        m, at = models[(shape, name)]
        r = m.config.r
        # the decoder graph is captured on a model's first call: stop_at is a fill of `at` inside it
        ops.stop_positions = lambda text, n: torch.full((text.shape[0],), at, dtype=torch.int32, device=text.device)
        try:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            m._marks = []
            _, out = m.inference(inputs[shape], train=False)
            if m.end_steps is None:
                audio.invert_spectrogram(out, r)
            else:
                audio.invert_speech(out, r, audio.stop_frames(m.end_steps, r, out.shape[1]))
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) * 1e3
        finally:
            ops.stop_positions = real_positions
        mk = dict(m._marks)
        m._marks = None
        return mk["encoder"].elapsed_time(mk["decoder"]), wall, out.shape[1]

    for key in models:                                     # warm-up: graph capture, weight packs, scratch buffers
        for _ in range(3):
            call(*key)
    times = {k: {"decoder_ms": [], "synthesis_ms": [], "steps": None} for k in models}
    for blk in range(args.blocks):
        for shape in SHAPES:
            names = [n for (s, n) in models if s == shape]
            for name in (names if blk % 2 == 0 else names[::-1]):
                for _ in range(args.per_block):
                    d, w, steps = call(shape, name)
                    times[(shape, name)]["decoder_ms"].append(d)
                    times[(shape, name)]["synthesis_ms"].append(w)
                    times[(shape, name)]["steps"] = steps
    out = {}
    for (shape, name), v in times.items():
        out.setdefault(shape, {})[name] = {"hold": models[(shape, name)][0].config.stop_at_end, "kept_steps": v["steps"],
                                           "decoder_ms_p50": statistics.median(v["decoder_ms"]),
                                           "decoder_ms_min": min(v["decoder_ms"]), "decoder_ms_max": max(v["decoder_ms"]),
                                           "synthesis_ms_p50": statistics.median(v["synthesis_ms"]),
                                           "synthesis_ms_min": min(v["synthesis_ms"]),
                                           "synthesis_ms_max": max(v["synthesis_ms"])}
    res["stop_rule"] = out
    res["card_after"] = card()
    s = json.dumps(res, indent=1)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
