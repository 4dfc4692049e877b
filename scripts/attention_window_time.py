"""Cost of the attention window (Config.attention_window) on the GPU, at two inference shapes (fp32x3, CUDA graphs, as
bench.py runs them):

  * c2:    the benchmark's inference step, B = 32, Tx = 128, T = 200, r = 5;
  * synth: the synthesis driver's batch, B = 32, Tx = 140 (data_input.MAX_TEXT_LEN), T = max_decode_iter = 180, r = 2.

For each shape, the decoder section (CUDA events around it) and the p50 of the decoder step (the kernel's %globaltimer
stamps, step_ns), window off against (2, 5), alternated in blocks in one process, medians.  With --base DIR: the
window-off decoder of this tree against a built checkout of another revision (e.g. the parent commit), on the same
inputs, in separate processes alternated in blocks.  The card's name, power limit and max SM clock are printed before
and after.

    python scripts/attention_window_time.py [--base DIR] [--blocks N] [--per-block N] [--out FILE]

Prints one JSON object; nothing is written unless --out is given."""
import argparse
import json
import os
import statistics
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = {"c2": (32, 128, 200, 5), "synth": (32, 140, 180, 2)}     # B, Tx, T, r


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def _setup(tree, window_names):
    """models[(shape, name)] and the inputs per shape, imported from the tree at `tree`"""
    sys.path.insert(0, tree)
    import torch
    from tacotron_b200 import Config, Tacotron
    if not torch.cuda.is_available():
        sys.exit("attention_window_time.py needs a CUDA device")
    models, inputs = {}, {}
    for shape, (B, TX, T, R) in SHAPES.items():
        g = torch.Generator().manual_seed(0)
        tl = torch.randint(TX // 2, TX + 1, (B,), generator=g, dtype=torch.int32)
        text = torch.randint(1, 64, (B, TX), generator=g, dtype=torch.int32) * (torch.arange(TX)[None, :] < tl[:, None]).to(torch.int32)
        inputs[shape] = {"text": text.cuda(), "text_length": tl.cuda()}
        for name, window in window_names:
            cfg = Config(r=R, vocab_size=64, max_decode_iter=T, cuda_graph=True)
            if window is not None:
                cfg.attention_window = window
            m = Tacotron(cfg, None, train=False, seed=1)
            m.step_ns = torch.zeros(T, dtype=torch.int64, device="cuda")
            models[(shape, name)] = m
    return torch, models, inputs


def _time(torch, m, inp):
    """(decoder section ms, per-step us list) of one inference call"""
    m._marks = []
    m.inference(inp, train=False)
    torch.cuda.synchronize()
    mk = dict(m._marks)
    m._marks = None
    ns = m.step_ns.cpu().numpy()
    return mk["encoder"].elapsed_time(mk["decoder"]), ((ns[1:] - ns[:-1]) / 1e3).tolist()


def _run(tree, window_names, blocks, per_block):
    torch, models, inputs = _setup(tree, window_names)
    for (shape, _), m in models.items():                   # warm-up: graph capture, weight packs, scratch buffers
        for _ in range(3):
            _time(torch, m, inputs[shape])
    res = {k: {"decoder_ms": [], "step_us": []} for k in models}
    names = [n for n, _ in window_names]
    for blk in range(blocks):
        for shape in SHAPES:
            for name in (names if blk % 2 == 0 else names[::-1]):
                for _ in range(per_block):
                    d, s = _time(torch, models[(shape, name)], inputs[shape])
                    res[(shape, name)]["decoder_ms"].append(d)
                    res[(shape, name)]["step_us"].extend(s)
    out = {}
    for (shape, name), v in res.items():
        out.setdefault(shape, {})[name] = {"decoder_ms_p50": statistics.median(v["decoder_ms"]),
                                           "decoder_ms_min": min(v["decoder_ms"]), "decoder_ms_max": max(v["decoder_ms"]),
                                           "step_us_p50": statistics.median(v["step_us"])}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", default=None, help="built checkout of the revision to compare the window-off decoder against")
    ap.add_argument("--blocks", type=int, default=6)
    ap.add_argument("--per-block", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:                                        # one block of the window-off decoder in the tree at --worker
        print(json.dumps(_run(args.worker, [("off", None)], 1, args.per_block)))
        return
    res = {"card": card(), "shapes": {k: dict(zip(("B", "Tx", "T", "r"), v)) for k, v in SHAPES.items()},
           "window": _run(HERE, [("off", None), ("win_2_5", (2, 5))], args.blocks, args.per_block)}
    if args.base:
        trees = [("this", HERE), ("base", os.path.abspath(args.base))]
        blk_res = {name: [] for name, _ in trees}
        for blk in range(args.blocks):
            for name, tree in (trees if blk % 2 == 0 else trees[::-1]):
                out = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", tree, "--per-block",
                                      str(args.per_block)], capture_output=True, text=True, cwd=tree)
                if out.returncode != 0:
                    raise RuntimeError(f"worker ({name}) failed:\n{out.stderr[-3000:]}")
                blk_res[name].append(json.loads(out.stdout.strip().splitlines()[-1]))
        res["base_off"] = {name: {shape: {k: statistics.median(b[shape]["off"][k] for b in blocks_)
                                          for k in ("decoder_ms_p50", "step_us_p50")} for shape in SHAPES}
                           for name, blocks_ in blk_res.items()}
        res["base_off_blocks"] = {name: [{s: b[s]["off"]["decoder_ms_p50"] for s in SHAPES} for b in blocks_]
                                  for name, blocks_ in blk_res.items()}
    res["card_after"] = card()
    s = json.dumps(res, indent=1)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
