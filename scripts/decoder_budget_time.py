"""Decoder CTA budgets on the GPU: the decoder section, the C2 inference call and the C2 training step at max_ctas = 128, 96,
64 and 32 (and the default), and the C5 latency (B = 1) of this tree against another build, alternated in blocks.

    python scripts/decoder_budget_time.py [--base DIR] [--out FILE]

--base DIR: a built checkout of another revision (e.g. the parent commit); its C5 p50 is measured in separate processes
alternating with this tree's.  A budget on a 132-SM H100 SXM reproduces the launch plan of a smaller part (an H100 PCIe
has 114 SMs), not its clocks or its memory.  Prints one JSON object; nothing is written unless --out is given."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def c5_worker(tree):
    """p50 of 50 C5 calls (B = 1, char 140, T = 100, r = 5, tf32, CUDA graphs, host in/out) of the tree at `tree`"""
    sys.path.insert(0, tree)
    import torch
    from tacotron_b200 import Config, Tacotron
    B, TX, T, R = 1, 140, 100, 5
    m = Tacotron(Config(r=R, vocab_size=64, max_decode_iter=T, precision="tf32", cuda_graph=True), None, train=False, seed=1)
    g = torch.Generator().manual_seed(0)
    text_h = torch.randint(1, 64, (B, TX), generator=g, dtype=torch.int32).pin_memory()
    len_h = torch.full((B,), 97, dtype=torch.int32).pin_memory()
    out_h = torch.empty((B, T, 1025 * R)).pin_memory()
    al_h = torch.empty((B, T, TX)).pin_memory()

    def once():
        ci = {"text": text_h.cuda(non_blocking=True), "text_length": len_h.cuda(non_blocking=True)}
        _, out = m.inference(ci, train=False)
        out_h.copy_(out, non_blocking=True)
        al_h.copy_(m.alignments, non_blocking=True)
        torch.cuda.synchronize()
    for _ in range(10):
        once()
    ts, dec = [], []
    for _ in range(50):
        m._marks = []
        t0 = time.perf_counter()
        once()
        ts.append((time.perf_counter() - t0) * 1e3)
        ev = dict(m._marks)
        dec.append(ev["encoder"].elapsed_time(ev["decoder"]))
    print(json.dumps({"p50_ms": statistics.median(ts), "decoder_ms": statistics.median(dec)}))


def c2_budgets(budgets):
    sys.path.insert(0, HERE)
    import torch
    from oracle import tacotron_oracle as O
    from tacotron_b200 import Config, Tacotron
    cfg = O.OracleConfig(r=5, vocab_size=64)
    p = O.init_params(cfg, seed=1, trained_like=True)
    inp = O.synthetic_inputs(cfg, 32, 128, 200, seed=0, ragged=True)
    gi = {k: v.cuda().contiguous() for k, v in inp.items()}
    res = {}
    for mc in budgets:
        m = Tacotron(Config(r=5, vocab_size=64, max_decode_iter=200, max_ctas=mc), None, train=False)
        m.load_params(p)
        ii = {"text": gi["text"], "text_length": gi["text_length"]}
        for _ in range(2):
            m.inference(ii, train=False)
        dec, tot = [], []
        for _ in range(10):
            m._marks = []
            m.inference(ii, train=False)
            torch.cuda.synchronize()
            ev = dict(m._marks)
            dec.append(ev["encoder"].elapsed_time(ev["decoder"]))
            tot.append(ev["start"].elapsed_time(ev["postnet"]))
        m._marks = None
        mt = Tacotron(Config(r=5, vocab_size=64, max_ctas=mc), None, train=True)
        mt.load_params(p)
        for _ in range(3):
            float(mt.train_step(gi, lr=1e-4))
        st = []
        for _ in range(8):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            float(mt.train_step(gi, lr=1e-4))
            st.append((time.perf_counter() - t0) * 1e3)
        res[str(mc)] = {"decoder_ms_p50": statistics.median(dec), "inference_ms_p50": statistics.median(tot),
                        "train_step_ms_p50": statistics.median(st)}
        del m, mt
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", default=None, help="built checkout of the revision to compare the C5 latency against")
    ap.add_argument("--blocks", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--c5-only", action="store_true", help="only the C5 comparison")
    ap.add_argument("--c5-worker", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.c5_worker:
        c5_worker(args.c5_worker)
        return
    res = {"card": card(), "c2": c2_budgets([None, 128, 96, 64, 32]) if not args.c5_only else None}
    trees = [("this", HERE)] + ([("base", os.path.abspath(args.base))] if args.base else [])
    c5 = {name: [] for name, _ in trees}
    c5_dec = {name: [] for name, _ in trees}
    for blk in range(args.blocks):
        for name, tree in (trees if blk % 2 == 0 else trees[::-1]):
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--c5-worker", tree], capture_output=True, text=True,
                                 cwd=tree)
            if out.returncode != 0:
                raise RuntimeError(f"C5 worker ({name}) failed:\n{out.stderr[-3000:]}")
            r = json.loads(out.stdout.strip().splitlines()[-1])
            c5[name].append(r["p50_ms"])
            c5_dec[name].append(r["decoder_ms"])
    res["c5_p50_ms_blocks"] = c5
    res["c5_decoder_ms_blocks"] = c5_dec
    res["card_after"] = card()
    s = json.dumps(res, indent=1)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
