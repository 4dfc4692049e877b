"""Cost of the guided attention loss on the GPU, at the benchmark's training shape (C2: B = 32, Tx = 128, T = 200, r = 5):

  * the training step with the loss off and on (lambda = 1), alternated in blocks, medians;
  * taco_guided_attention alone, and audio.speech_frames on the target stft (the driver's per-batch T_b), CUDA events;
  * with --base DIR: taco_decoder_bwd with dscore_add = NULL in this tree against a built checkout of another revision
    (e.g. the parent commit), on the same captured inputs, in separate processes alternated in blocks.

    python scripts/guided_attention_time.py [--base DIR] [--blocks N] [--out FILE]

Prints one JSON object; nothing is written unless --out is given."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, TX, T, R = 32, 128, 200, 5


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def _inputs(torch, O):
    cfg = O.OracleConfig(r=R, vocab_size=64)
    p = O.init_params(cfg, seed=1, trained_like=True)
    inp = O.synthetic_inputs(cfg, B, TX, T, seed=0, ragged=True)
    gi = {k: v.cuda().contiguous() for k, v in inp.items()}
    g = torch.Generator().manual_seed(11)
    gi["speech_steps"] = (torch.randint(1, T // 4 + 1, (B,), generator=g, dtype=torch.int32) * 4).cuda()
    return p, gi


def _events_ms(torch, fn, n):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def this_tree(blocks):
    sys.path.insert(0, HERE)
    import torch
    from oracle import tacotron_oracle as O
    from tacotron_b200 import Config, Tacotron, audio, kernels as K
    p, gi = _inputs(torch, O)
    models = {}
    for name, lam in (("off", 0.0), ("on", 1.0)):
        m = Tacotron(Config(r=R, vocab_size=64, guided_attention=lam), None, train=True)
        m.load_params(p)
        for _ in range(3):
            float(m.train_step(gi, lr=1e-4))
        models[name] = m
    steps = {"off": [], "on": []}
    for blk in range(blocks):
        for name in (("off", "on") if blk % 2 == 0 else ("on", "off")):
            for _ in range(5):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                float(models[name].train_step(gi, lr=1e-4))
                steps[name].append((time.perf_counter() - t0) * 1e3)
    al = models["on"].saved["dec/align"]
    ds, loss = torch.empty_like(al), torch.empty(1, device="cuda")
    part = torch.empty(B * T, device="cuda")
    ga_ms = _events_ms(torch, lambda: K.guided_attention(ds, loss, al, gi["text_length"], gi["speech_steps"], 0.2, 1.0, part), 200)
    mean = torch.zeros(1025 * R, device="cuda")
    std = torch.ones(1025 * R, device="cuda")
    sf_ms = _events_ms(torch, lambda: audio.speech_frames(gi["stft"], R, mean, std), 50)
    return {"train_step_ms_p50": {k: statistics.median(v) for k, v in steps.items()},
            "train_step_ms_blocks": steps,
            "guided_attention_ms": ga_ms, "speech_frames_ms": sf_ms,
            "stft_mbytes": gi["stft"].numel() * 4 / 1e6, "align_shape": list(al.shape)}


def dec_bwd_worker(tree):
    """median of taco_decoder_bwd (dscore_add = NULL) on the C2 backward's captured inputs, in the tree at `tree`"""
    sys.path.insert(0, tree)
    import torch
    from oracle import tacotron_oracle as O
    from tacotron_b200 import Config, Tacotron, kernels as K
    from tacotron_b200.models import ops
    p, gi = _inputs(torch, O)
    m = Tacotron(Config(r=R, vocab_size=64), None, train=True)
    m.load_params(p)
    S = {}
    with ops.saving(S):
        m.seq2seq_output, m.output = m.inference(gi, True)
    S.update(text=gi["text"], text_length=gi["text_length"], mel=gi["mel"], stft=gi["stft"])
    S["post/out"] = m.output
    S["_capture"] = {}
    m.backward(S)
    a = {k: v for k, v in S["_capture"]["decoder_bwd"].items() if not k.startswith("_")}
    assert a.get("dscore_add") is None
    K.set_gemm_impl(1)
    ts = [_events_ms(torch, lambda: K.decoder_bwd(a), 10) for _ in range(5)]
    print(json.dumps({"decoder_bwd_ms": statistics.median(ts)}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", default=None, help="built checkout of the revision to compare taco_decoder_bwd against")
    ap.add_argument("--blocks", type=int, default=6)
    ap.add_argument("--out", default=None)
    ap.add_argument("--dec-bwd-worker", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.dec_bwd_worker:
        dec_bwd_worker(args.dec_bwd_worker)
        return
    res = {"card": card(), "c2": this_tree(args.blocks)}
    if args.base:
        trees = [("this", HERE), ("base", os.path.abspath(args.base))]
        dec = {name: [] for name, _ in trees}
        for blk in range(args.blocks):
            for name, tree in (trees if blk % 2 == 0 else trees[::-1]):
                out = subprocess.run([sys.executable, os.path.abspath(__file__), "--dec-bwd-worker", tree], capture_output=True,
                                     text=True, cwd=tree)
                if out.returncode != 0:
                    raise RuntimeError(f"decoder_bwd worker ({name}) failed:\n{out.stderr[-3000:]}")
                dec[name].append(json.loads(out.stdout.strip().splitlines()[-1])["decoder_bwd_ms"])
        res["decoder_bwd_null_ms_blocks"] = dec
        res["decoder_bwd_null_ms_p50"] = {k: statistics.median(v) for k, v in dec.items()}
    res["card_after"] = card()
    s = json.dumps(res, indent=1)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
