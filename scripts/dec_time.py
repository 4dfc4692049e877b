"""Time only the decoder section of the C2 step (quick A/B of decoder variants).

    TACO_TRACE=1 python scripts/dec_time.py [--precision fp32x3|tf32|fp32] [--window BACK,AHEAD]

With TACO_TRACE set, the traced kernel instantiation also records per-slot and per-phase clocks of CTA 0, and per-warp
stage clocks of CTA 0 and CTA 48 (another row group) that split each slot into hop, barrier skew, epilogue and the rest;
--window times the decoder with that attention window (Config.attention_window)."""
import argparse, os, sys, statistics
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from tacotron_b200 import Config, Tacotron
ap = argparse.ArgumentParser()
ap.add_argument("--precision", default="fp32x3", choices=["fp32x3", "tf32", "fp32"], help="default: the benchmark's mode")
ap.add_argument("--window", default=None, help="attention window BACK,AHEAD (default: none)")
args = ap.parse_args()
window = None if args.window is None else tuple(int(v) for v in args.window.split(","))
B, TX, T, R = 32, 128, 200, 5
m = Tacotron(Config(r=R, vocab_size=64, max_decode_iter=T, precision=args.precision, attention_window=window), None,
             train=False, seed=1)
g = torch.Generator().manual_seed(0)
inp = {"text": torch.randint(1, 64, (B, TX), generator=g, dtype=torch.int32).cuda(), "text_length": torch.full((B,), TX, dtype=torch.int32).cuda()}
m.step_ns = torch.zeros(T, dtype=torch.int64, device="cuda")
for _ in range(3): m.inference(inp, train=False)
torch.cuda.synchronize()
dec = []
for _ in range(5):
    m._marks = []
    m.inference(inp, train=False)
    torch.cuda.synchronize()
    tt = dict(m._marks); m._marks = None
    dec.append(tt["encoder"].elapsed_time(tt["decoder"]))
ns = m.step_ns.cpu().numpy()
print("precision", args.precision, "window", window, "decoder ms", statistics.median(dec), "step p50 us", float(statistics.median(((ns[1:]-ns[:-1])/1e3).tolist())))
if os.environ.get("TACO_TRACE"):
    import numpy as np
    from tacotron_b200 import _lib as L
    ws = m.runtime.dec_ws.view(torch.int64).cpu().numpy()
    total = int(L.lib().taco_decoder_trace_offset())   # where the trace starts in the workspace (decoder.cu build_ws_layout)
    names = ["G1", "C1", "G2", "C2", "G3", "C3", "OQP", "A|P2"]
    n = 1 + len(names) * T
    tr = ws[total: total + n]
    assert (tr > 0).all() and (np.diff(tr) >= 0).all(), "the trace is not where taco_decoder_trace_offset says"
    d = np.diff(tr)                              # d[i] = time of entry i+1 - entry i; entry 0 = prologue
    d = d[: (len(d) // len(names)) * len(names)].reshape(-1, len(names))[5:]
    med = np.median(d, axis=0)
    print("per-slot median ns (CTA 0):", {n_: int(v) for n_, v in zip(names, med)}, "sum", int(med.sum()))
    ck = ws[total + 16 * T + 16: total + 16 * T + 16 + 4 * 20 * 8].reshape(4, 20, 8)
    inames = ["G1", "C1", "G2", "C2", "G3", "C3", "OQP", "AP2"]
    print("stage: start->on-chain loads issued | (off-chain half) ->on-chain weights | ->mma done | (finish) ->partials | ->sync | ->epilogue"
          "   [cycles, CTA0 thread0, median of steps 10..12]")
    for i, nm in enumerate(inames):
        if ck[1, i, 3] == 0: continue
        def f(a, b):
            v = [int(ck[st, i, a] - ck[st, i, b]) for st in range(3) if ck[st, i, a] and ck[st, i, b]]
            return int(statistics.median(v)) if v else -1
        nxt = [ck[st, i + 1, 3] if i + 1 < len(inames) else ck[st + 1, 0, 3] for st in range(3)]
        total = int(statistics.median([int(nxt[st] - ck[st, i, 3]) for st in range(3)]))
        print(f"  {nm:8s} {f(0,3):6d} {f(1,0):6d} {f(2,1):6d} | {f(4,2):6d} {f(5,4):6d} {f(6,5):6d} | total {total:6d}")
    c = ck[:3, 7]     # A|P2 stage records: attention on warp 0 / thread 0
    if c[1, 3]:
        print("attention (cycles from slot start): q arrived+exp %d | bar1 %d | scores %d | bar2 %d | stats+bar3 %d | ctx partial+push %d | merged ctx stored %d"
              % tuple(int(statistics.median([int(c[st, i] - c[st, 3]) for st in range(3)])) for i in (0, 1, 2, 4, 5, 6, 7)))
    # per-warp stage records [2 CTAs][3 steps][20 items][64]: [0,16) last on-chain word seen, [16,32) stage barrier
    # reached, [32,48) barrier passed, [48,64) epilogue done (decoder.cu, trace_words)
    wbase = int(L.lib().taco_decoder_trace_offset()) + 16 * T + 16 + 4 * 20 * 8 + 16
    wr = ws[wbase: wbase + 2 * 3 * 20 * 64].reshape(2, 3, 20, 64)
    epi = {"G1": 8, "C1": 2, "G2": 4, "C2": 2, "G3": 4, "C3": 2, "OQP": 8}     # warps with an epilogue role per stage
    print("per-warp stage split [cycles, median of steps 10..12]: hop = previous stage's store (its last epilogue warp done)"
          " -> last on-chain word seen by any warp | spread = first -> last warp's last word | skew = last word -> last warp at"
          " the barrier | bar = -> warp 0 past it | epi0 / epiN = epilogue of warp 0 / of the last epilogue warp | slot = store"
          " -> store")
    for c, cta in enumerate((0, 48)):
        if not (wr[c, :, :7, 48:64] > 0).all():
            continue
        print(f"  CTA {cta}:  stage    hop  spread   skew    bar   epi0   epiN   slot")
        for i, nm in enumerate(names[:7]):
            cols = []
            for st in range(3):
                r = wr[c, st, i].astype(np.int64)
                arr, reach, passed, done = r[0:16], r[16:32], r[32:48], r[48:64]
                ne = epi[nm]
                store = done[:ne].max()
                prev = wr[c, st, i - 1, 48:48 + epi[names[i - 1]]].astype(np.int64).max() if i > 0 else None
                cols.append([arr.max() - prev if prev is not None else -1, arr.max() - arr.min(), reach.max() - arr.max(),
                             passed[0] - reach.max(), done[0] - passed[0], done[ne - 1] - passed[ne - 1],
                             store - prev if prev is not None else -1])
            med = np.median(np.array(cols), axis=0).astype(int)
            print(f"          {nm:5s} " + " ".join(f"{v:6d}" for v in med))
