"""Where the time of the CBHG highway stacks goes, and what fusing them (taco_highway_stack_fwd) changes.

  1. one C2 inference step (B=32, Tx=128, T=200, r=5, fp32x3, eager) under torch.profiler (CUDA activities, a run of its
     own): the per-launch times of the encoder and post-net chains (highway layers + bi-GRU input products, and the
     post-net's width-fixing dense), i.e. every launch between each CBHG's last conv projection and its bi-GRU;
  2. the fused entry point against the unfused sequence (ops.highway x 4 + the xp ops.linear) on the same inputs, at
     the post-net C2 shape (32 000 x 80 rows) and the encoder C2 shape (4 096 x 128), alternated in blocks of --reps
     calls (one CUDA graph each, as the model replays them), CUDA events around each block; both must give the same
     bits;
  3. the card's name, power limit and max SM clock.

    python scripts/highway_stack_time.py [--blocks 10] [--reps 20] [--out FILE.json]"""
import argparse, json, os, statistics, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

ap = argparse.ArgumentParser()
ap.add_argument("--blocks", type=int, default=10)
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--out", default=None)
args = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("highway_stack_time.py needs a CUDA device")

from tacotron_b200 import Config, Tacotron
from tacotron_b200.models import ops
from tacotron_b200.params import ParamStore, cbhg_shapes

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print("card (name, power limit, max SM clock):", card)
summary = {"card": card}

# ---------------- 1. per-launch profile of one C2 step ----------------
B, TX, T, R = 32, 128, 200, 5
model = Tacotron(Config(r=R, vocab_size=64, max_decode_iter=T, precision="fp32x3", cuda_graph=False), None, train=False, seed=1)
g = torch.Generator().manual_seed(0)
inp = {"text": torch.randint(1, 64, (B, TX), generator=g, dtype=torch.int32).cuda(),
       "text_length": torch.full((B,), TX, dtype=torch.int32).cuda()}
for _ in range(2):
    model.inference(inp, train=False)
    model.inference(inp, train=False, trace={})
torch.cuda.synchronize()
profiles = {}
# a traced call keeps CBHG's layer-by-layer route (what the fused kernel replaces); an untraced one takes the fused route
for route, trace in (("layer_by_layer", {}), ("fused", None)):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        model.inference(inp, train=False, trace=trace)
        torch.cuda.synchronize()
    kern = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time > 0),
                  key=lambda e: e.time_range.start)
    names = [e.name for e in kern]
    gru = [i for i, n in enumerate(names) if "bigru_kernel" in n]
    assert len(gru) == 2, f"expected two bi-GRU launches (encoder, post-net), found {len(gru)}"
    chains = {}
    for sect, i, n_layered in (("encoder", gru[0], 5), ("postnet", gru[1], 6)):
        # fused: the one launch before the bi-GRU; layer by layer: (post-net: width-fixing dense) + 4 highway + xp
        n = 1 if "highway_stack_kernel" in names[i - 1] else n_layered
        rows = [{"kernel": e.name.replace("(anonymous namespace)::", "").split("(")[0], "us": round(e.device_time, 2)}
                for e in kern[i - n:i]]
        chains[sect] = {"launches": rows, "total_us": round(sum(r["us"] for r in rows), 2),
                        "span_us": round(kern[i - 1].time_range.end - kern[i - n].time_range.start, 2)}
        print(f"\n{route}, {sect} chain: {len(rows)} launch(es), kernel time {chains[sect]['total_us']:.1f} us, "
              f"first start to last end {chains[sect]['span_us']:.1f} us")
        for r in rows:
            print(f"  {r['us']:9.2f} us  {r['kernel']}")
    profiles[route] = chains
summary["step_profile"] = profiles
del model
torch.cuda.empty_cache()

# ---------------- 2. fused against unfused, alternated ----------------
def make_store(cin):
    st = ParamStore(cbhg_shapes("cbhg", cin, 16, [128, 128, cin]), "cuda")
    st.init_tf_default(seed=3)
    gg = torch.Generator().manual_seed(4)
    for n, (s, kind) in st.shapes.items():                # non-zero biases, so that every bias add is exercised
        if kind == "zeros":
            st.views[n].copy_(0.1 * torch.randn(s, generator=gg))
    st.version += 1
    return st


ab = {}
for label, (Bs, Ts, cin) in {"postnet_C2": (32, 1000, 80), "encoder_C2": (32, 128, 128)}.items():
    st = make_store(cin)
    rt = ops.runtime(st, "fp32x3")
    sc = ops.Scope(st, "cbhg")
    x = torch.randn(Bs, Ts, cin, generator=torch.Generator().manual_seed(5)).cuda()
    Wx, bx, Wxp = ops._gru_input_weights(rt, sc)

    def unfused():
        h = x
        for l in range(4):
            h = ops.highway(h, scope=sc.sub(f"highway{l}"))
        return ops.linear(rt, h, Wx, Wxp, 768, bias=bx, tag="ab_xp")

    def fused():
        return ops.highway_stack(x, 4, scope=sc)

    ref, got = unfused().clone(), fused().clone()
    torch.cuda.synchronize()
    same = torch.equal(ref.view(torch.int32), got.view(torch.int32))
    times = {"unfused": [], "fused": []}
    graphs = {}
    for name, f in (("unfused", unfused), ("fused", fused)):
        for _ in range(3):                                # warm-up (module load, kernel attributes)
            f()
        torch.cuda.synchronize()
        graphs[name] = torch.cuda.CUDAGraph()             # --reps calls per replay: device time, no host launch cost
        with torch.cuda.graph(graphs[name]):
            for _ in range(args.reps):
                f()
        graphs[name].replay()
    torch.cuda.synchronize()
    for _ in range(args.blocks):
        for name in ("unfused", "fused"):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            graphs[name].replay()
            b.record()
            torch.cuda.synchronize()
            times[name].append(a.elapsed_time(b) * 1e3 / args.reps)
    res = {k: {"median_us": round(statistics.median(v), 2), "min_us": round(min(v), 2), "max_us": round(max(v), 2)}
           for k, v in times.items()}
    res["rows"] = Bs * Ts
    res["in_channels"] = cin
    res["bit_identical"] = bool(same)
    res["saved_us"] = round(res["unfused"]["median_us"] - res["fused"]["median_us"], 2)
    ab[label] = res
    print(f"\n{label} ({Bs * Ts} x {cin}): unfused {res['unfused']['median_us']:.1f} us "
          f"[{res['unfused']['min_us']:.1f}, {res['unfused']['max_us']:.1f}], fused {res['fused']['median_us']:.1f} us "
          f"[{res['fused']['min_us']:.1f}, {res['fused']['max_us']:.1f}], bit-identical: {same}")
summary["fused_vs_unfused"] = ab
summary["blocks"], summary["reps_per_block"] = args.blocks, args.reps
print(json.dumps(summary, indent=1))
if args.out:
    with open(args.out, "w") as f:
        json.dump(summary, f, indent=1)
