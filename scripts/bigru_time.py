"""Where the time of the persistent bi-GRU forward (bigru_kernel, csrc/gru.cu) goes.

  1. one C2 inference step (B=32, Tx=128, T=200, r=5, fp32x3, eager) under torch.profiler (CUDA activities, a run of its
     own): the two bigru_kernel launches (encoder, post-net) and their share of the encoder and post-net sections
     (section times from the model's CUDA-event marks, median of 5 unprofiled steps);
  2. taco_bigru_fwd alone at the post-net shape (B=32, T=1000) and the encoder shape (B=32, T=128), and
     taco_bigru_fwd_h0 at the encoder shape: --blocks blocks of --reps calls, each block one CUDA-graph replay timed with
     CUDA events; median, min and max per call;
  3. the output of each against the float64 mirror of the kernel (tests/mirror_kernels_spk.bigru_fwd_h0);
  4. unless --no-trace: the per-phase %clock64 trace of thread 0 of CTA 0 (a library built from csrc/gru.cu with
     -DTACO_BIGRU_TRACE into a temporary directory), median cycles of steps 4..15 per phase;
  5. the card's name, power limit and max SM clock.

    python scripts/bigru_time.py [--blocks 10] [--reps 20] [--no-trace] [--out FILE.json]"""
import argparse, ctypes, json, os, statistics, subprocess, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

ap = argparse.ArgumentParser()
ap.add_argument("--blocks", type=int, default=10)
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--no-trace", action="store_true")
ap.add_argument("--out", default=None)
args = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bigru_time.py needs a CUDA device")

from tacotron_b200 import Config, Tacotron
from tacotron_b200 import _lib as L
from tests import mirror_kernels_spk as MK

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print("card (name, power limit, max SM clock):", card)
summary = {"card": card}

# ---------------- 1. the two launches in one C2 step ----------------
B, TX, T, R = 32, 128, 200, 5
model = Tacotron(Config(r=R, vocab_size=64, max_decode_iter=T, precision="fp32x3", cuda_graph=False), None, train=False, seed=1)
g = torch.Generator().manual_seed(0)
inp = {"text": torch.randint(1, 64, (B, TX), generator=g, dtype=torch.int32).cuda(),
       "text_length": torch.full((B,), TX, dtype=torch.int32).cuda()}
for _ in range(3):
    model.inference(inp, train=False)
torch.cuda.synchronize()
sect = {"encoder": [], "decoder": [], "postnet": []}
for _ in range(5):
    model._marks = []
    model.inference(inp, train=False)
    torch.cuda.synchronize()
    mk, model._marks = model._marks, None
    for (_, a), (name, b) in zip(mk[:-1], mk[1:]):
        sect[name].append(a.elapsed_time(b) * 1e3)
sect_us = {k: statistics.median(v) for k, v in sect.items()}
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    model.inference(inp, train=False)
    torch.cuda.synchronize()
kern = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time > 0),
              key=lambda e: e.time_range.start)
gru = [e.device_time for e in kern if "bigru_kernel" in e.name]
assert len(gru) == 2, f"expected two bi-GRU launches (encoder, post-net), found {len(gru)}"
step = {}
for name, us in zip(("encoder", "postnet"), gru):
    step[name] = {"bigru_us": round(us, 1), "section_us": round(sect_us[name], 1), "share": round(us / sect_us[name], 3)}
    print(f"C2 step, {name}: bigru_kernel {us:.1f} us of a {sect_us[name]:.1f} us section ({100 * us / sect_us[name]:.1f} %)")
step["decoder_section_us"] = round(sect_us["decoder"], 1)
summary["step_profile"] = step
del model
torch.cuda.empty_cache()

# ---------------- 2./3. the kernel alone, and against float64 ----------------
def case(Bs, Ts, with_h0, seed):
    gg = torch.Generator().manual_seed(seed)
    xp = torch.randn(Bs, Ts, 768, generator=gg)
    W = [torch.randn(128, 256, generator=gg) * 0.1, torch.randn(128, 128, generator=gg) * 0.1,
         torch.randn(128, 256, generator=gg) * 0.1, torch.randn(128, 128, generator=gg) * 0.1]
    h0 = [torch.randn(Bs, 128, generator=gg), torch.randn(Bs, 128, generator=gg)] if with_h0 else [None, None]
    return xp, W, h0


lib = L.lib()
P = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
res = {}
for label, (Bs, Ts, with_h0) in {"postnet_C2": (32, 1000, False), "encoder_C2": (32, 128, False),
                                 "encoder_C2_h0": (32, 128, True)}.items():
    xp, W, h0 = case(Bs, Ts, with_h0, 7)
    xd, Wd = xp.cuda(), [w.cuda() for w in W]
    hd = [None if h is None else h.cuda() for h in h0]
    out = torch.empty(Bs, Ts, 256, device="cuda")
    st = L.current_stream

    def call():
        if with_h0:
            rc = lib.taco_bigru_fwd_h0(P(xd), *[P(w) for w in Wd], P(hd[0]), P(hd[1]), P(out), Bs, Ts, st())
        else:
            rc = lib.taco_bigru_fwd(P(xd), *[P(w) for w in Wd], P(out), Bs, Ts, st())
        L.check(rc, "taco_bigru_fwd")
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    ref = torch.zeros(Bs, Ts, 256, dtype=torch.float64, device="cuda")
    zero = torch.zeros(Bs, 128, dtype=torch.float64, device="cuda")      # the mirror's own zero state lives on the CPU
    MK.bigru_fwd_h0(ref, xd.double(), *[w.double() for w in Wd], *[zero if h is None else h.double() for h in hd])
    err = (out.double() - ref).abs()
    acc = {"max_abs_err": float(err.max()), "mean_abs_err": float(err.mean()), "max_abs_ref": float(ref.abs().max())}
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(args.reps):
            call()
    graph.replay()
    torch.cuda.synchronize()
    times = []
    for _ in range(args.blocks):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        graph.replay()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) * 1e3 / args.reps)
    r = {"B": Bs, "T": Ts, "h0": with_h0, "median_us": round(statistics.median(times), 2), "min_us": round(min(times), 2),
         "max_us": round(max(times), 2), "ns_per_step": round(statistics.median(times) * 1e3 / Ts, 1), **acc}
    res[label] = r
    print(f"{label} (B={Bs}, T={Ts}{', h0' if with_h0 else ''}): {r['median_us']:.1f} us [{r['min_us']:.1f}, {r['max_us']:.1f}]"
          f" = {r['ns_per_step']:.0f} ns/step; vs float64: max {acc['max_abs_err']:.2e} mean {acc['mean_abs_err']:.2e}"
          f" (max |h| {acc['max_abs_ref']:.2f})")
summary["kernel"] = res
summary["blocks"], summary["reps_per_block"] = args.blocks, args.reps

# ---------------- 4. per-phase clock trace ----------------
if not args.no_trace:
    with tempfile.TemporaryDirectory() as d:
        shim = os.path.join(d, "trace.cu")
        with open(shim, "w") as f:      # the library's error hook and launch counter, which gru.cu links against
            f.write('#include <cstdarg>\n#include <cstdio>\nunsigned long long g_taco_launches = 0;\n'
                    'void taco_set_error(const char* fmt, ...) { va_list a; va_start(a, fmt); vfprintf(stderr, fmt, a); va_end(a); }\n'
                    f'#include "{os.path.join(ROOT, "tacotron_b200", "csrc", "gru.cu")}"\n')
        so = os.path.join(d, "libbigru_trace.so")
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                               "-DTACO_BIGRU_TRACE", "-Xcompiler", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"),
                               shim, "-o", so])
        tl = ctypes.CDLL(so)
    xp, W, _ = case(32, 1000, False, 7)
    xd, Wd = xp.cuda(), [w.cuda() for w in W]
    out = torch.empty(32, 1000, 256, device="cuda")
    for _ in range(2):
        assert tl.taco_bigru_fwd(P(xd), *[P(w) for w in Wd], P(out), 32, 1000, None) == 0
    torch.cuda.synchronize()
    import numpy as np
    buf = np.zeros(16 * 6, np.int64)
    assert tl.taco_bigru_trace_read(buf.ctypes.data_as(ctypes.c_void_p)) == 0
    ck = buf.reshape(16, 6)[4:]
    names = ["r products", "r reduction + u products + r*h stored", "barrier 1", "u, candidate + h stored", "barrier 2"]
    phase = {n: int(np.median(ck[:, i + 1] - ck[:, i])) for i, n in enumerate(names)}
    phase["step"] = int(np.median(ck[1:, 0] - ck[:-1, 0]))
    summary["trace_cycles"] = phase
    print("per-phase cycles (thread 0 of CTA 0, median of steps 4..15):", phase)

print(json.dumps(summary, indent=1))
if args.out:
    with open(args.out, "w") as f:
        json.dump(summary, f, indent=1)
