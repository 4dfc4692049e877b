"""Cost of the speaker-conditioned decoder (Config.speaker_decoder): the C2 inference step (B=32, Tx=128 ragged, T=200,
r=5, fp32x3) with its decoder section, and one training step (B=32, Tx=64, T=40, r=5), for a 109-speaker (VCTK) model with
the encoder-only speaker path and the same model with speaker_decoder=True, alternated in blocks in one process.  Prints
the card and its power limit with the figures.

    python scripts/speaker_decoder_time.py [--blocks 6] [--per-block 3] [--out FILE.json]"""
import argparse, json, os, statistics, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from tacotron_b200 import Config, Tacotron

ap = argparse.ArgumentParser()
ap.add_argument("--blocks", type=int, default=6)
ap.add_argument("--per-block", type=int, default=3)
ap.add_argument("--out", default=None)
args = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("speaker_decoder_time.py needs a CUDA device")
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print("card:", card)
g = torch.Generator().manual_seed(0)
B, TX, T, R, NSPK = 32, 128, 200, 5, 109
tl = torch.randint(TX // 2, TX + 1, (B,), generator=g, dtype=torch.int32)
text = torch.randint(1, 64, (B, TX), generator=g, dtype=torch.int32) * (torch.arange(TX)[None, :] < tl[:, None]).to(torch.int32)
spk = torch.randint(0, NSPK, (B,), generator=g, dtype=torch.int32)
inf_in = {"text": text.cuda(), "text_length": tl.cuda(), "speaker": spk.cuda()}
TT, TXT = 40, 64
tl2 = torch.randint(TXT // 2, TXT + 1, (B,), generator=g, dtype=torch.int32)
tr_in = {"text": torch.randint(1, 64, (B, TXT), generator=g, dtype=torch.int32).cuda(), "text_length": tl2.cuda(),
         "mel": torch.randn(B, TT, 80 * R, generator=g).cuda(), "stft": torch.randn(B, TT, 1025 * R, generator=g).cuda(),
         "speaker": spk.cuda()}
models = {}
for name, sd in (("encoder_only", False), ("speaker_decoder", True)):
    models[name] = (Tacotron(Config(r=R, vocab_size=64, max_decode_iter=T, num_speakers=NSPK, speaker_decoder=sd), None,
                             train=False, seed=1),
                    Tacotron(Config(r=R, vocab_size=64, num_speakers=NSPK, speaker_decoder=sd), None, train=True, seed=1))


def time_inference(m):
    m._marks = []
    m.inference(inf_in, train=False)
    torch.cuda.synchronize()
    mk = dict(m._marks); m._marks = None
    return mk["start"].elapsed_time(mk["postnet"]), mk["encoder"].elapsed_time(mk["decoder"])


def time_train(m):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    m.train_step(tr_in, lr=0.0)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


for mi, mt in models.values():                            # warm-up: module loads, weight packs, scratch buffers
    for _ in range(2):
        time_inference(mi); time_train(mt)
res = {n: {"step": [], "decoder": [], "train": []} for n in models}
for _ in range(args.blocks):
    for n, (mi, mt) in models.items():
        for _ in range(args.per_block):
            s, d = time_inference(mi)
            res[n]["step"].append(s); res[n]["decoder"].append(d)
        for _ in range(args.per_block):
            res[n]["train"].append(time_train(mt))
summary = {"card": card, "shape": {"inference": "C2: B=32 Tx=128 T=200 r=5 fp32x3", "train": "B=32 Tx=64 T=40 r=5"}}
for n in models:
    summary[n] = {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)} for k, v in res[n].items()}
print(json.dumps(summary, indent=1))
if args.out:
    with open(args.out, "w") as f:
        json.dump(summary, f, indent=1)
