"""GPU tests of long-form synthesis (csrc/audio.cu taco_speech_bounds and taco_join_segments;
tacotron_b200.audio.speech_bounds / join_speech; tacotron_b200.test --long-form): the speech bounds against the float64
oracle and bit for bit against speech_frames, the join within 2 ulp of its float64 mirror, and the driver end to end on
the toy model of test_gpu_z_summary.py."""
import os
import shutil

import numpy as np
import pytest
import torch
from scipy.io import wavfile

from tacotron_b200 import longform as LF
from tests import longform_oracle as LO
from tests import trim_oracle as TO
from tests.test_gpu_z_summary import _files, _train
from tests.test_summary import _events

pytestmark = pytest.mark.gpu
OUT = "log/toy/tacotron/test"


def _cuda(t):
    return None if t is None else torch.from_numpy(t).cuda()


@pytest.mark.parametrize("r", [1, 2, 5])
def test_speech_bounds_match_oracle_on_small_cases(r):
    from tacotron_b200 import audio
    T = {1: 24, 2: 16, 5: 8}[r]
    n = 4 * r * (T // 4)
    g = np.random.RandomState(r)
    scale, shift = (g.rand(1025 * r) * 2 + 1).astype(np.float32), (g.randn(1025 * r) * 2 - 5).astype(np.float32)
    starts, ends = [0, 3, n // 2, 0, n - 2, 0], [n // 2, n, n // 2 + 1, n, n - 1, 1]
    for sc, sh in ((None, None), (scale, shift)):
        spec = LO.speech_span_like(len(ends), T, r, starts, ends, seed=r, scale=sc, shift=sh)
        assert TO.margin_db(spec, r, sc, sh) >= 0.5
        got = audio.speech_bounds(_cuda(spec), r, stft_mean=_cuda(sh), stft_std=_cuda(sc))
        assert got.dtype == torch.int32 and got.is_cuda and got.shape == (len(ends), 3)
        frames = audio.speech_frames(_cuda(spec), r, stft_mean=_cuda(sh), stft_std=_cuda(sc))
        assert got.cpu().tolist() == LO.speech_bounds(spec, r, sc, sh).tolist()
        assert torch.equal(got[:, 2], frames)
    spec[1, 0, 3] = np.nan
    spec[2, T - 1, 5] = np.inf
    spec[3, 0, :1025] = -np.inf
    got = audio.speech_bounds(_cuda(spec), r).cpu()
    assert got[1:4].tolist() == [[0, n, n]] * 3
    assert got.tolist() == LO.speech_bounds(spec, r).tolist()


@pytest.mark.parametrize("r", [2, 5])
def test_speech_bounds_at_synthesis_size(r):
    """B = 32, full max_decode_iter (108000 / (300 r) decoder steps): [:, 2] is bit for bit speech_frames"""
    from tacotron_b200 import audio
    B, T = 32, 108000 // (300 * r)
    n = 4 * r * (T // 4)
    g = np.random.RandomState(10 + r)
    starts = [int(n * x) for x in np.linspace(0.0, 0.3, B)]
    ends = [int(n * x) for x in np.linspace(0.35, 1.0, B)]
    scale, shift = (g.rand(1025 * r) * 0.5 + 1.5).astype(np.float32), (g.randn(1025 * r) * 0.5 - 6).astype(np.float32)
    spec = LO.speech_span_like(B, T, r, starts, ends, seed=r, scale=scale, shift=shift)
    assert TO.margin_db(spec, r, scale, shift) >= 0.5
    sd, md, kd = _cuda(spec), _cuda(shift), _cuda(scale)
    want = LO.speech_bounds(spec, r, scale, shift)
    assert want[:, 0].tolist() == starts and want[:, 1].tolist() == ends
    for _ in range(2):
        got = audio.speech_bounds(sd, r, stft_mean=md, stft_std=kd)
        assert got.cpu().tolist() == want.tolist()
        assert torch.equal(got[:, 2], audio.speech_frames(sd, r, stft_mean=md, stft_std=kd))


@pytest.mark.parametrize("fade", [1, 160, 240])
def test_join_segments_within_two_ulp_of_the_float64_mirror(fade):
    from tacotron_b200 import audio, kernels as K
    g = np.random.RandomState(fade)
    src = (g.randn(200000) * np.exp(g.randn(200000))).astype(np.float32)
    lens = g.randint(1, 9000, size=40)
    lens[:3] = [1, 2 * fade - 1, 2 * fade + 1]
    seg, a, d = [], 0, 17
    for n in lens:
        seg.append((a, d, int(n)))
        a += int(n) + int(g.randint(0, 50))
        d += int(n) + int(g.randint(0, 300))
    seg = np.array(seg, dtype=np.int64)[g.permutation(len(lens))]
    out = torch.full((d + 5,), 3.5, device="cuda")
    K.join_segments(out, torch.from_numpy(src).cuda(), seg, fade)
    want = LO.join_segments(np.full(d + 5, 3.5), src, seg, fade)
    got = out.cpu().numpy().astype(np.float64)
    spacing = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    assert np.all(np.abs(got - want) <= 2 * spacing), float((np.abs(got - want) / spacing).max())
    out2 = torch.zeros(d + 5, device="cuda")                                             # the sr-derived fade of join_speech
    audio.join_speech(out2, torch.from_numpy(src).cuda(), seg, 16000)
    want2 = LO.join_segments(np.zeros(d + 5), src, seg, 160)
    assert np.all(np.abs(out2.cpu().numpy() - want2) <= 2 * np.spacing(np.abs(want2).astype(np.float32)))
    with pytest.raises(ValueError):
        K.join_segments(out, torch.from_numpy(src).cuda(), np.array([[0, 0, 10], [0, 5, 10]]), fade)


def _run(monkeypatch, prompts, **kw):
    """test.test on the toy model with the RNG seeded; spies on speech_bounds / speech_frames (spectrogram and result)"""
    from tacotron_b200 import audio
    from tacotron_b200 import test as synth
    from tacotron_b200.models.tacotron import Config, Tacotron
    seen = []
    reals = {name: getattr(audio, name) for name in ("speech_bounds", "speech_frames")}
    for name, real in reals.items():

        def spy(spec, r, _real=real, _name=name, **a):
            out = _real(spec, r, **a)
            seen.append((_name, spec.clone(), r, out.clone()))
            return out
        monkeypatch.setattr(audio, name, spy)
    logs = []
    cfg = Config()
    cfg.data_path, cfg.save_path = "data/toy/", "toy/tacotron"
    torch.manual_seed(0)
    waves = synth.test(Tacotron, cfg, prompts, log=logs.append, **kw)
    torch.cuda.synchronize()
    for name, real in reals.items():
        monkeypatch.setattr(audio, name, real)
    return waves, seen, logs


def _ulp_close(got, want, ulps=2):
    spacing = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    err = np.abs(np.asarray(got, np.float64) - want)
    assert np.all(err <= ulps * spacing), float((err / spacing).max())


def test_driver_without_the_flag_and_one_chunk_lines(tmp_path, monkeypatch):
    from tacotron_b200 import audio
    _train(str(tmp_path), monkeypatch, False)
    prompts = ["abcde\n", "helloyou\n", "abcde\n"]          # no break: a line voiced to its end is kept, not split again
    # 1. without the flag: every file byte-identical to a run that never passes it
    _run(monkeypatch, prompts)
    plain = _files(OUT)
    shutil.rmtree(OUT)
    _, seen, _ = _run(monkeypatch, prompts, long_form=False, summary_dir=None)
    assert not seen and _files(OUT) == plain
    shutil.rmtree(OUT)
    # 2. lines that fit in one chunk: the plain path's spectrograms, and each WAV is the trimmed waveform cut to the bounds
    trimmed, seen_t, _ = _run(monkeypatch, prompts, trim_tail=True)
    shutil.rmtree(OUT)
    waves, seen_l, _ = _run(monkeypatch, prompts, long_form=True)
    assert [s[0] for s in seen_t] == ["speech_frames"] and [s[0] for s in seen_l] == ["speech_bounds"]
    spec_t, r, frames = seen_t[0][1], seen_t[0][2], seen_t[0][3].cpu()
    spec_l, bounds = seen_l[0][1], seen_l[0][3].cpu()
    assert torch.equal(spec_t, spec_l) and torch.equal(bounds[:, 2], frames)
    for b in range(3):
        f0, f1, fr = bounds[b].tolist()
        a, e = audio.kept_samples(f0, f1, fr)
        want = LO.join_segments(np.zeros(e - a), trimmed[b].cpu().numpy(), [[a, 0, e - a]], 160)
        got = waves[b].cpu().numpy()
        assert got.shape == want.shape
        _ulp_close(got, want)
        rate, samples = wavfile.read(f"{OUT}/{b}.wav")
        assert rate == 16000 and samples.shape == got.shape
        al = np.load(f"{OUT}/{b}_attention.npy")
        assert al.shape == (fr // r, min(len(prompts[b]), 140))
        assert open(f"{OUT}/{b}.txt").read() == prompts[b].rstrip("\n")
        assert open(f"{OUT}/{b}_chunks.txt").read() == prompts[b].strip() + "\n"
    # --trim-tail with --long-form changes nothing
    shutil.rmtree(OUT)
    waves2, _, _ = _run(monkeypatch, prompts, long_form=True, trim_tail=True)
    assert all(torch.equal(x, y) for x, y in zip(waves, waves2))


def _controlled_inference(monkeypatch, threshold):
    """Tacotron.inference with every output row replaced: a chunk whose text_length is above `threshold` is voiced up to
    its last frame, any other is speech over frames [3, n/2) and the log(1e-8) padding elsewhere"""
    from tacotron_b200 import checkpoint
    from tacotron_b200.models.tacotron import Tacotron
    stats = {}
    real_restore, real_inf = checkpoint.restore, Tacotron.inference

    def restore(model, ck):
        stats["mean"], stats["std"] = (np.asarray(x, np.float32) for x in real_restore(model, ck))
        return stats["mean"], stats["std"]

    def inference(self, inputs, train=False):
        y, out = real_inf(self, inputs, train=train)
        B, T, W = out.shape
        r = W // 1025
        n = 4 * r * (T // 4)
        lens = inputs["text_length"].cpu().tolist()
        half = LO.speech_span_like(B, T, r, [3] * B, [n // 2] * B, seed=1, scale=stats["std"], shift=stats["mean"])
        for b, tl in enumerate(lens):
            if tl > threshold:
                half[b] = -stats["mean"] / stats["std"]                   # log magnitude 0 everywhere: every frame voiced
        out.copy_(torch.from_numpy(half).cuda())
        return y, out
    monkeypatch.setattr(checkpoint, "restore", restore)
    monkeypatch.setattr(Tacotron, "inference", inference)


def _paragraph(seed, words=90):
    rng = np.random.RandomState(seed)
    letters = list("abcdefghijklmnopqrs")
    ws = ["".join(rng.choice(letters, rng.randint(2, 8))) for _ in range(words)]
    punct = rng.choice(["", "", "", ",", ".", ";", " -"], words)
    return " ".join(w + p for w, p in zip(ws, punct)) + ".\n"


def test_driver_long_lines(tmp_path, monkeypatch):
    from tacotron_b200 import audio, data_input
    _train(str(tmp_path), monkeypatch, False)
    vocab = set(data_input.load_meta("data/toy/")["vocab"].values())
    lines = [_paragraph(1), "short one.\n", _paragraph(2, 120)]
    assert len(lines[0]) > 400 and len(lines[2]) > 400
    # 3. lines over 400 characters: chunks, joined length, attention, one audio and one image event per line
    _controlled_inference(monkeypatch, threshold=10 ** 9)
    waves, seen, _ = _run(monkeypatch, lines, long_form=True, summary_dir=OUT)
    r, T = seen[0][2], seen[0][1].shape[1]
    n, blk = 4 * r * (T // 4), 4 * r
    fr = blk * -(-(n // 2) // blk)
    a, e = audio.kept_samples(3, n // 2, fr)
    ev = _events(OUT)
    assert len(ev) == 1 + len(lines)
    for i, line in enumerate(lines):
        chunks = LF.split_line(line, vocab, i)
        assert open(f"{OUT}/{i}_chunks.txt").read() == "".join(c.text + "\n" for c in chunks)
        if i != 1:
            assert len(chunks) >= 3
        pauses = sum(LF.pause_samples(c.brk, 16000) for c in chunks[:-1])
        assert waves[i].numel() == len(chunks) * (e - a) + pauses
        rate, samples = wavfile.read(f"{OUT}/{i}.wav")
        assert rate == 16000 and samples.shape == (waves[i].numel(),)
        al = np.load(f"{OUT}/{i}_attention.npy")
        assert al.shape == (len(chunks) * fr // r, sum(min(len(c.prompt), 140) for c in chunks))
        vals = ev[i + 1][3]
        assert len(vals) == 2 and vals[0][0].endswith("/audio/0") and vals[1][0].endswith("/image/0")
        assert vals[0][1].audio.length_frames == waves[i].numel()
    total = sum(len(LF.split_line(x, vocab)) for x in lines)
    assert len([s for s in seen if s[0] == "speech_bounds"]) == -(-total // 32)


def test_driver_resplits_chunks_voiced_to_the_end(tmp_path, monkeypatch):
    from tacotron_b200 import data_input
    _train(str(tmp_path), monkeypatch, False)
    vocab = set(data_input.load_meta("data/toy/")["vocab"].values())
    thr = 30
    lines = [_paragraph(3), "abcdefghijklmnopqrsabcdefghijklmnopqrs\n", "ab cd.\n"]
    # 4. exactly the chunks above `thr` characters are split again; the one without a break is kept with a warning
    expect, warned = [], []

    def expand(c):
        if len(c.prompt) > thr:
            h = LF.resplit(c)
            if h is not None:
                return expand(h[0]) + expand(h[1])
            warned.append(c.text)
        return [c]
    for i, line in enumerate(lines):
        expect.append([x for c in LF.split_line(line, vocab, i) for x in expand(c)])
    assert warned == [lines[1].strip()]
    assert len(expect[0]) > len(LF.split_line(lines[0], vocab))
    _controlled_inference(monkeypatch, threshold=thr)
    _, seen, logs = _run(monkeypatch, lines, long_form=True)
    for i in range(len(lines)):
        assert open(f"{OUT}/{i}_chunks.txt").read() == "".join(c.text + "\n" for c in expect[i])
    warnings = [m for m in logs if "warning" in m]
    assert len(warnings) == 1 and lines[1].strip() in warnings[0]


def test_a_chunk_in_a_full_batch_equals_the_chunk_alone(tmp_path, monkeypatch):
    """5. rows of a batch are independent: the same text decodes to the same spectrogram in a batch of 32 and alone"""
    _train(str(tmp_path), monkeypatch, False)
    rng = np.random.RandomState(4)
    letters = list("abcdefghijklmnopqrs")
    lines = [" ".join("".join(rng.choice(letters, rng.randint(2, 8))) for _ in range(rng.randint(1, 6))) + "\n"
             for _ in range(32)]
    _, full, _ = _run(monkeypatch, lines, long_form=True)
    for k in (0, 17, 31):
        _, alone, _ = _run(monkeypatch, [lines[k]], long_form=True)
        assert full[0][1].shape[0] == 32 and alone[0][1].shape[0] == 1
        assert torch.equal(full[0][1][k], alone[0][1][0]), k
        assert torch.equal(full[0][3][k], alone[0][3][0]), k
