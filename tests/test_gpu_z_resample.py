"""GPU tests of resampling (csrc/resample.cu, audio.resample_batch, process_audio_batch(rates=...), preprocess
--resample): taco_resample bit for bit against its torch-CPU mirror with NaN-poisoned outputs at every ratio, a chunk
mixing source rates against its rate groups processed apart, and a 48 kHz VCTK corpus through the CLI against the same
corpus resampled by the oracle beforehand, then loaded and trained on with the multi-speaker model."""
import os

import numpy as np
import pytest
import torch

from tacotron_b200 import audio
from tests import mirror_kernels_resample as MKR
from tests import resample_oracle as RO
from tests.test_features import _write_wav
from tests.test_gpu_z_features import _compare_with_oracle, _run_preprocess, _utterance
from tests.test_resample import RATES, _case_lengths

pytestmark = pytest.mark.gpu


def _lengths(B, sr_orig, sr_new, rng):
    """B = 1: one long odd input (a zero tail wherever the ratio is not an integer); B = 64: the CPU test's edge cases,
    480000 samples and short random ones"""
    special = _case_lengths(sr_orig, sr_new) + [480000]
    return (special + list(rng.randint(1, 20000, size=B)))[:B] if B > 1 else [479999]


@pytest.mark.parametrize("B", [1, 64])
@pytest.mark.parametrize("sr_orig,sr_new", RATES)
def test_resample_kernel_against_mirror(sr_orig, sr_new, B):
    from tacotron_b200 import kernels as K
    rng = np.random.RandomState(B + sr_orig)
    lens = [int(n) for n in _lengths(B, sr_orig, sr_new, rng)]
    lens = [max(n, _case_lengths(sr_orig, sr_new)[0]) for n in lens]
    waves = [(rng.randn(n) * 0.3).astype(np.float32) for n in lens]
    ratio = float(sr_new) / sr_orig
    sizes = [audio.resample_lengths(n, sr_orig, sr_new) for n in lens]
    in_off = torch.tensor(np.concatenate([[0], np.cumsum(lens)]))
    out_off = torch.tensor(np.concatenate([[0], np.cumsum([s[1] for s in sizes])]))
    y = torch.from_numpy(np.concatenate(waves))
    wd, step = audio.resample_filter(sr_orig, sr_new)
    wd = torch.from_numpy(wd.copy())
    n_out = max(s[0] for s in sizes)
    treg = torch.from_numpy(audio.resample_register(ratio, n_out))
    got = torch.full((int(out_off[-1]),), float("nan"), device="cuda")
    K.resample(got, y.cuda(), in_off.cuda(), out_off.cuda(), wd.cuda(), step, ratio, treg.cuda())
    want = torch.empty(int(out_off[-1]))
    MKR.resample(want, y, in_off, out_off, wd, step, ratio, treg)
    got = got.cpu()
    assert not torch.isnan(got).any()
    assert torch.equal(got, want)
    assert sum(s[1] - s[0] for s in sizes) > 0 or sr_new % sr_orig == 0               # zero tails were written
    # the public form: the oracle's samples
    if B == 1:
        assert np.array_equal(audio.resample_batch(waves, [sr_orig], sr_new)[0], RO.resample(waves[0], sr_orig, sr_new))


def test_mixed_rate_chunk_equals_its_groups():
    rng = np.random.RandomState(11)
    rates = [48000, 24000, 48000, 24000, 24000, 48000]
    waves = [_utterance(rng, int(n), sr=q) for n, q in zip(rng.randint(20000, 200000, size=6), rates)]
    mel, stft, keep = audio.process_audio_batch(waves, 2, rates=rates, sr=24000)
    parts = {}
    for q in (48000, 24000):
        idx = [b for b, r in enumerate(rates) if r == q]
        parts[q] = (idx,) + audio.process_audio_batch([waves[b] for b in idx], 2, rates=[q] * len(idx), sr=24000)
    kept = np.flatnonzero(keep).tolist()
    for q, (idx, m, s, k) in parts.items():
        assert np.array_equal(k, keep[idx])
        for j, b in enumerate(i for i, kk in zip(idx, k) if kk):
            assert torch.equal(mel[kept.index(b)], m[j]) and torch.equal(stft[kept.index(b)], s[j])
    # utterances already at 24 kHz are exactly today's arithmetic
    m0, s0, k0 = audio.process_audio_batch([waves[b] for b in parts[24000][0]], 2)
    assert torch.equal(m0, parts[24000][1]) and torch.equal(s0, parts[24000][2])


def _vctk48(root, rng):
    """VCTK layout with the 48 kHz originals (int16), one utterance too long after resampling and trimming"""
    vctk = os.path.join(root, "vctk")
    os.makedirs(vctk)
    with open(os.path.join(vctk, "speaker-info.txt"), "w") as f:
        f.write("ID  AGE  GENDER  ACCENTS  REGION\n225  23  F  English  Southern\n226  22  M  English  Surrey\n")
    lengths = {"225": [60000, 280000, 41001], "226": [50000, 36000]}            # p225_002 is dropped
    for uid, ls in lengths.items():
        os.makedirs(os.path.join(vctk, "txt", f"p{uid}"))
        os.makedirs(os.path.join(vctk, "wav48", f"p{uid}"))
        for k, n in enumerate(ls):
            name = f"p{uid}_{k + 1:03d}"
            with open(os.path.join(vctk, "txt", f"p{uid}", name + ".txt"), "w") as f:
                f.write(f"Utterance {k} of speaker {uid}.\n")
            w = _utterance(rng, n, sr=48000)
            if n > 216000:
                w = (0.5 * np.sin(2 * np.pi * 220 * np.arange(n) / 48000)).astype(np.float32)
            _write_wav(os.path.join(vctk, "wav48", f"p{uid}", name + ".wav"), 48000, np.round(w * 32767).astype(np.int16))
    return vctk


def test_vctk_48k_corpus_resample_preprocess_train(tmp_path, monkeypatch):
    from tacotron_b200 import data_input, preprocess as P, train as trainer
    from tacotron_b200.models.tacotron import Config, Tacotron
    rng = np.random.RandomState(6)
    root, pre = str(tmp_path / "data"), str(tmp_path / "pre" / "data")
    vctk = _vctk48(root, rng)
    # the same corpus resampled by the oracle, written as float32 24 kHz files
    data = P.prepare_vctk(root)
    pre_vctk = os.path.join(pre, "vctk")
    for src in data["audio_files"] + [os.path.join(vctk, "speaker-info.txt")]:
        dst = src.replace(root, pre)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        if src.endswith(".wav"):
            x, rate = audio.read_wav(src)
            _write_wav(dst, 24000, RO.resample(x, rate, 24000))
        else:
            with open(src) as f, open(dst, "w") as g:
                g.write(f.read())
    for uid in ("225", "226"):
        os.makedirs(os.path.join(pre_vctk, "txt", f"p{uid}"), exist_ok=True)
        for name in os.listdir(os.path.join(vctk, "txt", f"p{uid}")):
            with open(os.path.join(vctk, "txt", f"p{uid}", name)) as f, open(os.path.join(pre_vctk, "txt", f"p{uid}", name), "w") as g:
                g.write(f.read())
    _run_preprocess(["vctk", "--data-dir", root, "-r", "2", "--resample"])
    _run_preprocess(["vctk", "--data-dir", pre, "-r", "2"])
    for k in ("texts", "text_lens", "speech_lens", "speakers", "mels", "stfts"):
        a, b = np.load(os.path.join(vctk, k + ".npy")), np.load(os.path.join(pre_vctk, k + ".npy"))
        assert a.dtype == b.dtype and np.array_equal(a, b), k
    with open(os.path.join(vctk, "meta.pkl"), "rb") as f, open(os.path.join(pre_vctk, "meta.pkl"), "rb") as g:
        assert f.read() == g.read()
    ref = _compare_with_oracle(pre_vctk, P.prepare_vctk(pre), 2, 24000)
    assert list(ref["kept"]) == [0, 2, 3, 4] and ref["meta"]["sr"] == 24000
    assert np.load(os.path.join(vctk, "speakers.npy")).tolist() == [0, 0, 1, 1]
    arrays, names, num_speakers, _, _ = data_input.load_from_npy(vctk + "/")
    assert num_speakers == 2 and arrays["stft"].shape[0] == 4
    monkeypatch.chdir(tmp_path)
    cfg = Config()
    cfg.data_path, cfg.save_path, cfg.restore = "data/vctk/", "vctk/tacotron", False
    m = trainer.train(Tacotron, cfg, num_steps=1, log=lambda *a: None, save_every=1000)
    assert m.config.num_speakers == 2 and m.global_step == 1 and np.isfinite(float(m.loss))
