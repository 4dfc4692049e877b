"""Generates tests/golden/reference_preprocess.npz.  Needs a checkout of the reference (barronalex/Tacotron): the
REFERENCE_DIR environment variable, by default a directory `reference` next to this repository.  The fixture is
committed, so the tests do not need the reference.

    REFERENCE_DIR=path/to/Tacotron python tests/golden/make_golden_features.py

Executes the reference's OWN preprocess.prepare_arctic / preprocess.preprocess and audio.process_audio (preprocess.py:41-60,
168-208; audio.py:38-65), unmodified, on a tiny synthetic ARCTIC-layout corpus written as 16-bit WAVs.  librosa's four
calls (load, effects.trim, stft, feature.melspectrogram) are stood in by the restatements of tests/feature_oracle.py, and
tensorflow / tqdm are stubbed, as make_golden.py::reference_griffinlim does.  This pins the WIRING: the trim / drop / pad /
pre-emphasis / log / reshape_frames statements, the vocabulary order (characters of a dropped utterance included), the
text padding, the float16 storage and meta.pkl.

The corpus: four utterances at 16 kHz, r = 2.  Utterance 2 is longer than maximum_audio_length after trimming, so it is
dropped, and it is the only one with the character 'Z'.  A speaker list is attached; the reference saves it whole.
"""
import os
import pickle
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REFERENCE_DIR = os.environ.get("REFERENCE_DIR", os.path.join(os.path.dirname(ROOT), "reference"))

PROMPTS = ["Hello world, it's me.", "a quick test", "Zebra Zone", "end of it!"]
SPEAKERS = [0, 1, 1, 0]


def corpus(seed=0):
    """four int16 waveforms: tone with quiet lead-in / tail, noise burst, a full-scale tone too long to keep, a chirp"""
    rng = np.random.RandomState(seed)
    t = lambda n: np.arange(n) / 16000.0
    quiet = lambda n: rng.randn(n) * 1e-4
    u0 = np.concatenate([quiet(3000), 0.5 * np.sin(2 * np.pi * 300 * t(14000)), quiet(2500)])
    u1 = np.concatenate([quiet(1800), 0.3 * rng.randn(12000), quiet(900)])
    u2 = 0.6 * np.sin(2 * np.pi * 100 * t(112000))
    u3 = 0.4 * np.sin(2 * np.pi * (200 + 900 * t(9000)) * t(9000))
    return [np.round(u * 32767).astype(np.int16) for u in (u0, u1, u2, u3)]


def write_arctic(root, waves):
    from scipy.io import wavfile
    os.makedirs(os.path.join(root, "arctic", "etc"), exist_ok=True)
    os.makedirs(os.path.join(root, "arctic", "wav"), exist_ok=True)
    with open(os.path.join(root, "arctic", "etc", "arctic.data"), "w") as f:
        for i, p in enumerate(PROMPTS):
            f.write(f'( arctic_a{i:04d} "{p}" )\n')
    for i, w in enumerate(waves):
        wavfile.write(os.path.join(root, "arctic", "wav", f"arctic_a{i:04d}.wav"), 16000, w)


def main():
    from tests import feature_oracle as FO
    from oracle import audio_oracle as A
    lib = types.ModuleType("librosa")
    lib.load = lambda f, mono=True, sr=22050: (FO.load(f, sr), sr)
    lib.effects = types.SimpleNamespace(trim=lambda y: FO.trim(y))
    lib.stft = lambda y, n_fft=2048, hop_length=None, win_length=None: A.stft(y, n_fft, hop_length, win_length)
    lib.feature = types.SimpleNamespace(melspectrogram=lambda S=None, n_mels=128: FO.melspectrogram(S))
    sys.modules["librosa"] = lib
    sys.modules["tensorflow"] = types.ModuleType("tensorflow")
    tq = types.ModuleType("tqdm")
    tq.tqdm = lambda x, **k: x
    sys.modules["tqdm"] = tq
    sys.path.insert(0, REFERENCE_DIR)
    import audio as ref_audio                      # the reference modules, unmodified
    import preprocess as ref_pre
    ref_audio.r = 2
    waves = corpus()
    out = {f"wave{i}": w for i, w in enumerate(waves)}
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as d:
        write_arctic(d, waves)
        ref_pre.DATA_DIR = d + "/"
        data = ref_pre.prepare_arctic()
        data["speakers"] = SPEAKERS
        os.makedirs(os.path.join(d, "data", "arctic"))
        os.chdir(d)
        try:
            ref_pre.preprocess(data, "arctic", sr=16000)
        finally:
            os.chdir(cwd)
        for name in ("texts", "text_lens", "mels", "stfts", "speech_lens", "speakers"):
            out[name] = np.load(os.path.join(d, "data", "arctic", name + ".npy"))
        with open(os.path.join(d, "data", "arctic", "meta.pkl"), "rb") as f:
            meta = pickle.load(f)
    out["prompts"] = np.array(PROMPTS)
    out["vocab_ids"] = np.array(sorted(meta["vocab"]))
    out["vocab_chars"] = np.array([meta["vocab"][k] for k in sorted(meta["vocab"])])
    out["r"], out["sr"] = np.array(meta["r"]), np.array(meta["sr"])
    np.savez_compressed(os.path.join(HERE, "reference_preprocess.npz"), **out)
    print("reference_preprocess.npz", {k: (v.shape, str(v.dtype)) for k, v in out.items()})


if __name__ == "__main__":
    main()
