"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY.  Preprocessing: the reference's ``audio.process_audio`` (audio.py:38-65) and
``preprocess.preprocess`` (preprocess.py:168-208) restated in float64 numpy, with librosa's four calls restated from their
published algorithms (librosa is not installed, and the release the reference ran is not recorded):

  load (librosa.load, mono=True, no resampling): float32 samples, 16-bit PCM as x / 32768, channels averaged.
  effects.trim (top_db=60, ref=np.max, frame_length=2048, hop_length=512): the time-domain RMS of librosa 0.6-0.9.  Frame
        energy = mean square over 2048 samples of the signal reflect-padded by 1024 (centre framing), 1 + len//512 frames;
        a frame is non-silent when 10 log10(max(1e-10, e)) - 10 log10(max(1e-10, max e)) > -60; the kept span is
        [first*512, min(len, (last+1)*512)), empty if no frame is non-silent.  Later releases compute the energy from a
        spectrogram; that choice is made here, and parity with librosa itself stays unpinned, as for the stft/istft
        restatements of oracle/audio_oracle.py (reused here for the stft).
  stft (n_fft=2048, win_length=1200, hop_length=300): oracle/audio_oracle.stft.
  feature.melspectrogram(S=stft, n_mels=80): mel_basis() . S, with the basis applied to the COMPLEX spectrum (S passes
        through unsquared) and built at librosa's default sr = 22050 whatever the file's rate: Slaney scale, fmax 11025,
        area-normalised (norm=1), rows stored as float32 before and after the normalisation (filters.mel(dtype=float32)).

Pinned by tests/golden/reference_preprocess.npz: the reference's own process_audio / preprocess, run unmodified with these
four restatements standing in for librosa, reproduced exactly (tests/test_features.py).  The mel basis is also checked
against torchaudio's independent implementation.
"""
from __future__ import annotations

import numpy as np

from oracle import audio_oracle as A
from oracle.tf12 import reshape_frames

MAX_LEN, HOP, WIN, N_FFT = 108000, 300, 1200, 2048       # audio.py:10-13


def load(path, sr):
    """librosa.load(path, mono=True, sr=sr) for a WAV already at sr -> float32"""
    from scipy.io import wavfile
    rate, x = wavfile.read(path)
    assert rate == sr, (path, rate, sr)
    scale = {np.dtype(np.int16): 2.0 ** 15, np.dtype(np.int32): 2.0 ** 31}
    if x.dtype == np.uint8:
        x = (x.astype(np.float64) - 128.0) / 128.0
    elif x.dtype in scale:
        x = x.astype(np.float64) / scale[x.dtype]
    x = x.astype(np.float32)
    return x.mean(axis=1, dtype=np.float32) if x.ndim == 2 else x


def trim(y, top_db=60, frame_length=2048, hop_length=512):
    """librosa.effects.trim(y) -> (y[start:end], np.array([start, end]))"""
    yp = np.pad(y.astype(np.float64), frame_length // 2, mode="reflect")
    nf = 1 + len(y) // hop_length
    e = np.array([np.mean(yp[f * hop_length:f * hop_length + frame_length] ** 2) for f in range(nf)])
    db = 10.0 * np.log10(np.maximum(1e-10, e)) - 10.0 * np.log10(np.maximum(1e-10, e.max()))
    nz = np.flatnonzero(db > -top_db)
    start, end = (nz[0] * hop_length, min(len(y), (nz[-1] + 1) * hop_length)) if nz.size else (0, 0)
    return y[start:end], np.array([start, end])


def mel_basis(sr=22050, n_fft=2048, n_mels=80):
    """librosa.filters.mel(sr, n_fft, n_mels) of librosa 0.6-0.9 (htk=False, norm=1, dtype=float32)"""
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    to_mel = lambda f: min_log_mel + np.log(f / min_log_hz) / logstep if f >= min_log_hz else f / f_sp
    mels = np.linspace(to_mel(0.0), to_mel(sr / 2.0), n_mels + 2)
    mel_f = f_sp * mels
    lg = mels >= min_log_mel
    mel_f[lg] = min_log_hz * np.exp(logstep * (mels[lg] - min_log_mel))
    fft_f = np.linspace(0, sr / 2.0, 1 + n_fft // 2, endpoint=True)
    w = np.zeros((n_mels, 1 + n_fft // 2), dtype=np.float32)
    for i in range(n_mels):
        lower = (fft_f - mel_f[i]) / (mel_f[i + 1] - mel_f[i])
        upper = (mel_f[i + 2] - fft_f) / (mel_f[i + 2] - mel_f[i + 1])
        w[i] = np.maximum(0, np.minimum(lower, upper))
    w *= (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]
    return w


_BASIS = None


def melspectrogram(S):
    global _BASIS
    if _BASIS is None:
        _BASIS = mel_basis()
    return np.dot(_BASIS, S)


def features(wave, r):
    """audio.py:41-63 after the load: (mel, stft) log-spectrograms [T, 80r] / [T, 1025r] in float64, or (None, None)"""
    wave, _ = trim(wave)
    if wave.shape[0] > MAX_LEN:
        return None, None
    wave = np.pad(wave, (0, MAX_LEN - wave.shape[0]), "constant", constant_values=0)
    wave = np.append(wave[0], wave[1:] - 0.97 * wave[:-1])          # float32, as numpy evaluates audio.py:54
    stft = A.stft(wave, N_FFT, HOP, WIN)
    mel = melspectrogram(stft)
    return (reshape_frames(np.log(np.abs(mel) + 1e-8), r, forward=True),
            reshape_frames(np.log(np.abs(stft) + 1e-8), r, forward=True))


def f16_ulp_distance(a, b):
    """elementwise distance in float16 steps between two float16 arrays (sign-magnitude bits mapped to a monotone integer)"""
    def ordered(x):
        bits = np.asarray(x, dtype=np.float16).view(np.int16).astype(np.int64)
        return np.where(bits < 0, -(bits & 0x7FFF), bits)
    return np.abs(ordered(a) - ordered(b))


def f16_close(a, b):
    """float16 log-spectrogram values within one float16 step of each other, or within 2^-11: near log = 0 (|X| ~ 1) a
    float16 step is finer than float32 error (one step of 1.0 is 2^-10, a relative error of 0.1 % in the linear domain)"""
    near = np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)) <= 2.0 ** -11
    return (f16_ulp_distance(a, b) <= 1) | near


def check_f16(got, ref, floor=1e-4):
    """float16 log-spectrogram `got` against the oracle's float16 `ref`: f16_close wherever the magnitude e^ref is at
    least `floor` of the utterance's maximum.  Returns the bit-identical fraction over the checked elements."""
    mask = np.exp(ref.astype(np.float64)) >= floor * np.exp(ref.astype(np.float64)).max()
    bad = ~f16_close(got, ref)[mask]
    assert not bad.any(), int(bad.sum())
    return float((f16_ulp_distance(got, ref)[mask] == 0).mean())


def preprocess(data, r, sr, waves=None):
    """preprocess.py:168-208 with the deviations of tacotron_b200/preprocess.py (speakers of kept utterances, meta sr).
    waves: the decoded waveforms, or None to load data['audio_files'].  Returns the arrays as written to disk + meta."""
    vocab, ivocab = {"<pad>": 0}, {0: "<pad>"}
    texts, mels, stfts, kept = [], [], [], []
    for i, text in enumerate(data["prompts"]):
        ids = []
        for c in text:
            if c not in vocab:
                vocab[c] = len(vocab)
                ivocab[vocab[c]] = c
            ids.append(vocab[c])
        w = waves[i] if waves is not None else load(data["audio_files"][i], sr)
        mel, stft = features(w, r)
        if mel is not None:
            texts.append(ids)
            mels.append(mel.astype(np.float16))
            stfts.append(stft.astype(np.float16))
            kept.append(i)
    out = {"texts": np.zeros((len(texts), max(len(t) for t in texts)), dtype=np.int64),
           "text_lens": np.array([len(t) for t in texts], dtype=np.int64),
           "mels": np.stack(mels), "stfts": np.stack(stfts),
           "speech_lens": np.array([m.shape[0] for m in mels], dtype=np.int64), "kept": np.array(kept)}
    for k, t in enumerate(texts):
        out["texts"][k, :len(t)] = t
    if "speakers" in data:
        out["speakers"] = np.asarray(data["speakers"], dtype=np.int64)[kept]
    out["meta"] = {"vocab": ivocab, "r": r, "sr": sr}
    return out
