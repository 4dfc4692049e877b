"""Preprocessing without a GPU: the float64 oracle (tests/feature_oracle.py) against the reference's own outputs, the mel
basis against torchaudio, trim bounds on hand-built signals, the WAV reader, the r check, the batched extraction and the
driver over the torch-CPU mirrors (tests/mirror_kernels_features.py), and the three kernel sources of csrc/features.cu under
the host emulation."""
import ctypes as C
import os
import pickle

import numpy as np
import pytest
import torch

from oracle import audio_oracle as A
from tacotron_b200 import audio, preprocess as P
from tests import feature_oracle as FO
from tests import mirror_kernels_features as MKF
from tests.emulator import emu  # noqa: F401  (the emulated library, built once per process)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_preprocess.npz")


def _fixture():
    fx = np.load(GOLDEN)
    waves = [fx[f"wave{i}"].astype(np.float32) / np.float32(32768) for i in range(4)]
    data = {"prompts": [str(p) for p in fx["prompts"]], "speakers": [0, 1, 1, 0]}
    return fx, waves, data


def _write_wav(path, sr, x, bits24=False):
    """scipy.io.wavfile.write, plus hand-built 24-bit PCM (which scipy reads but cannot write)"""
    from scipy.io import wavfile
    if not bits24:
        wavfile.write(path, sr, x)
        return
    ch = 1 if x.ndim == 1 else x.shape[1]
    raw = x.astype("<i4").reshape(-1).view(np.uint8).reshape(-1, 4)[:, 1:].tobytes()      # top 3 bytes of left-justified x
    fmt = (1).to_bytes(2, "little") + ch.to_bytes(2, "little") + sr.to_bytes(4, "little") + (sr * 3 * ch).to_bytes(4, "little") \
        + (3 * ch).to_bytes(2, "little") + (24).to_bytes(2, "little")
    body = b"WAVE" + b"fmt " + len(fmt).to_bytes(4, "little") + fmt + b"data" + len(raw).to_bytes(4, "little") + raw
    with open(path, "wb") as f:
        f.write(b"RIFF" + len(body).to_bytes(4, "little") + body)


def _arctic(root, waves, prompts, sr=16000):
    os.makedirs(os.path.join(root, "arctic", "etc"), exist_ok=True)
    os.makedirs(os.path.join(root, "arctic", "wav"), exist_ok=True)
    with open(os.path.join(root, "arctic", "etc", "arctic.data"), "w") as f:
        for i, p in enumerate(prompts):
            f.write(f'( arctic_a{i:04d} "{p}" )\n')
    for i, w in enumerate(waves):
        _write_wav(os.path.join(root, "arctic", "wav", f"arctic_a{i:04d}.wav"), sr, w)


def test_oracle_reproduces_reference_preprocess():
    fx, waves, data = _fixture()
    out = FO.preprocess(data, r=2, sr=16000, waves=waves)
    assert list(out["kept"]) == [0, 1, 3]                                     # utterance 2 is too long after trimming
    for k in ("texts", "text_lens", "mels", "stfts", "speech_lens"):
        assert out[k].dtype == fx[k].dtype and np.array_equal(out[k], fx[k]), k
    assert np.array_equal(out["speakers"], fx["speakers"][out["kept"]])        # the reference saves all four
    vocab = dict(zip(fx["vocab_ids"].tolist(), [str(c) for c in fx["vocab_chars"]]))
    assert out["meta"]["vocab"] == vocab and "Z" in vocab.values()             # a dropped utterance's characters count
    assert int(fx["r"]) == 2 and int(fx["sr"]) == 16000


def test_mel_basis_against_torchaudio_and_filter_ranges():
    ta = pytest.importorskip("torchaudio")
    ref = ta.functional.melscale_fbanks(1025, 0.0, 11025.0, 80, 22050, norm="slaney", mel_scale="slaney").t().double().numpy()
    ob = FO.mel_basis()
    basis, lo, hi = audio.mel_basis()
    assert basis.dtype == np.float32 and np.array_equal(basis, ob)
    assert np.abs(ob - ref).max() <= 1e-5 * ref.max()
    nz = basis != 0
    widths = nz.sum(1)
    assert (widths > 0).all() and widths.max() <= 83 and nz.sum(0).max() <= 2
    for m in range(80):
        idx = np.flatnonzero(nz[m])
        assert lo[m] == idx[0] and hi[m] == idx[-1] + 1 and hi[m] - lo[m] == len(idx)


def _tone_case(s0, s1, n):
    """square wave +-0.5 on [s0, s1), +-1e-4 (-74 dB) elsewhere; the expected trim span from the frame geometry:
    frame f sees samples [512 f - 1024, 512 f + 1024), and any loud sample makes it non-silent"""
    x = np.where(np.arange(n) % 2 == 0, 1e-4, -1e-4)
    x[s0:s1] = np.where(np.arange(s1 - s0) % 2 == 0, 0.5, -0.5)
    first = max(0, -(-(s0 - 1023) // 512))
    last = min(n // 512, (s1 - 1 + 1024) // 512)
    return x.astype(np.float32), (first * 512, min(n, (last + 1) * 512))


TRIM_CASES = [(512 * 5 + 1023, 40000 - 1500, 40000), (512 * 5 + 1024, 512 * 60 - 1024, 40000),
              (512 * 5 + 1022, 512 * 60 - 1023, 40000 + 7)]


def test_trim_bounds_hand_built():
    waves, expect = [], []
    for s0, s1, n in TRIM_CASES:
        x, e = _tone_case(s0, s1, n)
        waves.append(x); expect.append(e)
    waves.append(np.zeros(5000, np.float32)); expect.append((0, 5000))          # all zero: everything is kept
    for x, e in zip(waves, expect):
        assert tuple(FO.trim(x)[1]) == e
    offsets = torch.tensor(np.concatenate([[0], np.cumsum([len(w) for w in waves])]))
    bounds = torch.zeros(len(waves), 2, dtype=torch.int32)
    MKF.trim_bounds(bounds, torch.from_numpy(np.concatenate(waves)), offsets, 2048, 512, 60.0)
    assert [tuple(b) for b in bounds.tolist()] == expect


def test_wav_reader_formats(tmp_path):
    rng = np.random.RandomState(0)
    x16 = rng.randint(-32768, 32767, size=3000).astype(np.int16)
    x24 = rng.randint(-2 ** 23, 2 ** 23, size=3000).astype(np.int32) * 256      # 24-bit samples, left-justified
    x32 = rng.randint(-2 ** 31, 2 ** 31 - 1, size=3000).astype(np.int32)
    xu8 = rng.randint(0, 256, size=3000).astype(np.uint8)
    xf = (rng.randn(3000) * 0.3).astype(np.float32)
    st = rng.randint(-32768, 32767, size=(3000, 2)).astype(np.int16)
    cases = [("i16", x16, False, x16.astype(np.float64) / 32768), ("i24", x24, True, (x24 // 256).astype(np.float64) / 2 ** 23),
             ("i32", x32, False, x32.astype(np.float64) / 2 ** 31), ("u8", xu8, False, (xu8.astype(np.float64) - 128) / 128),
             ("f32", xf, False, xf.astype(np.float64)),
             ("stereo", st, False, ((st[:, 0].astype(np.float32) / 32768) + (st[:, 1].astype(np.float32) / 32768)) / 2)]
    for name, x, b24, want in cases:
        p = str(tmp_path / f"{name}.wav")
        _write_wav(p, 16000, x, bits24=b24)
        got = audio.load_wav(p, 16000)
        assert got.dtype == np.float32 and got.ndim == 1
        assert np.array_equal(got, np.asarray(want, dtype=np.float32)), name
        assert np.array_equal(got, FO.load(p, 16000)), name
    p = str(tmp_path / "rate.wav")
    _write_wav(p, 22050, x16)
    with pytest.raises(ValueError, match="rate.wav.*22050"):
        audio.load_wav(p, 16000)


def test_r4_and_unsupported_r_are_rejected(tmp_path):
    for r in (1, 2, 3, 5, 6):
        assert audio.feature_frames_per_utterance(r) == 108000 // (300 * r)
    for r in (4, 7, 0):
        with pytest.raises(ValueError, match=f"r = {r} is not supported"):
            audio.feature_frames_per_utterance(r)
    with pytest.raises(ValueError, match="r = 4"):
        P.main(["arctic", "--data-dir", str(tmp_path), "-r", "4"])


def test_short_utterance_is_rejected():
    with pytest.raises(ValueError, match="1024 samples"):
        audio.process_audio_batch([np.zeros(3000, np.float32), np.ones(1024, np.float32)], 2, K=MKF, device="cpu")


def _close_linear(got, ref, tol=2e-5):
    """|e^a - e^b| <= tol * max e^b over one utterance's log-spectrogram"""
    a, b = np.exp(np.asarray(got, np.float64)), np.exp(np.asarray(ref, np.float64))
    err = np.abs(a - b).max() / b.max()
    assert err <= tol, err


def test_process_audio_batch_over_mirrors_matches_oracle():
    fx, waves, _ = _fixture()
    for r in (2, 5):
        mel, stft, keep = audio.process_audio_batch(waves, r, K=MKF, device="cpu", out_dtype=torch.float32)
        assert keep.tolist() == [True, True, False, True]
        for j, i in enumerate((0, 1, 3)):
            om, os_ = FO.features(waves[i], r)
            assert mel[j].shape == om.shape and stft[j].shape == os_.shape
            _close_linear(mel[j].numpy(), om)
            _close_linear(stft[j].numpy(), os_)


def test_driver_over_mirrors(tmp_path):
    fx, waves, data = _fixture()
    root = str(tmp_path / "data")
    _arctic(root, [fx[f"wave{i}"] for i in range(4)], data["prompts"])
    d = P.prepare_arctic(root)
    assert d["prompts"] == data["prompts"]
    d["speakers"] = data["speakers"]
    out_dir = os.path.join(root, "arctic")
    n = P.preprocess(d, out_dir, r=2, sr=16000, chunk=3, K=MKF, device="cpu", log=lambda *a: None)
    assert n == 3
    ref = FO.preprocess(data, r=2, sr=16000, waves=waves)
    for k in ("texts", "text_lens", "speech_lens", "speakers"):
        got = np.load(os.path.join(out_dir, k + ".npy"))
        assert got.dtype == ref[k].dtype and np.array_equal(got, ref[k]), k
    for k in ("mels", "stfts"):
        got = np.load(os.path.join(out_dir, k + ".npy"))
        assert got.dtype == np.float16 and got.shape == ref[k].shape, k
        for j in range(n):
            # float32 arithmetic against float64: every element within one float16 step; near the 1e-4 floor a float32
            # error of ~1e-3 relative moves a value across a rounding boundary of float16 now and then (97.7 %
            # bit-identical measured on the quietest mel here)
            assert FO.check_f16(got[j], ref[k][j]) > 0.95
        assert os.path.getsize(os.path.join(out_dir, k + ".npy")) == 128 + got.nbytes
    with open(os.path.join(out_dir, "meta.pkl"), "rb") as f:
        assert pickle.load(f) == ref["meta"]
    from tacotron_b200 import data_input
    arrays, names, num_speakers, _, _ = data_input.load_from_npy(out_dir + "/")
    assert arrays["stft"].shape == (3, 180, 2050) and num_speakers == 2


# ---- the kernel sources under the host emulation ----
def _p(t):
    return C.c_void_p(t.data_ptr())


def test_feature_kernels_under_emulation(emu):
    ok = lambda rc: rc == 0 or pytest.fail(emu.taco_last_error().decode())
    # trim: the hand-built cases plus the all-zero signal, one CTA each
    waves = [_tone_case(*c)[0] for c in TRIM_CASES] + [np.zeros(3000, np.float32)]
    y = torch.from_numpy(np.concatenate(waves))
    offsets = torch.tensor(np.concatenate([[0], np.cumsum([len(w) for w in waves])]))
    want, got = torch.zeros(len(waves), 2, dtype=torch.int32), torch.full((len(waves), 2), -7, dtype=torch.int32)
    MKF.trim_bounds(want, y, offsets, 2048, 512, 60.0)
    ok(emu.taco_trim_bounds(_p(got), _p(y), _p(offsets), len(waves), 2048, 512, 60.0, None))
    assert torch.equal(got, want)
    # frames -> FFT -> spectra at a reduced max_len (11 frames), ragged spans, both output dtypes
    g = torch.Generator().manual_seed(4)
    max_len, hop, B = 3000, 300, 3
    n = 1 + max_len // hop
    y = torch.randn(9000, generator=g) * 0.3
    start = torch.tensor([0, 2500, 6000], dtype=torch.int64)
    length = torch.tensor([3000, 1025, 2200], dtype=torch.int32)
    fr_c, fr_e = torch.empty(B, n, 2048), torch.full((B, n, 2048), float("nan"))
    MKF.feature_frames(fr_c, y, start, length, max_len, hop, 1200, 0.97)
    ok(emu.taco_feature_frames(_p(fr_e), _p(y), _p(start), _p(length), B, n, max_len, hop, 2048, 1200, 0.97, None))
    assert (fr_e - fr_c).abs().max().item() <= 1e-6 * fr_c.abs().max().item()
    X = torch.empty(B, n, 1025, dtype=torch.complex64)
    ok(emu.taco_rfft2048(_p(X), _p(fr_e), B * n, None))
    basis, lo, hi = (torch.from_numpy(a) for a in audio.mel_basis())
    for r, dt in ((2, torch.float32), (1, torch.float16)):
        T = 4 * (n // (4 * r))
        s_c, m_c = torch.empty(B, T, 1025 * r, dtype=dt), torch.empty(B, T, 80 * r, dtype=dt)
        MKF.feature_spec(s_c, m_c, X, basis, lo, hi, r)
        s_e, m_e = torch.full_like(s_c, float("nan")), torch.full_like(m_c, float("nan"))
        ok(emu.taco_feature_spec(_p(s_e), _p(m_e), int(dt == torch.float16), _p(X), _p(basis), _p(lo), _p(hi), B, n, r, 80, None))
        for e_, c_ in ((s_e, s_c), (m_e, m_c)):
            assert not torch.isnan(e_).any()
            if dt == torch.float16:                  # the same float32 values up to rounding order, then one rounding each
                assert FO.f16_close(e_.numpy(), c_.numpy()).all()
            else:
                diff = (e_.double().exp() - c_.double().exp()).abs().max().item()
                assert diff <= 1e-5 * c_.double().exp().max().item(), (r, diff)
