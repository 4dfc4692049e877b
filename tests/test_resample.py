"""Resampling without a GPU: resampy's kaiser_best table and loop as restated in tests/resample_oracle.py (its filter,
its pass- and stopband, its pinned DC gains, its float64 time register), the torch-CPU mirror of taco_resample
(tests/mirror_kernels_resample.py) bit for bit against the oracle, the kernel source of csrc/resample.cu under the host
emulation, and resampling inside process_audio_batch and the preprocessing driver over the mirrors."""
import ctypes as C
import os
import pickle
from fractions import Fraction

import numpy as np
import pytest
import torch

from tacotron_b200 import audio, preprocess as P
from tests import feature_oracle as FO
from tests import mirror_kernels_resample as MKR
from tests import resample_oracle as RO
from tests.test_features import _close_linear, _write_wav
from tests.emulator import emu  # noqa: F401  (the emulated library, built once per process)

RATES = [(48000, 24000), (44100, 16000), (22050, 16000), (48000, 16000), (16000, 24000), (8000, 16000)]


def _noise(n, seed, amp=0.3):
    return (np.random.RandomState(seed).randn(n) * amp).astype(np.float32)


def _mirror(waves, sr_orig, sr_new):
    """resample_batch's arguments for one ratio, run through the mirror -> list of outputs"""
    ratio = float(sr_new) / sr_orig
    sizes = [audio.resample_lengths(len(w), sr_orig, sr_new) for w in waves]
    in_off = torch.tensor(np.concatenate([[0], np.cumsum([len(w) for w in waves])]))
    out_off = torch.tensor(np.concatenate([[0], np.cumsum([s[1] for s in sizes])]))
    out = torch.full((int(out_off[-1]),), float("nan"))
    wd, step = audio.resample_filter(sr_orig, sr_new)
    treg = torch.from_numpy(audio.resample_register(ratio, max(s[0] for s in sizes)))
    MKR.resample(out, torch.from_numpy(np.concatenate(waves)), in_off, out_off, torch.from_numpy(wd.copy()), step, ratio, treg)
    return [out[out_off[b]:out_off[b + 1]].numpy() for b in range(len(waves))]


def test_filter_table():
    win = RO.kaiser_best()
    assert win.shape == (32769,) and win[0] == RO.ROLLOFF and abs(win[-1]) < 1e-7         # the Kaiser taper's end
    for sr_orig, sr_new in RATES:
        ratio = float(sr_new) / sr_orig
        w, d = RO.filter_table(ratio)
        assert np.array_equal(w, win * ratio if ratio < 1 else win)
        assert d[-1] == 0 and np.array_equal(d[:-1], w[1:] - w[:-1])
        wd, step = audio.resample_filter(sr_orig, sr_new)
        assert wd.dtype == np.float64 and np.array_equal(wd[:, 0], w) and np.array_equal(wd[:, 1], d)
        assert step == int(min(1.0, ratio) * 512)
    assert [audio.resample_filter(*q)[1] for q in RATES] == [256, 185, 371, 170, 512, 512]


@pytest.mark.parametrize("sr_orig,sr_new", RATES)
def test_oracle_is_the_loop(sr_orig, sr_new):
    """the vectorised oracle keeps resample_f's tap order: equal, bit for bit, to the loop written out"""
    for n in (300, 7):
        x = _noise(n, n)
        assert np.array_equal(RO.resample(x, sr_orig, sr_new), RO.resample_loop(x, sr_orig, sr_new))


def _amplitude(y, f, sr):
    t = np.arange(len(y)) / sr
    A = np.stack([np.sin(2 * np.pi * f * t), np.cos(2 * np.pi * f * t)], 1)
    return float(np.hypot(*np.linalg.lstsq(A, y.astype(np.float64), rcond=None)[0]))


def _tone(f, n, sr, sr_new):
    y = RO.resample((0.5 * np.sin(2 * np.pi * f * np.arange(n) / sr)).astype(np.float32), sr, sr_new)
    return y[len(y) // 4:3 * len(y) // 4]


@pytest.mark.parametrize("sr_orig,sr_new,tol", [(48000, 24000, 4e-7), (16000, 24000, 1.7e-6)])
def test_passband(sr_orig, sr_new, tol):
    """tones up to 0.85 of the lower Nyquist keep their 0.5 amplitude (measured 1.2e-7 and 1.05e-6 off)"""
    low = min(sr_orig, sr_new) / 2
    for f in np.linspace(100, 0.85 * low, 12):
        assert abs(_amplitude(_tone(f, 24000, sr_orig, sr_new), f, sr_new) - 0.5) <= tol, f


def test_stopband_48_to_24():
    """tones above 1.05 x the 12 kHz target Nyquist are gone (measured peak 1.35e-7 of the signal's 0.5)"""
    for f in np.linspace(1.05 * 12000, 23000, 10):
        assert np.abs(_tone(f, 24000, 48000, 24000)).max() <= 2e-7, f


def test_matches_long_kaiser_resample_poly_48_to_24():
    """band-limited noise (below 0.7 x 12 kHz) through the oracle and through scipy's polyphase resampler with a long
    Kaiser low-pass agree within 2e-6 of max|x| (measured 8.7e-7)"""
    from scipy import signal
    b = signal.firwin(2001, 0.7 * 12000, fs=48000, window=("kaiser", 12.0))
    x = signal.lfilter(b, 1, np.random.RandomState(1).randn(96000))[4000:]
    x = (x / np.abs(x).max()).astype(np.float32)
    y = RO.resample(x, 48000, 24000)
    h = signal.firwin(2 * 128 * 2 + 1, 0.5, window=("kaiser", RO.BETA))
    z = signal.resample_poly(x.astype(np.float64), 1, 2, window=h)
    m = len(y)
    assert np.abs(y[m // 8:7 * m // 8] - z[m // 8:7 * m // 8]).max() <= 2e-6


@pytest.mark.parametrize("sr_orig,gain", [(44100, 1.00274), (48000, 1.00272), (22050, 1.00057)])
def test_pinned_dc_gain(sr_orig, gain):
    """resampy 0.2's truncated step (185.76 -> 185, 170.67 -> 170, 371.52 -> 371) over-samples the table: the DC gain
    peaks at these values.  This is the arithmetic being reproduced, not a defect to fix here."""
    y = RO.resample(np.ones(60000, np.float32), sr_orig, 16000)
    c = y[len(y) // 4:3 * len(y) // 4]
    assert abs(float(c.max()) - gain) <= 5e-6
    assert c.min() >= 1.0 + 0.6 * (gain - 1.0)


def test_time_register_is_the_sequential_sum():
    ratio = 16000 / 44100
    treg = audio.resample_register(ratio, 50000)
    assert np.array_equal(treg, RO.time_register(ratio, 50000))
    assert np.array_equal(audio.resample_register(ratio, 70000)[:50000], treg)          # growing keeps the prefix
    # exact rational positions t * 44100 / 16000 would not reproduce the register's arithmetic
    x = _noise(20000, 2)
    n_out = RO.lengths(len(x), 44100, 16000)[0]
    exact = np.array([float(Fraction(t * 44100, 16000)) for t in range(n_out)])
    assert not np.array_equal(exact, treg[:n_out])
    a, b = RO.resample(x, 44100, 16000), RO.resample(x, 44100, 16000, treg=exact)
    assert np.abs(a - b).max() > 1e-4


def _case_lengths(sr_orig, sr_new):
    """the fewest samples that give an output (one output, or two at 8 -> 16 kHz), shorter than a wing, odd (a zero
    tail wherever ratio * odd is not an integer), and long"""
    ratio = float(sr_new) / sr_orig
    one = 1
    while int(one * ratio) < 1:
        one += 1
    return [one, 100, 1001, 100001, 250000]


@pytest.mark.parametrize("sr_orig,sr_new", RATES)
def test_mirror_is_bit_identical_to_oracle(sr_orig, sr_new):
    lens = _case_lengths(sr_orig, sr_new)
    waves = [_noise(n, k) for k, n in enumerate(lens)]
    got = _mirror(waves, sr_orig, sr_new)
    tails = 0
    for w, g in zip(waves, got):
        n_out, n_fix = RO.lengths(len(w), sr_orig, sr_new)
        ref = RO.resample(w, sr_orig, sr_new)
        assert g.shape == ref.shape == (n_fix,) and np.array_equal(g, ref), len(w)
        tails += n_fix - n_out
    assert RO.lengths(lens[0], sr_orig, sr_new)[0] == (2 if sr_new == 2 * sr_orig else 1)
    assert tails > 0 or sr_new % sr_orig == 0


def test_too_short_to_resample_names_the_file(tmp_path):
    root = str(tmp_path / "data")
    waves = [_noise(30000, 0), _noise(1, 1)]
    from tests.test_features import _arctic
    _arctic(root, [w for w in waves], ["first one", "second"], sr=48000)
    with pytest.raises(ValueError, match="arctic_a0001.wav.*1 samples at 48000 Hz"):
        P.preprocess(P.prepare_arctic(root), os.path.join(root, "arctic"), sr=24000, K=MKR, device="cpu",
                     log=lambda *a: None, resample=True)
    with pytest.raises(ValueError, match="too few to resample"):
        audio.resample_lengths(2, 48000, 16000)


# ---- the kernel source under the host emulation ----
def _p(t):
    return C.c_void_p(t.data_ptr())


@pytest.mark.parametrize("sr_orig,sr_new", [(48000, 24000), (44100, 16000), (16000, 24000)])
def test_resample_kernel_under_emulation(emu, sr_orig, sr_new):
    ok = lambda rc: rc == 0 or pytest.fail(emu.taco_last_error().decode())
    ratio = float(sr_new) / sr_orig
    waves = [_noise(n, n) for n in (_case_lengths(sr_orig, sr_new)[0], 100, 1001)]
    sizes = [audio.resample_lengths(len(w), sr_orig, sr_new) for w in waves]
    in_off = torch.tensor(np.concatenate([[0], np.cumsum([len(w) for w in waves])]))
    out_off = torch.tensor(np.concatenate([[0], np.cumsum([s[1] for s in sizes])]))
    y = torch.from_numpy(np.concatenate(waves))
    wd, step = audio.resample_filter(sr_orig, sr_new)
    wd = torch.from_numpy(wd.copy())
    n_out = max(s[0] for s in sizes)
    treg = torch.from_numpy(audio.resample_register(ratio, n_out))
    want, got = torch.empty(int(out_off[-1])), torch.full((int(out_off[-1]),), float("nan"))
    MKR.resample(want, y, in_off, out_off, wd, step, ratio, treg)
    ok(emu.taco_resample(_p(got), _p(y), _p(in_off), _p(out_off), len(waves), _p(wd), wd.shape[0], step, ratio, _p(treg),
                         n_out, None))
    assert torch.equal(got, want)
    # argument checks
    assert emu.taco_resample(_p(got), _p(y), _p(in_off), _p(out_off), len(waves), _p(wd), wd.shape[0], 0, ratio, _p(treg),
                             n_out, None) != 0
    assert b"step" in emu.taco_last_error()
    assert emu.taco_resample(None, _p(y), _p(in_off), _p(out_off), len(waves), _p(wd), wd.shape[0], step, ratio, _p(treg),
                             n_out, None) != 0


# ---- resampling inside the feature extraction and the driver, over the mirrors ----
def _speech(n, sr, seed):
    rng = np.random.RandomState(seed)
    head, tail = n // 8, n // 10
    t = np.arange(n - head - tail) / sr
    x = 0.2 * rng.randn(len(t)) * (0.6 + 0.4 * np.sin(2 * np.pi * 3 * t)) + 0.3 * np.sin(2 * np.pi * rng.uniform(100, 400) * t)
    return np.concatenate([rng.randn(head) * 3e-5, x, rng.randn(tail) * 3e-5]).astype(np.float32)


def test_process_audio_batch_resamples_over_mirrors():
    waves = [_speech(60000, 48000, 0), _speech(30000, 24000, 1), _speech(40001, 48000, 2)]
    rates = [48000, 24000, 48000]
    mel, stft, keep = audio.process_audio_batch(waves, 2, K=MKR, device="cpu", out_dtype=torch.float32, rates=rates, sr=24000)
    assert keep.tolist() == [True, True, True]
    for j, (w, q) in enumerate(zip(waves, rates)):
        x = RO.resample(w, q, 24000) if q != 24000 else w
        om, os_ = FO.features(x, 2)
        _close_linear(mel[j].numpy(), om)
        _close_linear(stft[j].numpy(), os_)
    # the 1025-sample minimum applies after resampling: 2047 samples at 48 kHz give 1024 at 24 kHz
    with pytest.raises(ValueError, match="utterance 1 has 1024 samples"):
        audio.process_audio_batch([waves[1], _noise(2047, 3)], 2, K=MKR, device="cpu", rates=[24000, 48000], sr=24000)
    # resample_batch: the public form, an utterance already at sr is returned as it is
    out = audio.resample_batch(waves, rates, 24000, K=MKR, device="cpu")
    assert np.array_equal(out[1], waves[1]) and np.array_equal(out[0], RO.resample(waves[0], 48000, 24000))


def _vctk(root, rng_seed, sr):
    vctk = os.path.join(root, "vctk")
    os.makedirs(vctk)
    with open(os.path.join(vctk, "speaker-info.txt"), "w") as f:
        f.write("ID  AGE  GENDER  ACCENTS  REGION\n225  23  F  English  Southern\n226  22  M  English  Surrey\n")
    lengths = {"225": [40000, 260000], "226": [30000]}                                # p225_002 is too long: dropped
    k = 0
    for uid, ls in lengths.items():
        os.makedirs(os.path.join(vctk, "txt", f"p{uid}"))
        os.makedirs(os.path.join(vctk, "wav48", f"p{uid}"))
        for j, n in enumerate(ls):
            name = f"p{uid}_{j + 1:03d}"
            with open(os.path.join(vctk, "txt", f"p{uid}", name + ".txt"), "w") as f:
                f.write(f"Utterance {j} of speaker {uid}.\n")
            w = _speech(n, sr, rng_seed + k)
            if n > 216000:
                w = (0.5 * np.sin(2 * np.pi * 220 * np.arange(n) / sr)).astype(np.float32)
            _write_wav(os.path.join(vctk, "wav48", f"p{uid}", name + ".wav"), sr, np.round(w * 32767).astype(np.int16))
            k += 1
    return vctk


def test_driver_resamples_48k_vctk_over_mirrors(tmp_path):
    root = str(tmp_path / "data")
    vctk = _vctk(root, 10, 48000)
    data = P.prepare_vctk(root)
    with pytest.raises(ValueError, match=r"p225_001\.wav: sample rate 48000 Hz, expected 24000 Hz"):
        P.preprocess(data, vctk, r=5, sr=24000, K=MKR, device="cpu", log=lambda *a: None)
    n = P.preprocess(data, vctk, r=5, sr=24000, chunk=2, K=MKR, device="cpu", log=lambda *a: None, resample=True)
    assert n == 2
    waves = [RO.resample(FO.load(f, 48000), 48000, 24000) for f in data["audio_files"]]
    ref = FO.preprocess(data, r=5, sr=24000, waves=waves)
    assert list(ref["kept"]) == [0, 2]
    for k in ("texts", "text_lens", "speech_lens", "speakers"):
        got = np.load(os.path.join(vctk, k + ".npy"))
        assert got.dtype == ref[k].dtype and np.array_equal(got, ref[k]), k
    assert np.load(os.path.join(vctk, "speakers.npy")).tolist() == [0, 1]
    for k in ("mels", "stfts"):
        got = np.load(os.path.join(vctk, k + ".npy"))
        assert got.dtype == np.float16 and got.shape == ref[k].shape, k
        for j in range(n):
            assert FO.check_f16(got[j], ref[k][j]) > 0.95
    with open(os.path.join(vctk, "meta.pkl"), "rb") as f:
        meta = pickle.load(f)
    assert meta == ref["meta"] and meta["sr"] == 24000
