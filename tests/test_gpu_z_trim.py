"""GPU tests of the synthesis tail trim (csrc/audio.cu taco_speech_frames and the packed Griffin-Lim kernels;
tacotron_b200.audio.speech_frames / invert_speech; tacotron_b200.test --trim-tail): the end of speech against the
float64 oracle, the packed kernels against their mirrors, each packed utterance bit-identical to the padded inversion
of its truncated spectrogram, a 50-iteration run against the oracle, and the driver end to end."""
import math
import os

import numpy as np
import pytest
import torch
from scipy.io import wavfile

from oracle import audio_oracle as A
from tacotron_b200 import summary as S
from tests import mirror_kernels_trim as MKT
from tests import trim_oracle as TO
from tests.test_gpu_z_audio import _close
from tests.test_gpu_z_summary import _files, _train
from tests.test_summary import _events
from tests.test_trim import trim_cases

pytestmark = pytest.mark.gpu


def _cuda(t):
    return None if t is None else torch.from_numpy(t).cuda()


@pytest.mark.parametrize("r", [1, 2, 5])
def test_speech_frames_match_oracle_on_cpu_cases(r):
    from tacotron_b200 import audio
    for name, spec, scale, shift, want in trim_cases(r):
        got = audio.speech_frames(_cuda(spec), r, stft_mean=_cuda(shift), stft_std=_cuda(scale))
        assert got.dtype == torch.int32 and got.is_cuda
        assert got.cpu().tolist() == TO.speech_frames(spec, r, scale, shift).tolist() == want, name


@pytest.mark.parametrize("B,T,r", [(32, 180, 2), (4, 100, 5)])
def test_speech_frames_at_synthesis_size(B, T, r):
    from tacotron_b200 import audio
    n = 4 * r * (T // 4)
    rng = np.random.RandomState(B)
    ends = [int(n * x) for x in np.linspace(0.15, 1.0, B)]
    scale, shift = (rng.rand(1025 * r) * 2 + 1).astype(np.float32), (rng.randn(1025 * r) * 2 - 5).astype(np.float32)
    spec = TO.speech_like(B, T, r, ends, seed=r, scale=scale, shift=shift)
    assert TO.margin_db(spec, r, scale, shift) >= 0.5
    want = TO.speech_frames(spec, r, scale, shift)
    assert want.tolist() == [4 * r * -(-e // (4 * r)) for e in ends]
    sd = _cuda(spec)
    for _ in range(2):                                          # the same on every run
        got = audio.speech_frames(sd, r, stft_mean=_cuda(shift), stft_std=_cuda(scale))
        assert got.cpu().tolist() == want.tolist()


@pytest.mark.parametrize("r,T,frames", [(2, 12, [16, 8, 24]), (5, 8, [20, 40])])
def test_packed_kernels_match_mirror(r, T, frames):
    from tacotron_b200 import kernels as K
    g = torch.Generator().manual_seed(1)
    B, F = len(frames), 1025
    off = torch.tensor(np.concatenate([[0], np.cumsum(frames)]), dtype=torch.int64)
    N, nmax = int(off[-1]), max(frames)
    spec = torch.randn(B, T, F * r, generator=g) * 0.5
    scale, shift = torch.rand(F * r, generator=g) + 0.5, torch.randn(F * r, generator=g) * 0.1
    pu = torch.rand(N, F, generator=g)
    offd = off.cuda()
    for sc, sh in ((scale, shift), (None, None)):
        mag_c, full_c = torch.empty(N, F), torch.empty(N, F, dtype=torch.complex64)
        MKT.gl_init_packed(full_c, mag_c, spec, pu, off, r, nmax, sc, sh)
        mag_g, full_g = torch.full((N, F), math.nan, device="cuda"), torch.full((N, F), math.nan, dtype=torch.complex64, device="cuda")
        K.gl_init_packed(full_g, mag_g, spec.cuda(), pu.cuda(), offd, r, nmax, None if sc is None else sc.cuda(),
                         None if sh is None else sh.cuda())
        _close(mag_g, mag_c, 1e-5); _close(full_g, full_c, 1e-5)
    fr = torch.randn(N, 2048, generator=g)
    y_c = torch.empty(300 * (N - B)); MKT.gl_ola_packed(y_c, fr, off, nmax, 300, 1200)
    y_g = torch.full((300 * (N - B),), math.nan, device="cuda"); K.gl_ola_packed(y_g, fr.cuda(), offd, nmax, 300, 1200)
    _close(y_g, y_c, 1e-5)
    f_c = torch.empty(N, 2048); MKT.gl_frame_packed(f_c, y_c, off, nmax, 300, 1200)
    f_g = torch.full((N, 2048), math.nan, device="cuda"); K.gl_frame_packed(f_g, y_c.cuda(), offd, nmax, 300, 1200)
    _close(f_g, f_c, 1e-5)


@pytest.mark.parametrize("n_iter", [0, 3])
@pytest.mark.parametrize("r,T,frames", [(1, 12, [8, 12, 8]), (2, 12, [8, 24, 16]), (5, 8, [20, 40, 20])])
def test_packed_utterance_is_bit_identical_to_the_padded_inversion(r, T, frames, n_iter):
    from tacotron_b200 import audio
    g = torch.Generator().manual_seed(7)
    B, n = len(frames), 4 * r * (T // 4)
    spec = (torch.randn(B, T, 1025 * r, generator=g) * 0.5).cuda()
    mean, std = (torch.randn(1025 * r, generator=g) * 0.1).cuda(), (torch.rand(1025 * r, generator=g) + 0.5).cuda()
    pu = torch.rand(B, n, 1025, generator=g).cuda()
    packed = torch.cat([pu[b, :frames[b]] for b in range(B)])
    ys = audio.invert_speech(spec, r, torch.tensor(frames, dtype=torch.int32).cuda(), n_iter=n_iter, stft_mean=mean,
                             stft_std=std, phase_u=packed)
    for b in range(B):
        ref = audio.invert_spectrogram(spec[b:b + 1, :frames[b] // r], r, n_iter=n_iter, stft_mean=mean, stft_std=std,
                                       phase_u=pu[b:b + 1, :frames[b]])[0]
        assert ys[b].shape == (300 * (frames[b] - 1),)
        assert torch.equal(ys[b], ref), b


def test_fifty_iterations_on_the_kept_frames_converge_like_the_oracle():
    """C5-shaped (T = 100, r = 5): 300 frames of speech-like magnitude, then padding; speech_frames keeps 300 of the 500
    frames and 50 iterations over them reach the oracle's spectral convergence on the truncated spectrogram"""
    from tacotron_b200 import audio
    g = torch.Generator().manual_seed(11)
    r, T = 5, 100
    n, keep = 4 * r * (T // 4), 300
    t = torch.linspace(0, 1, n)[:, None]; k = torch.linspace(0, 1, 1025)[None, :]
    logmag = -3.0 * k + 1.5 * torch.sin(2 * math.pi * (3 * t + 8 * k * (1 + 0.3 * torch.sin(2 * math.pi * 2 * t)))) - 1.0
    logmag[keep:] = float(TO.PAD_LOG)
    spec = audio.reshape_frames(logmag.t().contiguous(), r, forward=True)[None].contiguous()          # [1, T, 1025*r]
    frames = audio.speech_frames(spec.cuda(), r)
    assert frames.cpu().tolist() == [keep]
    pu = torch.rand(keep, 1025, generator=g)
    y = audio.invert_speech(spec.cuda(), r, frames, n_iter=50, phase_u=pu.cuda())[0].cpu().double().numpy()
    assert y.shape == (300 * (keep - 1),)
    ref = A.invert_spectrogram(spec[0, :keep // r].double().numpy(), r, np.exp(2j * np.pi * pu.double().numpy().T), n_iter=50)
    mag = np.exp(logmag[:keep].double().numpy().T)

    def sc(w):
        return np.linalg.norm(np.abs(A.stft(w)) - mag) / np.linalg.norm(mag)
    s_gpu, s_ref = sc(y), sc(ref)
    assert abs(s_gpu - s_ref) <= 0.1 * s_ref + 1e-3, (s_gpu, s_ref)


def _synth(monkeypatch, **kw):
    from tacotron_b200 import audio
    from tacotron_b200 import test as synth
    from tacotron_b200.models.tacotron import Config, Tacotron
    seen = []
    real = audio.speech_frames

    def spy(spec, r, **a):
        out = real(spec, r, **a)
        seen.append((spec.clone(), r, a, out.clone()))
        return out
    monkeypatch.setattr(audio, "speech_frames", spy)
    cfg = Config()
    cfg.data_path, cfg.save_path = "data/toy/", "toy/tacotron"
    torch.manual_seed(0)
    waves = synth.test(Tacotron, cfg, ["abc de\n", "hello, you\n", "abc de\n"], log=lambda *a: None, **kw)
    torch.cuda.synchronize()
    monkeypatch.setattr(audio, "speech_frames", real)
    return waves, seen


def test_synthesis_driver_trim_tail(tmp_path, monkeypatch):
    import shutil
    from tacotron_b200 import audio
    _train(str(tmp_path), monkeypatch, False)
    out = "log/toy/tacotron/test"
    # without the flag: every file byte-identical to a run that never passes it
    _synth(monkeypatch)
    plain = _files(out)
    shutil.rmtree(out)
    _, seen = _synth(monkeypatch, trim_tail=False)
    assert not seen and _files(out) == plain
    shutil.rmtree(out)
    # with it: the files end where speech_frames says the speech ends
    waves, seen = _synth(monkeypatch, trim_tail=True, summary_dir=out)
    assert len(seen) == 1
    spec, r, a, frames = seen[0]
    assert a["stft_mean"] is not None and a["stft_std"] is not None
    frames = frames.cpu().tolist()
    assert frames == audio.speech_frames(spec, r, **a).cpu().tolist()
    n = 4 * r * (spec.shape[1] // 4)
    assert all(f % (4 * r) == 0 and 5 <= f <= n for f in frames)
    ev = _events(out)
    assert len(ev) == 4
    for b in range(3):
        wave, al = waves[b].cpu().numpy(), np.load(f"{out}/{b}_attention.npy")
        assert wave.shape == (300 * (frames[b] - 1),)
        assert al.shape[0] == frames[b] // r
        rate, samples = wavfile.read(f"{out}/{b}.wav")
        assert rate == 16000 and samples.shape == wave.shape
        au, im = ev[b + 1][3][0][1].audio, ev[b + 1][3][1][1].image
        assert au.encoded_audio_string == S.wav_bytes(wave, 16000) and au.length_frames == wave.size
        assert (im.height, im.width) == S.attention_rgba(al).shape[:2]
    assert os.path.exists(f"{out}/0.txt")
