"""-m gpu: fast Griffin-Lim (momentum) and de-emphasis of synthesised waveforms on the H100.

  1. taco_gl_phase_momentum against float64 over its whole range (zero, tiny and huge values; counts around the block and
     the grid stride);
  2. momentum inversions against the float64 oracle, the C5 shape's convergence, and the voiced test signal's ordering
     (25 momentum iterations closer than 50 plain ones);
  3. momentum = 0 given explicitly is the default call's bits (padded, packed, CUDA graph); packed = padded per
     utterance with momentum on; the graph replays equal eager;
  4. taco_de_emphasis against float64 lfilter on the layouts synthesis uses, its determinism, and pre-/de-emphasis
     round trips;
  5. the synthesis driver end to end with the flags, on the toy checkpoint."""
import math
import os
import shutil

import numpy as np
import pytest
import torch

from oracle import audio_oracle as A
from tacotron_b200 import audio
from tests import griffin_lim_oracle as G

pytestmark = pytest.mark.gpu
GRID_STRIDE = 132 * 32 * 256          # grid_for's largest grid times the block


def _K():
    from tacotron_b200 import kernels
    return kernels


# ---------------------------------------------------------------------------------------------------------------------
# 1. the phase update
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("count", [1, 255, 256, 257, GRID_STRIDE - 1, GRID_STRIDE, 2 * GRID_STRIDE + 77])
def test_gl_phase_momentum_against_float64(count):
    g = torch.Generator().manual_seed(count % 1000)
    scale = torch.tensor([0.0, 1e-30, 1e-6, 1.0, 1e6, 1e30])
    mag = torch.rand(count, generator=g) * scale[torch.randint(0, 6, (count,), generator=g)]
    vs = torch.tensor([0.0, 1e-20, 1e-3, 1.0, 1e3, 1e18])

    def cplx():
        s = vs[torch.randint(0, 6, (count,), generator=g)]
        return torch.complex(torch.randn(count, generator=g) * s, torch.randn(count, generator=g) * s)
    reb, prev = cplx(), cplx()
    reb[: min(count, 3)] = 0
    prev[: min(count, 2)] = 0                      # d = 0 in the first two elements
    K = _K()
    for beta in (0.0, 0.99 / 1.99, 0.5):
        got = torch.empty(count, dtype=torch.complex64, device="cuda")
        K.gl_phase_momentum(got, mag.cuda(), reb.cuda(), prev.cuda(), beta)
        got = got.cpu().numpy().astype(np.complex128)
        want = G.phase_momentum(mag.double().numpy(), reb.numpy(), prev.numpy(), float(np.float32(beta)))
        err = np.abs(got - want)
        assert (err <= 1e-5 * np.abs(want)).all(), (beta, err.max())
        if beta == 0.0:
            plain = torch.empty(count, dtype=torch.complex64, device="cuda")
            K.gl_phase(plain, mag.cuda(), reb.cuda())
            assert np.array_equal(plain.cpu().numpy(), got.astype(np.complex64))


# ---------------------------------------------------------------------------------------------------------------------
# 2. inversions against the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("r,T,n_iter", [(2, 8, 3), (5, 8, 2)])
def test_momentum_inversion_matches_oracle(r, T, n_iter):
    g = torch.Generator().manual_seed(7)
    B = 2
    spec = torch.randn(B, T, 1025 * r, generator=g) * 0.5
    mean, std = torch.randn(1025 * r, generator=g) * 0.1, torch.rand(1025 * r, generator=g) + 0.5
    n = 4 * r * (T // 4)
    pu = torch.rand(B, n, 1025, generator=g)
    y = audio.invert_spectrogram(spec.cuda(), r, n_iter=n_iter, stft_mean=mean.cuda(), stft_std=std.cuda(), phase_u=pu.cuda(),
                                 momentum=0.99)
    for b in range(B):
        ang0 = np.exp(2j * np.pi * pu[b].double().numpy().T)
        ref = G.invert_spectrogram((spec[b] * std + mean).double().numpy(), r, ang0, n_iter, 0.99)
        err = np.abs(y[b].cpu().double().numpy() - ref).max()
        assert err <= 1e-4 * np.abs(ref).max(), (err, np.abs(ref).max())


def test_fifty_momentum_iterations_converge_like_the_oracle():
    """C5-shaped: 500 frames (T=100, r=5), 50 iterations at momentum 0.99"""
    g = torch.Generator().manual_seed(11)
    r, T = 5, 100
    n = 4 * r * (T // 4)
    t = torch.linspace(0, 1, n)[:, None]; k = torch.linspace(0, 1, 1025)[None, :]
    logmag = -3.0 * k + 1.5 * torch.sin(2 * math.pi * (3 * t + 8 * k * (1 + 0.3 * torch.sin(2 * math.pi * 2 * t)))) - 1.0
    spec = audio.reshape_frames(logmag.t().contiguous(), r, forward=True)[None]
    pu = torch.rand(1, n, 1025, generator=g)
    y = audio.invert_spectrogram(spec.cuda().contiguous(), r, n_iter=50, phase_u=pu.cuda(), momentum=0.99)[0]
    ref = G.invert_spectrogram(spec[0].double().numpy(), r, np.exp(2j * np.pi * pu[0].double().numpy().T), 50, 0.99)
    mag = np.exp(logmag.double().numpy().T)
    s_gpu, s_ref = G.spectral_convergence(y.cpu().double().numpy(), mag), G.spectral_convergence(ref, mag)
    assert abs(s_gpu - s_ref) <= 0.1 * s_ref, (s_gpu, s_ref)


def _voiced(r):
    _, y, u = G.voiced_signal(r)
    mag = np.abs(A.stft(y))
    spec = audio.reshape_frames(torch.from_numpy(np.log(np.maximum(mag, 1e-30))).float(), r, forward=True)[None]
    return mag, spec.cuda().contiguous(), torch.from_numpy(u.T.copy()).float()[None].cuda()


def test_momentum_converges_faster_on_the_voiced_signal():
    mag, spec, pu = _voiced(2)
    sc = {}
    for n_iter, m in ((50, 0.0), (25, 0.99)):
        y = audio.invert_spectrogram(spec, 2, n_iter=n_iter, phase_u=pu, momentum=m)[0]
        sc[m] = G.spectral_convergence(y.cpu().double().numpy(), mag)
    assert sc[0.99] < sc[0.0], sc


# ---------------------------------------------------------------------------------------------------------------------
# 3. bits
# ---------------------------------------------------------------------------------------------------------------------
def _case(B, T, r, seed):
    g = torch.Generator().manual_seed(seed)
    spec = (torch.randn(B, T, 1025 * r, generator=g) * 0.5).cuda()
    mean, std = (torch.randn(1025 * r, generator=g) * 0.1).cuda(), (torch.rand(1025 * r, generator=g) + 0.5).cuda()
    return spec, mean, std, g


def test_zero_momentum_is_the_default_call():
    r, T, B = 2, 12, 3
    spec, mean, std, g = _case(B, T, r, 1)
    n = 4 * r * (T // 4)
    pu = torch.rand(B, n, 1025, generator=g).cuda()
    a = audio.griffinlim_batch(spec, r, n_iter=4, scale=std, shift=mean, phase_u=pu)
    b = audio.griffinlim_batch(spec, r, n_iter=4, scale=std, shift=mean, phase_u=pu, momentum=0)
    assert torch.equal(a, b)
    frames = [24, 8, 16]
    pp = torch.rand(sum(frames), 1025, generator=g).cuda()
    ya, sa = audio.invert_speech_packed(spec, r, frames, n_iter=4, stft_mean=mean, stft_std=std, phase_u=pp)
    yb, sb = audio.invert_speech_packed(spec, r, frames, n_iter=4, stft_mean=mean, stft_std=std, phase_u=pp, momentum=0.0)
    assert torch.equal(ya, yb) and np.array_equal(sa, sb)
    ga = audio.GriffinLimGraph(B, T, r, n_iter=4)(spec, stft_mean=mean, stft_std=std, phase_u=pu).clone()
    gb = audio.GriffinLimGraph(B, T, r, n_iter=4, momentum=0)(spec, stft_mean=mean, stft_std=std, phase_u=pu).clone()
    assert torch.equal(ga, gb) and torch.equal(ga, a)


def test_packed_equals_padded_with_momentum():
    r, T = 2, 12
    frames = [24, 8, 16]
    spec, mean, std, g = _case(3, T, r, 2)
    pp = torch.rand(sum(frames), 1025, generator=g).cuda()
    y, start = audio.invert_speech_packed(spec, r, frames, n_iter=5, stft_mean=mean, stft_std=std, phase_u=pp, momentum=0.99)
    off = np.concatenate([[0], np.cumsum(frames)])
    for b, f in enumerate(frames):
        one = audio.invert_spectrogram(spec[b:b + 1, :f // r].contiguous(), r, n_iter=5, stft_mean=mean, stft_std=std,
                                       phase_u=pp[off[b]:off[b + 1]][None].contiguous(), momentum=0.99)[0]
        assert torch.equal(y[start[b]:start[b + 1]], one), b


def test_graph_with_momentum_replays_eager():
    r, T, B = 2, 8, 2
    n = 4 * r * (T // 4)
    glg = audio.GriffinLimGraph(B, T, r, n_iter=5, momentum=0.99)
    assert isinstance(glg.rebuilt, tuple) and len(glg.rebuilt) == 2
    for seed in (1, 2):
        spec, mean, std, g = _case(B, T, r, 10 + seed)
        pu = torch.rand(B, n, 1025, generator=g).cuda()
        eager = audio.invert_spectrogram(spec, r, n_iter=5, stft_mean=mean, stft_std=std, phase_u=pu, momentum=0.99)
        graphed = glg(spec, stft_mean=mean, stft_std=std, phase_u=pu).clone()
        torch.cuda.synchronize()
        assert torch.equal(eager, graphed)


# ---------------------------------------------------------------------------------------------------------------------
# 4. de-emphasis
# ---------------------------------------------------------------------------------------------------------------------
def _check_de_emphasis(x, start, what):
    """x float32 numpy; de-emphasised on the GPU twice (bit-equal) and against float64 lfilter per segment"""
    y = torch.from_numpy(x).cuda()
    y2 = y.clone()
    audio.de_emphasis(y, start)
    audio.de_emphasis(y2, start)
    torch.cuda.synchronize()
    assert torch.equal(y, y2), what
    got = y.cpu().double().numpy()
    want = G.de_emphasis(x.astype(np.float64), start)
    for s, (a, b) in enumerate(zip(start[:-1], start[1:])):
        if b > a:
            err = np.abs(got[a:b] - want[a:b]).max()
            assert err <= 2e-6 * np.abs(want[a:b]).max(), (what, s, b - a, err)
    return got


def test_de_emphasis_padded_rows():
    x = (np.random.default_rng(0).standard_normal((32, 108000)) * 0.1).astype(np.float32)
    y = torch.from_numpy(x).cuda()
    audio.de_emphasis(y)
    want = G.de_emphasis(x.reshape(-1).astype(np.float64), np.arange(33) * 108000).reshape(32, 108000)
    assert np.abs(y.cpu().double().numpy() - want).max() <= 2e-6 * np.abs(want).max()
    _check_de_emphasis(x.reshape(-1), np.arange(33, dtype=np.int64) * 108000, "padded")


def test_de_emphasis_packed_offsets():
    spec, mean, std, g = _case(4, 12, 2, 3)
    y, start = audio.invert_speech_packed(spec, 2, [24, 8, 16, 24], n_iter=2, stft_mean=mean, stft_std=std)
    _check_de_emphasis(y.cpu().numpy(), start, "packed")


def test_de_emphasis_long_form_spans_and_empty_segments():
    rng = np.random.default_rng(1)
    lens = [0, 16000 * 600, 0, 1, 37, 8191, 8192, 8193, 0, 250000]              # one 10-minute line
    start = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    x = (rng.standard_normal(int(start[-1])) * 0.1).astype(np.float32)
    _check_de_emphasis(x, start, "spans")


def test_pre_then_de_emphasis_recovers_the_signal():
    clean, y, _ = G.voiced_signal(2)
    back = torch.from_numpy(y.astype(np.float32)).cuda()
    audio.de_emphasis(back, [0, len(y)])
    assert np.abs(back.cpu().double().numpy() - clean).max() <= 1e-5 * np.abs(clean).max()


# ---------------------------------------------------------------------------------------------------------------------
# 5. the synthesis driver
# ---------------------------------------------------------------------------------------------------------------------
def _drive(monkeypatch, argv, prompts):
    """python -m tacotron_b200.test argv on the toy checkpoint (seed 0) -> {file name: (WAV bytes, the float waveform
    write_wav got)}"""
    import io
    from tacotron_b200 import test as synth
    from tacotron_b200 import train as trainer
    got = {}
    real = trainer.write_wav

    def spy(path, wave, sr):
        real(path, wave, sr)
        got[os.path.basename(path)] = np.array(wave, dtype=np.float32)
    monkeypatch.setattr(trainer, "write_wav", spy)
    monkeypatch.setattr("sys.stdin", io.StringIO("".join(prompts)))
    torch.manual_seed(0)
    synth.main(["-t", "toy", *argv])
    torch.cuda.synchronize()
    monkeypatch.setattr(trainer, "write_wav", real)
    out = "log/toy/tacotron/test"
    files = {k: (open(os.path.join(out, k), "rb").read(), got[k]) for k in got}
    shutil.rmtree(out)
    return files


def test_synthesis_driver_flags(tmp_path, monkeypatch):
    from tests.test_gpu_z_summary import _train
    _train(str(tmp_path), monkeypatch, False)
    prompts = ["abc de\n", "hello, you. and abc de, again\n", "abc de\n"]
    plain = _drive(monkeypatch, [], prompts)
    spelled = _drive(monkeypatch, ["--griffin-lim-iters", "50", "--griffin-lim-momentum", "0"], prompts)
    assert plain.keys() == spelled.keys() and len(plain) == 3
    assert all(plain[k][0] == spelled[k][0] for k in plain)
    new = ["--griffin-lim-momentum", "--griffin-lim-iters", "25", "--de-emphasis"]
    for mode in ([], ["--trim-tail"], ["--stop-at-end"], ["--long-form"]):
        base = plain if not mode else _drive(monkeypatch, mode, prompts)
        opt = _drive(monkeypatch, mode + new, prompts)
        assert base.keys() == opt.keys()
        for k in base:
            assert base[k][1].shape == opt[k][1].shape, (mode, k)
            assert np.isfinite(opt[k][1]).all()
        if mode == ["--long-form"]:                       # per line: lfilter of that line's waveform, no state across lines
            de = _drive(monkeypatch, mode + ["--de-emphasis"], prompts)
            for k in base:
                want = G.de_emphasis(base[k][1].astype(np.float64), [0, base[k][1].size])
                assert np.abs(de[k][1] - want).max() <= 2e-6 * np.abs(want).max(), k
