"""The signal-path envelope checks (tests/stft_envelope_checks.py) on CPU, over the host emulation (tests/cuda_emu) of
csrc/audio.cu and csrc/features.cu at small sizes, so that the checks themselves are tested without a GPU.

The emulation runs one CTA after another with one OS thread per CUDA thread (about 20 ms per FFT row), so the FFT runs
one batch past the 528-CTA grid and otherwise a handful of rows; every gl_ola / gl_frame parameter set runs at its
smallest n.  Its sincospif / cospif are the float64 values rounded once (exact
at multiples of 1/2, as on the device), so the same bars hold with more margin.
"""
import pytest
import torch

from tacotron_b200 import audio
from tests import stft_envelope_checks as SE
from tests.emulator import KernelsOver, emu  # noqa: F401  (the emulated library, built once per process)

# (B, n, hop, n_fft, win_length): production at the smallest n gl_frame takes and at n = 2 (gl_ola only), win = n_fft,
# odd n_fft - win, hop not dividing win, hop in (win/2, win], hop = win, hop > win, the smallest L gl_frame takes
# (n_fft/2 + 1), smaller n_fft.  Launches past the 4224-CTA grid take minutes here; the device module runs them.
OLA_FRAME = [(2, 5, 300, 2048, 1200), (3, 2, 300, 2048, 1200), (1, 9, 300, 2048, 1200), (2, 6, 300, 2048, 2048),
             (2, 6, 300, 2048, 1201), (1, 6, 350, 2048, 1200), (2, 4, 700, 2048, 1200), (1, 3, 1200, 2048, 1200),
             (2, 3, 1500, 2048, 1200), (1, 2, 1025, 2048, 1200), (2, 10, 64, 256, 200), (1, 8, 128, 512, 512),
             (1, 7, 37, 256, 101)]


@pytest.fixture(scope="module")
def env(emu):  # noqa: F811
    return SE.Env(KernelsOver(emu), emu, "cpu")


def test_fft_forward_classes(env):
    sel = [0, 1, 2, 3, 255, 256, 511, 1023, 1024, 1025, 2046, 2047]
    SE.fft_forward(env, "impulse", len(sel), 0, sel)
    SE.fft_forward(env, "tone", 2 * 9, 0, [0, 1, 2, 255, 256, 512, 767, 1023, 1024])
    SE.fft_forward(env, "gauss", 3, 1)
    SE.fft_forward(env, "range", 3, 2)
    SE.fft_forward(env, "gauss", 1, 3)


def test_fft_past_the_grid(env):
    """529 rows: each of the 528 CTAs takes one row, CTA 0 a second one, which must give the same bits alone"""
    SE.fft_forward(env, "gauss", 529, 4)


def test_fft_inverse(env):
    SE.fft_inverse(env, "random", 3, 5)
    SE.fft_inverse(env, "hermitian", 3, 6)
    SE.fft_roundtrip(env, 3, 7)


def test_fft_laws(env):
    SE.fft_laws(env, 5, 8)
    SE.fft_empty(env)


@pytest.mark.parametrize("B,T,r,F", [(1, 4, 1, 7), (2, 6, 2, 1025), (1, 5, 3, 33), (2, 7, 5, 9)])
def test_gl_init(env, B, T, r, F):
    SE.gl_init_check(env, B, T, r, F, seed=B + T + r)
    SE.gl_init_mapping(env, B, T, r, min(F, 33))


@pytest.mark.parametrize("B,n,hop,n_fft,win", OLA_FRAME)
def test_gl_ola_frame(env, B, n, hop, n_fft, win):
    SE.gl_ola_frame_check(env, B, n, hop, n_fft, win, seed=n + hop)


def test_window(env):
    for n_fft, win in ((2048, 1200), (2048, 2048), (2048, 1201), (256, 101)):
        SE.window_of(env, n_fft, win)


def test_gl_phase(env):
    SE.gl_phase_check(env, 3000, 9)


def test_packed(env):
    SE.packed_check(env, [8, 20, 12], 5, 5, 300, 2048, 1200, seed=10)
    SE.packed_check(env, [5, 2, 9], 4, 3, 300, 2048, 1200, seed=11)
    SE.packed_check(env, [8, 20, 12], 5, 5, 300, 2048, 1200, seed=12, nan_utt=1)


def test_iterations_padded(env):
    spec = SE.speech_like(1, 8, 2, 13)
    w = SE.gl_iterations(env, spec, 2, 2, 14)
    assert set(w) == {"gl_init mag", "gl_init full", "irfft2048", "gl_ola", "gl_frame", "rfft2048", "gl_phase"}


def test_iterations_packed(env):
    spec = SE.speech_like(2, 8, 2, 15)
    g = torch.Generator().manual_seed(16)
    SE.gl_iterations(env, spec, 2, 1, 17, frames=[8, 16], scale=torch.rand(2 * 1025, generator=g) + 0.5,
                     shift=torch.randn(2 * 1025, generator=g))


def test_feature_frames(env):
    g = torch.Generator().manual_seed(18)
    y = torch.randn(9000, generator=g) * 0.3
    start = torch.tensor([0, 2500, 6000, 100], dtype=torch.int64)
    length = torch.tensor([3000, 1025, 2200, 1], dtype=torch.int32)
    SE.feature_frames_check(env, y, start, length, 3000)


@pytest.mark.parametrize("r,dtype", [(1, torch.float32), (2, torch.float16), (3, torch.float32), (5, torch.float16)])
def test_feature_spec(env, r, dtype):
    g = torch.Generator().manual_seed(19 + r)
    basis, lo, hi = (torch.from_numpy(a) for a in audio.mel_basis())
    n = 4 * r + 3
    y = torch.randn(6000, generator=g) * torch.exp(torch.randn(6000, generator=g))
    max_len = 300 * (n - 1)
    _, frw = SE.feature_frames_check(env, torch.cat([y, y]), torch.tensor([0, 6000]),
                                     torch.tensor([max_len, min(2100, max_len - 7)], dtype=torch.int32), max_len)
    X = SE.run_rfft(env, frw).view(2, n, 1025)
    SE.feature_spec_check(env, X, basis, lo, hi, r, dtype)
    rnd = torch.polar(torch.exp(torch.rand(2, n, 1025, generator=g) * 23 - 20), torch.rand(2, n, 1025, generator=g) * 6.3)
    SE.feature_spec_check(env, rnd.to(torch.complex64), basis, lo, hi, r, dtype)
    if dtype == torch.float32:
        SE.feature_spec_mapping(env, 2, n, r, basis, lo, hi)
