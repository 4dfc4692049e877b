"""The signal-path kernels over their whole envelope on the device, against float64 (the checks and the bars:
tests/stft_envelope_checks.py).

* FFT pair: a unit impulse at each of the 2048 positions, a cosine and a sine at each of the 1025 bins, Gaussian rows
  and rows spanning e^+-20, at 1, 527, 528, 529, 1057, 64 x 361 (preprocessing) and 32 000 (C2 Griffin-Lim) rows, so
  the 528-CTA grid-stride loop runs up to 61 rows per CTA; the inverse on random and on Hermitian spectra; the round
  trip; bit for bit: 2^k scaling, a row's bits at any position and alone, DC / Nyquist imaginary parts exactly 0 (forward)
  and ignored (inverse), NaN / Inf row isolation, determinism, rows = 0.
* gl_init with and without the affine at r = 1, 2, 3, 5, T not a multiple of 4 (the rows past 4*(T/4) are NaN), F = 1025
  and small; the frame -> (row, column block) map exactly.
* gl_ola / gl_frame at production parameters from n = 2 / 5 up to the C2 size (32 x 1000 frames, 65.5 M frame
  elements), win = n_fft, odd n_fft - win, hop not dividing win, hop in (win/2, win] and hop > win (samples covered only
  by window tails, or by none), L = n_fft/2 + 1, n_fft = 256 / 512, and B*n*n_fft past 4224 x 256; the reflect index
  exactly.  gl_phase with |z| from 1e-44 to 3e38 and signed zeros.
* packed: B = 1, 3, 64 and 4300 (past 4224, one x-block per utterance) with mixed lengths, bit-identical per utterance to
  the padded path alone, NaN isolation.
* every Griffin-Lim launch checked from its own operands: r = 2, T = 8; C5 (B = 1, T = 100, r = 5) for all 50
  iterations; C2 (B = 32, T = 200, r = 5) for 3; a packed batch of mixed lengths.
* feature_frames / feature_spec at the preprocessing shape, float32 and float16, r = 1, 2, 3, 5.

Measured on an NVIDIA H100 80GB HBM3 (power limit 700 W), worst element as a fraction of its bar:
  rfft2048       tones 0.376 per element, 0.518 normwise; Gaussian 0.068 / 0.377; e^+-20 rows 0.072; impulses 0.023
  irfft2048      random spectra 0.525, Hermitian 0.525; round trip 0.062
  gl_init        mag 0.463 (the fmaf rounding of v' at |v'| near 20 dominates), full 0.230
  gl_ola         production 0.085, other parameters (window tails, hop > win) 0.098
  gl_frame       0.201; feature_frames 0.200; hann_at's absolute error 0.342 of DW
  gl_phase       0.171
  packed         init 0.470 / 0.229, ola 0.087, frame 0.201
  iterations     gl_init 0.434 / 0.235, irfft2048 0.463, gl_ola 0.085, gl_frame 0.201, rfft2048 0.538, gl_phase 0.180
  feature_spec   stft 0.240 (float32), 0.060 (float16 beyond its rounding); mel 0.183 (float32), 0.001 (float16)
  module wall time: 32 s (53 tests)
"""
import pytest
import torch

from tacotron_b200 import _lib as L
from tacotron_b200 import audio
from tacotron_b200 import kernels as K
from tests import stft_envelope_checks as SE

pytestmark = pytest.mark.gpu
DEV = "cuda"
WORST = {}


def _note(key, w):
    WORST[key] = max(WORST.get(key, 0.0), w)


@pytest.fixture(scope="module")
def env():
    return SE.Env(K, L.lib(), DEV, L.current_stream())


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(WORST):                                   # shown with -s / -rA: the numbers of the docstring
        print(f"STFT ENVELOPE {k}: {WORST[k]:.4g}")


def test_fft_impulses_and_tones(env):
    e, en = SE.fft_forward(env, "impulse", 2048, 0)
    _note("rfft impulse per element", e)
    e, en = SE.fft_forward(env, "tone", 2050, 0, list(range(1025)))
    _note("rfft tone per element", e)
    _note("rfft tone normwise", en)


@pytest.mark.parametrize("rows", [1, 527, 528, 529, 1057, 64 * 361, 32000])
def test_fft_rows(env, rows):
    e, en = SE.fft_forward(env, "gauss", rows, rows)
    _note("rfft gauss per element", e)
    _note("rfft gauss normwise", en)
    e, en = SE.fft_forward(env, "range", rows, rows + 1)
    _note("rfft e^+-20 per element", e)
    _note("irfft random", SE.fft_inverse(env, "random", rows, rows + 2))
    _note("irfft hermitian", SE.fft_inverse(env, "hermitian", rows, rows + 3))
    if rows <= 1057:
        _note("round trip", SE.fft_roundtrip(env, rows, rows + 4))


@pytest.mark.parametrize("rows", [5, 1057])
def test_fft_laws(env, rows):
    SE.fft_laws(env, rows, rows)


def test_fft_empty(env):
    SE.fft_empty(env)


@pytest.mark.parametrize("B,T,r,F", [(1, 4, 1, 7), (2, 6, 2, 1025), (3, 7, 3, 1025), (2, 9, 5, 1025), (1, 5, 5, 33),
                                     (32, 200, 5, 1025)])
def test_gl_init(env, B, T, r, F):
    em, ef = SE.gl_init_check(env, B, T, r, F, seed=B + T + r)
    _note("gl_init mag", em)
    _note("gl_init full", ef)
    if B * T * F * r < 2 ** 18:
        SE.gl_init_mapping(env, B, T, r, F)


OLA_FRAME = [(2, 5, 300, 2048, 1200), (3, 2, 300, 2048, 1200), (1, 9, 300, 2048, 1200), (4, 100, 300, 2048, 1200),
             (32, 1000, 300, 2048, 1200), (2, 6, 300, 2048, 2048), (2, 40, 300, 2048, 1201), (3, 30, 350, 2048, 1200),
             (2, 20, 700, 2048, 1200), (1, 3, 1200, 2048, 1200), (2, 10, 1200, 2048, 1200), (2, 3, 1500, 2048, 1200),
             (2, 12, 1500, 2048, 1200), (1, 2, 1025, 2048, 1200), (2, 10, 64, 256, 200), (1, 8, 128, 512, 512),
             (1, 7, 37, 256, 101), (3, 1420, 256, 256, 256), (5, 2000, 100, 512, 400)]


@pytest.mark.parametrize("B,n,hop,n_fft,win", OLA_FRAME)
def test_gl_ola_frame(env, B, n, hop, n_fft, win):
    eo, ef = SE.gl_ola_frame_check(env, B, n, hop, n_fft, win, seed=n + hop)
    tag = "production" if (hop, n_fft, win) == (300, 2048, 1200) else "other parameters"
    _note(f"gl_ola {tag}", eo)
    _note(f"gl_frame {tag}", ef)


def test_window(env):
    for n_fft, win in ((2048, 1200), (2048, 2048), (2048, 1201), (256, 101), (512, 400)):
        _note("hann_at absolute error / DW", SE.window_of(env, n_fft, win)[1])


def test_gl_phase(env):
    _note("gl_phase", SE.gl_phase_check(env, 1 << 22, 9))


@pytest.mark.parametrize("B", [1, 3, 64, 4300])
def test_packed(env, B):
    g = torch.Generator().manual_seed(B)
    T, r = (200, 5) if B <= 64 else (5, 5)
    nfull = 4 * r * (T // 4)
    lengths = torch.randint(5, nfull + 1, (B,), generator=g).tolist()
    lengths[0] = nfull
    if B > 1:
        lengths[1] = 5
    sample = None if B <= 64 else set(range(0, B, 97)) | {B - 1}
    w = SE.packed_check(env, lengths, T, r, 300, 2048, 1200, seed=B, sample=sample)
    for k, v in w.items():
        _note(f"packed {k}", v)
    if B in (3, 64):
        SE.packed_check(env, lengths, T, r, 300, 2048, 1200, seed=B + 1, nan_utt=B // 2,
                        sample=set(range(0, B, 7)))


@pytest.mark.parametrize("B,T,r,n_iter,frames", [(1, 8, 2, 5, None), (1, 100, 5, 50, None), (32, 200, 5, 3, None),
                                                 (4, 40, 5, 4, [20, 200, 100, 40])])
def test_iterations(env, B, T, r, n_iter, frames):
    spec = SE.speech_like(B, T, r, B + T)
    g = torch.Generator().manual_seed(T)
    sc, sh = (torch.rand(r * 1025, generator=g) + 0.5, torch.randn(r * 1025, generator=g)) if frames else (None, None)
    if frames:
        spec = SE.speech_like(B, 200, r, B + T)
    w = SE.gl_iterations(env, spec, r, n_iter, T, frames=frames, scale=sc, shift=sh)
    for k, v in w.items():
        _note(f"iteration {k}", v)
    torch.cuda.empty_cache()


def test_feature_frames(env):
    g = torch.Generator().manual_seed(18)
    y = torch.randn(400000, generator=g) * 0.3
    start = torch.tensor([0, 108000, 150001, 260000, 300000, 399000], dtype=torch.int64)
    length = torch.tensor([108000, 1025, 100000, 37, 99999, 1000], dtype=torch.int32)
    _note("feature_frames", SE.feature_frames_check(env, y, start, length, 108000)[0])


@pytest.mark.parametrize("r,dtype", [(1, torch.float32), (2, torch.float32), (3, torch.float16), (5, torch.float16),
                                     (2, torch.float16), (5, torch.float32)])
def test_feature_spec(env, r, dtype):
    g = torch.Generator().manual_seed(19 + r)
    basis, lo, hi = (torch.from_numpy(a) for a in audio.mel_basis())
    n = audio.STFT_FRAMES
    y = torch.randn(4 * 108000, generator=g) * torch.exp(torch.randn(4 * 108000, generator=g))
    start = torch.tensor([0, 108000, 216000, 324000], dtype=torch.int64)
    length = torch.tensor([108000, 50000, 1025, 80000], dtype=torch.int32)
    e, frw = SE.feature_frames_check(env, y, start, length, 108000)
    _note("feature_frames", e)
    X = SE.run_rfft(env, frw).view(4, n, 1025)
    es, em = SE.feature_spec_check(env, X, basis, lo, hi, r, dtype)
    tag = "f16" if dtype == torch.float16 else "f32"
    _note(f"feature_spec stft {tag}", es)
    _note(f"feature_spec mel {tag}", em)
    rnd = torch.polar(torch.exp(torch.rand(4, n, 1025, generator=g) * 23 - 20), torch.rand(4, n, 1025, generator=g) * 6.3)
    es, em = SE.feature_spec_check(env, rnd.to(torch.complex64), basis, lo, hi, r, dtype)
    _note(f"feature_spec stft {tag}", es)
    _note(f"feature_spec mel {tag}", em)
    if dtype == torch.float32:
        SE.feature_spec_mapping(env, 2, 4 * r + 3, r, basis, lo, hi)
