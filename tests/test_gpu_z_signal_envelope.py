"""The trim, speech-end, segment-join, de-emphasis and resampling kernels over their whole envelope on the device,
against float64 (the checks, the decision rule and the bars: tests/signal_envelope_checks.py).

* taco_trim_bounds: frame_length/hop 2048/512, 2048/2048, 2048/128, 1024/256 and 32/2 (per = 4, 1, 16, 4, 16) at
  frame_length/2 + 1, multiples of hop +- 1 and nf = 255 ... 513 frames; a 10-minute file at 16 kHz; a loud frame at
  every f of a 520-frame utterance (per = 1 and 16), so first and last cross both tile edges and reach nf - 1 (end
  clipped to len); frames planted at -60 +- 0.01 dB; all-zero utterances (kept whole); NaN isolation; 2000 utterances
  from a base offset of 13 (NaN before it).
* taco_speech_frames / taco_speech_bounds: the index-coded map (one loud frame per utterance at every f < n, r = 1 ... 6,
  T = 5, 14, 23, rows past 4 (T/4) NaN); frames exactly at the float32 threshold (>=) and one step below, r = 1 ... 6;
  frames planted at top_db +- 0.01 dB (60 and 30 dB); 16 000, 16 896 (the 132 x 16 x 8-warp grid exactly), 17 424,
  32 000 (B = 32, T = 200, r = 5: guided attention's batch), 49 600 and 64 000 frames, with and without the affine;
  NaN, +Inf and all -Inf frames isolated per utterance; both entry points' frame counts bit-identical.
* taco_join_segments: fade 1, 60, 240 and 10^6 over lengths 0, 1, 2, around 2 fade and up; S = 1, 40 and 200 with
  segments past 256 x 4224 / S (the grid-stride loop); S = 65 535; shuffled rows, untouched gaps; rows outside out
  skipped through the C ABI.
* taco_de_emphasis: segment lengths 0 ... 3 x 8192 + 5 from an odd start, c = 0, 0.5, 0.97, 0.999 and 1 - 2^-24, noise,
  DC and +-1; 14.4 M samples (10 min at 24 kHz); a loud burst and 10^5 quiet samples; NaN isolation, a segment alone,
  samples outside [start[0], start[S]) untouched; 70 000 segments of 1 to 3 samples.
* taco_resample: the six production rate pairs and 96 -> 24, 44.1 -> 24, 22.05 -> 24, 32 -> 16 and 11.025 -> 16 kHz, at
  lengths from one output through both tap clamps (bit for bit against resample_loop itself) and 100 001 samples; one
  utterance of 16 800 001 outputs (past the 65 535 x 256 grid); a short register through the C ABI.
* sensitivity: each check run on a kernel with one parameter off.

Measured on an NVIDIA H100 80GB HBM3 (power limit 700 W), worst element as a fraction of its bar, and the utterances
whose answer hung on an undecided frame:
  trim_bounds    0 undecided: every bound bit for bit feature_oracle.trim's
  speech         0 undecided: every bound longform_oracle.speech_bounds', every frame count trim_oracle.speech_frames'
  join           1.000 of (half an ulp + tol): rounding to nearest, bit for bit float32(ref) except 348 samples that
                 took the neighbour inside the reference's own cancellation tolerance (4 u64 / w at small fade weights)
  de_emphasis    c = 0.5: 0.022, 0.97: 0.031, 0.999: 0.017, 1 - 2^-24: 0.026; 14.4 M samples 0.031 (0.97) and 0.026
                 (1 - 2^-24); burst and quiet tail 0.017; 70 000 segments 0.016; c = 0 the input bit for bit
  resample       bit for bit the loop at every output checked; 0.556 of taps u sum |w x| (0.045 past the grid)
  sensitivity    trim: a reference hop of 256 or 1024 against the kernel's 512 is flagged; speech: top_db +-0.0105 dB
                 flagged on frames planted at +-0.01 dB; join: fade 239 and 241 against 240 flagged; de_emphasis:
                 c (1 + 2^-20) flagged at c = 0.97, c (1 + 2^-19) at 0.999; resample: the register of ratio one ulp up
                 flips 99 998 of 100 000 outputs
  module wall time: 40 s (59 tests)
"""
import numpy as np
import pytest
import torch

from tacotron_b200 import _lib as L
from tacotron_b200 import kernels as K
from tests import signal_envelope_checks as SG

pytestmark = pytest.mark.gpu
DEV = "cuda"
WORST = {}


def _note(key, w):
    WORST[key] = max(WORST.get(key, 0.0), w)


@pytest.fixture(scope="module")
def env():
    return SG.Env(K, L.lib(), DEV, L.current_stream())


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(WORST):                                   # shown with -s / -rA: the numbers of the docstring
        print(f"SIGNAL ENVELOPE {k}: {WORST[k]:.4g}")


# ---- taco_trim_bounds ----
@pytest.mark.parametrize("fl,hop", [(2048, 512), (2048, 2048), (2048, 128), (1024, 256), (32, 2)])
def test_trim_lengths(env, fl, hop):
    waves = [SG.envelope_wave(n, seed=n) for n in SG.trim_lengths(fl, hop)]
    _, und = SG.trim_check(env, waves, fl, hop)
    _note("trim undecided", und)


def test_trim_ten_minutes(env):
    x = SG.envelope_wave(16000 * 600, seed=600)
    x[:50000] *= 1e-4                                         # a quiet lead-in and tail, so the span is a cut
    x[-70000:] *= 1e-4
    got, und = SG.trim_check(env, [x], 2048, 512)
    assert 0 < got[0, 0] and got[0, 1] < len(x)
    _note("trim undecided", und)


@pytest.mark.parametrize("fl,hop,step", [(8, 8, 1), (32, 2, 3)])
def test_trim_every_frame(env, fl, hop, step):
    frames = sorted(set(range(0, 520, step)) | {254, 255, 256, 257, 511, 512, 513, 518, 519})
    _, und = SG.trim_check(env, SG.impulse_waves(520, fl, hop, frames, seed=hop), fl, hop)
    _note("trim undecided", und)


def test_trim_planted_zero_nan(env):
    for fl, hop in ((64, 64), (2048, 512), (32, 2), (2048, 128)):
        up = SG.trim_check(env, [SG.planted_waves(fl, hop, d, 1) for d in (0.01, -0.01)], fl, hop)[0]
        assert up[0, 0] < up[1, 0] and up[0, 1] > up[1, 1], "the planted frames did not decide the bounds"
    waves = [SG.envelope_wave(n, seed=n) for n in (3000, 50000, 1025, 77777)] + [np.zeros(4000, np.float32)]
    got, _ = SG.trim_check(env, waves, 2048, 512, base=13)
    assert tuple(got[4]) == (0, 4000), "an all-zero utterance is kept whole"
    waves[1] = waves[1].copy()
    waves[1][25000] = np.nan
    nan = SG.run_trim(env, waves, 2048, 512, 60.0, base=13)
    assert np.array_equal(np.delete(nan, 1, 0), np.delete(got, 1, 0)), "a NaN utterance changed another"


def test_trim_thousands(env):
    g = np.random.RandomState(2000)
    waves = [SG.envelope_wave(int(n), seed=int(n) + i) for i, n in enumerate(g.randint(1025, 12000, size=2000))]
    _, und = SG.trim_check(env, waves, 2048, 512, base=13)
    _note("trim undecided", und)


def test_trim_sensitivity(env):
    waves = SG.impulse_waves(300, 2048, 512, [0, 5, 255, 256, 299], seed=2)
    for ref_hop in (256, 1024):
        with pytest.raises(AssertionError):
            SG.trim_check(env, waves, 2048, 512, ref_hop=ref_hop)


# ---- taco_speech_frames / taco_speech_bounds ----
@pytest.mark.parametrize("r", [1, 2, 3, 4, 5, 6])
def test_speech_map(env, r):
    for T in (5, 14, 23):
        SG.speech_map(env, T, r, 1025 if T == 14 else 33, seed=r + T)
    SG.speech_at_threshold(env, r)
    SG.speech_at_threshold(env, r, top_db=37.5)


def test_speech_planted(env):
    for top_db, r in ((60.0, 2), (30.0, 5), (60.0, 1)):
        bd, und = SG.speech_check(env, SG.planted_spec(14, r, 1025, 0.01, top_db), r, top_db=top_db)
        assert und == 0 and bd[0, 0] == 1 and bd[1, 0] > 1, "the planted frames did not decide the bounds"


@pytest.mark.parametrize("B,T,r,affine", [(16, 200, 5, False), (32, 266, 2, False), (33, 266, 2, True),
                                          (32, 200, 5, True), (32, 200, 5, False), (64, 200, 5, False),
                                          (40, 250, 5, True)])
def test_speech_totals(env, B, T, r, affine):
    g = torch.Generator().manual_seed(B + T)
    spec = SG.ramp_spec(B, T, r, 1025, B * T)
    sc, sh = (torch.rand(1025 * r, generator=g) * 1.5 + 0.25, torch.randn(1025 * r, generator=g)) if affine else (None, None)
    _, und = SG.speech_check(env, spec, r, sc, sh)
    _note("speech undecided", und)
    torch.cuda.empty_cache()


def test_speech_nonfinite(env):
    SG.speech_nonfinite(env, 8, 200, 5, 1025, 7)


def test_speech_sensitivity(env):
    spec = SG.planted_spec(14, 5, 1025, 0.01)
    flagged = set()
    for d in (0.02, -0.02, 0.015, -0.015, 0.012, -0.012, 0.0105, -0.0105):
        try:
            SG.speech_check(env, spec, 5, top_db=60.0 + d, ref_top_db=60.0)
        except AssertionError:
            flagged.add(d)
    assert {0.02, -0.02} <= flagged, f"top_db +-0.02 on frames planted at +-0.01 dB: only {sorted(flagged)} flagged"
    print(f"SIGNAL ENVELOPE speech sensitivity: top_db perturbations flagged: {sorted(flagged)} dB")


# ---- taco_join_segments ----
JOIN_LENS = [0, 1, 2, 3, 100, 119, 120, 121, 239, 240, 241, 479, 480, 481, 700, 2500]


@pytest.mark.parametrize("fade", [1, 60, 240, 10 ** 6])
def test_join(env, fade):
    src = np.random.RandomState(fade % 1000).randn(20000).astype(np.float32)
    seg, out_len = SG.make_segments(JOIN_LENS, len(src), seed=fade % 1000)
    w, nb = SG.join_check(env, src, seg, out_len, fade)
    _note("join", w)
    _note("join neighbours", nb)


@pytest.mark.parametrize("S,n", [(1, 1100000), (40, 27000), (200, 6000)])
def test_join_grid_stride(env, S, n):
    assert n > 256 * (SG.SMS * 32 // S)
    g = np.random.RandomState(S)
    src = g.randn(n + 5000).astype(np.float32)
    lens = [n] + list(g.randint(0, n + 1, size=S - 1))
    seg, out_len = SG.make_segments(lens, len(src), seed=S)
    w, nb = SG.join_check(env, src, seg, out_len, 240)
    _note("join", w)
    _note("join neighbours", nb)


def test_join_max_segments(env):
    g = np.random.RandomState(65535)
    src = g.randn(1000).astype(np.float32)
    seg, out_len = SG.make_segments(list(g.randint(0, 5, size=65535)), len(src), seed=7, gap=2)
    w, nb = SG.join_check(env, src, seg, out_len, 2)
    _note("join", w)


def test_join_abi_and_sensitivity(env):
    SG.join_abi_skips(env)
    src = np.random.RandomState(9).randn(30000).astype(np.float32)
    seg, out_len = SG.make_segments([400, 900, 37, 5000], len(src), seed=9)
    for f in (239, 241):
        with pytest.raises(AssertionError):
            SG.join_check(env, src, seg, out_len, f, ref_fade=240)


# ---- taco_de_emphasis ----
C_TOP = float(np.nextafter(np.float32(1), np.float32(0)))


@pytest.mark.parametrize("c", [0.0, 0.5, 0.97, 0.999, C_TOP])
def test_de_emphasis_lengths(env, c):
    start, N = SG.de_segments(SG.DE_LENGTHS)
    for kind in ("noise", "dc", "alt"):
        _note(f"de_emphasis c={c:.9g}", SG.de_check(env, SG.de_signal(kind, N, 1), start, c))


@pytest.mark.parametrize("c", [0.97, C_TOP])
def test_de_emphasis_ten_minutes(env, c):
    start, N = SG.de_segments([24000 * 600], first=5)
    for kind in ("noise", "dc"):
        _note(f"de_emphasis 14.4M c={c:.9g}", SG.de_check(env, SG.de_signal(kind, N, 2), start, c))


def test_de_emphasis_burst_and_laws(env):
    start, N = SG.de_segments([102000], first=1)
    for c in (0.97, 0.999):
        _note("de_emphasis burst", SG.de_check(env, SG.de_signal("burst", N, 2), start, c))
    start, N = SG.de_segments(SG.DE_LENGTHS, first=7)
    SG.de_laws(env, SG.de_signal("noise", N, 3), start, 0.97, picks=[1, 5, 6, 7, 10])


def test_de_emphasis_many_segments(env):
    g = np.random.RandomState(70000)
    start, N = SG.de_segments(list(g.randint(1, 4, size=70000)), first=11)
    _note("de_emphasis 70000 segments", SG.de_check(env, SG.de_signal("noise", N, 4), start, 0.97))


def test_de_emphasis_sensitivity(env):
    start, N = SG.de_segments([102000], first=1)
    for c in (0.97, 0.999):
        k = SG.de_sensitivity(env, SG.de_signal("burst", N, 4), start, c, range(14, 25))
        print(f"SIGNAL ENVELOPE de_emphasis sensitivity c={c}: c (1 + 2^-k) flagged down to k = {k}")
        assert k is not None and k >= 18, k


# ---- taco_resample ----
RATES = [(48000, 24000), (44100, 16000), (22050, 16000), (48000, 16000), (16000, 24000), (8000, 16000),
         (96000, 24000), (44100, 24000), (22050, 24000), (32000, 16000), (11025, 16000)]


@pytest.mark.parametrize("sr_orig,sr_new", RATES)
def test_resample(env, sr_orig, sr_new):
    g = np.random.RandomState(sr_orig % 1000 + sr_new % 997)
    waves = [(g.randn(n) * 0.3).astype(np.float32) for n in SG.resample_lengths(sr_orig, sr_new)]
    _note("resample", SG.resample_check(env, waves, sr_orig, sr_new, loop=True))
    long = [(g.randn(100001) * 0.3).astype(np.float32), (g.randn(3001) * 0.3).astype(np.float32)]
    pick = lambda b, n: np.concatenate([np.arange(min(n, 3000)), np.arange(max(0, n - 3000), n),  # noqa: E731
                                        g.randint(0, n, size=min(n, 20000))])
    _note("resample", SG.resample_check(env, long, sr_orig, sr_new, sample=pick))


def test_resample_past_the_grid(env):
    n_in = 3 * 16800000 + 3
    x = (np.random.RandomState(17).randn(n_in) * 0.3).astype(np.float32)
    n_out = n_in // 3
    assert n_out > SG.RS_GRID
    g = np.random.RandomState(18)
    pick = lambda b, n: np.concatenate([np.arange(SG.RS_GRID - 2000, n), g.randint(0, n, size=100000)])  # noqa: E731
    _note("resample 16.8M outputs", SG.resample_check(env, [x], 48000, 16000, sample=pick))
    torch.cuda.empty_cache()


def test_resample_abi_and_sensitivity(env):
    SG.resample_abi_nan(env)
    x = (np.random.RandomState(8).randn(3000000) * 0.3).astype(np.float32)
    n = SG.resample_sensitivity(env, x, 48000, 16000, np.arange(900000, 1000000))
    print(f"SIGNAL ENVELOPE resample sensitivity: ratio one ulp up in the register flips {n} of 100000 outputs")
    assert n > 0
