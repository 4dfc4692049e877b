"""The signal envelope checks (tests/signal_envelope_checks.py) on CPU, over the host emulation (tests/cuda_emu) of
csrc/features.cu, csrc/audio.cu and csrc/resample.cu at small sizes, so that the checks themselves are tested without a
GPU.  The emulation runs one CTA after another with one OS thread per CUDA thread, so every case here keeps to a few
hundred CTAs; the device module runs the sizes where the grids stride."""
import numpy as np
import pytest
import torch

from tests import signal_envelope_checks as SG
from tests.emulator import KernelsOver, emu  # noqa: F401  (the emulated library, built once per process)


@pytest.fixture(scope="module")
def env(emu):  # noqa: F811
    return SG.Env(KernelsOver(emu), emu, "cpu")


# ---- trim ----
@pytest.mark.parametrize("fl,hop", [(2048, 512), (2048, 2048), (2048, 128), (1024, 256), (32, 2)])
def test_trim_lengths(env, fl, hop):
    lens = SG.trim_lengths(fl, hop)
    if hop >= 512:
        lens = [n for n in lens if n < 40 * hop] + [256 * hop - 1]
    waves = [SG.envelope_wave(n, seed=n) for n in lens]
    _, und = SG.trim_check(env, waves, fl, hop)
    assert und == 0


def test_trim_tile_edges(env):
    """first / last at frames around the 256-frame tile edge and at nf - 1 (end clipped to len); per = 1 and 16"""
    frames = [0, 1, 254, 255, 256, 257, 259]
    for fl, hop in ((8, 8), (32, 2)):
        _, und = SG.trim_check(env, SG.impulse_waves(260, fl, hop, frames, seed=hop), fl, hop)
        assert und == 0


def test_trim_planted_zero_nan_base(env):
    for fl, hop in ((64, 64), (2048, 512)):
        up = SG.trim_check(env, [SG.planted_waves(fl, hop, d, 1) for d in (0.01, -0.01)], fl, hop)[0]
        assert up[0, 0] < up[1, 0] and up[0, 1] > up[1, 1], "the planted frames did not decide the bounds"
    waves = [SG.envelope_wave(n, seed=n) for n in (3000, 5000, 1025, 7777)] + [np.zeros(4000, np.float32)]
    got, _ = SG.trim_check(env, waves, 2048, 512, base=13)
    assert tuple(got[4]) == (0, 4000), "an all-zero utterance is kept whole"
    waves[1] = waves[1].copy()
    waves[1][2500] = np.nan
    nan = SG.run_trim(env, waves, 2048, 512, 60.0, base=13)
    assert np.array_equal(np.delete(nan, 1, 0), np.delete(got, 1, 0)), "a NaN utterance changed another"


def test_trim_sensitivity(env):
    waves = SG.impulse_waves(40, 2048, 512, [0, 5, 39], seed=2)
    for ref_hop in (256, 1024):
        with pytest.raises(AssertionError):
            SG.trim_check(env, waves, 2048, 512, ref_hop=ref_hop)


# ---- speech frames / bounds ----
@pytest.mark.parametrize("r,T", [(1, 5), (1, 14), (2, 10), (3, 6)])
def test_speech_map(env, r, T):
    SG.speech_map(env, T, r, 33, seed=r + T)


@pytest.mark.parametrize("r", [1, 5])
def test_speech_threshold(env, r):
    SG.speech_at_threshold(env, r)
    SG.speech_at_threshold(env, r, top_db=37.5)


def test_speech_planted_and_ramps(env):
    for top_db in (60.0, 30.0):
        bd, und = SG.speech_check(env, SG.planted_spec(10, 2, 1025, 0.01, top_db), 2, top_db=top_db)
        assert und == 0 and bd[0, 0] == 1 and bd[1, 0] > 1, "the planted frames did not decide the bounds"
    g = torch.Generator().manual_seed(5)
    spec = SG.ramp_spec(3, 9, 2, 70, 6)
    sc, sh = torch.rand(140, generator=g) * 1.5 + 0.25, torch.randn(140, generator=g)
    for a, b in ((None, None), (sc, sh)):
        assert SG.speech_check(env, spec, 2, a, b)[1] == 0


def test_speech_nonfinite(env):
    SG.speech_nonfinite(env, 5, 9, 2, 40, 7)


def test_speech_sensitivity(env):
    spec = SG.planted_spec(10, 2, 1025, 0.01)
    for d in (0.02, -0.02):
        with pytest.raises(AssertionError):
            SG.speech_check(env, spec, 2, top_db=60.0 + d, ref_top_db=60.0)


# ---- join ----
@pytest.mark.parametrize("fade", [1, 4, 60, 300])
def test_join(env, fade):
    src = np.random.RandomState(fade).randn(5000).astype(np.float32)
    lens = [0, 1, 2, 3, 100, 119, 120, 121, 250, 700, 1100]           # fade >= len / 2, fade >= len, len <= 2
    seg, out_len = SG.make_segments(lens, len(src), seed=fade)
    SG.join_check(env, src, seg, out_len, fade)


def test_join_abi_and_sensitivity(env):
    SG.join_abi_skips(env)
    src = np.random.RandomState(9).randn(3000).astype(np.float32)
    seg, out_len = SG.make_segments([400, 900, 37], len(src), seed=9)
    for f in (59, 61):
        with pytest.raises(AssertionError):
            SG.join_check(env, src, seg, out_len, f, ref_fade=60)


# ---- de-emphasis ----
@pytest.mark.parametrize("c", [0.0, 0.5, 0.97, 0.999, float(np.nextafter(np.float32(1), np.float32(0)))])
def test_de_emphasis_lengths(env, c):
    start, N = SG.de_segments(SG.DE_LENGTHS)
    for kind in ("noise", "dc", "alt"):
        SG.de_check(env, SG.de_signal(kind, N, 1), start, c)


def test_de_emphasis_burst_and_laws(env):
    start, N = SG.de_segments([40000], first=1)
    SG.de_check(env, SG.de_signal("burst", N, 2), start, 0.97)
    start, N = SG.de_segments([17, 8193, 0, 300, 5], first=2)
    SG.de_laws(env, SG.de_signal("noise", N, 3), start, 0.97, picks=[1, 3])


def test_de_emphasis_sensitivity(env):
    start, N = SG.de_segments([20000], first=1)
    k = SG.de_sensitivity(env, SG.de_signal("burst", N, 4), start, 0.97, range(16, 24))
    assert k is not None and k >= 18, k


# ---- resample ----
RATES = [(48000, 24000), (44100, 16000), (16000, 24000), (8000, 16000), (96000, 24000), (44100, 24000),
         (22050, 24000), (32000, 16000), (11025, 16000)]


@pytest.mark.parametrize("sr_orig,sr_new", RATES)
def test_resample(env, sr_orig, sr_new):
    g = np.random.RandomState(sr_orig % 1000 + sr_new % 997)
    lens = SG.resample_lengths(sr_orig, sr_new)[:6]
    waves = [(g.randn(n) * 0.3).astype(np.float32) for n in lens]
    SG.resample_check(env, waves, sr_orig, sr_new, loop=True)


def test_resample_abi_and_sensitivity(env):
    SG.resample_abi_nan(env)
    x = np.random.RandomState(8).randn(60000).astype(np.float32)
    n = SG.resample_sensitivity(env, x, 48000, 16000, np.arange(10000, 20000))
    assert n > 0
