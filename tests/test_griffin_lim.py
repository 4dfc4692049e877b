"""Fast Griffin-Lim (momentum) and de-emphasis of synthesised waveforms, without a GPU: the float64 statements against
the reference's plain loop and the convergence claim on the voiced test signal; taco_gl_phase_momentum and
taco_de_emphasis under the host emulation through the kernels.py wrappers, and a tiny momentum inversion through
audio.invert_spectrogram; the host checks and their messages; the synthesis driver's flags."""
import ctypes as C
import io

import numpy as np
import pytest
import torch

from oracle import audio_oracle as A
from tacotron_b200 import _lib as L
from tacotron_b200 import audio, kernels
from tests import griffin_lim_oracle as G
from tests.emulator import KernelsOver, emu  # noqa: F401  (the emulated library, built once per process)


# ---------------------------------------------------------------------------------------------------------------------
# the float64 statements
# ---------------------------------------------------------------------------------------------------------------------
def test_zero_momentum_is_the_reference_loop():
    rng = np.random.default_rng(3)
    mag = np.exp(rng.standard_normal((1025, 16)))
    ang = np.exp(2j * np.pi * rng.random((1025, 16)))
    for n_iter in (0, 1, 3):
        assert np.array_equal(G.fast_griffinlim(mag, ang, n_iter, 0.0), A.griffinlim(mag, ang, n_iter))


def test_momentum_converges_faster_on_the_voiced_signal():
    """momentum 0.99 after 25 iterations is closer to the target magnitude than plain Griffin-Lim after 50"""
    _, y, u = G.voiced_signal(2)
    mag = np.abs(A.stft(y))
    ang = np.exp(2j * np.pi * u)
    plain50 = G.spectral_convergence(G.fast_griffinlim(mag, ang, 50), mag)
    fast25 = G.spectral_convergence(G.fast_griffinlim(mag, ang, 25, 0.99), mag)
    assert fast25 < plain50, (fast25, plain50)


def test_de_emphasis_inverts_pre_emphasis():
    x = np.random.default_rng(0).standard_normal(3000)
    assert np.abs(G.de_emphasis(G.pre_emphasis(x), [0, 3000]) - x).max() < 1e-12


# ---------------------------------------------------------------------------------------------------------------------
# the kernels under the host emulation
# ---------------------------------------------------------------------------------------------------------------------
def _phase_case(n, seed):
    g = torch.Generator().manual_seed(seed)
    mag = torch.rand(n, generator=g) * 3
    reb = torch.complex(torch.randn(n, generator=g), torch.randn(n, generator=g))
    prev = torch.complex(torch.randn(n, generator=g), torch.randn(n, generator=g))
    reb[:7] = 0
    prev[:4] = 0                       # d = 0 exactly in 4 elements, d = -beta prev in 3
    reb[10:13] = prev[10:13] * 0.5     # d = 0 exactly at beta = 0.5
    return mag, reb, prev


@pytest.mark.parametrize("beta", [0.0, 0.25, 0.99 / 1.99, 0.5])
def test_gl_phase_momentum_under_emulation(emu, beta):
    K = KernelsOver(emu)
    n = 1000
    mag, reb, prev = _phase_case(n, 1)
    got = torch.empty(n, dtype=torch.complex64)
    K.gl_phase_momentum(got, mag, reb, prev, beta)
    want = G.phase_momentum(mag.double().numpy(), reb.numpy(), prev.numpy(), np.float32(beta))
    err = np.abs(got.numpy().astype(np.complex128) - want)
    assert (err <= 1e-5 * np.maximum(np.abs(want), 1e-30)).all(), err.max()
    zero = (reb - np.float32(beta) * prev).abs() == 0
    assert zero[:4].all() and torch.equal(got[zero], torch.complex(mag[zero], torch.zeros_like(mag[zero])))
    if beta == 0.0:
        plain = torch.empty(n, dtype=torch.complex64)
        K.gl_phase(plain, mag, reb)
        assert torch.equal(got, plain)


SEGMENTS = [0, 1, 2, 31, 32, 33, 1023, 1024, 1025, 5000, 0, 20000]


def test_de_emphasis_under_emulation(emu):
    """every length around the warp and tile edges, empty segments, one segment over several tiles, a gap left alone"""
    K = KernelsOver(emu)
    start = np.concatenate([[5], 5 + np.cumsum(SEGMENTS)]).astype(np.int64)
    x = torch.from_numpy(np.random.default_rng(2).standard_normal(int(start[-1]) + 9).astype(np.float32))
    y = x.clone()
    K.de_emphasis(y, start, audio.PRE_EMPHASIS)
    want = G.de_emphasis(x.double().numpy(), start)
    assert torch.equal(y[:5], x[:5]) and torch.equal(y[start[-1]:], x[start[-1]:])       # outside the segments
    err = np.abs(y.double().numpy() - want)
    for a, b in zip(start[:-1], start[1:]):
        if b > a:
            assert err[a:b].max() <= 2e-6 * np.abs(want[a:b]).max(), (b - a, err[a:b].max())
    y2 = x.clone()
    K.de_emphasis(y2, start, audio.PRE_EMPHASIS)
    assert torch.equal(y, y2)
    y0 = x.clone()
    K.de_emphasis(y0, start, 0.0)
    assert torch.equal(y0, x)


def test_audio_de_emphasis_rows_under_emulation(emu):
    x = torch.from_numpy(np.random.default_rng(4).standard_normal((3, 700)).astype(np.float32))
    y = audio.de_emphasis(x.clone(), K=KernelsOver(emu))
    want = G.de_emphasis(x.double().numpy().reshape(-1), np.arange(4) * 700).reshape(3, 700)
    assert np.abs(y.double().numpy() - want).max() <= 2e-6 * np.abs(want).max()


def test_momentum_inversion_under_emulation(emu):
    """audio.invert_spectrogram(momentum=0.9) -- the ping-pong of the two rebuilt buffers -- against the oracle"""
    r, T, n_iter = 2, 8, 3
    g = torch.Generator().manual_seed(7)
    spec = torch.randn(1, T, 1025 * r, generator=g) * 0.5
    n = 4 * r * (T // 4)
    pu = torch.rand(1, n, 1025, generator=g)
    y = audio.invert_spectrogram(spec, r, n_iter=n_iter, phase_u=pu, K=KernelsOver(emu), momentum=0.9)
    ref = G.invert_spectrogram(spec[0].double().numpy(), r, np.exp(2j * np.pi * pu[0].double().numpy().T), n_iter, 0.9)
    assert np.abs(y[0].double().numpy() - ref).max() <= 1e-4 * np.abs(ref).max()
    plain = G.invert_spectrogram(spec[0].double().numpy(), r, np.exp(2j * np.pi * pu[0].double().numpy().T), n_iter)
    assert np.abs(plain - ref).max() > 1e-2 * np.abs(ref).max()           # the momentum took effect


# ---------------------------------------------------------------------------------------------------------------------
# host checks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [-0.01, 1.01, float("nan"), float("inf"), "a", None, True])
def test_momentum_outside_the_range_is_refused(m):
    with pytest.raises(ValueError, match=r"momentum = .* must be a number in \[0, 1\]") as e:
        audio.gl_check(50, m)
    assert repr(m) in str(e.value)


def test_momentum_range_and_beta():
    assert audio.gl_check(50, 0) == 0.0 and audio.gl_check(0, 1.0) == 0.5
    assert audio.gl_check(3, 0.99) == pytest.approx(0.99 / 1.99)


@pytest.mark.parametrize("n", [-1, 2.0, True])
def test_bad_iterations_are_refused(n):
    with pytest.raises(ValueError, match="n_iter = .* must be an integer >= 0"):
        audio.gl_check(n, 0.0)


def test_inversions_refuse_before_launching():
    spec = torch.zeros(1, 8, 2050)
    for call in (lambda: audio.invert_spectrogram(spec, 2, momentum=1.5),
                 lambda: audio.griffinlim_batch(spec, 2, n_iter=-2),
                 lambda: audio.invert_speech(spec, 2, [16], momentum=-1),
                 lambda: audio.invert_speech_packed(spec, 2, [16], n_iter=-1)):
        with pytest.raises(ValueError):
            call()


@pytest.mark.parametrize("start,word", [([3, 2], "below start"), ([0, 5, 4, 9], r"start\[2\] = 4 is below"),
                                        ([-1, 4], "negative"), ([0, 11], "past the end"), ([], "1-D integer"),
                                        ([[0, 1]], "1-D integer"), ([0.0, 1.0], "1-D integer")])
def test_bad_offsets_are_refused(start, word):
    with pytest.raises(ValueError, match=word):
        kernels.check_offsets(start, 10)


def test_offsets_accepted():
    assert kernels.check_offsets([0], 0).tolist() == [0]
    assert kernels.check_offsets(np.array([2, 2, 7, 10], np.int32), 10).dtype == np.int64


def test_c_entry_points_refuse(emu):
    y = torch.zeros(8)
    st = torch.tensor([0, 8], dtype=torch.int64)
    p = lambda t: C.c_void_p(t.data_ptr())                                 # noqa: E731
    for coef in (1.0, 1.5, -0.1, float("nan")):
        assert emu.taco_de_emphasis(p(y), p(st), 1, coef, None) != 0
        assert "coef" in emu.taco_last_error().decode()
    assert emu.taco_de_emphasis(None, p(st), 1, 0.97, None) != 0
    assert emu.taco_de_emphasis(p(y), None, 1, 0.97, None) != 0
    assert emu.taco_de_emphasis(p(y), p(st), -1, 0.97, None) != 0
    assert emu.taco_de_emphasis(p(y), p(st), 0, 0.97, None) == 0
    c = torch.zeros(4, dtype=torch.complex64)
    m = torch.zeros(4)
    assert emu.taco_gl_phase_momentum(p(c), p(m), p(c), None, 0.3, 4, None) != 0
    assert emu.taco_gl_phase_momentum(p(c), p(m), p(c), p(c), 0.6, 4, None) != 0
    assert emu.taco_gl_phase_momentum(p(c), p(m), p(c), p(c), 0.3, -1, None) != 0


def test_entry_points_declared():
    assert {"taco_gl_phase_momentum", "taco_de_emphasis"} <= set(L.EXPORTS)


# ---------------------------------------------------------------------------------------------------------------------
# the synthesis driver
# ---------------------------------------------------------------------------------------------------------------------
def test_cli_flag_forms(monkeypatch):
    """bare and valued flags, the defaults, forwarding next to every other synthesis flag, refusals before any model"""
    from tacotron_b200 import test as drv
    seen = []
    monkeypatch.setattr(drv, "test", lambda cls, config, prompts, **kw: seen.append(
        (kw["griffin_lim_iters"], kw["griffin_lim_momentum"], kw["de_emphasis"], kw["trim_tail"], kw["long_form"],
         config.stop_at_end, config.attention_window, config.max_ctas, kw["speaker"], kw["summary_dir"] is not None)))
    monkeypatch.setattr("sys.stdin", io.StringIO("hello\n"))
    drv.main(["-t", "x"])
    drv.main(["-t", "x", "--griffin-lim-momentum"])
    drv.main(["-t", "x", "--griffin-lim-momentum", "0.5", "--griffin-lim-iters", "25", "--de-emphasis"])
    drv.main(["-t", "x", "--griffin-lim-iters", "0", "--griffin-lim-momentum", "--de-emphasis", "--trim-tail",
              "--long-form", "--stop-at-end", "2", "--attention-window", "--max-ctas", "32", "-s", "1", "--summaries"])
    drv.main(["-t", "x", "--griffin-lim-momentum", "1", "--griffin-lim-iters", "50", "--griffin-lim-momentum", "0"])
    assert seen == [(50, 0.0, False, False, False, None, None, None, 0, False),
                    (50, 0.99, False, False, False, None, None, None, 0, False),
                    (25, 0.5, True, False, False, None, None, None, 0, False),
                    (0, 0.99, True, True, True, 2, (2, 5), 32, 1, True),
                    (50, 0.0, False, False, False, None, None, None, 0, False)]
    for bad in (["--griffin-lim-iters", "-1"], ["--griffin-lim-iters", "2.5"], ["--griffin-lim-momentum", "1.5"],
                ["--griffin-lim-momentum", "-0.1"], ["--griffin-lim-momentum", "x"]):
        with pytest.raises(SystemExit):
            drv.main(["-t", "x", *bad])
    assert len(seen) == 5


def test_cli_parsers():
    from tacotron_b200.test import parse_gl_iters, parse_gl_momentum
    import argparse
    assert parse_gl_iters("0") == 0 and parse_gl_iters("100") == 100
    assert parse_gl_momentum("0") == 0.0 and parse_gl_momentum("1") == 1.0 and parse_gl_momentum("0.99") == 0.99
    for bad in ("nan", "inf", "-0.5", "2"):
        with pytest.raises(argparse.ArgumentTypeError):
            parse_gl_momentum(bad)
