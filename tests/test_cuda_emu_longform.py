"""The long-form kernels of csrc/audio.cu under the host emulation (tests/cuda_emu/emu.h; see tests/test_cuda_emu.py):
taco_speech_bounds against the float64 oracle and against taco_speech_frames, taco_join_segments against its float64
mirror, and the argument checks of both.  Checks their indexing without a GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import longform_oracle as LO
from tests import trim_oracle as TO
from tests.emulator import emu  # noqa: F401  (the emulated library, built once per process)


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _ok(lib, rc):
    assert rc == 0, lib.taco_last_error().decode()


@pytest.mark.parametrize("r,T", [(1, 12), (2, 8), (5, 8)])
def test_speech_bounds_under_emulation(emu, r, T):
    n = 4 * r * (T // 4)
    g = np.random.RandomState(r)
    scale, shift = (g.rand(1025 * r) + 1.0).astype(np.float32), (g.randn(1025 * r) - 5.0).astype(np.float32)
    starts, ends = [0, 3, n // 2, 0], [n // 2 - 1, n, n // 2 + 1, 1]
    for sc, sh in ((None, None), (scale, shift)):
        spec = torch.from_numpy(LO.speech_span_like(4, T, r, starts, ends, seed=r, scale=sc, shift=sh))
        assert TO.margin_db(spec.numpy(), r, sc, sh) >= 0.5
        tsc, tsh = (None, None) if sc is None else (torch.from_numpy(sc), torch.from_numpy(sh))
        got = torch.full((4, 3), -7, dtype=torch.int32)
        _ok(emu, emu.taco_speech_bounds(_p(got), _p(spec), 4, T, r, 1025, _p(tsc), _p(tsh), 60.0, None))
        frames = torch.full((4,), -7, dtype=torch.int32)
        _ok(emu, emu.taco_speech_frames(_p(frames), _p(spec), 4, T, r, 1025, _p(tsc), _p(tsh), 60.0, None))
        assert got.tolist() == LO.speech_bounds(spec.numpy(), r, sc, sh).tolist()
        assert got[:, 0].tolist() == starts and got[:, 1].tolist() == ends
        assert got[:, 2].tolist() == frames.tolist()
    spec[1, 0, 3] = float("nan")
    spec[2, T - 1, 5] = float("inf")
    _ok(emu, emu.taco_speech_bounds(_p(got), _p(spec), 4, T, r, 1025, None, None, 60.0, None))
    assert got[1].tolist() == got[2].tolist() == [0, n, n]


def test_speech_bounds_argument_checks(emu):
    spec = torch.zeros(1, 8, 2050)
    got = torch.zeros(1, 3, dtype=torch.int32)
    sc = torch.ones(2050)
    for args in ((None, _p(spec), 1, 8, 2, 1025, None, None, 60.0), (_p(got), None, 1, 8, 2, 1025, None, None, 60.0),
                 (_p(got), _p(spec), 0, 8, 2, 1025, None, None, 60.0), (_p(got), _p(spec), 1, 3, 2, 1025, None, None, 60.0),
                 (_p(got), _p(spec), 1, 8, 0, 1025, None, None, 60.0), (_p(got), _p(spec), 1, 8, 2, 0, None, None, 60.0),
                 (_p(got), _p(spec), 1, 8, 2, 1025, None, _p(sc), 60.0), (_p(got), _p(spec), 1, 8, 2, 1025, None, None, -1.0),
                 (_p(got), _p(spec), 1, 8, 2, 1025, None, None, float("nan"))):
        assert emu.taco_speech_bounds(*args, None) != 0


def _ulp_close(got, want, ulps):
    """|got - want| <= ulps float32 ulps of want (want float64)"""
    spacing = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    err = np.abs(got.astype(np.float64) - want)
    assert np.all(err <= ulps * spacing), float((err / spacing).max())


@pytest.mark.parametrize("fade", [1, 4, 160])
def test_join_segments_under_emulation(emu, fade):
    g = np.random.RandomState(fade)
    src = torch.from_numpy(g.randn(3000).astype(np.float32))
    seg = np.array([[0, 10, 700], [900, 800, 333], [1500, 1200, 5], [2000, 1300, 1000]], dtype=np.int64)
    out = torch.full((2400,), 7.0)
    _ok(emu, emu.taco_join_segments(_p(out), 2400, _p(src), _p(torch.from_numpy(seg)), len(seg), 1000, fade, None))
    want = LO.join_segments(np.full(2400, 7.0), src.numpy(), seg, fade)
    _ulp_close(out.numpy(), want, 1)
    assert np.all(out.numpy()[:10] == 7.0) and np.all(out.numpy()[2300:] == 7.0)


def test_join_segments_argument_checks(emu):
    src, out = torch.zeros(100), torch.full((50,), 3.0)
    seg = torch.tensor([[0, 0, 10]], dtype=torch.int64)
    for args in ((None, 50, _p(src), _p(seg), 1, 10, 4), (_p(out), 50, None, _p(seg), 1, 10, 4),
                 (_p(out), 50, _p(src), None, 1, 10, 4), (_p(out), 50, _p(src), _p(seg), 0, 10, 4),
                 (_p(out), 50, _p(src), _p(seg), 65536, 10, 4), (_p(out), -1, _p(src), _p(seg), 1, 10, 4),
                 (_p(out), 50, _p(src), _p(seg), 1, -1, 4), (_p(out), 50, _p(src), _p(seg), 1, 10, 0)):
        assert emu.taco_join_segments(*args, None) != 0
    bad = torch.tensor([[0, 45, 10], [0, -1, 10], [-1, 0, 10]], dtype=torch.int64)      # outside out: skipped
    _ok(emu, emu.taco_join_segments(_p(out), 50, _p(src), _p(bad), 3, 10, 4, None))
    assert torch.all(out == 3.0)
