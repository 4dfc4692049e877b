"""The tail-trim kernels of csrc/audio.cu under the host emulation (tests/cuda_emu/emu.h; see tests/test_cuda_emu.py):
taco_speech_frames and the three packed Griffin-Lim entry points against the torch mirrors, for two utterances of
different lengths.  Checks their indexing without a GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import mirror_kernels_trim as MKT
from tests import trim_oracle as TO
from tests.emulator import emu  # noqa: F401  (the emulated library, built once per process)


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _ok(lib, rc):
    assert rc == 0, lib.taco_last_error().decode()


@pytest.mark.parametrize("r,T", [(1, 12), (2, 8), (5, 8)])
def test_speech_frames_under_emulation(emu, r, T):
    n = 4 * r * (T // 4)
    scale, shift = (torch.rand(1025 * r, generator=torch.Generator().manual_seed(r)) + 1.0,
                    torch.randn(1025 * r, generator=torch.Generator().manual_seed(r + 1)) - 5.0)
    for sc, sh in ((None, None), (scale, shift)):
        npsc = None if sc is None else sc.numpy()
        npsh = None if sh is None else sh.numpy()
        spec = torch.from_numpy(TO.speech_like(2, T, r, [n // 2 - 1, 1], seed=r, scale=npsc, shift=npsh))
        assert TO.margin_db(spec.numpy(), r, npsc, npsh) >= 0.5
        want = torch.empty(2, dtype=torch.int32)
        MKT.speech_frames(want, spec, r, sc, sh)
        got = torch.full((2,), -7, dtype=torch.int32)
        _ok(emu, emu.taco_speech_frames(_p(got), _p(spec), 2, T, r, 1025, _p(sc), _p(sh), 60.0, None))
        assert got.tolist() == want.tolist() == TO.speech_frames(spec.numpy(), r, npsc, npsh).tolist()
    spec[1, 0, 3] = float("nan")
    _ok(emu, emu.taco_speech_frames(_p(got), _p(spec), 2, T, r, 1025, None, None, 60.0, None))
    assert got[1].item() == n


def test_speech_frames_argument_checks(emu):
    spec = torch.zeros(1, 8, 2050)
    got = torch.zeros(1, dtype=torch.int32)
    sc = torch.ones(2050)
    for args in ((None, _p(spec), 1, 8, 2, 1025, None, None, 60.0), (_p(got), _p(spec), 0, 8, 2, 1025, None, None, 60.0),
                 (_p(got), _p(spec), 1, 3, 2, 1025, None, None, 60.0), (_p(got), _p(spec), 1, 8, 0, 1025, None, None, 60.0),
                 (_p(got), _p(spec), 1, 8, 2, 1025, _p(sc), None, 60.0), (_p(got), _p(spec), 1, 8, 2, 1025, None, None, 0.0),
                 (_p(got), _p(spec), 1, 8, 2, 1025, None, None, float("inf"))):
        assert emu.taco_speech_frames(*args, None) != 0


@pytest.mark.parametrize("r,T,frames", [(2, 8, [16, 8]), (5, 8, [20, 40])])
def test_packed_gl_kernels_under_emulation(emu, r, T, frames):
    g = torch.Generator().manual_seed(3)
    B, F = len(frames), 1025
    off = torch.tensor(np.concatenate([[0], np.cumsum(frames)]), dtype=torch.int64)
    N, nmax = int(off[-1]), max(frames)
    spec = torch.randn(B, T, F * r, generator=g) * 0.5
    scale, shift = torch.rand(F * r, generator=g) + 0.5, torch.randn(F * r, generator=g) * 0.1
    pu = torch.rand(N, F, generator=g)

    def close(a, b, tol):
        a = torch.view_as_real(a) if a.is_complex() else a
        b = torch.view_as_real(b) if b.is_complex() else b
        assert (a - b).abs().max().item() <= tol * (b.abs().max().item() + 1e-6)
    for sc, sh in ((scale, shift), (None, None)):
        mag_c, full_c = torch.empty(N, F), torch.empty(N, F, dtype=torch.complex64)
        MKT.gl_init_packed(full_c, mag_c, spec, pu, off, r, nmax, sc, sh)
        mag_e, full_e = torch.full((N, F), float("nan")), torch.full((N, F), float("nan"), dtype=torch.complex64)
        _ok(emu, emu.taco_gl_init_packed(_p(full_e), _p(mag_e), _p(spec), _p(pu), _p(off), B, T, r, F, nmax, _p(sc), _p(sh), None))
        close(mag_e, mag_c, 2e-6); close(full_e, full_c, 1e-5)
    fr = torch.randn(N, 2048, generator=g)
    y_c, y_e = torch.empty(300 * (N - B)), torch.full((300 * (N - B),), float("nan"))
    MKT.gl_ola_packed(y_c, fr, off, nmax, 300, 1200)
    _ok(emu, emu.taco_gl_ola_packed(_p(y_e), _p(fr), _p(off), B, nmax, 300, 2048, 1200, None))
    close(y_e, y_c, 1e-5)
    f_c, f_e = torch.empty(N, 2048), torch.full((N, 2048), float("nan"))
    MKT.gl_frame_packed(f_c, y_c, off, nmax, 300, 1200)
    _ok(emu, emu.taco_gl_frame_packed(_p(f_e), _p(y_c), _p(off), B, nmax, 300, 2048, 1200, None))
    close(f_e, f_c, 1e-5)
