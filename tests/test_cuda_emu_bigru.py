"""The persistent bi-GRU forward kernel (csrc/gru.cu) under the host emulation (tests/cuda_emu/emu.h), against the float64
mirror: the lane mapping, the select-free transposing butterflies and the 3-step prefetch rotation, checked without a
GPU.  T = 1..4 and 7 cover every tail of the 3-step unrolled loop; B = 3 puts utterances at non-zero offsets."""
import ctypes as C

import pytest
import torch

from tests import mirror_kernels_spk as MK
from tests.emulator import emu  # noqa: F401  (the emulated library, built once per process)


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _case(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    xp = torch.randn(B, T, 768, generator=g)
    # distinct scales per column block, so that a gate, unit or direction taken from the wrong column shows
    W = [torch.randn(128, 256, generator=g) * 0.15, torch.randn(128, 128, generator=g) * 0.1,
         torch.randn(128, 256, generator=g) * 0.12, torch.randn(128, 128, generator=g) * 0.08]
    h0 = (torch.randn(B, 128, generator=g), torch.randn(B, 128, generator=g))
    return xp, W, h0


def _ref(xp, W, h0f, h0b):
    B, T, _ = xp.shape
    ref = torch.zeros(B, T, 256, dtype=torch.float64)
    dbl = lambda t: None if t is None else t.double()
    MK.bigru_fwd_h0(ref, xp.double(), *[w.double() for w in W], dbl(h0f), dbl(h0b))
    return ref


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("T", [1, 2, 3, 4, 7])
def test_bigru_fwd_kernel_under_emulation(emu, B, T):
    xp, W, _ = _case(B, T, 100 + 10 * B + T)
    got = torch.full((B, T, 256), float("nan"))
    assert emu.taco_bigru_fwd(_p(xp), *[_p(w) for w in W], _p(got), B, T, None) == 0, emu.taco_last_error().decode()
    ref = _ref(xp, W, None, None)
    assert (torch.nan_to_num(got.double(), nan=1e30) - ref).abs().max().item() <= 2e-6 * max(1.0, T)


def test_bigru_fwd_h0_kernel_under_emulation(emu):
    B, T = 3, 7
    xp, W, (h0f, h0b) = _case(B, T, 9)
    got = torch.full((B, T, 256), float("nan"))
    assert emu.taco_bigru_fwd_h0(_p(xp), *[_p(w) for w in W], _p(h0f), _p(h0b), _p(got), B, T, None) == 0, \
        emu.taco_last_error().decode()
    ref = _ref(xp, W, h0f, h0b)
    assert (torch.nan_to_num(got.double(), nan=1e30) - ref).abs().max().item() <= 2e-5
