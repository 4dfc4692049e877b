"""The bi-GRU envelope checks (tests/bigru_envelope_checks.py) on CPU, over the host emulation (tests/cuda_emu) of
csrc/gru.cu and csrc/gru_bwd.cu at small sizes, so that the checks themselves are tested without a GPU.

T in {0..5, 7, 9} covers every tail of the forward's two-step loop and its prefetch; B in {1, 2, 3} puts utterances at
non-zero offsets.  The emulation computes the activations with expf and a true division, so the local bars use its
own bounds: sigmoid within 2^-23 and tanh within 2^-22 (one rounding of the quotient and of 1 - quotient, plus expf's).
"""
import pytest
import torch

from tests import bigru_envelope_checks as BG
from tests.emulator import KernelsOver, emu  # noqa: F401  (the emulated library, built once per process)

SHAPES = [(1, 0), (3, 0), (0, 5), (1, 1), (2, 1), (3, 2), (1, 3), (2, 4), (3, 5), (2, 7), (1, 9)]


@pytest.fixture(scope="module")
def env(emu):  # noqa: F811
    return BG.Env(KernelsOver(emu), emu, "cpu", None, eps_sig=2.0 ** -23, eps_tanh=2.0 ** -22)


def _cases():
    """each shape with one h0 setting and one input regime, cycling so that every setting and regime meets several T"""
    out = []
    for i, (B, T) in enumerate(SHAPES):
        out.append((B, T, BG.H0_MODES[i % 4], ("typical", "expansive", "saturating")[i % 3]))
    return out


@pytest.mark.parametrize("B,T,h0_mode,regime", _cases())
def test_fwd_local_and_laws(env, B, T, h0_mode, regime):
    xp, W, h0f, h0b = BG.fwd_inputs(B, T, regime, h0_mode, seed=10 * B + T)
    out = BG.run_fwd(env, xp, W, h0f, h0b)
    BG.fwd_local(env, xp, W, h0f, h0b, out)
    if regime == "typical":
        BG.fwd_free(xp, W, h0f, h0b, out)
    BG.fwd_laws(env, xp, W, h0f, h0b, out, restarts=T <= 5 or regime == "typical")
    if B > 1:
        BG.fwd_utterances(env, xp, W, h0f, h0b, out)


@pytest.mark.parametrize("B,T", [(2, 5), (1, 20)])
def test_fwd_exact_class(env, B, T):
    BG.fwd_exact(env, B, T, seed=T)


def test_fwd_abi(env):
    BG.fwd_abi(env)


@pytest.mark.parametrize("B,T,h0_mode", [(1, 0, "diff"), (3, 0, "half"), (0, 5, "same"), (1, 1, "none"), (2, 2, "diff"),
                                         (3, 3, "same"), (1, 4, "half"), (2, 5, "none"), (3, 7, "diff"), (2, 9, "half")])
def test_bwd(env, B, T, h0_mode):
    I = BG.bwd_inputs(env, B, T, h0_mode, seed=20 * B + T)
    dxp, dh0 = BG.run_bwd(env, I["dOut"], I["out"], I["ACT"], I["W"], I["h0f"], I["h0b"])
    BG.bwd_free(env, I, dxp, dh0)
    BG.bwd_local_dr(env, I, dxp)
    if B and T > 1:
        BG.bwd_compose(env, I, dxp, dh0, BG.splits_for(T, n_random=0))
    BG.bwd_laws(env, I, dxp, dh0)
    if B > 1:
        BG.bwd_utterances(env, I, dxp, dh0)


def test_bwd_exact_classes(env):
    BG.bwd_exact_long(env, 2, 9, seed=1)
    BG.bwd_exact_short(env, 2, 3, seed=2)


def test_bwd_abi(env):
    BG.bwd_abi(env)
