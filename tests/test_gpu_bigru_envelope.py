"""The bi-GRU forward (taco_bigru_fwd_h0, csrc/gru.cu) and BPTT (taco_bigru_bwd_h0, csrc/gru_bwd.cu) kernels over their
whole envelope on the device, against float64 (the checks: tests/bigru_envelope_checks.py).

Forward, every shape below with four initial-state settings (NULL/NULL, h/h as models/ops.py passes it, h_fw != h_bw,
NULL/h) and three input regimes (typical, expansive weights x3, saturating |xp| <= 90 with +-inf):
* local: at every (b, direction, t, unit) one GRU step in float64 from the kernel's own previous state, within twice
      e_h = |h - c| e_u + (1 - u) e_c + 4u (|u h| + |(1 - u) c| + |h'|),  e_r, e_u = gamma S / 4 + eps_sigmoid,
      e_c = (1 - c^2)(gamma S_c + sum_k |h_k| e_r,k |Wc[k, j]|) + eps_tanh
  (gamma = 2^-20: a 128-term fp32 dot product at most 16 roundings deep; the kernel's depth is 13; eps_sigmoid = 2.5e-7
  and eps_tanh = 5e-7 as csrc/common.cuh states them);
* free running (typical regime): against the float64 mirror, absolute, within FREE_FWD_TOL;
* bit for bit: determinism, time reversal, restart at s = 1, 2, 3, T/2, T-1, direction and NaN isolation, zero state =
  NULL, utterance independence at B = 67 and 200 (more CTAs than SMs), an exact class (gate inputs in {-inf, 0, +inf},
  candidate inputs +-inf) equal to float64;
* guards: operands in NaN bands, out in a sentinel pattern; T = 0 / B = 0 untouched; B*T = 2 796 202 (B = 2,
  T = 1 398 101, 8.6 GB of xp) accepted and locally right on its first and last 4096 steps, one more refused.
Backward, the same shapes (its offsets are 64-bit) and initial states, on a real forward's out and ACT, dOut random with
one row in 8 x64: composition of split runs bit for bit (dh0 is the carry, h0 is hprev); dr_pre at every step and
du_pre / dc_pre at the split steps in float64 (local bars); every row of dxp and dh0 against the float64 mirror relative
to that row's max |ref| (FREE_BWD_TOL); the bit-for-bit laws; two exact classes; the guards.
NULL-pointer and negative-size refusals are checked under the host emulation (tests/test_bigru_envelope_host.py).

Measured on an NVIDIA H100 80GB HBM3 (power limit 700 W), worst element as a fraction of its bar:
  forward local  typical 0.134, expansive 0.126, saturating 0.116, at the B*T limit 0.079
  forward free   2.95e-7 absolute (2.74e-7 at the post-net C2 shape, B = 32, T = 1000): FREE_FWD_TOL = 1e-6, a margin of 3.4
  backward local dr_pre 0.064, du_pre / dc_pre 0.349
  backward free  8.9e-7 of the row's max |ref|: FREE_BWD_TOL = 1e-5, a margin of 11
  module wall time: 124 s (343 tests)
"""
import pytest
import torch

from tacotron_b200 import _lib as L
from tacotron_b200 import kernels as K
from tests import bigru_envelope_checks as BG

pytestmark = pytest.mark.gpu
DEV = "cuda"
WORST = {}
SHAPES = [(1, 0), (3, 0), (0, 5),
          (1, 1), (2, 2), (3, 3), (1, 4), (2, 5), (3, 1), (1, 2), (2, 3), (3, 4), (1, 5),
          (32, 128), (1, 140), (1, 500), (32, 1000), (33, 1000),
          (67, 64), (200, 37),
          (5, 4001)]
REGIMES = ("typical", "expansive", "saturating")


def _note(key, w):
    WORST[key] = max(WORST.get(key, 0.0), w)


@pytest.fixture(scope="module")
def env():
    return BG.Env(K, L.lib(), DEV, L.current_stream())


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(WORST):                                   # shown with -s / -rA: the numbers of the docstring
        print(f"BIGRU ENVELOPE {k}: {WORST[k]:.4g}")


def _seed(B, T, *tags):
    return (1000 * B + T + 7 * sum(len(t) * (i + 1) for i, t in enumerate(tags))) % (2 ** 31)


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("h0_mode", BG.H0_MODES)
@pytest.mark.parametrize("B,T", SHAPES)
def test_fwd(env, B, T, h0_mode, regime):
    xp, W, h0f, h0b = BG.fwd_inputs(B, T, regime, h0_mode, _seed(B, T, h0_mode, regime))
    out = BG.run_fwd(env, xp, W, h0f, h0b)
    _note(f"fwd local {regime}", BG.fwd_local(env, xp.to(DEV), W, h0f, h0b, out))
    if regime == "typical":
        e = BG.fwd_free(xp, W, h0f, h0b, out)
        _note("fwd free abs error" + (" (post-net C2, B=32 T=1000)" if (B, T) == (32, 1000) else ""), e)
    BG.fwd_laws(env, xp, W, h0f, h0b, out, restarts=regime == "typical")
    if B in (67, 200) and regime == "typical":
        BG.fwd_utterances(env, xp, W, h0f, h0b, out)


@pytest.mark.parametrize("B,T", [(2, 5), (3, 16), (33, 1000)])
def test_fwd_exact_class(env, B, T):
    BG.fwd_exact(env, B, T, seed=T)


def test_fwd_abi(env):
    BG.fwd_abi(env, refusals=False)


def test_fwd_limit(env):
    free, _ = torch.cuda.mem_get_info()
    if free < 16 * 2 ** 30:
        pytest.skip(f"the B*T = 2 796 202 case needs 16 GB free, {free / 2 ** 30:.1f} GB are")
    _note("fwd local at the B*T limit", BG.fwd_limit(env))
    torch.cuda.empty_cache()


@pytest.mark.parametrize("h0_mode", BG.H0_MODES)
@pytest.mark.parametrize("B,T", SHAPES)
def test_bwd(env, B, T, h0_mode):
    I = BG.bwd_inputs(env, B, T, h0_mode, _seed(B, T, h0_mode))
    dxp, dh0 = BG.run_bwd(env, I["dOut"], I["out"], I["ACT"], I["W"], I["h0f"], I["h0b"])
    _note("bwd free (of each row's max)", BG.bwd_free(env, I, dxp, dh0))
    _note("bwd local dr_pre", BG.bwd_local_dr(env, I, dxp))
    if B and T > 1:
        _note("bwd local du_pre / dc_pre", BG.bwd_compose(env, I, dxp, dh0, BG.splits_for(T, seed=T)))
    BG.bwd_laws(env, I, dxp, dh0)
    if B in (67, 200) and h0_mode == "diff":
        BG.bwd_utterances(env, I, dxp, dh0)


def test_bwd_exact_classes(env):
    BG.bwd_exact_long(env, 32, 1000, seed=1)
    BG.bwd_exact_short(env, 3, 3, seed=2)


def test_bwd_abi(env):
    BG.bwd_abi(env, refusals=False)
