"""The training-kernel envelope on CPU: which taco_gemm forms the backward issues, where split-K puts its chunk
boundaries, and every kernel of csrc/train.cu under the host emulation (tests/cuda_emu) against float64.

* Call-site accounting: models/grad.py runs over the float64 mirror namespace with a recorder around `gemm` (single- and
  multi-speaker models, the speaker-conditioned decoder, r = 2 and 5, scheduled sampling on and off).  Every recorded
  addressing form must have a case in tests/train_envelope_cases.py, so a new form in the backward fails here until it
  gets an envelope case.
* Split reach: the cases reach 1, 2 and >= 8 splits, and chunk boundaries inside a `period` block and a tap segment.
* Emulation: the case list at reduced sizes (`Case.emu`) through both GEMM implementations -- the FFMA kernel in the
  integer class, bit for bit; the 3xTF32 kernel in the float class, per element (a dropped hi*lo product is invisible to
  integers, whose lo parts are 0) -- with NaN guards around the operands and sentinels around C; the element-wise,
  reduction and optimizer kernels at their tiny sizes and edges.  An emulated launch of a wrapping grid (> 540,672
  threads) takes about 20 s on one CPU, so only taco_l1_bwd_ld (the 1028-pitch spectrogram gradient) and taco_sumsq
  (whose fixed grid wraps from 303,104 elements) wrap here; bias_act, mul_shift, epi_bwd, epi_fwd_keep, maxpool_bwd,
  highway_fwd / bwd, l1_bwd, scatter_add_rows, dec_inputs and adam_step wrap only in tests/test_gpu_train_envelope.py.
"""
import pytest
import torch

from oracle import tacotron_oracle as O
from tacotron_b200 import kernels
from tacotron_b200.models import grad
from tests import grad_util, grad_util_spk, mirror_kernels_spkdec as MKD, speaker_decoder_oracle as SD, speaker_oracle as SO
from tests import train_envelope_cases as TE
from tests import train_envelope_checks as CH
from tests.emulator import KernelsOver, emu  # noqa: F401  (the emulated library, built once per process)


# ------------------------------------------------------------------------------------------------------------------
# call-site accounting
# ------------------------------------------------------------------------------------------------------------------
class _Recorder:
    """the mirror namespace with every gemm (conv_dx included) reduced to its addressing form"""

    def __init__(self, K):
        self.K, self.forms = K, {}

    def __getattr__(self, name):
        return getattr(self.K, name)

    def gemm(self, Cm, A, B, **kw):
        k = dict(ta=False, tb=False, beta=0.0, shift=0, period=0, taps=1, batch=1, a_bstride=0, b_bstride=0, c_bstride=0,
                 bshift=0)
        k.update(kw)
        sliced = lambda t: t.shape[0] > 1 and t.stride(0) != t.shape[1]
        f = TE.form(k["ta"], k["tb"], k["beta"], k["shift"], k["period"], k["taps"], k["batch"], k["a_bstride"],
                    k["b_bstride"], k["c_bstride"], k["bshift"], sliced(Cm), sliced(A), sliced(B))
        self.forms.setdefault(f, (tuple(Cm.shape), tuple(A.shape), tuple(B.shape), kw))
        return self.K.gemm(Cm, A, B, **kw)

    def conv_dx(self, dX, dZ, W, T, beta=0.0):                  # kernels.conv_dx on the taco_gemm route
        taps, Cin, Cout = W.shape
        self.gemm(dX, dZ, W.reshape(taps * Cin, Cout)[:Cin], tb=True, beta=beta, shift=(taps - 1) // 2, dshift=-1, kper=Cout,
                  taps=taps, b_tap_stride=Cin * Cout, period=T)


def _backward(rec, kind, r, sched, B=2, Tx=8, T=5):
    if kind == "single":
        cfg = O.OracleConfig(r=r, vocab_size=20)
        p, fwd = O.init_params(cfg, seed=1, trained_like=True, dtype=torch.float64), grad_util.saving_forward
    elif kind == "speaker":
        cfg = SO.SpkOracleConfig(r=r, vocab_size=20, num_speakers=3)
        p, fwd = SO.init_params(cfg, seed=1, trained_like=True, dtype=torch.float64), grad_util_spk.saving_forward_spk
    else:
        cfg = SD.SpkDecOracleConfig(r=r, vocab_size=20, num_speakers=3)
        p, fwd = SD.init_params(cfg, seed=1, trained_like=True, dtype=torch.float64), SD.saving_forward
    inp = O.synthetic_inputs(cfg, B, Tx, T, seed=0, ragged=True)
    inp = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in inp.items()}
    if kind != "single":
        inp["speaker"] = torch.tensor([0, 2][:B], dtype=torch.int32)
    enc_m, dec_m = O.dropout_masks(cfg, B, Tx, T, seed=2)
    sm = O.sched_mask(cfg, B, T, seed=3) if sched else None
    S, _, _ = fwd(p, inp, cfg, enc_m, dec_m, sm)
    grad.model_bwd(rec, p, {k: torch.zeros_like(v) for k, v in p.items()}, S, cfg)


def test_every_gemm_form_of_the_backward_has_an_envelope_case():
    rec = _Recorder(MKD)
    for kind in ("single", "speaker", "speaker_decoder"):
        for r in (2, 5):
            for sched in (True, False):
                _backward(rec, kind, r, sched)
    covered = {c.form() for c in TE.CASES}
    missing = {f: ex for f, ex in rec.forms.items() if f not in covered}
    assert len(rec.forms) >= 20, sorted(rec.forms)
    assert not missing, "taco_gemm forms without an envelope case (form: C, A, B shapes, arguments):\n" + \
        "\n".join(f"{f}: {ex}" for f, ex in missing.items())


# ------------------------------------------------------------------------------------------------------------------
# split-K reach
# ------------------------------------------------------------------------------------------------------------------
def _reach(cases):
    splits, in_period, in_tap = set(), False, False
    for c in cases:
        s, _ = TE.split_k(c.M, c.N, c.K, c.batch, c.beta)
        splits.add(s)
        for b in TE.boundaries(c):
            in_period |= c.ta and c.period > 0 and b % c.period != 0
            in_tap |= c.taps > 1 and c.beta == 1.0 and c.taps * c.kper > 512 and b % c.kper != 0
    return splits, in_period, in_tap


def test_split_k_restatement():
    assert TE.split_k(128, 256, 32000, 1, 1.0) == (56, 576)     # post-net bi-GRU dW_h in fp32 mode: 56 splits of 576 rows
    assert TE.split_k(70, 45, 600, 1, 0.0) == (1, 608)          # beta = 0: never split
    assert TE.split_k(64, 64, 0, 1, 1.0) == (1, 16)
    assert TE.split_k(7100, 128, 768, 1, 1.0) == (2, 384)


@pytest.mark.parametrize("which", ["device", "emulation"])
def test_split_k_reach(which):
    cases = TE.CASES if which == "device" else [c.for_emulation() for c in TE.CASES]
    splits, in_period, in_tap = _reach(cases)
    assert 1 in splits and (2 if which == "device" else 3) in splits and max(splits) >= 8, sorted(splits)
    assert in_period, "no chunk boundary inside a period block"
    assert in_tap, "no chunk boundary inside a tap segment"


def test_layouts_are_disjoint_and_guarded():
    for c in TE.CASES:
        lay = TE.Layout(c)
        for op in (lay.A, lay.B, lay.C):
            m = op.mask()
            assert int(m.sum()) == op.nb * op.rows * op.cols, c.name                # entries do not overlap
            assert not bool(m[:op.off - op.col0].any()) and not bool(m[-TE.GUARD * op.ld:].any()), c.name


# ------------------------------------------------------------------------------------------------------------------
# emulation
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", [0, 1])
def test_gemm_envelope_under_emulation(emu, impl):
    prev = emu.taco_set_gemm_impl(impl)
    try:
        for c in TE.CASES:                                      # (the device module runs both classes on both kernels)
            if impl == 0:
                CH.run_gemm(emu, c.for_emulation(), impl, "exact", "cpu")
            else:                                               # the float class is what sees a dropped split term
                CH.run_gemm(emu, c.for_emulation(), impl, "float", "cpu", seed=1)
    finally:
        emu.taco_set_gemm_impl(prev)


def test_elementwise_kernels_under_emulation(emu):
    K = KernelsOver(emu)
    for act in (kernels.ACT_NONE, kernels.ACT_RELU):
        CH.check_bias_act(K, "cpu", "tiny", act, "exact")
    for act in (kernels.ACT_SIGMOID, kernels.ACT_TANH):
        CH.check_bias_act(K, "cpu", "tiny", act, "float")
    for sh, per in ((-1, 2), (1, 2), (0, 0), (-1, 0)):
        CH.check_mul_shift(K, "cpu", "tiny", sh, per)
    for form in ("plain", "relu", "relu_bn", "relu_bn_res"):
        CH.check_epi_bwd(K, "cpu", "tiny", form)
    CH.check_epi_fwd_keep(K, "cpu", "tiny")
    CH.check_bn_param_grad(K, "cpu", "tiny")
    CH.check_bn_param_grad(K, "cpu", "c2")
    CH.check_highway(K, "cpu", "tiny")
    for beta in (0.0, 1.0):
        CH.check_l1_bwd(K, "cpu", "tiny", beta, padded=False)
        CH.check_l1_bwd(K, "cpu", "tiny", beta, padded=True)
    CH.check_scatter_add_rows(K, "cpu", "tiny")
    for form in ("sum", "dot", "dot_res"):
        CH.check_colsum(K, "cpu", "tiny", form)
    for period in (1, 2, 7, 128):
        CH.check_colsum_seg(K, "cpu", "tiny", period)
    for r in range(1, 7):
        for sched in (False, True):
            CH.check_dec_inputs(K, "cpu", "tiny", r, sched)
    CH.check_attn_bwd_post(K, "cpu", "tiny")
    for clip in ("active", "inactive", "off"):
        CH.check_adam(K, "cpu", 1000, clip)


def test_shaped_kernels_under_emulation(emu):
    """multi-row shapes the tiny edges do not reach: shifts inside several period blocks, maxpool ties across rows,
    colsum over several row blocks, attention over several steps, the 1028-pitch gradient over many rows"""
    K = KernelsOver(emu)
    g = torch.Generator().manual_seed(0)
    CH.check_maxpool_bwd(K, "cpu", "tiny")
    sizes = {"mp": (2, 9, 128)}
    B, T, Cc = sizes["mp"]
    x = torch.randint(-1, 2, (B, T, Cc), generator=g).float()
    dp = torch.randint(-8, 9, (B, T, Cc), generator=g).float()
    dX = torch.empty(B, T, Cc)
    K.maxpool_bwd(dX, dp, x)
    ref = torch.empty(B, T, Cc, dtype=torch.float64)
    CH.MK.maxpool_bwd(ref, dp.double(), x.double())
    assert torch.equal(dX.double(), ref)
    M, N = 130, 45
    X, H = torch.randn(M, N, generator=g), torch.randn(M, N, generator=g)
    for sh, per in ((-1, 13), (1, 13), (-4, 0)):
        out = torch.empty(M, N)
        K.mul_shift(out, X, H, sh, per)
        ref = torch.empty(M, N, dtype=torch.float64)
        CH.MK.mul_shift(ref, X.double(), H.double(), sh, per)
        assert torch.equal(out.double(), ref.float().double())
    A = torch.randint(-3, 4, (700, 37), generator=g).float()
    out = torch.zeros(37)
    K.colsum(out, A)
    assert torch.equal(out.double(), A.double().sum(0))


def test_grid_stride_wrap_under_emulation(emu):
    """two launches whose grid wraps: l1_bwd_ld over the [rows][1025] gradient in its 1028 pitch, sumsq over its fixed
    1184-block grid (303,104 threads) -- run once each"""
    K = KernelsOver(emu)
    CH.check_l1_bwd(K, "cpu", "wrap", 1.0, padded=True)
    CH.check_sumsq(K, "cpu", 1184 * 256 + 777, repeat=False)
