"""The training path's own kernels over their whole envelope on the device, against float64.

taco_gemm, both implementations (0 = FFMA, 1 = 3xTF32 mma.sync), is called directly (not through kernels.gemm, so the
wgmma routes never take a case) over every case of tests/train_envelope_cases.py at its full size, in two classes
(tests/train_envelope_checks.py): small integers, bit-identical to float64, and random fp32 with some large rows, each
element within tol[impl] * S (S = float64 sum |a||b| (+ |C|)).  A, B and the input C sit in NaN guard buffers, C's
surroundings hold a sentinel that must survive, and with beta = 0 C is prefilled with NaN, so it must not be read.  The
bars of tests/train_checks.check_gemm (1e-4 FFMA, 2e-5 mma.sync, of max|ref|) hold on every case too.

tol[impl] started from the linear envelope's constants, 2^-20 (FFMA) and 2^-16 (truncating 3xTF32).  The FFMA bar is
2^-19: its worst element, the post-net conv data gradient at C2 size (K = 3 x 256 in one fp32 accumulator chain),
measured 1.002 of 2^-20.  No split-K case needs an allowance beyond it.

The element-wise, reduction and optimizer kernels run at a tiny edge, a size that wraps the grid-stride loop more than
three times, and their C2 call-site shape; sumsq, l1_loss_fwd and colsum_seg are run twice and must be bit-identical.

Measured on an NVIDIA H100 80GB HBM3 (power limit 700 W), worst element as a fraction of its bar:
  taco_gemm float class   FFMA 0.501 of 2^-19 S (0.018 of the global 1e-4 max|ref|)
                          3xTF32 0.337 of 2^-16 S (0.747 of the global 2e-5 max|ref|)
  bias_act sigmoid 0.313, tanh 0.347;  highway fwd / bwd 0.585;  attn_bwd_post 0.033;  bn_param_grad 0.433
  colsum_seg (float rows) 0.167;  sumsq 0.064;  l1_loss_fwd 0.020;  adam 0.507
  (every other kernel: bit-identical to float64 rounded once)
  module wall time: 40 s (222 tests)
"""
import pytest
import torch

from tacotron_b200 import _lib as L
from tacotron_b200 import kernels as K
from tests import train_envelope_cases as TE
from tests import train_envelope_checks as CH

pytestmark = pytest.mark.gpu
DEV = "cuda"
WORST = {}


def _note(key, w):
    WORST[key] = max(WORST.get(key, 0.0), w)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(WORST):                                   # shown with -s / -rA: the numbers of the docstring
        print(f"ENVELOPE {k}: {WORST[k]:.4f}")


@pytest.fixture
def impl(request):
    prev = K.set_gemm_impl(request.param)
    yield request.param
    K.set_gemm_impl(prev)


@pytest.mark.parametrize("impl", [0, 1], indirect=True)
@pytest.mark.parametrize("case", TE.CASES, ids=[c.name for c in TE.CASES])
def test_gemm_envelope(impl, case):
    CH.run_gemm(L.lib(), case, impl, "exact", DEV, L.current_stream())
    w, gw = CH.run_gemm(L.lib(), case, impl, "float", DEV, L.current_stream(), seed=1)
    _note(f"gemm impl{impl} tol*S", w)
    _note(f"gemm impl{impl} global", gw)
    assert gw <= 1.0, f"{case.name}: max error at {gw:.3f} of the global bar"


SIZES = ["tiny", "wrap", "c2"]


@pytest.mark.parametrize("size", SIZES)
def test_bias_act(size):
    for act in (K.ACT_NONE, K.ACT_RELU):
        CH.check_bias_act(K, DEV, size, act, "exact")
    for act in (K.ACT_SIGMOID, K.ACT_TANH):
        _note(f"bias_act[{act}]", CH.check_bias_act(K, DEV, size, act, "float"))


@pytest.mark.parametrize("size", SIZES)
def test_mul_shift(size):
    for sh, per in ((-1, 2), (1, 2), (-1, 1000), (1, 1000), (-32, 0), (0, 0)):
        CH.check_mul_shift(K, DEV, size, sh, per)


@pytest.mark.parametrize("size", SIZES)
def test_epi(size):
    for form in ("plain", "relu", "relu_bn", "relu_bn_res"):
        CH.check_epi_bwd(K, DEV, size, form)
    CH.check_epi_fwd_keep(K, DEV, size)


@pytest.mark.parametrize("size", SIZES)
def test_bn_param_grad(size):
    _note("bn_param_grad", CH.check_bn_param_grad(K, DEV, size))


@pytest.mark.parametrize("size", SIZES)
def test_maxpool_bwd(size):
    CH.check_maxpool_bwd(K, DEV, size)


@pytest.mark.parametrize("size", SIZES)
def test_highway(size):
    _note("highway", CH.check_highway(K, DEV, size))


@pytest.mark.parametrize("size", SIZES)
def test_l1_bwd(size):
    for beta in (0.0, 1.0):
        for padded in (False, True):
            CH.check_l1_bwd(K, DEV, size, beta, padded)


@pytest.mark.parametrize("size", SIZES)
def test_scatter_add_rows(size):
    CH.check_scatter_add_rows(K, DEV, size)


@pytest.mark.parametrize("size", SIZES)
def test_colsum(size):
    for form in ("sum", "dot", "dot_res"):
        CH.check_colsum(K, DEV, size, form)


@pytest.mark.parametrize("size", SIZES)
def test_colsum_seg(size):
    for period in (1, 2, 7, 128):
        _note("colsum_seg", CH.check_colsum_seg(K, DEV, size, period))


@pytest.mark.parametrize("size", SIZES)
def test_dec_inputs(size):
    for r in range(1, 7):
        for sched in (False, True):
            CH.check_dec_inputs(K, DEV, size, r, sched)


@pytest.mark.parametrize("size", SIZES)
def test_attn_bwd_post(size):
    _note("attn_bwd_post", CH.check_attn_bwd_post(K, DEV, size))


@pytest.mark.parametrize("size", SIZES)
def test_mask_rows(size):
    CH.check_mask_rows(K, DEV, size)


@pytest.mark.parametrize("n", [0, 1, 7, 303104, 303104 + 777, CH.WRAP, 7_000_001, 32000 * 1025])
def test_sumsq(n):
    _note("sumsq", CH.check_sumsq(K, DEV, n))


@pytest.mark.parametrize("n", [0, 1, 2, 3, 4, 5, 6, 7, 1056 * 256 * 4 + 3, CH.WRAP + 2, 32000 * 80, 32000 * 1025 + 1])
def test_l1_loss_fwd(n):
    _note("l1_loss_fwd", CH.check_l1_loss_fwd(L.lib(), DEV, n, L.current_stream()))


@pytest.mark.parametrize("n", [1, CH.WRAP, 7_000_001])
def test_adam(n):
    for clip in ("active", "inactive", "off"):
        _note("adam", CH.check_adam(K, DEV, n, clip))
