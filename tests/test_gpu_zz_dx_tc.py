"""GPU tests of the opt-in wgmma route for data gradients (kernels.DX_TC / Config.grad_dx_tc): a conv1d('same') data
gradient is itself a convolution of dZ with the taps reversed and the weights transposed, so it can run on the forward's
tensor-core kernel (taco_linear_fwd).  These per-call checks run the 3xTF32 route (DX_TC_IMPL's default) against the
single-pass bar of 3e-3 of max|ref|; tests/test_gpu_zz_bwd_tc_envelope.py holds both DX_TC_IMPL values to per-element
float64 bars.  The whole-model test runs Config.grad_dx_tc in 'tf32' mode (single-pass TF32 data gradients) and holds
the gradients to the global bar of the TF32 forward test (relative L2 <= 0.15, cosine >= 0.98)."""
import pytest
import torch

from tests import mirror_kernels as MK, train_checks as TC

pytestmark = pytest.mark.gpu


@pytest.fixture()
def dx_tc():
    from tacotron_b200 import kernels as K
    prev, K.DX_TC = K.DX_TC, True
    try:
        yield K
    finally:
        K.DX_TC = prev


@pytest.mark.parametrize("taps,Cin,Cout,B,T", [(1, 256, 1028, 4, 50), (3, 1024, 256, 2, 40), (3, 256, 80, 2, 40), (2, 80, 128, 3, 17),
                                               (7, 128, 128, 2, 33), (16, 128, 128, 2, 40)])
def test_conv_dx_on_tensor_cores(dx_tc, taps, Cin, Cout, B, T):
    K = dx_tc
    g = torch.Generator().manual_seed(taps)
    W = torch.randn(taps, Cin, Cout, generator=g) * 0.1
    dZ = torch.randn(B * T, Cout, generator=g)
    for beta in (0.0, 1.0):
        ref = torch.randn(B * T, Cin, generator=g)
        got = ref.cuda()
        MK.conv_dx(ref, dZ, W, T, beta=beta)
        K.conv_dx(got, dZ.cuda(), W.cuda(), T, beta=beta)
        torch.cuda.synchronize()
        err = (got.cpu() - ref).abs().max().item()
        assert err <= 3e-3 * ref.abs().max().item(), (taps, beta, err)


def test_conv_dx_bank_slice(dx_tc):
    """dZ as a column slice of the wide bank gradient (row stride 8*128), accumulated into dX like the bank loop does"""
    K = dx_tc
    g = torch.Generator().manual_seed(9)
    B, T, Cin = 2, 24, 80
    wide = torch.randn(B * T, 8 * 128, generator=g)
    ref = torch.zeros(B * T, Cin)
    got = ref.cuda()
    wide_g = wide.cuda()
    for k in range(1, 9):
        W = torch.randn(k, Cin, 128, generator=g) * 0.1
        MK.conv_dx(ref, wide[:, (k - 1) * 128:k * 128], W, T, beta=1.0)
        K.conv_dx(got, wide_g[:, (k - 1) * 128:k * 128], W.cuda(), T, beta=1.0)
    torch.cuda.synchronize()
    assert (got.cpu() - ref).abs().max().item() <= 3e-3 * ref.abs().max().item()


def test_model_backward_with_tc_data_gradients():
    from tacotron_b200 import kernels as K
    prev, K.DX_TC = K.DX_TC, False
    try:
        import tacotron_b200.models.tacotron as TM
        orig = TM.Config.grad_dx_tc if hasattr(TM.Config, "grad_dx_tc") else None
        TM.Config.grad_dx_tc = True
        try:
            res = TC.check_model_bwd(5, True, "tf32")
        finally:
            if orig is None:
                del TM.Config.grad_dx_tc
            else:
                TM.Config.grad_dx_tc = orig
    finally:
        K.DX_TC = prev
    assert res["_rel_l2"][0] <= 0.15 and res["_cosine"][0] >= 0.98, (res["_rel_l2"], res["_cosine"])
