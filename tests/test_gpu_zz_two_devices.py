"""-m gpu: two devices in one process.  The wgmma launchers set their kernels' dynamic shared-memory limit and the decoder
sizes its grid per device; a setting made for the first device only would make the second one refuse its launches.  The
fp32x3 untraced forward (the fused highway stack among its kernels) and one taco_conv_dw call run on cuda:0, then on
cuda:1 in the same process, and must give the same bits (same card model).  Skipped with fewer than two GPUs."""
import pytest
import torch

from oracle import tacotron_oracle as O
from tacotron_b200 import Config, Tacotron
from tacotron_b200 import _lib as L

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs in one process")]


def _forward(dev, p, inp):
    with torch.cuda.device(dev):
        m = Tacotron(Config(r=5, vocab_size=64, max_decode_iter=20, precision="fp32x3"), None, train=False)
        m.load_params(p)
        y, out = m.inference({k: v.to(f"cuda:{dev}") for k, v in inp.items()}, train=False)
        torch.cuda.synchronize()
        return y.cpu(), m.alignments.cpu(), out.cpu()


def _conv_dw(dev, X, Z, B, T, taps):
    """dW [taps][C][N] of small-integer X [B T, C] and dZ [B T, N] (exact sums: the atomics' order does not matter)"""
    with torch.cuda.device(dev):
        Xd, Zd = X.to(f"cuda:{dev}"), Z.to(f"cuda:{dev}")
        Cc, N = X.shape[1], Z.shape[1]
        dW = torch.zeros(taps, Cc, N, device=f"cuda:{dev}")
        rc = L.lib().taco_conv_dw(L.ptr(dW), N, Cc * N, L.ptr(Xd), Cc, L.ptr(Zd), N, B, T, Cc, N, taps, -(taps // 2),
                                  L.current_stream())
        assert rc == 0, L.lib().taco_last_error().decode()
        torch.cuda.synchronize()
        return dW.cpu()


def test_two_devices_same_bits():
    cfg = O.OracleConfig(r=5, max_decode_iter=20, vocab_size=64)
    p = O.init_params(cfg, seed=1, trained_like=True)
    inp = O.synthetic_inputs(cfg, 4, 32, 20, seed=0, ragged=True, with_targets=False)
    g = torch.Generator().manual_seed(3)
    B, T, taps = 4, 100, 3
    X = torch.randint(-4, 5, (B * T, 128), generator=g).float()
    Z = torch.randint(-4, 5, (B * T, 256), generator=g).float()
    try:
        res = [_forward(d, p, inp) + (_conv_dw(d, X, Z, B, T, taps),) for d in (0, 1)]
    finally:
        torch.cuda.set_device(0)
    for a, b, name in zip(res[0], res[1], ("seq2seq_output", "alignments", "output", "conv_dw")):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"{name}: cuda:1 differs from cuda:0"
