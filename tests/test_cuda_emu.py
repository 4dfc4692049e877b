"""Functional check of CUDA kernels WITHOUT a GPU: the product's own kernel sources are compiled for the host over
tests/cuda_emu/emu.h by tests/emulator.py (a thread-per-thread host emulation: real barriers, shuffles, a warp-collective mma defined from the
PTX fragment layout) and driven through the same C-ABI entry points with host pointers, against the torch-CPU mirrors.

What it is for: kernels written after the round's GPU budget was spent (the Griffin-Lim glue kernels, the float16
normalisation, the 3xTF32 mma.sync GEMM variant) get their INDEXING checked here; the FFMA GEMM, which has passed on
hardware, doubles as the check that the emulator itself behaves.  It does not stand in for a hardware run (memory
ordering, real instruction behaviour, performance) -- those tests keep their `gpu` markers.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import data_oracle as DO
from tests import mirror_kernels as MK
from tests.emulator import KernelsOver, emu  # noqa: F401  (the emulated library, built once per process)


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _gemm_cases():
    g = torch.Generator().manual_seed(1)
    rn = lambda *s: torch.randn(*s, generator=g)
    M, N, Kd = 70, 45, 37
    taps, Cin, Cout, Bt, T = 3, 24, 16, 4, 9
    W = rn(taps, Cin, Cout)
    W4 = rn(4, Cin, Cout)
    ident = lambda t: t
    return [
        ("plain", torch.zeros(M, N), rn(M, Kd), rn(Kd, N), ident, ident, ident, {}),
        ("beta1", rn(M, N), rn(M, Kd), rn(Kd, N), ident, ident, ident, dict(beta=1.0)),
        ("tb", torch.zeros(M, N), rn(M, Kd), rn(N, Kd), ident, ident, ident, dict(tb=True)),
        ("ta", torch.zeros(M, N), rn(Kd, M), rn(Kd, N), ident, ident, ident, dict(ta=True)),
        ("ta_tb_beta1", rn(M, N), rn(Kd, M), rn(N, Kd), ident, ident, ident, dict(ta=True, tb=True, beta=1.0)),
        ("strided", torch.zeros(M, 2 * N), rn(M, 3 * Kd), rn(Kd, 2 * N), lambda t: t[:, N:], lambda t: t[:, Kd:2 * Kd], lambda t: t[:, :N], {}),
        ("shift-1", torch.zeros(72, N), rn(72, Kd), rn(Kd, N), ident, ident, ident, dict(shift=-1, period=12)),
        ("shift+1", torch.zeros(72, N), rn(72, Kd), rn(Kd, N), ident, ident, ident, dict(shift=1, period=12)),
        ("ta_shift", rn(20, N), rn(72, 20), rn(72, N), ident, ident, ident, dict(ta=True, shift=-1, period=12, beta=1.0)),
        ("conv_dx", torch.zeros(Bt * T, Cin), rn(Bt * T, Cout), W.reshape(taps * Cin, Cout), ident, ident, lambda t: t[:Cin],
         dict(tb=True, shift=1, dshift=-1, kper=Cout, taps=taps, b_tap_stride=Cin * Cout, period=T)),
        ("conv_dx_k4", torch.zeros(Bt * T, Cin), rn(Bt * T, Cout), W4.reshape(4 * Cin, Cout), ident, ident, lambda t: t[:Cin],
         dict(tb=True, shift=1, dshift=-1, kper=Cout, taps=4, b_tap_stride=Cin * Cout, period=T)),
        ("conv_dw_splitk", rn(taps * Cin, Cout), rn(16 * 40, Cin), rn(16 * 40, Cout), lambda t: t[:Cin], ident, ident,
         dict(ta=True, beta=1.0, shift=-1, bshift=1, batch=taps, c_bstride=Cin * Cout, period=40)),
    ]


@pytest.mark.parametrize("impl,tol", [(0, 2e-6), (1, 2e-5)])
def test_gemm_kernels_under_emulation(emu, impl, tol):
    """impl 0 = the FFMA kernel (green on hardware: validates the emulator); impl 1 = the 3xTF32 mma.sync kernel"""
    K = KernelsOver(emu)
    prev = emu.taco_set_gemm_impl(impl)
    try:
        for name, Cs, As, Bs, cv, av, bv, kw in _gemm_cases():
            Cref, Cemu = Cs.clone(), Cs.clone()
            MK.gemm(cv(Cref), av(As), bv(Bs), **kw)
            K.gemm(cv(Cemu), av(As.clone()), bv(Bs.clone()), **kw)
            err = (Cemu - Cref).abs().max().item()
            assert err <= tol * (Cref.abs().max().item() + 1e-6), (name, impl, err)
    finally:
        emu.taco_set_gemm_impl(prev)


@pytest.mark.parametrize("r,T", [(2, 8), (5, 4)])
def test_griffinlim_kernels_under_emulation(emu, r, T):
    g = torch.Generator().manual_seed(1)
    B, F = 2, 1025
    n = 4 * r * (T // 4)
    Ls = 300 * (n - 1)
    spec = torch.randn(B, T, F * r, generator=g) * 0.5
    scale, shift = torch.rand(F * r, generator=g) + 0.5, torch.randn(F * r, generator=g) * 0.1
    pu = torch.rand(B, n, F, generator=g)

    def close(a, b, tol=2e-6):
        a = torch.view_as_real(a) if a.is_complex() else a
        b = torch.view_as_real(b) if b.is_complex() else b
        assert (a - b).abs().max().item() <= tol * (b.abs().max().item() + 1e-6)
    for sc, sh in ((scale, shift), (None, None)):
        mag_c, full_c = torch.empty(B, n, F), torch.empty(B, n, F, dtype=torch.complex64)
        MK.gl_init(full_c, mag_c, spec, pu, r, sc, sh)
        mag_e, full_e = torch.empty(B, n, F), torch.empty(B, n, F, dtype=torch.complex64)
        assert emu.taco_gl_init(_p(full_e), _p(mag_e), _p(spec), _p(pu), B, T, n, r, F, _p(sc), _p(sh), None) == 0
        close(mag_e, mag_c); close(full_e, full_c, 1e-5)
    fr = torch.randn(B, n, 2048, generator=g)
    y_c, y_e = torch.empty(B, Ls), torch.empty(B, Ls)
    MK.gl_ola(y_c, fr, 300, 1200)
    assert emu.taco_gl_ola(_p(y_e), _p(fr), B, n, 300, 2048, 1200, None) == 0
    close(y_e, y_c, 1e-5)
    f_c, f_e = torch.empty(B, n, 2048), torch.empty(B, n, 2048)
    MK.gl_frame(f_c, y_c, 300, 1200)
    assert emu.taco_gl_frame(_p(f_e), _p(y_c), B, n, 300, 2048, 1200, None) == 0
    close(f_e, f_c, 1e-5)
    reb = torch.complex(torch.randn(B, n, F, generator=g), torch.randn(B, n, F, generator=g))
    reb[0, 0, :5] = 0
    p_c, p_e = torch.empty(B, n, F, dtype=torch.complex64), torch.empty(B, n, F, dtype=torch.complex64)
    MK.gl_phase(p_c, mag_c, reb)
    assert emu.taco_gl_phase(_p(p_e), _p(mag_c), _p(reb), mag_c.numel(), None) == 0
    close(p_e, p_c, 1e-5)


@pytest.mark.parametrize("r,sched", [(2, True), (5, False)])
def test_decoder_bwd_kernel_under_emulation(emu, r, sched):
    """the cooperative decoder-backward kernel (green on hardware) as a one-CTA grid: shared-memory staging, the column
    dealing, all 11 stages and the attention block reductions against the mirror"""
    import copy
    from tacotron_b200.models import grad
    from tests import grad_util, train_checks as TC
    B, Tx, T = 2, 8, 4
    cfg, p, inp, enc_m, dec_m, sm = TC._small_case(r, sched, B, Tx, T)
    S, y, out = grad_util.saving_forward(p, inp, cfg, enc_m, dec_m, sm)
    S["_capture"] = {}
    G = {k: torch.zeros_like(v) for k, v in p.items()}
    dY = torch.randn(B, T, 80 * r, generator=torch.Generator().manual_seed(5))
    grad.decoder_bwd(MK, p, G, S, cfg, dY)
    a = S["_capture"]["decoder_bwd"]                          # inputs + the mirror's outputs
    outs = ("DATT", "DY", "DPQ", "DSCORE", "DCTX", "DZ", "DPN2", "DPN1", "DX")
    e = {k: copy.deepcopy(v) for k, v in a.items() if not k.startswith("_")}
    for k in outs:
        e[k].fill_(float("nan"))
    for i in range(3):
        e["DG"][i].fill_(float("nan")); e["DC"][i].fill_(float("nan"))
    for k in ("Wg", "Wc", "RU", "C", "H", "DG", "DC"):
        for i in range(3):
            e[k][i] = e[k][i].contiguous()
    KernelsOver(emu).decoder_bwd(e)
    for k in outs:
        got, ref = torch.nan_to_num(e[k], nan=1e30), a[k]
        assert (got - ref).abs().max().item() <= 2e-5 * (ref.abs().max().item() + 1e-6), k
    for i in range(3):
        for k in ("DG", "DC"):
            got, ref = torch.nan_to_num(e[k][i], nan=1e30), a[k][i]
            assert (got - ref).abs().max().item() <= 2e-5 * (ref.abs().max().item() + 1e-6), (k, i)


def test_fft2048_kernels_under_emulation(emu):
    """the shared-memory Stockham FFT pair of the Griffin-Lim loop (csrc/audio.cu) against torch.fft"""
    g = torch.Generator().manual_seed(11)
    x = torch.randn(3, 2048, generator=g)
    X = torch.empty(3, 1025, dtype=torch.complex64)
    assert emu.taco_rfft2048(_p(X), _p(x), 3, None) == 0, emu.taco_last_error().decode()
    ref = torch.fft.rfft(x.double(), dim=-1)
    assert (X.to(torch.complex128) - ref).abs().max().item() <= 2e-6 * ref.abs().max().item()
    Y = torch.randn(3, 1025, generator=g) + 1j * torch.randn(3, 1025, generator=g)
    Y = Y.to(torch.complex64).contiguous()
    y = torch.empty(3, 2048)
    assert emu.taco_irfft2048(_p(y), _p(Y), 3, None) == 0, emu.taco_last_error().decode()
    refy = torch.fft.irfft(Y.to(torch.complex128), n=2048, dim=-1)
    assert (y.double() - refy).abs().max().item() <= 2e-6 * refy.abs().max().item()


def test_bigru_bwd_kernel_under_emulation(emu):
    """the register-resident bi-GRU BPTT kernel (green on hardware): 512-thread CTAs, butterfly shuffles"""
    g = torch.Generator().manual_seed(3)
    B, T = 2, 5
    out = torch.tanh(torch.randn(B, T, 256, generator=g))
    ACT = torch.rand(B, T, 768, generator=g)
    ACT[:, :, 256:384] = ACT[:, :, 256:384] * 2 - 1
    ACT[:, :, 640:768] = ACT[:, :, 640:768] * 2 - 1
    dOut = torch.randn(B, T, 256, generator=g)
    W = [torch.randn(128, 256, generator=g) * 0.1, torch.randn(128, 128, generator=g) * 0.1,
         torch.randn(128, 256, generator=g) * 0.1, torch.randn(128, 128, generator=g) * 0.1]
    ref = torch.zeros(B, T, 768)
    MK.bigru_bwd(ref, dOut, out, ACT, *W)
    got = torch.full((B, T, 768), float("nan"))
    assert emu.taco_bigru_bwd(_p(got), _p(dOut), _p(out), _p(ACT), *[_p(w) for w in W], B, T, None) == 0
    assert (torch.nan_to_num(got, nan=1e30) - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()


def test_normalize_f16_under_emulation_is_bit_exact(emu):
    rng = np.random.RandomState(1)
    for shape in ((6, 5, 2050), (3, 7, 161), (1, 1, 161)):                          # even / odd widths and totals
        x = (rng.randn(*shape) * 3 - 2).astype(np.float16)
        x.reshape(-1)[:4] = [65504, -65504, 6e-8, 0]
        mean, std = DO.sample_stats(x, rng.randint(len(x), size=100))
        ref = DO.normalize_explicit(x, mean, std)
        xt, mt, st = torch.from_numpy(x), torch.from_numpy(mean), torch.from_numpy(std)
        out = torch.empty(shape, dtype=torch.float32)
        assert emu.taco_normalize_f16(_p(out), _p(xt), _p(mt), _p(st), x.size // shape[-1], shape[-1], None) == 0
        assert np.array_equal(out.numpy(), ref, equal_nan=True)
