"""Tensor-level namespace over the training entry points of libtaco_b200.so (include/taco_b200.h, "Training path").

This is the `K` that tacotron_b200/models/grad.py is written against: every function takes CUDA fp32 tensors
(2-D views may be strided in their leading dimension), extracts pointers / leading strides and calls the C-ABI on
the current stream.  There is NO fallback: a missing library or a non-CUDA tensor raises.
Semantics = the docstrings of the same names in tests/mirror_kernels.py (the kernels are tested against them).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib as L

ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_TANH = 0, 1, 2, 3


def _on_device(t):
    """whether tensor t lives where the library's kernels run: every 'is a CUDA tensor' check goes through here"""
    return t.is_cuda


def _chk2(t, name):
    if not (_on_device(t) and t.dtype == torch.float32 and t.dim() == 2 and (t.shape[1] == 1 or t.stride(1) == 1)):
        raise L.TacoError(f"{name}: expected a CUDA fp32 [M,N] view with unit inner stride, got {tuple(t.shape)} "
                          f"{t.dtype} {t.device} strides {t.stride()}")
    return t


def _ld(t):
    return t.stride(0) if t.shape[0] > 1 else max(t.shape[1], t.stride(0))


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _st():
    return L.current_stream()


def empty(shape, like, dtype=None):
    return torch.empty(shape, dtype=dtype or like.dtype, device=like.device)


def padded_rows(rows, cols, like):
    """[rows, cols] view of a buffer whose row pitch is rounded up to 4 floats (16 bytes): TMA-readable rows for odd widths"""
    ld = (cols + 3) // 4 * 4
    return torch.empty((rows, ld), dtype=like.dtype, device=like.device)[:, :cols]


def zeros(shape, like, dtype=None):
    return torch.zeros(shape, dtype=dtype or like.dtype, device=like.device)


def gemm(Cm, A, B, *, ta=False, tb=False, beta=0.0, shift=0, period=0, taps=1, dshift=0, kper=0, b_tap_stride=0,
         batch=1, a_bstride=0, b_bstride=0, c_bstride=0, bshift=0):
    _chk2(Cm, "gemm C"); _chk2(A, "gemm A"); _chk2(B, "gemm B")
    M, N = Cm.shape
    if ta:
        K, Ma = A.shape
        assert Ma == M, (A.shape, Cm.shape)
    else:
        Ma, Kseg = A.shape
        assert Ma == M, (A.shape, Cm.shape)
        K = Kseg * taps
        if taps > 1:
            assert kper == Kseg
    if tb:
        assert B.shape[0] == N and B.shape[1] * taps == K, (B.shape, N, K)
    else:
        assert B.shape == (K, N), (B.shape, K, N)
    if (not ta) and GEMM_TC and _gemm_tc_ok(Cm, A, B, beta, period, taps, dshift, kper, batch):
        _gemm_tc(Cm, A, B, tb, beta, shift, period)
        return
    if ta and DW_TC and _dw_tc_ok(Cm, A, B, tb, beta, period, taps, dshift, kper, batch, a_bstride, b_bstride, c_bstride, bshift):
        # weight gradient on the wgmma kernel: rows of A / B are (utterance, time), batch entries are the conv taps
        T = period if period > 0 else K
        if beta == 0.0:
            for z in range(batch):
                _offset2(Cm, z * c_bstride).zero_()
        L.check(L.lib().taco_conv_dw(_p(Cm), _ld(Cm), c_bstride, _p(A), _ld(A), _p(B), _ld(B), K // T, T, M, N, batch,
                                     shift, _st()), "taco_conv_dw")
        return
    d = L.GemmDesc()
    d.A = A.data_ptr(); d.lda = _ld(A); d.B = B.data_ptr(); d.ldb = _ld(B); d.C = Cm.data_ptr(); d.ldc = _ld(Cm)
    d.M = M; d.N = N; d.K = K; d.ta = int(ta); d.tb = int(tb); d.beta = float(beta)
    d.shift = shift; d.period = period; d.taps = taps; d.dshift = dshift; d.kper = kper; d.b_tap_stride = b_tap_stride
    d.batch = batch; d.a_bstride = a_bstride; d.b_bstride = b_bstride; d.c_bstride = c_bstride; d.bshift = bshift
    L.check(L.lib().taco_gemm(C.byref(d), _st()), "taco_gemm")


# Data gradient of conv1d('same') / dense.  DX_TC = False: taco_gemm (K-segmented, row-shifted form on the mma.sync / FFMA
# GEMM).  DX_TC = True routes it through the wgmma forward kernel instead (taco_linear_fwd on dZ with the taps reversed and
# the weights transposed: a conv data gradient IS a convolution).  DX_TC_IMPL picks the arithmetic of that route:
# TACO_IMPL_TC3 (3xTF32, fp32-grade -- what Tacotron.backward uses in 'fp32x3' mode) or TACO_IMPL_TC (single-pass TF32).
DX_TC = False
DX_TC_IMPL = L.IMPL_TC3
# DW_TC = True routes the weight gradients (gemm(..., ta=True): dW = X^T dZ over the rows) through taco_conv_dw: 3xTF32 on the
# wgmma tensor cores (fp32-grade) instead of the mma.sync / FFMA GEMM.  Tacotron.backward turns it on outside 'fp32' mode.
DW_TC = False
DW_TC_MIN_ROWS = 512      # below this the launch is all prologue: keep the plain GEMM


def _dw_tc_ok(Cm, A, B, tb, beta, period, taps, dshift, kper, batch, a_bstride, b_bstride, c_bstride, bshift):
    K = A.shape[0]
    if tb or taps != 1 or dshift != 0 or kper != 0 or beta not in (0.0, 1.0) or K < DW_TC_MIN_ROWS:
        return False
    if batch > 1 and (bshift != 1 or a_bstride != 0 or b_bstride != 0):
        return False
    if period > 0 and K % period != 0:
        return False
    return (A.stride(0) % 4 == 0 and B.stride(0) % 4 == 0 and A.data_ptr() % 16 == 0 and B.data_ptr() % 16 == 0
            and A.stride(1) == 1 and B.stride(1) == 1 and Cm.stride(1) == 1)


# GEMM_TC = True routes the plain products of the backward (activation recomputation y = x.W, data gradients dx = dy.W^T, with
# the row shift / period of the recurrent layers) through the wgmma forward kernel: a row-shifted product is a 1-tap
# convolution with tap offset `shift`, accumulation is the kernel's residual input.  Arithmetic = DX_TC_IMPL.
GEMM_TC = False
GEMM_TC_MIN_ROWS = 2048


def _gemm_tc_ok(Cm, A, B, beta, period, taps, dshift, kper, batch):
    M = A.shape[0]
    if taps != 1 or dshift != 0 or kper != 0 or batch != 1 or beta not in (0.0, 1.0) or M < GEMM_TC_MIN_ROWS:
        return False
    if period > 0 and M % period != 0:
        return False
    return (A.stride(1) == 1 and A.stride(0) % 4 == 0 and A.data_ptr() % 16 == 0 and Cm.stride(1) == 1 and Cm.stride(0) % 4 == 0
            and Cm.data_ptr() % 16 == 0 and Cm.shape[1] % 4 == 0)


def _gemm_tc(Cm, A, B, tb, beta, shift, period):
    M, Kc = A.shape
    N = Cm.shape[1]
    W = (B.t() if tb else B).contiguous()                        # TF layout [K][N] (a transpose is a small copy: <= 512 x 1024 floats)
    ld = _cpad(Kc)
    x3 = DX_TC_IMPL == L.IMPL_TC3
    Wp = torch.zeros(((2 if x3 else 1) * N, ld), dtype=torch.float32, device=A.device)
    if x3:
        L.check(L.lib().taco_pack_weight_x3(_p(W), 1, Kc, N, _p(Wp), C.c_void_p(Wp.data_ptr() + N * ld * 4), ld, _st()), "taco_pack_weight_x3")
    else:
        L.check(L.lib().taco_pack_weight(_p(W), 1, Kc, N, _p(Wp), ld, _st()), "taco_pack_weight")
    T = period if period > 0 else M
    d = L.LinearDesc()
    d.X = A.data_ptr(); d.ldx = A.stride(0); d.B = M // T; d.T = T; d.C = Kc
    d.taps = 1; d.tap0 = shift; d.N = N
    d.W = W.data_ptr(); d.Wp = Wp.data_ptr(); d.ldwp = ld
    d.Y = Cm.data_ptr(); d.ldy = Cm.stride(0)
    d.act = ACT_NONE; d.keep_scale = 1.0
    if beta != 0.0:
        d.residual = Cm.data_ptr(); d.ldr = Cm.stride(0)           # accumulate: each element is read then written by one thread
    d.impl = DX_TC_IMPL
    L.check(L.lib().taco_linear_fwd(C.byref(d), _st()), "taco_linear_fwd[gemm]")


def _offset2(t, off):
    return t if off == 0 else torch.as_strided(t, t.shape, t.stride(), t.storage_offset() + off)


def _cpad(c):
    return (c + 31) // 32 * 32


def conv_dx(dX, dZ, W, T, beta=0.0):
    taps, Cin, Cout = W.shape
    tap0 = -((taps - 1) // 2)
    M = dZ.shape[0]
    tma_ok = (dZ.stride(0) * 4) % 16 == 0 and dZ.data_ptr() % 16 == 0 and M % T == 0
    if DX_TC and tma_ok:
        Wt = W.flip(0).transpose(1, 2).contiguous()                    # [taps, Cout, Cin]: taps reversed, weights transposed
        ld = taps * _cpad(Cout)
        x3 = DX_TC_IMPL == L.IMPL_TC3
        Wp = torch.zeros(((2 if x3 else 1) * Cin, ld), dtype=torch.float32, device=W.device)
        if x3:
            L.check(L.lib().taco_pack_weight_x3(_p(Wt), taps, Cout, Cin, _p(Wp), C.c_void_p(Wp.data_ptr() + Cin * ld * 4), ld, _st()),
                    "taco_pack_weight_x3")
        else:
            L.check(L.lib().taco_pack_weight(_p(Wt), taps, Cout, Cin, _p(Wp), ld, _st()), "taco_pack_weight")
        d = L.LinearDesc()
        d.X = dZ.data_ptr(); d.ldx = dZ.stride(0); d.B = M // T; d.T = T; d.C = Cout
        d.taps = taps; d.tap0 = -(tap0 + taps - 1); d.N = Cin
        d.W = Wt.data_ptr(); d.Wp = Wp.data_ptr(); d.ldwp = ld
        d.Y = dX.data_ptr(); d.ldy = dX.stride(0)
        d.act = ACT_NONE; d.keep_scale = 1.0
        if beta != 0.0:
            assert beta == 1.0
            d.residual = dX.data_ptr(); d.ldr = dX.stride(0)             # accumulate: each element is read then written by one thread
        d.impl = DX_TC_IMPL
        L.check(L.lib().taco_linear_fwd(C.byref(d), _st()), "taco_linear_fwd[conv_dx]")
        return
    gemm(dX, dZ, W.reshape(taps * Cin, Cout)[:Cin], tb=True, beta=beta, shift=-tap0, dshift=-1, kper=Cout, taps=taps,
         b_tap_stride=Cin * Cout, period=T)


def set_gemm_impl(impl):
    """0 = exact-product FFMA GEMM (default), 1 = 3xTF32 mma.sync tensor-core GEMM; returns the previous setting"""
    return L.lib().taco_set_gemm_impl(int(impl))


def colsum(out, A, Bm=None, R=None, beta=1.0):
    _chk2(A, "colsum A")
    M, N = A.shape
    assert out.is_contiguous() and out.numel() == N
    if beta == 0.0:
        out.zero_()
    else:
        assert beta == 1.0
    L.check(L.lib().taco_colsum(_p(out), _p(A), _ld(A), _p(Bm), _ld(Bm) if Bm is not None else 0, _p(R),
                                _ld(R) if R is not None else 0, M, N, _st()), "taco_colsum")


def bias_act_(Cm, bias, act):
    _chk2(Cm, "bias_act C")
    L.check(L.lib().taco_bias_act(_p(Cm), _ld(Cm), Cm.shape[0], Cm.shape[1], _p(bias), act, _st()), "taco_bias_act")


def mul_shift(out, X, Hm, shift, period):
    _chk2(out, "mul_shift out"); _chk2(X, "mul_shift X"); _chk2(Hm, "mul_shift H")
    M, N = out.shape
    L.check(L.lib().taco_mul_shift(_p(out), _ld(out), _p(X), _ld(X), _p(Hm), _ld(Hm), M, N, shift, period, _st()), "taco_mul_shift")


def epi_bwd(dZ, dY, Y, relu, scale=None, shift=None, gain=1.0, R=None):
    _chk2(dZ, "epi_bwd dZ"); _chk2(dY, "epi_bwd dY")
    M, N = dY.shape
    L.check(L.lib().taco_epi_bwd(_p(dZ), _ld(dZ), _p(dY), _ld(dY), _p(Y), _ld(Y) if Y is not None else 0, _p(R),
                                 _ld(R) if R is not None else 0, M, N, int(bool(relu)), _p(scale), _p(shift), float(gain), _st()),
            "taco_epi_bwd")


def epi_fwd_keep_(X, keep, gain):
    _chk2(X, "epi_fwd_keep X")
    assert keep.dtype == torch.uint8 and keep.is_contiguous() and keep.numel() == X.numel()
    L.check(L.lib().taco_epi_fwd_keep(_p(X), _ld(X), _p(keep), X.shape[0], X.shape[1], float(gain), _st()), "taco_epi_fwd_keep")


def bn_param_grad(dgamma, dbeta, S1, S2, gamma, beta):
    L.check(L.lib().taco_bn_param_grad(_p(dgamma), _p(dbeta), _p(S1), _p(S2), _p(gamma), _p(beta), gamma.numel(), _st()),
            "taco_bn_param_grad")


def maxpool_bwd(dX, dP, X):
    B, T, Cc = X.shape
    assert dX.is_contiguous() and dP.is_contiguous() and X.is_contiguous()
    L.check(L.lib().taco_maxpool_bwd(_p(dX), _p(dP), _p(X), B, T, Cc, _st()), "taco_maxpool_bwd")


def highway_fwd(Y, Pm, X):
    _chk2(Y, "highway_fwd Y"); _chk2(Pm, "highway_fwd P"); _chk2(X, "highway_fwd X")
    M, U = X.shape
    L.check(L.lib().taco_highway_fwd(_p(Y), _ld(Y), _p(Pm), _ld(Pm), _p(X), _ld(X), M, U, _st()), "taco_highway_fwd")


def highway_bwd(dP, dXd, dY, Pm, X):
    M, U = X.shape
    L.check(L.lib().taco_highway_bwd(_p(dP), _ld(dP), _p(dXd), _ld(dXd), _p(dY), _ld(dY), _p(Pm), _ld(Pm), _p(X), _ld(X), M, U,
                                     _st()), "taco_highway_bwd")


def l1_bwd(dA, A, Bt, beta=0.0):
    if not dA.is_contiguous():          # row-padded gradient buffer (see padded_rows)
        assert dA.dim() == 2 and dA.stride(1) == 1 and A.is_contiguous() and Bt.is_contiguous() and A.shape == Bt.shape == dA.shape
        L.check(L.lib().taco_l1_bwd_ld(_p(dA), dA.stride(0), _p(A), _p(Bt), dA.shape[0], dA.shape[1], float(beta), _st()), "taco_l1_bwd_ld")
        return
    assert dA.is_contiguous() and A.is_contiguous() and Bt.is_contiguous() and A.numel() == Bt.numel() == dA.numel()
    L.check(L.lib().taco_l1_bwd(_p(dA), _p(A), _p(Bt), A.numel(), float(beta), _st()), "taco_l1_bwd")


def scatter_add_rows(dTable, ids, dRows):
    assert ids.dtype == torch.int32 and ids.is_contiguous() and dRows.is_contiguous() and dTable.is_contiguous()
    V, W = dTable.shape
    L.check(L.lib().taco_scatter_add_rows(_p(dTable), _p(ids), _p(dRows), ids.numel(), W, V, _st()), "taco_scatter_add_rows")


def bigru_bwd(dxp, dOut, out, ACT, Wg_h_fw, Wc_h_fw, Wg_h_bw, Wc_h_bw):
    B, T, _ = out.shape
    for t in (dxp, dOut, out, ACT, Wg_h_fw, Wc_h_fw, Wg_h_bw, Wc_h_bw):
        assert t.is_contiguous() and _on_device(t)
    L.check(L.lib().taco_bigru_bwd(_p(dxp), _p(dOut), _p(out), _p(ACT), _p(Wg_h_fw), _p(Wc_h_fw), _p(Wg_h_bw), _p(Wc_h_bw), B, T,
                                   _st()), "taco_bigru_bwd")


def bigru_bwd_h0(dxp, dOut, out, ACT, Wg_h_fw, Wc_h_fw, Wg_h_bw, Wc_h_bw, h0_fw, h0_bw, dh0):
    B, T, _ = out.shape
    for t in (dxp, dOut, out, ACT, Wg_h_fw, Wc_h_fw, Wg_h_bw, Wc_h_bw, h0_fw, h0_bw, dh0):
        assert t is None or (t.is_contiguous() and _on_device(t))
    for t in (h0_fw, h0_bw):
        assert t is None or tuple(t.shape) == (B, 128)
    assert dh0 is None or tuple(dh0.shape) == (B, 2, 128)
    L.check(L.lib().taco_bigru_bwd_h0(_p(dxp), _p(dOut), _p(out), _p(ACT), _p(Wg_h_fw), _p(Wc_h_fw), _p(Wg_h_bw), _p(Wc_h_bw),
                                      _p(h0_fw), _p(h0_bw), _p(dh0), B, T, _st()), "taco_bigru_bwd_h0")


def bigru_fwd_h0(out, xp, Wg_h_fw, Wc_h_fw, Wg_h_bw, Wc_h_bw, h0_fw, h0_bw):
    B, T, _ = out.shape
    for t in (out, xp, Wg_h_fw, Wc_h_fw, Wg_h_bw, Wc_h_bw, h0_fw, h0_bw):
        assert t is None or (t.is_contiguous() and _on_device(t))
    for t in (h0_fw, h0_bw):
        assert t is None or tuple(t.shape) == (B, 128)
    L.check(L.lib().taco_bigru_fwd_h0(_p(xp), _p(Wg_h_fw), _p(Wc_h_fw), _p(Wg_h_bw), _p(Wc_h_bw), _p(h0_fw), _p(h0_bw), _p(out),
                                      B, T, _st()), "taco_bigru_fwd_h0")


def colsum_seg(out, A, period):
    _chk2(A, "colsum_seg A"); _chk2(out, "colsum_seg out")
    M, N = A.shape
    assert M % period == 0 and tuple(out.shape) == (M // period, N), (out.shape, A.shape, period)
    L.check(L.lib().taco_colsum_seg(_p(out), _ld(out), _p(A), _ld(A), M, N, period, _st()), "taco_colsum_seg")


def dec_inputs(Xin, sel, mel, y, sample_mask, r, sched):
    T, B, mf = Xin.shape
    assert mf == 80 and sel.dtype == torch.uint8 and mel.is_contiguous() and y.is_contiguous()
    L.check(L.lib().taco_dec_inputs(_p(Xin), _p(sel), _p(mel), _p(y), _p(sample_mask), B, T, r, int(bool(sched)), _st()),
            "taco_dec_inputs")


def decoder_bwd(a):
    T, B, OUT = a["dy_ext"].shape
    Tx = a["align"].shape[2]
    d = L.DecoderBwdArgs()
    d.B, d.T, d.Tx, d.r, d.keep_scale = B, T, Tx, OUT // 80, float(a["keep_scale"])
    for k in ("W_a", "W_q", "W_out", "W_in", "W1", "W2", "v", "dy_ext", "align", "values", "keys", "PQ", "PN1", "PN2", "sel",
              "DATT", "DY", "DPQ", "DSCORE", "DCTX", "DZ", "DPN2", "DPN1", "DX"):
        assert a[k].is_contiguous() and _on_device(a[k]), k
        setattr(d, k, a[k].data_ptr())
    for k in ("Wg", "Wc", "RU", "C", "H", "DG", "DC"):
        for i in range(3):
            assert a[k][i].is_contiguous(), k
            getattr(d, k)[i] = a[k][i].data_ptr()
    if a.get("H0") is not None:                              # initial GRU states h_i(-1) [B][256] (speaker-conditioned decoder)
        for i in range(3):
            assert a["H0"][i].is_contiguous() and _on_device(a["H0"][i]) and tuple(a["H0"][i].shape) == (B, 256)
            d.H0[i] = a["H0"][i].data_ptr()
    if a.get("DH0") is not None:                             # out: d(loss)/d(h_i(-1)) [3][B][256]
        assert a["DH0"].is_contiguous() and _on_device(a["DH0"]) and tuple(a["DH0"].shape) == (3, B, 256)
        d.DH0 = a["DH0"].data_ptr()
    if a.get("dscore_add") is not None:                      # [B][T][Tx] added to every step's dscore (guided attention)
        assert a["dscore_add"].is_contiguous() and _on_device(a["dscore_add"]) and a["dscore_add"].shape == a["align"].shape
        d.dscore_add = a["dscore_add"].data_ptr()
    ws = torch.empty(L.lib().taco_decoder_bwd_workspace_bytes() // 4, dtype=torch.float32, device=a["dy_ext"].device)
    d.workspace = ws.data_ptr()
    d.max_ctas = int(a.get("max_ctas") or 0)                 # CTA budget, 0 = the device's capacity
    L.check(L.lib().taco_decoder_bwd(C.byref(d), _st()), "taco_decoder_bwd")
    a["_ws"] = ws                                            # keep the scratch alive until the stream has consumed it


def guided_attention(dscore, loss, align, text_length, speech_steps, g, lam, partial=None):
    """Guided attention loss (include/taco_b200.h taco_guided_attention; tests/mirror_kernels_guided.py): dscore fp32
    [B,T,Tx] <- d(loss)/d(attention scores), loss fp32 [1] <- lam * sum align * W, for the alignments align [B,T,Tx],
    text_length and speech_steps int32 [B].  partial: fp32 scratch of taco_guided_attention_partial_count(B, T) floats
    (allocated when None)."""
    B, T, Tx = align.shape
    _f32c(align, "guided_attention align"); _f32c(dscore, "guided_attention dscore"); _f32c(loss, "guided_attention loss")
    _cuda_c(text_length, torch.int32, "guided_attention text_length")
    _cuda_c(speech_steps, torch.int32, "guided_attention speech_steps")
    if dscore.shape != align.shape or loss.numel() != 1 or text_length.shape != (B,) or speech_steps.shape != (B,):
        raise L.TacoError(f"guided_attention: align [B,T,Tx] = {tuple(align.shape)} needs dscore of that shape, a 1-element "
                          f"loss and [B] lengths, got {tuple(dscore.shape)}, {tuple(loss.shape)}, "
                          f"{tuple(text_length.shape)}, {tuple(speech_steps.shape)}")
    n = L.lib().taco_guided_attention_partial_count(B, T)
    if partial is None:
        partial = torch.empty(n, dtype=torch.float32, device=align.device)
    _f32c(partial, "guided_attention partial")
    if partial.numel() < n:
        raise L.TacoError(f"guided_attention: partial holds {partial.numel()} floats, needs {n}")
    L.check(L.lib().taco_guided_attention(_p(dscore), _p(loss), _p(align), _p(text_length), _p(speech_steps), B, T, Tx,
                                          float(g), float(lam), _p(partial), _st()), "taco_guided_attention")


def decoder_capacity():
    """(forward, backward): the co-resident CTAs of the two persistent decoder kernels on the current device.  The forward
    runs 32 CTAs per row group of 8 utterances (at most 4 row groups per launch), the backward min(budget, capacity, 128)."""
    f, b = C.c_int(0), C.c_int(0)
    L.check(L.lib().taco_decoder_capacity(C.byref(f), C.byref(b)), "taco_decoder_capacity")
    return f.value, b.value


def attn_bwd_post(dkeys, dv, DSCORE, keys, PQ, v):
    B, T, Tx = DSCORE.shape
    assert keys.shape[2] == 256
    L.check(L.lib().taco_attn_bwd_post(_p(dkeys), _p(dv), _p(DSCORE), _p(keys), _p(PQ), _p(v), B, T, Tx, _st()), "taco_attn_bwd_post")


def mask_rows(dst, src, length):
    B, T, Cc = src.shape
    L.check(L.lib().taco_mask_rows(_p(src), _p(length), _p(dst), B, T, Cc, _st()), "taco_mask_rows")


# ---- Griffin-Lim glue (tacotron_b200/audio.py) ----
def _f32c(t, name):
    if not (_on_device(t) and t.is_contiguous() and t.dtype in (torch.float32, torch.complex64)):
        raise L.TacoError(f"{name}: expected a contiguous CUDA fp32/complex64 tensor, got {t.dtype} {t.device}")
    return t


def gl_init(full, mag, spec, phase_u, r, scale=None, shift=None):
    B, n, F = mag.shape
    T = spec.shape[1]
    for t, nm in ((full, "full"), (mag, "mag"), (spec, "spec"), (phase_u, "phase_u")):
        _f32c(t, f"gl_init {nm}")
    assert full.dtype == torch.complex64 and spec.shape == (B, T, F * r) and phase_u.shape == mag.shape
    L.check(L.lib().taco_gl_init(_p(full), _p(mag), _p(spec), _p(phase_u), B, T, n, r, F, _p(scale), _p(shift), _st()), "taco_gl_init")


def gl_ola(y, fr, hop, win_length):
    B, n, n_fft = fr.shape
    _f32c(y, "gl_ola y"); _f32c(fr, "gl_ola fr")
    assert y.shape == (B, hop * (n - 1)) and fr.dtype == torch.float32
    L.check(L.lib().taco_gl_ola(_p(y), _p(fr), B, n, hop, n_fft, win_length, _st()), "taco_gl_ola")


def gl_frame(frw, y, hop, win_length):
    B, n, n_fft = frw.shape
    _f32c(y, "gl_frame y"); _f32c(frw, "gl_frame frw")
    assert y.shape == (B, hop * (n - 1))
    L.check(L.lib().taco_gl_frame(_p(frw), _p(y), B, n, hop, n_fft, win_length, _st()), "taco_gl_frame")


def gl_phase(full, mag, rebuilt):
    _f32c(full, "gl_phase full"); _f32c(mag, "gl_phase mag"); _f32c(rebuilt, "gl_phase rebuilt")
    assert full.dtype == torch.complex64 and rebuilt.dtype == torch.complex64 and full.shape == rebuilt.shape == mag.shape
    L.check(L.lib().taco_gl_phase(_p(full), _p(mag), _p(rebuilt), mag.numel(), _st()), "taco_gl_phase")


def gl_phase_momentum(full, mag, rebuilt, prev, beta):
    """full = mag * d/|d|, d = rebuilt - beta*prev (mag + 0i where d == 0): fast Griffin-Lim's phase update"""
    for t, nm in ((full, "full"), (mag, "mag"), (rebuilt, "rebuilt"), (prev, "prev")):
        _f32c(t, f"gl_phase_momentum {nm}")
    assert full.dtype == rebuilt.dtype == prev.dtype == torch.complex64 and mag.dtype == torch.float32
    assert full.shape == rebuilt.shape == prev.shape == mag.shape
    L.check(L.lib().taco_gl_phase_momentum(_p(full), _p(mag), _p(rebuilt), _p(prev), float(beta), mag.numel(), _st()),
            "taco_gl_phase_momentum")


def check_offsets(start, n, name="de_emphasis"):
    """start int64 [S+1] (host): segment s = [start[s], start[s+1]) of a buffer of n samples, 0 <= start[0] and
    non-decreasing up to start[S] <= n; raises ValueError naming the first entry that is not"""
    s = np.asarray(start)
    if s.ndim != 1 or s.size < 1 or s.dtype.kind not in "iu":
        raise ValueError(f"{name}: start must be a 1-D integer array of S+1 offsets, got {s.dtype} {s.shape}")
    s = s.astype(np.int64)
    if s[0] < 0:
        raise ValueError(f"{name}: start[0] = {int(s[0])} is negative")
    down = np.flatnonzero(s[1:] < s[:-1])
    if down.size:
        i = int(down[0]) + 1
        raise ValueError(f"{name}: start[{i}] = {int(s[i])} is below start[{i - 1}] = {int(s[i - 1])}")
    if s[-1] > n:
        raise ValueError(f"{name}: start[{s.size - 1}] = {int(s[-1])} is past the end of the {n}-sample buffer")
    return s


def de_emphasis(y, start, coef):
    """in place: y[i] = x[i] + coef*y[i-1] over each segment [start[s], start[s+1]) of y (contiguous fp32), zero state
    before start[s] (scipy.signal.lfilter([1], [1, -coef], .) per segment).  start (host, int64 [S+1]) is checked on the
    host, then copied to the device: one launch."""
    _cuda_c(y, torch.float32, "de_emphasis y")
    s = check_offsets(start, y.numel())
    if s.size - 1 > 2**31 - 1:
        raise ValueError(f"de_emphasis: {s.size - 1} segments, at most 2^31 - 1 per launch")
    start_d = torch.from_numpy(np.ascontiguousarray(s)).to(y.device)
    L.check(L.lib().taco_de_emphasis(_p(y), _p(start_d), s.size - 1, float(coef), _st()), "taco_de_emphasis")


def rfft2048(X, x):
    """X complex64 [..., 1025] = rfft(x fp32 [..., 2048]) over the last axis (unnormalised) -- librosa.stft's transform"""
    _f32c(X, "rfft2048 X"); _f32c(x, "rfft2048 x")
    assert X.dtype == torch.complex64 and x.dtype == torch.float32 and x.shape[-1] == 2048 and X.shape[-1] == 1025
    assert X.numel() // 1025 == x.numel() // 2048
    L.check(L.lib().taco_rfft2048(_p(X), _p(x), x.numel() // 2048, _st()), "taco_rfft2048")


def irfft2048(x, X):
    """x fp32 [..., 2048] = irfft(X complex64 [..., 1025], n=2048) over the last axis (1/n scaling) -- librosa.istft's transform"""
    _f32c(X, "irfft2048 X"); _f32c(x, "irfft2048 x")
    assert X.dtype == torch.complex64 and x.dtype == torch.float32 and x.shape[-1] == 2048 and X.shape[-1] == 1025
    assert X.numel() // 1025 == x.numel() // 2048
    L.check(L.lib().taco_irfft2048(_p(x), _p(X), x.numel() // 2048, _st()), "taco_irfft2048")


def _affine(scale, shift, W, name):
    if (scale is None) != (shift is None):
        raise L.TacoError(f"{name}: scale and shift go together")
    for t, nm in ((scale, "scale"), (shift, "shift")):
        if t is not None:
            _f32c(t, f"{name} {nm}")
            if t.dtype != torch.float32 or t.numel() != W:
                raise L.TacoError(f"{name}: {nm} must be fp32 [{W}], got {t.dtype} {tuple(t.shape)}")


def speech_frames(frames, spec, r, scale=None, shift=None, top_db=60.0):
    """frames int32 [B] = STFT frames to keep of each utterance of spec fp32 [B, T, F*r] (the post-net output): whole
    blocks of 4r frames up to the last one within top_db of the utterance's loudest (tests/mirror_kernels_trim.py)"""
    B, T, W = spec.shape
    _f32c(spec, "speech_frames spec"); _cuda_c(frames, torch.int32, "speech_frames frames")
    if spec.dtype != torch.float32 or W % r or frames.shape != (B,):
        raise L.TacoError(f"speech_frames: spec fp32 [B, T, F*r] (r={r}) and frames [B], got {spec.dtype} "
                          f"{tuple(spec.shape)} and {tuple(frames.shape)}")
    _affine(scale, shift, W, "speech_frames")
    L.check(L.lib().taco_speech_frames(_p(frames), _p(spec), B, T, r, W // r, _p(scale), _p(shift), float(top_db), _st()),
            "taco_speech_frames")


def speech_bounds(bounds, spec, r, scale=None, shift=None, top_db=60.0):
    """bounds int32 [B, 3] = {first voiced frame, last voiced frame + 1, speech_frames' frame count} of each utterance of
    spec fp32 [B, T, F*r] (tests/longform_oracle.py speech_bounds)"""
    B, T, W = spec.shape
    _f32c(spec, "speech_bounds spec"); _cuda_c(bounds, torch.int32, "speech_bounds bounds")
    if spec.dtype != torch.float32 or W % r or bounds.shape != (B, 3):
        raise L.TacoError(f"speech_bounds: spec fp32 [B, T, F*r] (r={r}) and bounds [B, 3], got {spec.dtype} "
                          f"{tuple(spec.shape)} and {tuple(bounds.shape)}")
    _affine(scale, shift, W, "speech_bounds")
    L.check(L.lib().taco_speech_bounds(_p(bounds), _p(spec), B, T, r, W // r, _p(scale), _p(shift), float(top_db), _st()),
            "taco_speech_bounds")


def check_segments(seg, src_len, out_len):
    """seg int64 [S, 3] rows {src_start, dst_start, len}: every segment inside src [0, src_len) and out [0, out_len),
    no two overlapping in out; raises ValueError naming the first that is not"""
    seg = np.asarray(seg, dtype=np.int64).reshape(-1, 3)
    for s, (a, d, n) in enumerate(seg.tolist()):
        if n < 0 or a < 0 or d < 0 or a + n > src_len or d + n > out_len:
            raise ValueError(f"join_segments: segment {s} = (src {a}, dst {d}, len {n}) outside src [0, {src_len}) or "
                             f"out [0, {out_len})")
    order = np.argsort(seg[:, 1], kind="stable")
    ends = seg[order, 1] + seg[order, 2]
    clash = np.flatnonzero(seg[order[1:], 1] < ends[:-1])
    if clash.size:
        i, j = int(order[clash[0]]), int(order[clash[0] + 1])
        raise ValueError(f"join_segments: segments {i} and {j} overlap in out")
    return seg


def join_segments(out, src, seg, fade):
    """out fp32 [out_len]: out[d + i] = src[a + i] * w(i) for every host row {a, d, len} of seg int64 [S, 3], w the
    raised-cosine fade of `fade` samples at both ends (tests/longform_oracle.py join_segments); other samples of out are
    left as they are.  The segments are checked on the host, then copied to the device: one launch."""
    _f32c(out, "join_segments out"); _f32c(src, "join_segments src")
    if out.dtype != torch.float32 or src.dtype != torch.float32 or out.dim() != 1 or src.dim() != 1:
        raise L.TacoError(f"join_segments: out and src must be 1-D fp32, got {out.dtype} {tuple(out.shape)} and "
                          f"{src.dtype} {tuple(src.shape)}")
    seg = check_segments(seg, src.numel(), out.numel())
    if len(seg) == 0:
        return
    if len(seg) > 65535 or int(seg[:, 2].max()) > 2**31 - 1:
        raise ValueError(f"join_segments: at most 65535 segments of < 2^31 samples per launch, got {len(seg)}")
    seg_d = torch.from_numpy(np.ascontiguousarray(seg)).to(out.device)
    L.check(L.lib().taco_join_segments(_p(out), out.numel(), _p(src), _p(seg_d), len(seg), int(seg[:, 2].max()), int(fade),
                                       _st()), "taco_join_segments")


def _packed(off, name):
    _cuda_c(off, torch.int64, f"{name} off")
    if off.dim() != 1 or off.numel() < 2:
        raise L.TacoError(f"{name}: off must be int64 [B+1], got {tuple(off.shape)}")
    return off.numel() - 1


def gl_init_packed(full, mag, spec, phase_u, off, r, max_frames, scale=None, shift=None):
    """gl_init over the packed layout: utterance b owns rows off[b]:off[b+1] of mag / full / phase_u [N, F]"""
    N, F = mag.shape
    for t, nm in ((full, "full"), (mag, "mag"), (spec, "spec"), (phase_u, "phase_u")):
        _f32c(t, f"gl_init_packed {nm}")
    B = _packed(off, "gl_init_packed")
    assert full.dtype == torch.complex64 and spec.dtype == mag.dtype == phase_u.dtype == torch.float32
    assert full.shape == phase_u.shape == (N, F) and spec.dim() == 3 and spec.shape[0] == B and spec.shape[2] == F * r
    _affine(scale, shift, F * r, "gl_init_packed")
    L.check(L.lib().taco_gl_init_packed(_p(full), _p(mag), _p(spec), _p(phase_u), _p(off), B, spec.shape[1], r, F, int(max_frames),
                                        _p(scale), _p(shift), _st()), "taco_gl_init_packed")


def gl_ola_packed(y, fr, off, max_frames, hop, win_length):
    """gl_ola over the packed layout: fr [N, n_fft] -> y [hop*(N - B)], utterance b's samples from hop*(off[b] - b)"""
    N, n_fft = fr.shape
    _f32c(y, "gl_ola_packed y"); _f32c(fr, "gl_ola_packed fr")
    B = _packed(off, "gl_ola_packed")
    assert y.dtype == fr.dtype == torch.float32 and y.shape == (hop * (N - B),)
    L.check(L.lib().taco_gl_ola_packed(_p(y), _p(fr), _p(off), B, int(max_frames), hop, n_fft, win_length, _st()), "taco_gl_ola_packed")


def gl_frame_packed(frw, y, off, max_frames, hop, win_length):
    """gl_frame over the packed layout: y [hop*(N - B)] -> frw [N, n_fft]"""
    N, n_fft = frw.shape
    _f32c(y, "gl_frame_packed y"); _f32c(frw, "gl_frame_packed frw")
    B = _packed(off, "gl_frame_packed")
    assert y.dtype == frw.dtype == torch.float32 and y.shape == (hop * (N - B),)
    L.check(L.lib().taco_gl_frame_packed(_p(frw), _p(y), _p(off), B, int(max_frames), hop, n_fft, win_length, _st()),
            "taco_gl_frame_packed")


def normalize_f16(out, x, mean, std):
    """out fp32 [..., W] = the reference's in-place float16 normalisation of x (float16) followed by the float32 cast"""
    W = x.shape[-1]
    assert _on_device(x) and x.dtype == torch.float16 and x.is_contiguous() and out.dtype == torch.float32 and out.is_contiguous()
    assert mean.dtype == torch.float16 and std.dtype == torch.float32 and mean.numel() == W == std.numel() and out.shape == x.shape
    L.check(L.lib().taco_normalize_f16(_p(out), _p(x), _p(mean), _p(std), x.numel() // W, W, _st()), "taco_normalize_f16")


# ---- feature extraction (tacotron_b200/audio.py process_audio_batch) ----
def _cuda_c(t, dtype, name):
    if not (_on_device(t) and t.is_contiguous() and t.dtype == dtype):
        raise L.TacoError(f"{name}: expected a contiguous CUDA {dtype} tensor, got {t.dtype} {t.device}")
    return t


def trim_bounds(bounds, y, offsets, frame_length, hop, top_db):
    """bounds int32 [B, 2] = librosa.effects.trim's kept span of each utterance y[offsets[b]:offsets[b+1]] (fp32 y)"""
    B = offsets.numel() - 1
    _cuda_c(bounds, torch.int32, "trim_bounds bounds"); _cuda_c(y, torch.float32, "trim_bounds y")
    _cuda_c(offsets, torch.int64, "trim_bounds offsets")
    assert bounds.shape == (B, 2)
    L.check(L.lib().taco_trim_bounds(_p(bounds), _p(y), _p(offsets), B, frame_length, hop, float(top_db), _st()), "taco_trim_bounds")


def feature_frames(frw, y, start, length, max_len, hop, win_length, preemph):
    """frw fp32 [B, n, n_fft] = windowed frames of the pre-emphasised, zero-padded span y[start[b]:start[b]+length[b]]"""
    B, n, n_fft = frw.shape
    _f32c(frw, "feature_frames frw"); _cuda_c(y, torch.float32, "feature_frames y")
    _cuda_c(start, torch.int64, "feature_frames start"); _cuda_c(length, torch.int32, "feature_frames length")
    assert start.shape == (B,) and length.shape == (B,)
    L.check(L.lib().taco_feature_frames(_p(frw), _p(y), _p(start), _p(length), B, n, max_len, hop, n_fft, win_length,
                                        float(preemph), _st()), "taco_feature_frames")


def feature_spec(stft_out, mel_out, X, basis, lo, hi, r):
    """log |X| and log |basis . X| of X complex64 [B, n, 1025] in the reshape_frames layout: stft_out [B, T, 1025 r],
    mel_out [B, T, n_mels r], both float16 or both float32"""
    B, n, F = X.shape
    n_mels = basis.shape[0]
    f16 = stft_out.dtype == torch.float16
    for t, nm in ((stft_out, "stft_out"), (mel_out, "mel_out")):
        _cuda_c(t, torch.float16 if f16 else torch.float32, f"feature_spec {nm}")
    _cuda_c(X, torch.complex64, "feature_spec X"); _cuda_c(basis, torch.float32, "feature_spec basis")
    _cuda_c(lo, torch.int32, "feature_spec lo"); _cuda_c(hi, torch.int32, "feature_spec hi")
    T = 4 * (n // (4 * r))
    assert F == 1025 and basis.shape == (n_mels, F) and stft_out.shape == (B, T, F * r) and mel_out.shape == (B, T, n_mels * r)
    L.check(L.lib().taco_feature_spec(_p(stft_out), _p(mel_out), int(f16), _p(X), _p(basis), _p(lo), _p(hi), B, n, r, n_mels,
                                      _st()), "taco_feature_spec")


def resample(out, y, in_off, out_off, win_delta, step, ratio, treg):
    """out fp32 = librosa's kaiser_best resampling of each y[in_off[b]:in_off[b+1]] by one ratio into
    out[out_off[b]:out_off[b+1]] (ceil(n_in*ratio) samples, zeros after int(n_in*ratio)).  win_delta float64 [nwin, 2],
    treg float64 [>= the longest int(n_in*ratio)]: audio.resample_filter / audio.resample_register."""
    B = in_off.numel() - 1
    _cuda_c(out, torch.float32, "resample out"); _cuda_c(y, torch.float32, "resample y")
    _cuda_c(in_off, torch.int64, "resample in_off"); _cuda_c(out_off, torch.int64, "resample out_off")
    _cuda_c(win_delta, torch.float64, "resample win_delta"); _cuda_c(treg, torch.float64, "resample treg")
    assert out_off.shape == (B + 1,) and win_delta.dim() == 2 and win_delta.shape[1] == 2 and treg.dim() == 1
    L.check(L.lib().taco_resample(_p(out), _p(y), _p(in_off), _p(out_off), B, _p(win_delta), win_delta.shape[0], int(step),
                                  float(ratio), _p(treg), treg.numel(), _st()), "taco_resample")


# ---- training summaries (tacotron_b200/summary.py) ----
_hist_ws = {}


def histogram(res, x, limits):
    """TF 1.2's histogram of x (contiguous CUDA fp32, 16-byte aligned) into res int64 [nlim + 5]: res[:nlim] the bucket
    counts (a finite value goes to upper_bound(limits, value)), res[nlim] the NaN / Inf count (not binned),
    res[nlim+1:].view(float64) = {min, max, sum, sum of squares} of the finite values.  limits float64 [nlim] on the
    device = summary.histogram_limits()."""
    nlim = limits.numel()
    _cuda_c(x, torch.float32, "histogram x"); _cuda_c(res, torch.int64, "histogram res"); _cuda_c(limits, torch.float64, "histogram limits")
    assert res.shape == (nlim + 5,)
    ws = _hist_ws.get(x.device)
    if ws is None:
        ws = _hist_ws[x.device] = torch.empty(L.lib().taco_histogram_workspace_bytes(), dtype=torch.uint8, device=x.device)
    L.check(L.lib().taco_histogram(_p(x), x.numel(), _p(limits), nlim, _p(ws), _p(res), C.c_void_p(res.data_ptr() + 8 * (nlim + 1)),
                                   C.c_void_p(res.data_ptr() + 8 * nlim), _st()), "taco_histogram")


_ss_ws = {}


def sumsq(out, x):
    ws = _ss_ws.get(x.device)
    if ws is None:
        ws = _ss_ws[x.device] = torch.empty(2048, dtype=torch.float32, device=x.device)
    L.check(L.lib().taco_sumsq(_p(x), x.numel(), _p(ws), _p(out), _st()), "taco_sumsq")


def adam_step(p, g, m, v, lr_t, b1, b2, eps, clip, sumsq_t):
    for t in (p, g, m, v):
        assert t.is_contiguous() and _on_device(t) and t.dtype == torch.float32
    L.check(L.lib().taco_adam_step(_p(p), _p(g), _p(m), _p(v), p.numel(), float(lr_t), float(b1), float(b2), float(eps),
                                   float(clip), _p(sumsq_t), _st()), "taco_adam_step")
