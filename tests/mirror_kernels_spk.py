"""TEST INFRASTRUCTURE ONLY -- tests/mirror_kernels.py plus the torch-CPU restatements of the multi-speaker entry points
(taco_bigru_fwd_h0, taco_bigru_bwd_h0, taco_colsum_seg, taco_linear_fwd's per-utterance bias).  This module is the
kernel namespace `K` that tacotron_b200/models/grad.py runs over on CPU for a multi-speaker model; the docstrings are the
specification of the CUDA kernels of the same names."""
from __future__ import annotations

import torch

from tests.mirror_kernels import *            # noqa: F401,F403  (the single-speaker namespace, unchanged)
from tests.mirror_kernels import ACT_NONE, bias_act_


def bigru_bwd_h0(dxp, dOut, out, ACT, Wg_h_fw, Wc_h_fw, Wg_h_bw, Wc_h_bw, h0_fw, h0_bw, dh0):
    """bigru_bwd for a forward that started from h0_fw / h0_bw [B,128] (None = zero): h0 is hprev of the first processed
    step (t = 0 fw, t = T-1 bw); dh0 [B,2,128] (or None) <- the carry left after the last step = d(loss)/d(h0) per direction."""
    B, T, _ = out.shape
    Hn = 128
    for d, (Wg, Wc, h0) in enumerate(((Wg_h_fw, Wc_h_fw, h0_fw), (Wg_h_bw, Wc_h_bw, h0_bw))):
        carry = torch.zeros(B, Hn, dtype=out.dtype, device=out.device)
        order = range(T - 1, -1, -1) if d == 0 else range(T)
        for t in order:
            tp = t - 1 if d == 0 else t + 1
            if 0 <= tp < T:
                hprev = out[:, tp, d * Hn:(d + 1) * Hn]
            else:
                hprev = h0 if h0 is not None else torch.zeros(B, Hn, dtype=out.dtype, device=out.device)
            a = ACT[:, t, d * 384:(d + 1) * 384]
            r, u, c = a[:, :Hn], a[:, Hn:2 * Hn], a[:, 2 * Hn:]
            dh = dOut[:, t, d * Hn:(d + 1) * Hn] + carry
            du_pre = dh * (hprev - c) * u * (1 - u)
            dc_pre = dh * (1 - u) * (1 - c * c)
            drh = dc_pre @ Wc.t()
            dr_pre = drh * hprev * r * (1 - r)
            carry = dh * u + drh * r + torch.cat([dr_pre, du_pre], -1) @ Wg.t()
            dxp[:, t, d * 384:(d + 1) * 384] = torch.cat([dr_pre, du_pre, dc_pre], -1)
        if dh0 is not None:
            dh0[:, d] = carry


def bigru_fwd_h0(out, xp, Wg_h_fw, Wc_h_fw, Wg_h_bw, Wc_h_bw, h0_fw, h0_bw):
    """taco_bigru_fwd_h0: xp [B,T,768] = hoisted input products + biases (fw gates | fw cand | bw gates | bw cand);
    out [B,T,256] = fw | bw states of GRUCell(128) started from h0_fw / h0_bw [B,128] (None = zero state)."""
    B, T, _ = out.shape
    Hn = 128
    for d, (Wg, Wc, h0) in enumerate(((Wg_h_fw, Wc_h_fw, h0_fw), (Wg_h_bw, Wc_h_bw, h0_bw))):
        h = h0 if h0 is not None else torch.zeros(B, Hn, dtype=out.dtype, device=out.device)
        for t in (range(T) if d == 0 else range(T - 1, -1, -1)):
            x = xp[:, t, d * 384:(d + 1) * 384]
            g = torch.sigmoid(x[:, :2 * Hn] + h @ Wg)
            r, u = g[:, :Hn], g[:, Hn:]
            c = torch.tanh(x[:, 2 * Hn:] + (r * h) @ Wc)
            h = u * h + (1 - u) * c
            out[:, t, d * Hn:(d + 1) * Hn] = h


def colsum_seg(out, A, period):
    """out[m // period, n] += sum of A[m, n] over the rows m of segment m // period  (A [M,N], M % period == 0)"""
    M, N = A.shape
    out.add_(A.reshape(M // period, period, N).sum(1))


def linear_bias_utt(X, W, bias, bias_utt, act=ACT_NONE):
    """taco_linear_fwd (dense) with a per-utterance bias: Y[b,t,n] = act(X[b,t].W[:,n] + (bias[n] + bias_utt[b,n]))"""
    v = X @ W
    bb = bias_utt[:, None, :] if bias is None else bias + bias_utt[:, None, :]
    Y = (v + bb).contiguous()
    bias_act_(Y.view(-1, Y.shape[-1]), None, act)
    return Y
