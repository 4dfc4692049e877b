"""TEST INFRASTRUCTURE ONLY -- float64 statement of the guided attention loss (Tachibana et al. 2017, "Efficiently
Trainable Text-to-Speech System Based on Deep Convolutional Networks with Guided Attention", arXiv:1710.08969), the
specification of taco_guided_attention and of Config.guided_attention.  The reference has no such term.

For utterance b with N_b = min(text_length[b], Tx) characters and T_b = speech_steps[b] voiced decoder steps:
    W[b,t,j] = 1 - exp(-(j/N_b - t/T_b)^2 / (2 g^2))   for t < T_b and j < N_b (0-based), else 0
    L_ga     = lam * sum_{b,t,j} align[b,t,j] * W[b,t,j]
and, per (b, t) row with s = sum_j align W, the gradient with respect to the attention scores (softmax backward of
lam * W) is lam * align * (W - s) inside the mask and 0 outside it."""
from __future__ import annotations

import torch


def band(text_length, speech_steps, T, Tx, g, dtype=torch.float64):
    """(W [B,T,Tx], mask [B,T,Tx] bool): the penalty weights and the positions t < T_b, j < N_b they are defined on"""
    B = len(text_length)
    W = torch.zeros(B, T, Tx, dtype=torch.float64)
    mask = torch.zeros(B, T, Tx, dtype=torch.bool)
    for b in range(B):
        n = min(int(text_length[b]), Tx)
        tb = int(speech_steps[b])
        if n < 1 or tb < 1:
            continue
        t = torch.arange(min(tb, T), dtype=torch.float64)[:, None]
        j = torch.arange(n, dtype=torch.float64)[None, :]
        W[b, :min(tb, T), :n] = 1.0 - torch.exp(-(j / n - t / tb) ** 2 / (2.0 * g * g))
        mask[b, :min(tb, T), :n] = True
    return W.to(dtype), mask


def loss(align, text_length, speech_steps, g, lam):
    """L_ga of align [B,T,Tx] (differentiable in align)"""
    W, _ = band(text_length, speech_steps, align.shape[1], align.shape[2], g, align.dtype)
    return lam * (align * W).sum()


def dscore(align, text_length, speech_steps, g, lam):
    """d(L_ga)/d(attention score) [B,T,Tx]: lam * align * (W - s) on the mask, 0 elsewhere"""
    W, mask = band(text_length, speech_steps, align.shape[1], align.shape[2], g, align.dtype)
    s = (align * W).sum(-1, keepdim=True)
    return torch.where(mask, lam * align * (W - s), torch.zeros_like(align))
