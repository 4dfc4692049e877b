"""TEST INFRASTRUCTURE ONLY -- free-running decoding with an attention window (Config.attention_window), in float64 over
the oracles of oracle/tacotron_oracle.py and tests/speaker_decoder_oracle.py.

The reference has no window, so this restatement is its specification.  For utterance b, N_b = min(text_length_b, Tx),
a window (back >= 0, ahead >= 1) and p(-1) = 0:
    W_t  = { j : max(0, p(t-1) - back) <= j <= p(t-1) + ahead, j < N_b }
    e_t  = the Bahdanau scores as without a window; e_tj = -inf for j not in W_t; alpha(t) = softmax(e_t)
    p(t) = the lowest j maximising e_tj over W_t (p(t-1) when W_t is empty, i.e. N_b = 0)
Everything else (context, attention vector, next input) follows alpha(t) exactly as without a window."""
from __future__ import annotations

import math

import torch

from oracle import tacotron_oracle as O
from oracle import tf12


def window_mask(p_prev, N, Tx, back, ahead):
    """[B, Tx] bool: the allowed positions W_t of each row, from p(t-1) [B] and N [B]"""
    j = torch.arange(Tx)[None, :]
    lo = (p_prev - back).clamp_min(0)[:, None]
    return (j >= lo) & (j <= (p_prev + ahead)[:, None]) & (j < N[:, None])


def window_step(score, N, p_prev, back, ahead):
    """score [B, Tx] (unmasked) -> (alpha [B, Tx], p [B], masked score [B, Tx])"""
    allowed = window_mask(p_prev, N, score.shape[1], back, ahead)
    e = torch.where(allowed, score, torch.full_like(score, -math.inf))
    any_ = allowed.any(1)
    alpha = torch.where(any_[:, None], torch.softmax(torch.where(any_[:, None], e, torch.zeros_like(e)), -1),
                        torch.zeros_like(e))
    alpha = torch.where(allowed, alpha, torch.zeros_like(alpha))
    p = torch.where(any_, torch.argmax(e, 1), p_prev)          # torch.argmax returns the first maximal index
    return alpha, p, e


def decoder(encoded, text_length, p, cfg, T, window, h0=None, att0=None, peaks=None, trace=None):
    """Free-running decoder (InferenceHelper) with the attention window (back, ahead).  h0 [3,B,256] / att0 [B,256]: the
    speaker-conditioned initial state (speaker_decoder_oracle.initial_state), None = zero.  peaks [B,T] (optional): the
    window of step t is built around peaks[:, t-1] instead of the oracle's own p(t-1) (t >= 1).  trace (optional)
    receives 'score' [B,T,Tx], the windowed scores (-inf outside W_t).  Returns (y [B,T,80r], alpha [B,T,Tx], p [B,T]):
    p is the oracle's own peak of every step, also when forced."""
    back, ahead = window
    B, Tx, _ = encoded.shape
    dt = encoded.dtype
    U = cfg.decoder_units
    mf, r = cfg.mel_features, cfg.r
    values, keys, _ = tf12.attention_prepare(encoded, text_length, p["dec/attn/W_mem"])
    N = text_length.to(torch.int64).clamp(max=Tx)
    h = [torch.zeros(B, U, dtype=dt) for _ in range(3)] if h0 is None else [h0[i] for i in range(3)]
    attn = torch.zeros(B, cfg.attention_units, dtype=dt) if att0 is None else att0
    x = torch.zeros(B, mf * r, dtype=dt)
    p_prev = torch.zeros(B, dtype=torch.int64)
    ys, als, ps, es = [], [], [], []
    for t in range(T):
        pn = O.pre_net(x[:, (r - 1) * mf:], p, "dec/prenet", cfg.audio_dropout_prob, None)
        z = tf12.dense(torch.cat([pn, attn], -1), p["dec/in_proj/W"], p["dec/in_proj/b"])
        inp = z
        for i in range(3):
            h[i] = tf12.gru_cell(inp, h[i], p[f"dec/gru{i+1}/Wg"], p[f"dec/gru{i+1}/bg"], p[f"dec/gru{i+1}/Wc"], p[f"dec/gru{i+1}/bc"])
            inp = h[i]
        y = tf12.dense(z + inp, p["dec/out_proj/W"], p["dec/out_proj/b"])
        pq = y @ p["dec/attn/W_q"]
        score = (p["dec/attn/v"] * torch.tanh(keys + pq[:, None, :])).sum(-1)
        if peaks is not None and t > 0:
            p_prev = peaks[:, t - 1].to(torch.int64)
        a, p_t, e = window_step(score, N, p_prev, back, ahead)
        ctx = torch.bmm(a[:, None, :], values)[:, 0]
        attn = torch.cat([y, ctx], -1) @ p["dec/attn/W_a"]
        ys.append(y)
        als.append(a)
        ps.append(p_t)
        es.append(e)
        p_prev = p_t
        x = y
    if trace is not None:
        trace["score"] = torch.stack(es, 1)
    return torch.stack(ys, 1), torch.stack(als, 1), torch.stack(ps, 1)


def inference(p, inputs, cfg, T, window, peaks=None):
    """O.inference (train=False) with the windowed decoder: (y, out, alpha, p)"""
    text = inputs["text"].to(torch.int64)
    emb = p["embedding"][text]
    pre = O.pre_net(emb, p, "enc/prenet", cfg.char_dropout_prob, None)
    encoded = O.cbhg(pre, p, "enc/cbhg", cfg.enc_K)
    y, align, pk = decoder(encoded, inputs["text_length"], p, cfg, T, window, peaks=peaks)
    B = y.shape[0]
    post = O.cbhg(y.reshape(B, -1, cfg.mel_features), p, "post/cbhg", cfg.post_K)
    out = tf12.dense(post, p["post/dense/W"], p["post/dense/b"]).reshape(B, -1, cfg.fft_size * cfg.r)
    return y, out, align, pk


def top_two_gap(score):
    """[..., Tx] windowed scores -> [...] difference between the highest and the second highest finite score (inf when a
    row has fewer than two allowed positions)"""
    if score.shape[-1] < 2:
        return torch.full(score.shape[:-1], math.inf, dtype=score.dtype)
    top = torch.topk(score, 2, dim=-1).values
    gap = top[..., 0] - top[..., 1]
    return torch.where(torch.isfinite(gap), gap, torch.full_like(gap, math.inf))
