"""TEST INFRASTRUCTURE ONLY -- the speaker-conditioned decoder (Config.speaker_decoder) over the oracles of
oracle/tacotron_oracle.py and tests/speaker_oracle.py, which it reuses unchanged for everything else.

The reference leaves this path commented out (models/tacotron.py:96-97), so this float64 restatement is its specification.
With e = speaker/embed[speaker] [B,16]:
    a(-1)   = e.Wa + ba                     initial attention vector (dec/spk/attn)
    h_i(-1) = relu(e.Wh_i + bh_i), i = 1..3  initial state of decoder GRU i (dec/spk/h{i}), the form of ops.py:111-113
Nothing else changes: step 0 computes z(0) = [p2(0), a(-1)].W_in + b_in and starts GRU i from h_i(-1)."""
from __future__ import annotations

from dataclasses import dataclass

import torch

from oracle import tacotron_oracle as O
from oracle import tf12
from tests import speaker_oracle as SO


@dataclass
class SpkDecOracleConfig(SO.SpkOracleConfig):
    speaker_decoder: bool = True


def decoder_speaker_param_shapes(cfg):
    """same names and order as tacotron_b200.params.decoder_speaker_shapes"""
    E = cfg.speaker_embed_dim
    P = [("dec/spk/attn/W", (E, cfg.attention_units), "dense"), ("dec/spk/attn/b", (cfg.attention_units,), "zeros")]
    for i in (1, 2, 3):
        P += [(f"dec/spk/h{i}/W", (E, cfg.decoder_units), "dense"), (f"dec/spk/h{i}/b", (cfg.decoder_units,), "zeros")]
    return P


def param_shapes(cfg):
    return SO.param_shapes(cfg) + decoder_speaker_param_shapes(cfg)


def init_params(cfg, seed=1, trained_like=False, dtype=torch.float32, zero=False):
    """SO.init_params (same values as an encoder-only multi-speaker model with this seed), then the decoder's speaker
    variables from a generator of their own: glorot kernels, biases 0 (or ~0.1 N(0,1) when trained_like); zero=True sets
    all of them to zero (a(-1) = h_i(-1) = 0: the encoder-only model)."""
    params = SO.init_params(cfg, seed=seed, trained_like=trained_like, dtype=dtype)
    gen = torch.Generator().manual_seed(seed + 2000)
    for name, shape, kind in decoder_speaker_param_shapes(cfg):
        if kind == "dense":
            t = O._glorot(gen, shape, shape[0], shape[1], dtype)
        else:
            t = torch.zeros(shape, dtype=dtype)
            if trained_like:
                t = (0.1 * torch.randn(shape, generator=gen, dtype=torch.float64)).to(dtype)
        params[name] = torch.zeros(shape, dtype=dtype) if zero else t
    return params


def initial_state(p, e):
    """(h0 [3,B,256], att0 [B,256]) of speaker rows e [B,16]"""
    att0 = tf12.dense(e, p["dec/spk/attn/W"], p["dec/spk/attn/b"])
    h0 = torch.stack([tf12.dense(e, p[f"dec/spk/h{i}/W"], p[f"dec/spk/h{i}/b"], torch.relu) for i in (1, 2, 3)])
    return h0, att0


def decoder(encoded, text_length, p, cfg, mode, T, h0, att0, mel=None, drop_masks=None, sample_mask=None, trace=None):
    """O.decoder started from h_i(-1) = h0[i] and a(-1) = att0 instead of zeros.  trace (optional) receives 'dec/z0'
    (z(0)), 'dec/H' ([3,T,B,256] state sequences), 'dec/keys', 'dec/values'."""
    B, Tx, _ = encoded.shape
    dt = encoded.dtype
    U = cfg.decoder_units
    mf, r = cfg.mel_features, cfg.r
    values, keys, mask = tf12.attention_prepare(encoded, text_length, p["dec/attn/W_mem"])
    h = [h0[i] for i in range(3)]
    attn = att0
    x = torch.zeros(B, mf * r, dtype=dt) if mode == "infer" else mel[:, 0]
    ys, als, hs = [], [], []
    for t in range(T):
        dm = None if drop_masks is None else (drop_masks[0][t], drop_masks[1][t])
        pn = O.pre_net(x[:, (r - 1) * mf:], p, "dec/prenet", cfg.audio_dropout_prob, dm)
        z = tf12.dense(torch.cat([pn, attn], -1), p["dec/in_proj/W"], p["dec/in_proj/b"])
        if t == 0 and trace is not None:
            trace["dec/z0"] = z
        inp = z
        for i in range(3):
            h[i] = tf12.gru_cell(inp, h[i], p[f"dec/gru{i+1}/Wg"], p[f"dec/gru{i+1}/bg"], p[f"dec/gru{i+1}/Wc"], p[f"dec/gru{i+1}/bc"])
            inp = h[i]
        hs.append(torch.stack(h))
        y = tf12.dense(z + inp, p["dec/out_proj/W"], p["dec/out_proj/b"])
        a = tf12.bahdanau_alignments(y, keys, mask, p["dec/attn/W_q"], p["dec/attn/v"])
        ctx = torch.bmm(a[:, None, :], values)[:, 0]
        attn = torch.cat([y, ctx], -1) @ p["dec/attn/W_a"]
        ys.append(y)
        als.append(a)
        if mode == "infer":
            x = y
        else:
            nxt = mel[:, t + 1] if t + 1 < T else torch.zeros_like(y)
            x = torch.where(sample_mask[t].to(torch.bool)[:, None], y, nxt) if mode == "sched" else nxt
    if trace is not None:
        trace["dec/H"] = torch.stack(hs, 1)
        trace["dec/keys"], trace["dec/values"] = keys, values
    return torch.stack(ys, 1), torch.stack(als, 1)


def inference(p, inputs, cfg, train=False, enc_drop_masks=None, dec_drop_masks=None, sample_mask=None, T=None, trace=None):
    """SO.inference with the speaker-conditioned decoder"""
    text = inputs["text"].to(torch.int64)
    emb = p["embedding"][text]
    e = p["speaker/embed"][inputs["speaker"].to(torch.int64)]
    pre = O.pre_net(emb, p, "enc/prenet", cfg.char_dropout_prob, enc_drop_masks)
    encoded = SO.cbhg_spk(pre, p, "enc/cbhg", cfg.enc_K, e, trace=trace)
    if train:
        mel = inputs["mel"]
        T = mel.shape[1] if T is None else T
        mode = "sched" if sample_mask is not None else "teacher"
    else:
        mel = None
        T = cfg.max_decode_iter if T is None else T
        mode = "infer"
    h0, att0 = initial_state(p, e)
    y, align = decoder(encoded, inputs["text_length"], p, cfg, mode, T, h0, att0, mel=mel, drop_masks=dec_drop_masks,
                       sample_mask=sample_mask, trace=trace)
    B = y.shape[0]
    post = O.cbhg(y.reshape(B, -1, cfg.mel_features), p, "post/cbhg", cfg.post_K, trace=trace)
    out = tf12.dense(post, p["post/dense/W"], p["post/dense/b"]).reshape(B, -1, cfg.fft_size * cfg.r)
    if trace is not None:
        trace["encoded"] = encoded
    return y, out, align


def loss_and_grads(p, inputs, cfg, enc_drop_masks=None, dec_drop_masks=None, sample_mask=None):
    """O.loss_and_grads over the speaker-conditioned forward"""
    q = {k: v.detach().clone().requires_grad_(not k.endswith(O.NON_TRAINABLE_SUFFIXES)) for k, v in p.items()}
    y, out, _ = inference(q, inputs, cfg, train=True, enc_drop_masks=enc_drop_masks, dec_drop_masks=dec_drop_masks,
                          sample_mask=sample_mask)
    total, _, _ = O.loss(y, out, inputs["mel"].to(y.dtype), inputs["stft"].to(y.dtype))
    names = [k for k, v in q.items() if v.requires_grad]
    grads = torch.autograd.grad(total, [q[k] for k in names])
    return total.detach(), dict(zip(names, grads))


def saving_forward(p, inputs, cfg, enc_masks, dec_masks, sample_mask):
    """tests/grad_util_spk.saving_forward_spk for a speaker-conditioned decoder: also records what its backward reads
    (dec/spk_e, dec/spk_s = [a(-1) | h_1(-1) | h_2(-1) | h_3(-1)], dec/h0 [3,B,256], dec/att0)."""
    from tests import grad_util, grad_util_spk
    S = {"text": inputs["text"], "text_length": inputs["text_length"], "mel": inputs["mel"], "stft": inputs["stft"],
         "speaker": inputs["speaker"]}
    text = inputs["text"].to(torch.int64)
    ks = 1.0 / (1.0 - cfg.char_dropout_prob)
    t1 = torch.relu(p["embedding"] @ p["enc/prenet/W1"] + p["enc/prenet/b1"])
    l1 = t1[text] * enc_masks[0].to(t1.dtype) * ks
    l2 = torch.relu(l1 @ p["enc/prenet/W2"] + p["enc/prenet/b2"]) * enc_masks[1].to(t1.dtype) * ks
    S["enc/prenet/t1"], S["enc/prenet/l1"], S["enc/prenet/l2"] = t1, l1, l2
    e = p["speaker/embed"][inputs["speaker"].to(torch.int64)]
    encoded = grad_util_spk.cbhg_saving_spk(l2, p, "enc/cbhg", cfg.enc_K, S, e)
    T = inputs["mel"].shape[1]
    S["dec/keep1"], S["dec/keep2"] = dec_masks
    if sample_mask is not None:
        S["dec/sample_mask"] = sample_mask
    h0, att0 = initial_state(p, e)
    S["dec/spk_e"], S["dec/spk_s"] = e, torch.cat([att0, *h0], 1)
    S["dec/h0"], S["dec/att0"] = h0.contiguous(), att0.contiguous()
    tr = {}
    y, align = decoder(encoded, inputs["text_length"], p, cfg, "sched" if sample_mask is not None else "teacher", T, h0, att0,
                       mel=inputs["mel"], drop_masks=dec_masks, sample_mask=sample_mask, trace=tr)
    S["dec/values"], S["dec/keys"] = tr["dec/values"], tr["dec/keys"]
    S["dec/y"], S["dec/align"] = y.contiguous(), align.contiguous()
    S["dec/H"] = tr["dec/H"].contiguous()
    B = y.shape[0]
    post = grad_util.cbhg_saving(y.reshape(B, -1, cfg.mel_features), p, "post/cbhg", cfg.post_K, S)
    out = tf12.dense(post, p["post/dense/W"], p["post/dense/b"]).reshape(B, -1, cfg.fft_size * cfg.r)
    S["post/out"] = out
    return S, y, out
