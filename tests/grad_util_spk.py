"""Test helper: the multi-speaker counterpart of tests/grad_util.py -- an oracle forward that also returns the
activations the train-mode CUDA forward of a multi-speaker model saves (names = the S[...] keys of
tacotron_b200/models/grad.py), built from oracle/tf12.py primitives."""
from __future__ import annotations

import torch

from oracle import tf12
from tests import speaker_oracle as SO
from tests.grad_util import _bn, cbhg_saving, decoder_saving
def cbhg_saving_spk(x, p, prefix, K, S, e):
    """cbhg_saving for a speaker-conditioned CBHG (ops.py:101-115), e [B,16]; records what the multi-speaker backward
    reads: spk_e, spk_s = relu(e.[Ws_0..Ws_3 | Ws_init] + bs), h0, and per highway layer its outer input hw{l}_x."""
    B, T, Cin = x.shape
    S[f"{prefix}/x_in"] = x
    bank = torch.cat([tf12.conv1d_same(x, p[f"{prefix}/bank/W{k}"], p[f"{prefix}/bank/b{k}"], torch.relu)
                      for k in range(1, K + 1)], -1)
    bank_bn = _bn(p, f"{prefix}/bank", bank, S)
    S[f"{prefix}/bank_bn"] = bank_bn
    pool = tf12.max_pool_2_1_same(bank_bn)
    S[f"{prefix}/bank_pool"] = pool
    p1 = _bn(p, f"{prefix}/proj1", tf12.conv1d_same(pool, p[f"{prefix}/proj1/W"], p[f"{prefix}/proj1/b"], torch.relu), S)
    S[f"{prefix}/proj1"] = p1
    res = _bn(p, f"{prefix}/proj2", tf12.conv1d_same(p1, p[f"{prefix}/proj2/W"], p[f"{prefix}/proj2/b"]), S) + x
    S[f"{prefix}/res"] = res
    names = [f"highway{l}" for l in range(4)] + ["gru_init"]
    Sv = torch.relu(e @ torch.cat([p[f"{prefix}/{n}/Ws"] for n in names], 1) + torch.cat([p[f"{prefix}/{n}/bs"] for n in names]))
    S[f"{prefix}/spk_e"], S[f"{prefix}/spk_s"] = e, Sv
    h = res
    for l in range(4):
        pre = f"{prefix}/highway{l}"
        S[f"{prefix}/hw{l}_x"] = h
        u = Sv[:, 128 * l:128 * (l + 1)] @ p[f"{pre}/Wd"][128:] + p[f"{pre}/bd"]
        h = h @ p[f"{pre}/Wd"][:128] + u[:, None, :]
        S[f"{prefix}/hw{l}_in"] = h
        Pm = torch.cat([tf12.dense(h, p[f"{pre}/WH"], p[f"{pre}/bH"]), tf12.dense(h, p[f"{pre}/WT"], p[f"{pre}/bT"])], -1)
        S[f"{prefix}/hw{l}_P"] = Pm
        h = torch.relu(Pm[..., :128]) * torch.sigmoid(Pm[..., 128:]) + h * (1 - torch.sigmoid(Pm[..., 128:]))
    S[f"{prefix}/hw_out"] = h
    h0 = Sv[:, 512:].contiguous()
    S[f"{prefix}/h0"] = h0
    fw = tuple(p[f"{prefix}/gru_fw/{n}"] for n in ("Wg", "bg", "Wc", "bc"))
    bw = tuple(p[f"{prefix}/gru_bw/{n}"] for n in ("Wg", "bg", "Wc", "bc"))
    Wx = torch.cat([fw[0][:128], fw[2][:128], bw[0][:128], bw[2][:128]], 1)
    bx = torch.cat([fw[1], fw[3], bw[1], bw[3]])
    S[f"{prefix}/xp"] = h @ Wx + bx
    out = SO.bidirectional_gru_h0(h, fw, bw, h0)
    S[f"{prefix}/gru_out"] = out
    return out


def saving_forward_spk(p, inputs, cfg, enc_masks, dec_masks, sample_mask):
    """saving_forward for a multi-speaker model (inputs['speaker'] int [B])."""
    S = {"text": inputs["text"], "text_length": inputs["text_length"], "mel": inputs["mel"], "stft": inputs["stft"],
         "speaker": inputs["speaker"]}
    text = inputs["text"].to(torch.int64)
    ks = 1.0 / (1.0 - cfg.char_dropout_prob)
    t1 = torch.relu(p["embedding"] @ p["enc/prenet/W1"] + p["enc/prenet/b1"])
    l1 = t1[text] * enc_masks[0].to(t1.dtype) * ks
    l2 = torch.relu(l1 @ p["enc/prenet/W2"] + p["enc/prenet/b2"]) * enc_masks[1].to(t1.dtype) * ks
    S["enc/prenet/t1"], S["enc/prenet/l1"], S["enc/prenet/l2"] = t1, l1, l2
    e = p["speaker/embed"][inputs["speaker"].to(torch.int64)]
    encoded = cbhg_saving_spk(l2, p, "enc/cbhg", cfg.enc_K, S, e)
    T = inputs["mel"].shape[1]
    S["dec/keep1"], S["dec/keep2"] = dec_masks
    if sample_mask is not None:
        S["dec/sample_mask"] = sample_mask
    y = decoder_saving(encoded, inputs["text_length"], p, cfg, T, inputs["mel"], dec_masks, sample_mask, S)
    B = y.shape[0]
    post = cbhg_saving(y.reshape(B, -1, cfg.mel_features), p, "post/cbhg", cfg.post_K, S)
    out = tf12.dense(post, p["post/dense/W"], p["post/dense/b"]).reshape(B, -1, cfg.fft_size * cfg.r)
    S["post/out"] = out
    return S, y, out
