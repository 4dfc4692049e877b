"""TEST INFRASTRUCTURE ONLY -- the multi-speaker path of the reference model (models/tacotron.py:116-124,
models/ops.py:101-126) over the oracle of oracle/tacotron_oracle.py, which it reuses unchanged for everything the speaker
does not touch (pre-nets, conv bank / projections, highway, decoder, post-net, loss).

S = num_speakers, e[b] = speaker/embed[speaker[b]] ([S,16]).  Only the encoder CBHG is conditioned: highway layer l sees
[h | tile(relu(e.Ws_l + bs_l))] (256 wide, so highway's width-fixing dense Wd_l [256,128] applies, ops.py:29-30), and the
bi-GRU starts both directions from relu(e.Wg + bg) (ops.py:111-126)."""
from __future__ import annotations

from dataclasses import dataclass

import torch

from oracle import tacotron_oracle as O
from oracle import tf12


@dataclass
class SpkOracleConfig(O.OracleConfig):
    num_speakers: int = 3
    speaker_embed_dim: int = 16


def speaker_param_shapes(cfg):
    """the multi-speaker variables, after the single-speaker ones (same names as tacotron_b200.params.speaker_shapes)"""
    E, U = cfg.speaker_embed_dim, 128
    P = [("speaker/embed", (cfg.num_speakers, E), "dense")]
    for l in range(cfg.num_highway_layers):
        P += [(f"enc/cbhg/highway{l}/Ws", (E, U), "dense"), (f"enc/cbhg/highway{l}/bs", (U,), "zeros"),
              (f"enc/cbhg/highway{l}/Wd", (2 * U, U), "dense"), (f"enc/cbhg/highway{l}/bd", (U,), "zeros")]
    P += [("enc/cbhg/gru_init/Ws", (E, cfg.gru_units), "dense"), ("enc/cbhg/gru_init/bs", (cfg.gru_units,), "zeros")]
    return P


def param_shapes(cfg):
    return O.param_shapes(cfg) + speaker_param_shapes(cfg)


def init_params(cfg, seed=1, trained_like=False, dtype=torch.float32):
    """O.init_params for the single-speaker variables (same values as a single-speaker model with this seed), then the
    speaker variables from a generator of their own: glorot kernels, biases 0 (or ~0.1 N(0,1) when trained_like)."""
    params = O.init_params(cfg, seed=seed, trained_like=trained_like, dtype=dtype)
    gen = torch.Generator().manual_seed(seed + 1000)
    for name, shape, kind in speaker_param_shapes(cfg):
        if kind == "dense":
            params[name] = O._glorot(gen, shape, shape[0], shape[1], dtype)
        else:
            t = torch.zeros(shape, dtype=dtype)
            if trained_like:
                t = (0.1 * torch.randn(shape, generator=gen, dtype=torch.float64)).to(dtype)
            params[name] = t
    return params


def bidirectional_gru_h0(x, fw, bw, h0):
    """tf12.bidirectional_gru with initial_state_fw = initial_state_bw = h0 [B,n] (ops.py:118-126)"""
    B, T, _ = x.shape
    hf, hb = h0, h0
    of, ob = [None] * T, [None] * T
    for t in range(T):
        hf = tf12.gru_cell(x[:, t], hf, *fw)
        of[t] = hf
        tb = T - 1 - t
        hb = tf12.gru_cell(x[:, tb], hb, *bw)
        ob[tb] = hb
    return torch.cat([torch.stack(of, 1), torch.stack(ob, 1)], -1)


def cbhg_spk(x, p, prefix, K, e, n_proj=2, n_hw=4, trace=None):
    """O.cbhg with speaker_embed e [B,16] (ops.py:48-132)"""
    def bn(t, pre):
        return tf12.batch_norm_inference(t, p[f"{pre}/bn_gamma"], p[f"{pre}/bn_beta"], p[f"{pre}/bn_mean"], p[f"{pre}/bn_var"])
    bank = torch.cat([tf12.conv1d_same(x, p[f"{prefix}/bank/W{k}"], p[f"{prefix}/bank/b{k}"], torch.relu)
                      for k in range(1, K + 1)], -1)
    bank = tf12.max_pool_2_1_same(bn(bank, f"{prefix}/bank"))
    proj = bank
    for i in range(1, n_proj + 1):
        act = None if i == n_proj else torch.relu
        proj = bn(tf12.conv1d_same(proj, p[f"{prefix}/proj{i}/W"], p[f"{prefix}/proj{i}/b"], act), f"{prefix}/proj{i}")
    h = proj + x
    for l in range(n_hw):                                       # ops.py:97-107
        s = tf12.dense(e, p[f"{prefix}/highway{l}/Ws"], p[f"{prefix}/highway{l}/bs"], torch.relu)
        h = torch.cat([h, s[:, None, :].expand(-1, h.shape[1], -1)], 2)
        h = O.highway(h, p, f"{prefix}/highway{l}")
    fw = tuple(p[f"{prefix}/gru_fw/{n}"] for n in ("Wg", "bg", "Wc", "bc"))
    bw = tuple(p[f"{prefix}/gru_bw/{n}"] for n in ("Wg", "bg", "Wc", "bc"))
    h0 = tf12.dense(e, p[f"{prefix}/gru_init/Ws"], p[f"{prefix}/gru_init/bs"], torch.relu)
    out = bidirectional_gru_h0(h, fw, bw, h0)
    if trace is not None:
        trace[f"{prefix}/highway_out"] = h
        trace[f"{prefix}/out"] = out
    return out


def inference(p, inputs, cfg, train=False, enc_drop_masks=None, dec_drop_masks=None, sample_mask=None, T=None, trace=None):
    """O.inference for a multi-speaker model: inputs['speaker'] int [B] selects the rows of speaker/embed"""
    text = inputs["text"].to(torch.int64)
    emb = p["embedding"][text]
    e = p["speaker/embed"][inputs["speaker"].to(torch.int64)]                          # tacotron.py:116-124
    pre = O.pre_net(emb, p, "enc/prenet", cfg.char_dropout_prob, enc_drop_masks)
    encoded = cbhg_spk(pre, p, "enc/cbhg", cfg.enc_K, e, trace=trace)
    if train:
        mel = inputs["mel"]
        T = mel.shape[1] if T is None else T
        mode = "sched" if sample_mask is not None else "teacher"
    else:
        mel = None
        T = cfg.max_decode_iter if T is None else T
        mode = "infer"
    y, align = O.decoder(encoded, inputs["text_length"], p, cfg, mode, T, mel=mel, drop_masks=dec_drop_masks,
                         sample_mask=sample_mask, trace=trace)
    B = y.shape[0]
    post = O.cbhg(y.reshape(B, -1, cfg.mel_features), p, "post/cbhg", cfg.post_K, trace=trace)
    out = tf12.dense(post, p["post/dense/W"], p["post/dense/b"]).reshape(B, -1, cfg.fft_size * cfg.r)
    if trace is not None:
        trace["encoded"] = encoded
    return y, out, align


def loss_and_grads(p, inputs, cfg, enc_drop_masks=None, dec_drop_masks=None, sample_mask=None):
    """O.loss_and_grads over the multi-speaker forward"""
    q = {k: v.detach().clone().requires_grad_(not k.endswith(O.NON_TRAINABLE_SUFFIXES)) for k, v in p.items()}
    y, out, _ = inference(q, inputs, cfg, train=True, enc_drop_masks=enc_drop_masks, dec_drop_masks=dec_drop_masks,
                          sample_mask=sample_mask)
    total, _, _ = O.loss(y, out, inputs["mel"].to(y.dtype), inputs["stft"].to(y.dtype))
    names = [k for k, v in q.items() if v.requires_grad]
    grads = torch.autograd.grad(total, [q[k] for k in names])
    return total.detach(), dict(zip(names, grads))
