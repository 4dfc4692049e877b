"""Parameter store for the H100 Tacotron path.

All variables of the hot path (reference: models/tacotron.py:107-154, models/ops.py:27-132; inventory
SURVEY.md section 8a) live in ONE flat fp32 device buffer in their TensorFlow layouts -- dense [in,out],
conv [k,Cin,Cout], GRU gates [in+n,2n] / candidate [in+n,n] -- so that (a) a TF checkpoint maps
1:1 by name, (b) the data-parallel gradient all-reduce and the fused Adam step see one bucket.
Kernel-side operand layouts (TF32 K-major packs, folded batch-norm affines, per-CTA decoder
slices, concatenated GRU input weights) are *derived* buffers refreshed after every update.
"""
from __future__ import annotations

import math
from collections import OrderedDict

import torch

BN_EPS = 1e-3   # tf.layers.batch_normalization default epsilon (models/ops.py:64,87)


def cbhg_shapes(prefix, cin, K, c, gru_units=128, n_hw=4):
    """Variables of one ops.CBHG call (models/ops.py:48-132).  The K bank filters are stored back
    to back (W1..WK, then b1..bK) so the grouped bank kernel sees one tensor."""
    out = []
    for k in range(1, K + 1):
        out.append((f"{prefix}/bank/W{k}", (k, cin, c[0]), "conv"))
    for k in range(1, K + 1):
        out.append((f"{prefix}/bank/b{k}", (c[0],), "zeros"))
    ch = K * c[0]
    for nm in ("gamma", "beta", "mean", "var"):
        out.append((f"{prefix}/bank/bn_{nm}", (ch,), nm))
    prev = ch
    for i, co in enumerate(c[1:], start=1):
        out.append((f"{prefix}/proj{i}/W", (3, prev, co), "conv"))
        out.append((f"{prefix}/proj{i}/b", (co,), "zeros"))
        for nm in ("gamma", "beta", "mean", "var"):
            out.append((f"{prefix}/proj{i}/bn_{nm}", (co,), nm))
        prev = co
    units = 128                                   # ops.highway(units=128)
    d = cin
    for l in range(n_hw):
        if d != units:                            # ops.py:29-30
            out.append((f"{prefix}/highway{l}/Wd", (d, units), "dense"))
            out.append((f"{prefix}/highway{l}/bd", (units,), "zeros"))
            d = units
        out.append((f"{prefix}/highway{l}/WT", (units, units), "dense"))
        out.append((f"{prefix}/highway{l}/bT", (units,), "zeros"))
        out.append((f"{prefix}/highway{l}/WH", (units, units), "dense"))
        out.append((f"{prefix}/highway{l}/bH", (units,), "zeros"))
    for dn in ("gru_fw", "gru_bw"):
        out.append((f"{prefix}/{dn}/Wg", (units + gru_units, 2 * gru_units), "dense"))
        out.append((f"{prefix}/{dn}/bg", (2 * gru_units,), "ones"))
        out.append((f"{prefix}/{dn}/Wc", (units + gru_units, gru_units), "dense"))
        out.append((f"{prefix}/{dn}/bc", (gru_units,), "zeros"))
    return out


def model_shapes(cfg):
    mel_out = cfg.mel_features * cfg.r
    U, A = cfg.decoder_units, cfg.attention_units
    P = [("embedding", (cfg.vocab_size, cfg.embed_dim), "dense")]
    P += [("enc/prenet/W1", (cfg.embed_dim, 256), "dense"), ("enc/prenet/b1", (256,), "zeros"),
          ("enc/prenet/W2", (256, 128), "dense"), ("enc/prenet/b2", (128,), "zeros")]
    P += cbhg_shapes("enc/cbhg", 128, 16, (128, 128, 128))
    P += [("dec/attn/W_mem", (256, A), "dense"), ("dec/attn/W_q", (mel_out, A), "dense"),
          ("dec/attn/v", (A,), "attn_v"), ("dec/attn/W_a", (mel_out + 256, A), "dense")]
    P += [("dec/prenet/W1", (cfg.mel_features, 256), "dense"), ("dec/prenet/b1", (256,), "zeros"),
          ("dec/prenet/W2", (256, 128), "dense"), ("dec/prenet/b2", (128,), "zeros")]
    P += [("dec/in_proj/W", (128 + A, U), "dense"), ("dec/in_proj/b", (U,), "zeros")]
    for i in (1, 2, 3):
        P += [(f"dec/gru{i}/Wg", (2 * U, 2 * U), "dense"), (f"dec/gru{i}/bg", (2 * U,), "ones"),
              (f"dec/gru{i}/Wc", (2 * U, U), "dense"), (f"dec/gru{i}/bc", (U,), "zeros")]
    P += [("dec/out_proj/W", (U, mel_out), "dense"), ("dec/out_proj/b", (mel_out,), "zeros")]
    P += cbhg_shapes("post/cbhg", cfg.mel_features, 8, (128, 256, 80))
    P += [("post/dense/W", (256, cfg.fft_size), "dense"), ("post/dense/b", (cfg.fft_size,), "zeros")]
    if getattr(cfg, "num_speakers", 1) > 1:
        P += speaker_shapes(cfg.num_speakers, getattr(cfg, "speaker_embed_dim", 16))
    if getattr(cfg, "speaker_decoder", False):
        if getattr(cfg, "num_speakers", 1) <= 1:
            raise ValueError("speaker_decoder needs a multi-speaker model (num_speakers > 1): there is no speaker embedding")
        P += decoder_speaker_shapes(getattr(cfg, "speaker_embed_dim", 16), U, A)
    return P


def speaker_shapes(num_speakers, E=16, n_hw=4, units=128):
    """Multi-speaker variables (tacotron.py:116-124, ops.py:101-115), stored after the single-speaker ones so that the
    layout of those does not depend on the speaker count: the speaker table; per encoder highway layer the speaker dense
    Ws/bs (E -> 128, relu) and the width-fixing dense Wd/bd of the [h | s] input (256 -> 128, ops.py:29-30); the dense
    gru_init/Ws,bs giving the initial state of both bi-GRU directions."""
    P = [("speaker/embed", (num_speakers, E), "dense")]
    for l in range(n_hw):
        P += [(f"enc/cbhg/highway{l}/Ws", (E, units), "dense"), (f"enc/cbhg/highway{l}/bs", (units,), "zeros"),
              (f"enc/cbhg/highway{l}/Wd", (2 * units, units), "dense"), (f"enc/cbhg/highway{l}/bd", (units,), "zeros")]
    P += [("enc/cbhg/gru_init/Ws", (E, units), "dense"), ("enc/cbhg/gru_init/bs", (units,), "zeros")]
    return P


def decoder_speaker_shapes(E=16, units=256, attention_units=256):
    """Speaker conditioning of the decoder (Config.speaker_decoder), stored after the other speaker variables: the dense
    giving the initial attention vector a(-1) = e.W + b (the reference's commented-out line, models/tacotron.py:96-97) and
    one dense per decoder GRU giving its initial state h_i(-1) = relu(e.W + b) (the form of ops.py:111-113)."""
    P = [("dec/spk/attn/W", (E, attention_units), "dense"), ("dec/spk/attn/b", (attention_units,), "zeros")]
    for i in (1, 2, 3):
        P += [(f"dec/spk/h{i}/W", (E, units), "dense"), (f"dec/spk/h{i}/b", (units,), "zeros")]
    return P


def _numel(shape):
    n = 1
    for s in shape:
        n *= s
    return n


class ParamStore:
    """Flat fp32 buffer + named views (each view 16-byte aligned)."""

    def __init__(self, shapes, device):
        self.device = torch.device(device)
        self.shapes = OrderedDict((n, (tuple(s), k)) for n, s, k in shapes)
        self.offsets = OrderedDict()
        off = 0
        for n, (s, _) in self.shapes.items():
            self.offsets[n] = off
            off += (_numel(s) + 3) // 4 * 4
        self.flat = torch.zeros(off, dtype=torch.float32, device=self.device)
        self.views = {n: self.flat[o:o + _numel(self.shapes[n][0])].view(self.shapes[n][0])
                      for n, o in self.offsets.items()}
        self.version = 0

    def __getitem__(self, name):
        return self.views[name]

    def __contains__(self, name):
        return name in self.views

    def names(self):
        return list(self.shapes.keys())

    def trainable(self):
        return [n for n in self.shapes if not (n.endswith("bn_mean") or n.endswith("bn_var"))]

    def span(self, first, last):
        """Contiguous flat slice covering variables first..last (inclusive); valid only when the
        variables in between are stored back to back without padding."""
        a = self.offsets[first]
        b = self.offsets[last] + _numel(self.shapes[last][0])
        return self.flat[a:b]

    def init_tf_default(self, seed=1):
        """glorot-uniform kernels, zero biases, GRU gate bias 1.0, BN gamma=1 beta=0 mean=0 var=1
        (TF-1.2 defaults; tacotron.py:111 xavier embedding)."""
        g = torch.Generator().manual_seed(seed)
        for n, (s, kind) in self.shapes.items():
            if kind in ("dense", "conv", "attn_v"):
                if kind == "dense":
                    fi, fo = s[0], s[1]
                elif kind == "conv":
                    fi, fo = s[0] * s[1], s[0] * s[2]
                else:
                    fi = fo = s[0]
                lim = math.sqrt(6.0 / (fi + fo))
                t = (torch.rand(s, generator=g, dtype=torch.float64) * 2 - 1) * lim
            elif kind in ("zeros", "beta", "mean"):
                t = torch.zeros(s, dtype=torch.float64)
            else:
                t = torch.ones(s, dtype=torch.float64)
            self.views[n].copy_(t.to(torch.float32))
        self.version += 1

    def load(self, params):
        """Copy a name -> tensor dict (any device / float dtype) into the store."""
        missing = [n for n in self.shapes if n not in params]
        if missing:
            raise KeyError(f"missing parameters: {missing[:5]}{'...' if len(missing) > 5 else ''}")
        for n in self.shapes:
            src = params[n]
            if tuple(src.shape) != self.shapes[n][0]:
                raise ValueError(f"{n}: shape {tuple(src.shape)} != {self.shapes[n][0]}")
            self.views[n].copy_(src.to(device=self.device, dtype=torch.float32))
        self.version += 1

    def state_dict(self):
        return {n: v.detach().cpu().clone() for n, v in self.views.items()}
