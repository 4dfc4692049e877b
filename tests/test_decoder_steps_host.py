"""The decoder's step-by-step check (tests/decoder_step_checks.py) on the CPU: it passes decoders computed in float32 and
reports float64 ones at float64 level, its infer-mode rebuild is the oracle's free-running step, one corrupted element is
reported at exactly its place, and its bars restate the derivation on a case small enough to follow by hand."""
import math

import pytest
import torch

from oracle import tacotron_oracle as O
from tests import decoder_step_checks as DC
from tests import speaker_decoder_oracle as SD
from tests.util import ocfg


def _run(dtype, mode, r, state, B=4, Tx=13, T=9):
    """a decoder in `dtype` through the float64-capable oracle (speaker_decoder_oracle.decoder: O.decoder from an initial
    state, zero when `state` is False) and its state sequences.  Tx = 13: attention quarters of 4, lengths 13, 4, 5, 9
    end on and just past quarter boundaries."""
    cfg = ocfg(r=r, T=T, vocab=20)
    p = {k: v.to(dtype) for k, v in O.init_params(cfg, seed=1, trained_like=True).items()}
    g = torch.Generator().manual_seed(0)
    enc = (torch.randn(B, Tx, 256, generator=g) * 0.5).to(dtype)
    tl = torch.tensor([13, 4, 5, 9][:B], dtype=torch.int32)
    mel = O.synthetic_inputs(cfg, B, Tx, T, seed=0, ragged=True)["mel"].to(dtype)
    _, dm = O.dropout_masks(cfg, B, Tx, T, seed=2)
    sm = O.sched_mask(cfg, B, T, seed=3)
    h0 = (torch.rand(3, B, 256, generator=g) * 0.6).to(dtype) if state else torch.zeros(3, B, 256, dtype=dtype)
    att0 = torch.randn(B, 256, generator=g).to(dtype) if state else torch.zeros(B, 256, dtype=dtype)
    drop = None if mode == "infer" else dm
    tr = {}
    y, a = SD.decoder(enc, tl, p, cfg, mode, T, h0, att0, mel=mel, drop_masks=drop,
                      sample_mask=sm if mode == "sched" else None, trace=tr)
    kw = dict(mel=mel, sample_mask=sm, keep=drop, keep_scale=1.0 / (1.0 - cfg.audio_dropout_prob),
              h0=h0 if state else None, att0=att0 if state else None)
    return dict(y=y, align=a, H=tr["dec/H"], p=p, keys=tr["dec/keys"], values=tr["dec/values"], tl=tl, r=r, mode=mode,
                kw=kw, cfg=cfg, enc=enc)


def _check(d, **over):
    args = dict(y=d["y"], align=d["align"], H=d["H"])
    args.update(over)
    return DC.check(args["y"], args["align"], args["H"], d["p"], d["keys"], d["values"], d["tl"], d["r"], d["mode"], **d["kw"])


@pytest.mark.parametrize("state", [False, True])
@pytest.mark.parametrize("r", [2, 5])
@pytest.mark.parametrize("mode", ["infer", "teacher", "sched"])
def test_float32_decoder_passes_float64_is_exact(mode, r, state):
    rep = _check(_run(torch.float32, mode, r, state))
    assert rep.first is None, rep.first
    assert all(v < 0.5 for v in rep.worst.values()), rep
    rep = _check(_run(torch.float64, mode, r, state))
    assert rep.first is None and all(v < 1e-6 for v in rep.worst.values()), rep


def test_infer_rebuild_is_the_oracles_free_running_step():
    d = _run(torch.float64, "infer", 5, False)
    y_o, a_o = O.decoder(d["enc"], d["tl"], d["p"], d["cfg"], "infer", d["y"].shape[1])
    assert torch.allclose(d["y"], y_o, rtol=0, atol=1e-12) and torch.allclose(d["align"], a_o, rtol=0, atol=1e-12)
    rep = _check(d)
    scale = y_o.abs().max()
    assert (rep.ref["y"] - y_o.transpose(0, 1)).abs().max() <= 1e-12 * scale
    assert (rep.ref["align"] - a_o.transpose(0, 1)).abs().max() <= 1e-12
    for i in range(3):
        assert (rep.ref[f"h{i+1}"] - d["H"][i]).abs().max() <= 1e-12


@pytest.mark.parametrize("stage,t,b,n", [("h2", 3, 1, 17), ("y", 2, 2, 33), ("align", 4, 0, None)])
def test_one_corrupted_element_is_the_first_failure(stage, t, b, n):
    d = _run(torch.float32, "sched", 2, True)
    rep = _check(d)
    assert rep.first is None
    if n is None:                                   # the row's largest weight: far from the flush floor
        n = int(d["align"][b, t].argmax())
    bar = float(rep.bar[stage][t, b, n])
    over = {}
    if stage == "h2":
        H = d["H"].clone().double()
        H[1, t, b, n] += 8 * bar
        over["H"] = H
    else:
        X = d[stage].clone().double()
        X[b, t, n] += 8 * bar
        over[stage] = X
    f = _check(d, **over).first
    assert f is not None and (f.t, f.stage, f.b, f.unit) == (t, stage, b, n), f


def test_bars_restated_by_hand():
    """one unit and two keys"""
    u, eps = 2.0 ** -24, 2.0 ** -20
    # GRU: r = 0.4, u = 0.7, c = -0.2, h(t-1) = 0.5, S_g = (2, 3), S_c = 1.5, |Wc_h| = 0.8, C = 2
    RU, cc, hp = torch.tensor([[0.4, 0.7]], dtype=torch.float64), torch.tensor([[-0.2]], dtype=torch.float64), torch.tensor([[0.5]], dtype=torch.float64)
    h, bar = DC.gru_bar(RU, cc, hp, torch.tensor([[2.0, 3.0]], dtype=torch.float64), torch.tensor([[1.5]], dtype=torch.float64),
                        torch.tensor([[0.8]], dtype=torch.float64), c=2.0)
    d_r = 0.4 * 0.6 * 2 * eps * 2.0 + 2.5e-7                      # sigma (1 - sigma) C 2^-20 S_g + 2.5e-7
    d_u = 0.7 * 0.3 * 2 * eps * 3.0 + 2.5e-7
    d_c = (1 - 0.04) * (2 * eps * 1.5 + d_r * 0.5 * 0.8) + 5e-7    # (1 - c^2) (C 2^-20 S_c + |dr| |h| |Wc_h|) + 5e-7
    hv = 0.7 * 0.5 + 0.3 * -0.2
    want = abs(0.5 + 0.2) * d_u + 0.3 * d_c + 2 * u * (abs(0.3 * -0.2) + abs(0.7 * 0.5) + abs(hv))
    assert float(h) == pytest.approx(0.29, rel=1e-15) and float(bar) == pytest.approx(want, rel=1e-12)
    assert want == pytest.approx(2.2078e-6, rel=1e-4)
    # scores: v = 0.5, q = 0.4 (bar 1e-6), keys 0.3 and -1.2
    k = torch.tensor([[0.3], [-1.2]], dtype=torch.float64)
    q, v = 0.4, torch.tensor([0.5], dtype=torch.float64)
    th = torch.tanh(k + q)
    e = (th * v).sum(-1)
    dE = DC.score_bar(th, e, v, 1e-6, k.abs(), abs(q))
    t0, t1 = math.tanh(0.7), math.tanh(-0.8)
    want = [0.5 * (1 - t ** 2) * (1e-6 + u * (abs(kk) + 0.4 + 2)) + 7 * u * 0.5 * (1 - t) + u * (4 * 0.5 + abs(0.5 * t))
            for t, kk in ((t0, 0.3), (t1, -1.2))]
    assert dE.tolist() == pytest.approx(want, rel=1e-12)
    assert want == pytest.approx([5.8820e-07, 8.2565e-07], rel=1e-4)
    # softmax of the two scores
    a = torch.softmax(e, -1)
    dist = (e - e.max()).abs()
    bar = DC.softmax_bar(a, dE, dist)
    a0, a1 = a.tolist()
    s_de = a0 * want[0] + a1 * want[1]
    s_dist = a1 * abs(0.5 * (t1 - t0))
    want_a = [a0 * (want[0] + s_de + u * (0 + 3 * s_dist + 24)) + 2.0 ** -126,
              a1 * (want[1] + s_de + u * (3 * abs(0.5 * (t1 - t0)) + 3 * s_dist + 24)) + 2.0 ** -126]
    assert bar.tolist() == pytest.approx(want_a, rel=1e-12)


def _tf32(x):
    """x with its fp32 mantissa cut to TF32's 10 bits (the tensor core's single-pass operand), as float64"""
    i = x.float().contiguous().view(torch.int32) & ~0x1FFF
    return i.view(torch.float32).double()


@pytest.mark.parametrize("stage", ["h1", "y", "align"])
def test_tf32_grade_stage_is_flagged(stage):
    """a stage whose products lost fp32 grade (single-pass TF32, no correction term) is flagged at step 0, at that stage:
    h1 from TF32 gate and candidate products, y = s . W_out in TF32, align from a TF32 q = y . W_q"""
    from types import SimpleNamespace
    from tacotron_b200.models import grad
    from tests import mirror_kernels as MK
    d = _run(torch.float32, "infer", 2, False)
    p = {k: v.double() for k, v in d["p"].items()}
    T, B = d["y"].shape[1], d["y"].shape[0]
    S = {"dec/y": d["y"].double(), "dec/align": d["align"].double(), "dec/H": d["H"].double(),
         "dec/values": d["values"].double(), "mel": torch.zeros_like(d["y"], dtype=torch.float64),
         "dec/sample_mask": torch.ones(T, B, dtype=torch.uint8), "dec/keep1": torch.ones(T, B, 256, dtype=torch.uint8),
         "dec/keep2": torch.ones(T, B, 128, dtype=torch.uint8)}
    R = grad.decoder_recompute(MK, p, S, SimpleNamespace(mel_features=80, r=2, audio_dropout_prob=0.0))
    Z = R["Z"].view(T, B, 256)
    over = {}
    if stage == "h1":
        hp = torch.cat([torch.zeros(1, B, 256, dtype=torch.float64), S["dec/H"][0][:-1]])
        Wg, Wc = _tf32(p["dec/gru1/Wg"]), _tf32(p["dec/gru1/Wc"])
        ru = torch.sigmoid(_tf32(Z) @ Wg[:256] + _tf32(hp) @ Wg[256:] + p["dec/gru1/bg"])
        cand = torch.tanh(_tf32(Z) @ Wc[:256] + _tf32(ru[..., :256] * hp) @ Wc[256:] + p["dec/gru1/bc"])
        H = S["dec/H"].clone()
        H[0] = ru[..., 256:] * hp + (1 - ru[..., 256:]) * cand
        over["H"] = H
    elif stage == "y":
        over["y"] = (_tf32(Z + S["dec/H"][2]) @ _tf32(p["dec/out_proj/W"]) + p["dec/out_proj/b"]).transpose(0, 1)
    else:
        q = _tf32(S["dec/y"]) @ _tf32(p["dec/attn/W_q"])                            # [B,T,256]
        e = (p["dec/attn/v"] * torch.tanh(d["keys"].double()[:, None] + q[:, :, None])).sum(-1)
        mask = torch.arange(e.shape[-1])[None, None] < d["tl"][:, None, None].to(torch.int64)
        over["align"] = torch.softmax(torch.where(mask, e, torch.full_like(e, -math.inf)), -1)
    f = _check(d, **over).first
    assert f is not None and (f.t, f.stage) == (0, stage), f
