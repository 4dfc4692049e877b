"""Guided attention loss (Config.guided_attention) without a GPU: the float64 oracle on hand-checked cases, the
hand-written backward over the kernel mirrors against torch.autograd of the oracle loss plus the guided attention term,
lambda = 0 against the path without the feature, the kernel sources under the host emulation, the argument checks and
the training driver's command line."""
import copy
import ctypes as C
import math
import types

import pytest
import torch

from oracle import tacotron_oracle as O
from tacotron_b200 import _lib as L
from tacotron_b200.models import grad
from tacotron_b200.models.tacotron import Config, Tacotron
from tests import grad_util, guided_attention_oracle as GA, mirror_kernels_guided as MKG, speaker_decoder_oracle as SD
from tests.emulator import emu  # noqa: F401  (the emulated library, built once per process)

G_PAPER = 0.2


# ---- the oracle on hand-checked cases ----
def test_weights_vanish_on_the_diagonal_and_approach_one_far_from_it():
    N, Tb = 10, 20
    W, mask = GA.band([N], [Tb], Tb, N, G_PAPER)
    for t in range(0, Tb, 2):                       # j/N = t/Tb exactly at j = t/2
        assert W[0, t, t // 2] == 0.0
    assert W[0, 0, N - 1] > 0.99 and W[0, Tb - 1, 0] > 0.99
    # one point by hand: j = 3, t = 10 -> d = 0.3 - 0.5
    assert math.isclose(float(W[0, 10, 3]), 1 - math.exp(-0.04 / 0.08), rel_tol=1e-15)
    assert mask.all()


def test_mask_stops_at_the_voiced_steps_and_the_text_length():
    W, mask = GA.band([5, 3], [4, 7], 8, 6, G_PAPER)
    assert mask[0, :4, :5].all() and not mask[0, 4:].any() and not mask[0, :, 5:].any()
    assert mask[1, :7, :3].all() and not mask[1, 7:].any() and not mask[1, :, 3:].any()
    assert (W[~mask] == 0).all()
    al = torch.rand(2, 8, 6, dtype=torch.float64)
    d = GA.dscore(al, [5, 3], [4, 7], G_PAPER, 2.0)
    assert (d[~mask] == 0).all() and (d[mask] != 0).any()


def test_text_length_beyond_the_width_is_clipped():
    W1, m1 = GA.band([9], [6], 6, 5, G_PAPER)
    W2, m2 = GA.band([5], [6], 6, 5, G_PAPER)
    assert torch.equal(W1, W2) and torch.equal(m1, m2)


def test_dscore_is_the_softmax_backward_of_the_loss():
    g = torch.Generator().manual_seed(0)
    score = torch.randn(3, 7, 9, generator=g, dtype=torch.float64, requires_grad=True)
    tl, steps = [9, 4, 12], [7, 3, 5]
    text_mask = torch.arange(9)[None, None, :] < torch.tensor([9, 4, 9])[:, None, None]    # the decoder's memory mask
    al = torch.softmax(score.masked_fill(~text_mask, -float("inf")), -1)
    (ds,) = torch.autograd.grad(GA.loss(al, tl, steps, 0.3, 1.7), score)
    assert torch.allclose(GA.dscore(al.detach(), tl, steps, 0.3, 1.7), ds, rtol=0, atol=1e-14)


# ---- the backward over the mirrors against autograd ----
def _setup(r, sched, spk, B=2, Tx=8, T=5):
    if spk:
        cfg = SD.SpkDecOracleConfig(r=r, vocab_size=20, num_speakers=3)
        p = SD.init_params(cfg, seed=1, trained_like=True, dtype=torch.float64)
    else:
        cfg = O.OracleConfig(r=r, vocab_size=20)
        p = O.init_params(cfg, seed=1, trained_like=True, dtype=torch.float64)
    inp = O.synthetic_inputs(cfg, B, Tx, T, seed=0, ragged=True)
    inp = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in inp.items()}
    if spk:
        inp["speaker"] = torch.tensor([0, 2, 1, 2][:B], dtype=torch.int32)
    inp["speech_steps"] = torch.tensor([T, T - 2, T - 1, 1][:B], dtype=torch.int32)
    enc_m, dec_m = O.dropout_masks(cfg, B, Tx, T, seed=2)
    sm = O.sched_mask(cfg, B, T, seed=3) if sched else None
    return cfg, p, inp, enc_m, dec_m, sm


def _autograd(cfg, p, inp, enc_m, dec_m, sm, spk, lam, g):
    q = {k: v.detach().clone().requires_grad_(not k.endswith(O.NON_TRAINABLE_SUFFIXES)) for k, v in p.items()}
    y, out, align = (SD if spk else O).inference(q, inp, cfg, train=True, enc_drop_masks=enc_m, dec_drop_masks=dec_m,
                                                 sample_mask=sm)
    total, _, _ = O.loss(y, out, inp["mel"], inp["stft"])
    total = total + GA.loss(align, inp["text_length"], inp["speech_steps"], g, lam)
    names = [k for k, v in q.items() if v.requires_grad]
    return dict(zip(names, torch.autograd.grad(total, [q[k] for k in names])))


def _mirror_backward(cfg, p, inp, enc_m, dec_m, sm, spk, lam, g):
    """(G, S): grad.model_bwd over the mirrors, with the guided attention gradient of the mirror kernel when lam is not
    None (lam = None: the path without the feature)"""
    S, _, _ = (SD if spk else grad_util).saving_forward(p, inp, cfg, enc_m, dec_m, sm)
    if lam is not None:
        al = S["dec/align"]
        ds, ga = torch.empty_like(al), torch.empty(1, dtype=al.dtype)
        MKG.guided_attention(ds, ga, al, inp["text_length"], inp["speech_steps"], g, lam)
        S["dec/dscore_ga"] = ds
        S["_ga"] = ga
    G = {k: torch.zeros_like(v) for k, v in p.items()}
    grad.model_bwd(MKG, p, G, S, cfg)
    return G, S


@pytest.mark.parametrize("r,sched,spk", [(2, False, False), (2, True, False), (5, False, False), (5, True, False),
                                         (2, True, True), (5, False, True)])
def test_backward_matches_autograd(r, sched, spk):
    case = _setup(r, sched, spk)
    lam, g = 40.0, 0.25
    g_ref = _autograd(*case, spk, lam, g)
    G, S = _mirror_backward(*case, spk, lam, g)
    G0, _ = _mirror_backward(*case, spk, None, g)
    moved = 0
    for k, ref in g_ref.items():
        err = (G[k] - ref).abs().max().item()
        assert err <= 1e-8 * (1.0 + ref.abs().max().item()), f"{k}: max err {err:.3e}"
        moved += bool((G[k] - G0[k]).abs().max().item() > 1e-6 * (1.0 + ref.abs().max().item()))
    assert moved >= 10, moved                                       # the term reaches the decoder and the encoder
    # the loss the mirror kernel reports is the oracle's
    ga = GA.loss(S["dec/align"], case[2]["text_length"], case[2]["speech_steps"], g, lam)
    assert math.isclose(float(S["_ga"]), float(ga), rel_tol=1e-12)


@pytest.mark.parametrize("spk", [False, True])
def test_zero_lambda_gives_the_gradients_without_the_feature(spk):
    case = _setup(5, True, spk)
    G0, _ = _mirror_backward(*case, spk, None, G_PAPER)
    G1, S = _mirror_backward(*case, spk, 0.0, G_PAPER)
    assert float(S["_ga"]) == 0.0 and not S["dec/dscore_ga"].any()
    for k in G0:
        assert torch.equal(G0[k], G1[k]), k


# ---- the kernel sources under the host emulation (tests/cuda_emu/emu.h) ----
def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _emu_ga(emu, al, tl, steps, g, lam):
    B, T, Tx = al.shape
    ds = torch.full_like(al, float("nan"))
    loss = torch.full((1,), float("nan"))
    part = torch.empty(emu.taco_guided_attention_partial_count(B, T))
    rc = emu.taco_guided_attention(_p(ds), _p(loss), _p(al), _p(tl), _p(steps), B, T, Tx, g, lam, _p(part), None)
    assert rc == 0, emu.taco_last_error().decode()
    return ds, loss


def test_guided_attention_kernel_under_emulation(emu):
    gen = torch.Generator().manual_seed(4)
    B, T, Tx = 3, 9, 70                          # Tx > 64: three positions per lane, the last lane group ragged
    tl = torch.tensor([70, 33, 200], dtype=torch.int32)     # the last one beyond Tx (clipped)
    steps = torch.tensor([9, 4, 1], dtype=torch.int32)
    mask = torch.arange(Tx)[None, None, :] < torch.tensor([70, 33, 70])[:, None, None]
    al = torch.softmax(torch.randn(B, T, Tx, generator=gen).masked_fill(~mask, -float("inf")), -1).contiguous()
    ds, loss = _emu_ga(emu, al, tl, steps, 0.2, 3.0)
    ds64, loss64 = torch.empty(B, T, Tx, dtype=torch.float64), torch.empty(1, dtype=torch.float64)
    MKG.guided_attention(ds64, loss64, al.double(), tl, steps, 0.2, 3.0)
    assert not torch.isnan(ds).any()
    assert (ds.double() - ds64).abs().max().item() <= 1e-6 * ds64.abs().max().item()
    assert math.isclose(float(loss), float(loss64), rel_tol=1e-6)
    _, mk = GA.band(tl, steps, T, Tx, 0.2)
    assert (ds[~mk] == 0).all()
    # run to run: the same bits
    ds2, loss2 = _emu_ga(emu, al, tl, steps, 0.2, 3.0)
    assert torch.equal(ds, ds2) and torch.equal(loss, loss2)


def test_guided_attention_kernel_rejects_bad_arguments(emu):
    B, T, Tx = 2, 4, 8
    al = torch.full((B, T, Tx), 1.0 / Tx)
    tl = torch.tensor([8, 5], dtype=torch.int32)
    steps = torch.tensor([4, 2], dtype=torch.int32)
    ds, loss, part = torch.empty_like(al), torch.empty(1), torch.empty(B * T)
    args = lambda **kw: dict(dict(ds=_p(ds), loss=_p(loss), al=_p(al), tl=_p(tl), steps=_p(steps), B=B, T=T, Tx=Tx, g=0.2,
                                  lam=1.0, part=_p(part)), **kw)
    call = lambda a: emu.taco_guided_attention(a["ds"], a["loss"], a["al"], a["tl"], a["steps"], a["B"], a["T"], a["Tx"],
                                               a["g"], a["lam"], a["part"], None)
    assert call(args()) == 0
    for bad, msg in ((dict(g=0.0), b"g="), (dict(g=-1.0), b"g="), (dict(g=float("nan")), b"g="),
                     (dict(lam=-0.5), b"lam="), (dict(lam=float("inf")), b"lam="), (dict(Tx=257), b"Tx"),
                     (dict(B=0), b"sizes"), (dict(steps=None), b"NULL"), (dict(part=None), b"NULL")):
        assert call(args(**bad)) != 0, bad
        assert msg in emu.taco_last_error(), (bad, emu.taco_last_error())
    assert emu.taco_guided_attention_partial_count(32, 200) == 6400


@pytest.mark.parametrize("r,sched,spk", [(2, True, False), (5, False, True)])
def test_decoder_bwd_kernel_with_dscore_add_under_emulation(emu, r, sched, spk):
    B, Tx, T = 2, 8, 4
    cfg, p, inp, enc_m, dec_m, sm = _setup(r, sched, spk, B=B, Tx=Tx, T=T)
    p = {k: v.float() for k, v in p.items()}
    inp = {k: (v.float() if v.dtype.is_floating_point else v) for k, v in inp.items()}
    S, _, _ = (SD if spk else grad_util).saving_forward(p, inp, cfg, enc_m, dec_m, sm)
    al = S["dec/align"]
    ds_ga, ga = torch.empty_like(al), torch.empty(1)
    MKG.guided_attention(ds_ga, ga, al, inp["text_length"], inp["speech_steps"], 0.2, 30.0)
    S["dec/dscore_ga"] = ds_ga
    S["_capture"] = {}
    G = {k: torch.zeros_like(v) for k, v in p.items()}
    grad.decoder_bwd(MKG, p, G, S, cfg, torch.randn(B, T, 80 * r, generator=torch.Generator().manual_seed(5)))
    a = S["_capture"]["decoder_bwd"]                            # inputs + the mirror's outputs
    outs = ("DATT", "DY", "DPQ", "DSCORE", "DCTX", "DZ", "DPN2", "DPN1", "DX") + (("DH0",) if spk else ())
    e = {k: copy.deepcopy(v) for k, v in a.items() if not k.startswith("_")}
    for k in outs:
        e[k].fill_(float("nan"))
    for i in range(3):
        e["DG"][i].fill_(float("nan")); e["DC"][i].fill_(float("nan"))
    d = L.DecoderBwdArgs()
    d.B, d.T, d.Tx, d.r, d.keep_scale = B, T, Tx, r, float(a["keep_scale"])
    for k in ("W_a", "W_q", "W_out", "W_in", "W1", "W2", "v", "dy_ext", "align", "values", "keys", "PQ", "PN1", "PN2", "sel",
              "dscore_add", *outs):
        e[k] = e[k].contiguous()
        setattr(d, k, e[k].data_ptr())
    for k in ("Wg", "Wc", "RU", "C", "H", "DG", "DC") + (("H0",) if spk else ()):
        for i in range(3):
            e[k][i] = e[k][i].contiguous()
            getattr(d, k)[i] = e[k][i].data_ptr()
    ws = torch.empty(emu.taco_decoder_bwd_workspace_bytes() // 4)
    d.workspace = ws.data_ptr()
    assert emu.taco_decoder_bwd(C.byref(d), None) == 0, emu.taco_last_error().decode()
    for k in outs:
        got, ref = torch.nan_to_num(e[k], nan=1e30), a[k]
        assert (got - ref).abs().max().item() <= 2e-5 * (ref.abs().max().item() + 1e-6), k
    for i in range(3):
        for k in ("DG", "DC"):
            got, ref = torch.nan_to_num(e[k][i], nan=1e30), a[k][i]
            assert (got - ref).abs().max().item() <= 2e-5 * (ref.abs().max().item() + 1e-6), (k, i)
    # without dscore_add the kernel is today's: its attention gradients differ
    e2 = {k: v.clone() for k, v in e.items() if torch.is_tensor(v)}
    d.dscore_add = None
    d.DSCORE = e2["DSCORE"].data_ptr()
    assert emu.taco_decoder_bwd(C.byref(d), None) == 0, emu.taco_last_error().decode()
    assert not torch.allclose(e2["DSCORE"], e["DSCORE"])


# ---- argument checks of the model and the driver's command line ----
def _lam(**kw):
    m = types.SimpleNamespace(config=Config(**kw))
    inp = {"mel": torch.zeros(2, 6, 160)}
    return lambda extra=None: Tacotron._guided_attention_lambda(m, dict(inp, **(extra or {})))


def test_model_argument_checks():
    assert _lam()() == 0.0                                      # off: speech_steps is not needed
    assert _lam(guided_attention=0.0, guided_attention_g=-1.0)() == 0.0
    with pytest.raises(ValueError, match="guided_attention = -1"):
        _lam(guided_attention=-1.0)()
    with pytest.raises(ValueError, match="finite"):
        _lam(guided_attention=float("nan"))()
    with pytest.raises(ValueError, match="guided_attention_g"):
        _lam(guided_attention=1.0, guided_attention_g=0.0)()
    with pytest.raises(ValueError, match="needs inputs\\['speech_steps'\\]"):
        _lam(guided_attention=1.0)()
    with pytest.raises(ValueError, match="int32 CUDA tensor of shape \\[2\\]"):
        _lam(guided_attention=1.0)({"speech_steps": torch.tensor([6, 4], dtype=torch.int32)})
    assert Config.guided_attention == 0.0 and Config.guided_attention_g == 0.2


def test_driver_command_line():
    from tacotron_b200 import train as TR
    cfg, args = TR.config_from_args(["-t", "arctic"])
    assert cfg.guided_attention == 0.0 and cfg.guided_attention_g == 0.2
    cfg, args = TR.config_from_args(["-t", "arctic", "--guided-attention", "2.5", "--guided-attention-g", "0.3", "--summaries"])
    assert (cfg.guided_attention, cfg.guided_attention_g, args.summaries) == (2.5, 0.3, True)
    assert cfg.data_path == "data/arctic/"
    for bad in (["--guided-attention", "-1"], ["--guided-attention", "nan"], ["--guided-attention-g", "0"],
                ["--guided-attention-g", "-0.2"]):
        with pytest.raises(SystemExit):
            TR.config_from_args(bad)
