"""-m gpu: the guided attention loss (Config.guided_attention, csrc/train.cu taco_guided_attention, the dscore_add input
of csrc/decoder_bwd.cu).

  * the kernel against the float64 mirror at the benchmark's training shape and at ragged N_b / T_b, B = 1, 7 and 32;
    the loss within 1e-6 of the float64 sum, bit-identical run to run;
  * taco_decoder_bwd with dscore_add on the inputs the model's backward captured, against the float64 mirror, and
    bit-identical across CTA budgets of 128, 64 and 32;
  * the full-size training backward with the loss on, against the float64 mirror of the same host code on the GPU's
    saved activations (as test_gpu_train_fullsize.py does), with and without the speaker-conditioned decoder;
  * the feature off and lambda = 0 launch the same kernels and give the same loss bits; a NULL or zero dscore_add gives
    the decoder backward's outputs bit for bit;
  * on a seeded toy batch with a large lambda, the loss falls below half its first value within a few dozen Adam steps;
  * the training driver on a synthetic WAV corpus with --guided-attention and --summaries.
"""
import math
import os

import numpy as np
import pytest
import torch

from oracle import tacotron_oracle as O
from tests import guided_attention_oracle as GA, mirror_kernels_guided as MKG, speaker_decoder_oracle as SD
from tests.test_gpu_train_fullsize import B as B_C2, R as R_C2, T as T_C2, TX as TX_C2, _cuda, _f64, _log_rel_l2
from tests.util import assert_close

pytestmark = pytest.mark.gpu
G_PAPER = 0.2


def _steps(B, T, seed):
    """ragged voiced decoder steps: multiples of 4 in [4, T], as audio.speech_frames // r gives them, and one utterance
    voiced to its last step"""
    g = torch.Generator().manual_seed(seed)
    s = torch.randint(1, T // 4 + 1, (B,), generator=g, dtype=torch.int32) * 4
    s[0] = T
    return s


def _alignments(B, T, Tx, tl, seed):
    g = torch.Generator().manual_seed(seed)
    mask = torch.arange(Tx)[None, None, :] < torch.clamp(tl, max=Tx).to(torch.int64)[:, None, None]
    return torch.softmax((3 * torch.randn(B, T, Tx, generator=g)).masked_fill(~mask, -float("inf")), -1).contiguous()


def _run_kernel(al, tl, steps, g, lam):
    from tacotron_b200 import kernels as K
    ds = torch.full_like(al, float("nan"))
    loss = torch.full((1,), float("nan"), device="cuda")
    K.guided_attention(ds, loss, al, tl, steps, g, lam)
    torch.cuda.synchronize()
    return ds, loss


# ---------------------------------------------------------------------------------------------------------------------
# the kernel
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,T,Tx", [(B_C2, T_C2, TX_C2), (1, 37, 5), (7, 90, 67), (32, 64, 256)])
def test_kernel_matches_float64_mirror(B, T, Tx):
    g = torch.Generator().manual_seed(B + T)
    tl = torch.randint(max(1, Tx // 2), Tx + 1, (B,), generator=g, dtype=torch.int32)
    tl[-1] = Tx + 9                                                  # beyond the width: clipped to Tx
    steps = _steps(B, T, B)
    al = _alignments(B, T, Tx, tl, 1)
    lam = 2.5
    ds, loss = _run_kernel(al.cuda(), tl.cuda(), steps.cuda(), G_PAPER, lam)
    ds64, loss64 = torch.empty(B, T, Tx, dtype=torch.float64), torch.empty(1, dtype=torch.float64)
    MKG.guided_attention(ds64, loss64, al.double(), tl, steps, G_PAPER, lam)
    assert not torch.isnan(ds).any()
    assert_close(ds.cpu(), ds64, 1e-5, f"guided_attention dscore B={B} T={T} Tx={Tx}")
    W, mask = GA.band(tl, steps, T, Tx, G_PAPER)
    fsum = lam * math.fsum((al.double() * W).reshape(-1).tolist())
    assert abs(float(loss) - fsum) <= 1e-6 * abs(fsum), (float(loss), fsum)
    assert (ds.cpu()[~mask] == 0).all()
    ds2, loss2 = _run_kernel(al.cuda(), tl.cuda(), steps.cuda(), G_PAPER, lam)
    assert torch.equal(ds, ds2) and torch.equal(loss, loss2)


def test_kernel_argument_errors():
    from tacotron_b200 import _lib as L, kernels as K
    al = torch.full((2, 4, 8), 0.125, device="cuda")
    tl = torch.tensor([8, 5], dtype=torch.int32, device="cuda")
    st = torch.tensor([4, 2], dtype=torch.int32, device="cuda")
    ds, loss = torch.empty_like(al), torch.empty(1, device="cuda")
    with pytest.raises(L.TacoError, match="g="):
        K.guided_attention(ds, loss, al, tl, st, 0.0, 1.0)
    with pytest.raises(L.TacoError, match="lam="):
        K.guided_attention(ds, loss, al, tl, st, 0.2, -1.0)
    with pytest.raises(L.TacoError, match="int32"):
        K.guided_attention(ds, loss, al, tl, st.long(), 0.2, 1.0)
    with pytest.raises(L.TacoError, match="partial"):
        K.guided_attention(ds, loss, al, tl, st, 0.2, 1.0, partial=torch.empty(3, device="cuda"))


# ---------------------------------------------------------------------------------------------------------------------
# the model at the benchmark's training shape
# ---------------------------------------------------------------------------------------------------------------------
def _case(spk):
    if spk:
        cfg = SD.SpkDecOracleConfig(r=R_C2, vocab_size=64, num_speakers=109)
        p = SD.init_params(cfg, seed=1, trained_like=True)
    else:
        cfg = O.OracleConfig(r=R_C2, vocab_size=64)
        p = O.init_params(cfg, seed=1, trained_like=True)
    inp = O.synthetic_inputs(cfg, B_C2, TX_C2, T_C2, seed=0, ragged=True)
    if spk:
        inp["speaker"] = torch.randint(0, 109, (B_C2,), generator=torch.Generator().manual_seed(7), dtype=torch.int32)
    inp["speech_steps"] = _steps(B_C2, T_C2, 11)
    enc_m, dec_m = O.dropout_masks(cfg, B_C2, TX_C2, T_C2, seed=2)
    return cfg, p, inp, enc_m, dec_m, O.sched_mask(cfg, B_C2, T_C2, seed=3)


def _model(cfg, precision="fp32x3", **kw):
    from tacotron_b200 import Config, Tacotron
    nspk = getattr(cfg, "num_speakers", 1)
    return Tacotron(Config(r=cfg.r, vocab_size=cfg.vocab_size, precision=precision, num_speakers=nspk,
                           speaker_decoder=nspk > 1, scheduled_sample=cfg.scheduled_sample, **kw), None, train=True)


def _forward_with_ga(case, lam, precision="fp32x3"):
    """train-mode forward with saved activations and, for lam > 0, the guided attention gradient in S"""
    from tacotron_b200 import kernels as K
    from tacotron_b200.models import ops
    cfg, p, inp, enc_m, dec_m, sm = case
    m = _model(cfg, precision)
    m.load_params(p)
    gi = {k: v.cuda().contiguous() for k, v in inp.items()}
    S = {}
    with ops.saving(S):
        m.seq2seq_output, m.output = m.inference(gi, True, enc_drop_masks=_cuda(enc_m), dec_drop_masks=_cuda(dec_m),
                                                 sample_mask=sm.cuda())
    S.update(text=gi["text"], text_length=gi["text_length"], mel=gi["mel"], stft=gi["stft"])
    if "speaker" in gi:
        S["speaker"] = gi["speaker"]
    S["post/out"] = m.output
    if lam > 0:
        al = S["dec/align"]
        ds, ga = torch.empty_like(al), torch.empty(1, device="cuda")
        K.guided_attention(ds, ga, al, gi["text_length"], gi["speech_steps"], G_PAPER, lam)
        S["dec/dscore_ga"] = ds
    return m, S


LAM_C2 = 200.0      # large enough that the term moves the whole gradient (asserted below), so the mirror checks it


@pytest.mark.parametrize("spk", [False, True])
def test_fullsize_backward_matches_fp64_mirror(spk):
    from tacotron_b200.models import grad
    case = _case(spk)
    m, S = _forward_with_ga(case, LAM_C2)
    G = m.backward(S)
    torch.cuda.synchronize()
    S64 = {k: _f64(v) for k, v in S.items()}
    P64 = {n: _f64(m.store[n]) for n in m.store.names()}
    G64 = {n: torch.zeros_like(v) for n, v in P64.items()}
    grad.model_bwd(MKG, P64, G64, S64, case[0])
    names = m.store.trainable()
    bad = []
    for n in names:
        try:
            assert_close(G[n], G64[n], 2e-4, f"guided attention fullsize bwd spk={spk} {n}")
        except AssertionError as ex:
            bad.append(str(ex))
    assert not bad, "\n".join(bad)
    a = torch.cat([G[n].detach().double().cpu().reshape(-1) for n in names])
    b = torch.cat([G64[n].reshape(-1) for n in names])
    assert _log_rel_l2(f"guided attention fullsize bwd spk={spk} whole-gradient rel L2", a, b, 3e-5) <= 3e-5
    # the term moves the gradient: the float64 mirror without it differs
    S64.pop("dec/dscore_ga")
    G0 = {n: torch.zeros_like(v) for n, v in P64.items()}
    grad.model_bwd(MKG, P64, G0, S64, case[0])
    b0 = torch.cat([G0[n].reshape(-1) for n in names])
    assert ((b - b0).norm() / b.norm()).item() > 1e-3


DEC_OUTS = ("DATT", "DY", "DPQ", "DSCORE", "DCTX", "DZ", "DPN2", "DPN1", "DX")


def test_decoder_bwd_with_dscore_add_on_captured_inputs():
    from tacotron_b200 import kernels as K
    m, S = _forward_with_ga(_case(False), LAM_C2)
    S["_capture"] = {}
    m.backward(S)
    torch.cuda.synchronize()
    cap = {k: v for k, v in S["_capture"]["decoder_bwd"].items() if not k.startswith("_")}
    assert cap["dscore_add"] is S["dec/dscore_ga"]
    runs = {}
    prev = K.set_gemm_impl(1)                                       # the GEMM the fp32x3 backward selected
    try:
        for ctas in (128, 64, 32):
            a = {k: ([t.clone() for t in v] if isinstance(v, list) else v.clone() if torch.is_tensor(v) else v)
                 for k, v in cap.items()}
            for k in DEC_OUTS:
                a[k].fill_(float("nan"))
            for i in range(3):
                a["DG"][i].fill_(float("nan")); a["DC"][i].fill_(float("nan"))
            a["max_ctas"] = ctas
            K.decoder_bwd(a)
            torch.cuda.synchronize()
            runs[ctas] = a
    finally:
        K.set_gemm_impl(prev)
    a64 = {k: _f64(v) for k, v in cap.items()}
    MKG.decoder_bwd(a64)
    for k in DEC_OUTS:
        assert not torch.isnan(runs[128][k]).any(), f"{k}: cells left unwritten"
        assert_close(runs[128][k], a64[k], 2e-4, f"guided attention decoder_bwd {k}")
    for i in range(3):
        assert_close(runs[128]["DG"][i], a64["DG"][i], 2e-4, f"guided attention decoder_bwd DG{i}")
        assert_close(runs[128]["DC"][i], a64["DC"][i], 2e-4, f"guided attention decoder_bwd DC{i}")
    for ctas in (64, 32):
        for k in DEC_OUTS:
            assert torch.equal(runs[ctas][k], runs[128][k]), (ctas, k)
        for i in range(3):
            assert torch.equal(runs[ctas]["DG"][i], runs[128]["DG"][i]) and torch.equal(runs[ctas]["DC"][i], runs[128]["DC"][i])


def _rerun_decoder_bwd(cap, **kw):
    from tacotron_b200 import kernels as K
    a = {k: ([t.clone() for t in v] if isinstance(v, list) else v.clone() if torch.is_tensor(v) else v)
         for k, v in cap.items() if not k.startswith("_")}
    a.update(kw)
    for k in DEC_OUTS:
        a[k].fill_(float("nan"))
    for i in range(3):
        a["DG"][i].fill_(float("nan")); a["DC"][i].fill_(float("nan"))
    prev = K.set_gemm_impl(1)                                       # the GEMM the fp32x3 backward selected
    try:
        K.decoder_bwd(a)
        torch.cuda.synchronize()
    finally:
        K.set_gemm_impl(prev)
    return a


def test_null_and_zero_dscore_add_are_bit_identical_to_the_path_without_it():
    """the decoder backward kernel is deterministic (each output column has one owner CTA), so its outputs compare bit for
    bit; the model's weight gradients do not (split-K and dv / embedding gradients add with float atomics)"""
    m, S = _forward_with_ga(_case(False), 0.0)
    S["_capture"] = {}
    m.backward(S)
    torch.cuda.synchronize()
    cap = S["_capture"]["decoder_bwd"]
    assert cap.get("dscore_add") is None
    runs = [_rerun_decoder_bwd(cap), _rerun_decoder_bwd(cap, dscore_add=torch.zeros_like(cap["align"]))]
    for a in runs:
        for k in DEC_OUTS:
            assert torch.equal(a[k], cap[k]), k
        for i in range(3):
            assert torch.equal(a["DG"][i], cap["DG"][i]) and torch.equal(a["DC"][i], cap["DC"][i]), i


# ---------------------------------------------------------------------------------------------------------------------
# train_step: off, lambda = 0, the errors, and the loss falling on a toy batch
# ---------------------------------------------------------------------------------------------------------------------
def _toy(B=4, Tx=12, T=24, r=2, seed=0):
    cfg = O.OracleConfig(r=r, vocab_size=20)
    inp = O.synthetic_inputs(cfg, B, Tx, T, seed=seed, ragged=True)
    gi = {k: v.cuda().contiguous() for k, v in inp.items()}
    gi["speech_steps"] = torch.tensor([T, 16, 20, 8][:B], dtype=torch.int32, device="cuda")
    return cfg, gi


def _steps_of(cfg, gi, n, lr=1e-3, **kw):
    from tacotron_b200 import _lib as L
    m = _model(cfg, "fp32x3", **kw)
    torch.manual_seed(5)
    n0 = L.lib().taco_launch_count()
    losses, ga = [], []
    for _ in range(n):
        losses.append(float(m.train_step(gi, lr)))
        ga.append(None if m.guided_attention_loss is None else float(m.guided_attention_loss))
    torch.cuda.synchronize()
    return m, losses, ga, L.lib().taco_launch_count() - n0


def test_off_and_zero_lambda_are_identical_and_launch_nothing_more():
    cfg, gi = _toy()
    m0, l0, ga0, n0 = _steps_of(cfg, {k: v for k, v in gi.items() if k != "speech_steps"}, 1)
    m1, l1, ga1, n1 = _steps_of(cfg, gi, 1, guided_attention=0.0)
    assert l0 == l1 and n0 == n1 and ga0 == ga1 == [None]          # same launches, the same loss bits
    # the update: the same arithmetic; the float atomics of the weight gradients may round differently run to run
    assert_close(m1.store.flat, m0.store.flat, 1e-6, "guided attention lambda = 0 vs off: parameters after one step")
    m2, l2, ga2, n2 = _steps_of(cfg, gi, 1, guided_attention=10.0)
    assert n2 == n1 + 2                                            # the loss kernel's two launches
    assert ga2[0] > 0 and (m2.store.flat - m1.store.flat).abs().max().item() > 1e-6
    assert abs(l2[0] - (l1[0] + ga2[0])) <= 1e-6 * l2[0]            # same first forward, plus the term


def test_train_step_errors():
    cfg, gi = _toy()
    m = _model(cfg, "fp32x3", guided_attention=1.0)
    with pytest.raises(ValueError, match="needs inputs\\['speech_steps'\\]"):
        m.train_step({k: v for k, v in gi.items() if k != "speech_steps"})
    for bad in ([0, 16, 20, 8], [24, 25, 20, 8]):
        with pytest.raises(ValueError, match="must lie in \\[1, 24\\]"):
            m.train_step(dict(gi, speech_steps=torch.tensor(bad, dtype=torch.int32, device="cuda")))
    assert m.global_step == 0


# Measured on an H100 80GB HBM3 (700 W power limit), 60 steps of this batch at lr 1e-3: with lambda = 1e4 (3.9e5 at the
# first step) the loss first fell below half its first value at step 18; with lambda = 1e3 at step 21.  The bar leaves room for the run-to-run rounding of the weight gradients' float atomics.
DESCENT_STEPS, DESCENT_LAMBDA, DESCENT_LR = 30, 1e4, 1e-3


def test_loss_falls_on_a_toy_batch():
    cfg, gi = _toy()
    _, _, ga, _ = _steps_of(cfg, gi, DESCENT_STEPS, lr=DESCENT_LR, guided_attention=DESCENT_LAMBDA)
    print("guided attention loss per step:", [f"{g:.1f}" for g in ga])
    assert min(ga) < 0.5 * ga[0], ga


# ---------------------------------------------------------------------------------------------------------------------
# the driver
# ---------------------------------------------------------------------------------------------------------------------
def test_driver_on_a_wav_corpus(tmp_path, monkeypatch):
    from tacotron_b200 import summary as SUM, train as trainer
    from tacotron_b200.models.tacotron import Tacotron
    from tests.test_gpu_z_features import _corpus_arctic, _run_preprocess
    from tests.test_summary import _events
    root = str(tmp_path / "data")
    _corpus_arctic(root, np.random.RandomState(3))
    _run_preprocess(["arctic", "--data-dir", root])
    monkeypatch.chdir(tmp_path)
    seen = []

    class Spy(Tacotron):
        def train_step(self, inputs, lr=None, **kw):
            seen.append((inputs["speech_steps"].cpu(), inputs["mel"].shape[1]))
            return super().train_step(inputs, lr, **kw)

    cfg, args = trainer.config_from_args(["-t", "arctic", "--guided-attention", "5", "--summaries"])
    cfg.save_path = "arctic/tacotron"
    logs = []
    m = trainer.train(Spy, cfg, num_steps=3, log=logs.append, save_every=100, summary_dir="log/arctic/train")
    assert m.global_step == 3 and np.isfinite(float(m.loss)) and float(m.guided_attention_loss) > 0
    for steps, T in seen:
        assert steps.dtype == torch.int32 and (steps % 4 == 0).all() and (steps >= 4).all() and (steps <= T).all()
        assert (steps < T).any(), (steps, T)                       # the padded utterances end before the padding
    ev = _events("log/arctic/train")
    tags = [t for _, _, _, vals in ev[1:] for t, _ in vals]
    assert tags.count(SUM.GUIDED_ATTENTION_TAG) == 3
    last = {t: v for step, _, _, vals in ev[1:] if step == 3 for t, v in vals}
    assert last[SUM.GUIDED_ATTENTION_TAG].simple_value == float(m.guided_attention_loss)
    assert last["loss"].simple_value == float(m.loss)
