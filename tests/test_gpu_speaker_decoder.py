"""-m gpu: the speaker-conditioned decoder (Config.speaker_decoder) on the H100: taco_decoder_fwd with initial states
against the float64 oracle, NULL / zero-state / CTA-budget bit-identity, taco_decoder_bwd with H0 / DH0 against the
float64 mirror, whole-model inference and CUDA-graph replay, training gradients, and the two drivers."""
import os

import numpy as np
import pytest
import torch

from oracle import tacotron_oracle as O
from tacotron_b200 import _lib as L
from tacotron_b200 import kernels as K
from tacotron_b200.models import grad, ops
from tacotron_b200.params import ParamStore, model_shapes
from tests import mirror_kernels_spkdec as MK, speaker_decoder_oracle as SD
from tests.test_gpu_multispeaker import _bar, _cuda, _dataset
from tests.util import assert_close

pytestmark = pytest.mark.gpu
NSPK = 4
TOL = {"fp32": 2e-4, "fp32x3": 2e-4, "tf32": 5e-3}
MODES = {"infer": L.DEC_INFER, "teacher": L.DEC_TEACHER, "sched": L.DEC_SCHED}


def _config(r, **kw):
    from tacotron_b200 import Config
    return Config(r=r, vocab_size=20, num_speakers=NSPK, speaker_decoder=True, **kw)


def _dec_case(r, B, Tx, T, seed=0):
    cfg = SD.SpkDecOracleConfig(r=r, max_decode_iter=T, vocab_size=20, num_speakers=NSPK)
    p = SD.init_params(cfg, seed=1, trained_like=True)
    g = torch.Generator().manual_seed(seed)
    encoded = torch.randn(B, Tx, 256, generator=g) * 0.5
    inp = O.synthetic_inputs(cfg, B, Tx, T, seed=seed, ragged=True)
    _, dec_m = O.dropout_masks(cfg, B, Tx, T, seed=2)
    sm = O.sched_mask(cfg, B, T, seed=3)
    e = p["speaker/embed"][torch.randint(0, NSPK, (B,), generator=g)]
    h0, att0 = SD.initial_state(p, e)
    st = ParamStore(model_shapes(_config(r)), "cuda")
    st.load(p)
    ops.runtime(st, "fp32")
    return cfg, p, encoded, inp, dec_m, sm, h0, att0, st


def _run(st, r, T, mode, encoded, inp, dec_m, sm, h0, att0, max_ctas=None):
    y, a = ops.attention_decoder(encoded.cuda(), inp["text_length"].cuda(), r, T, mode=MODES[mode],
                                 mel=None if mode == "infer" else inp["mel"].cuda(),
                                 sample_mask=sm.cuda() if mode == "sched" else None,
                                 drop_masks=None if mode == "infer" else (dec_m[0].cuda(), dec_m[1].cuda()),
                                 scope=ops.Scope(st, "dec"), max_ctas=max_ctas,
                                 h0=None if h0 is None else h0.float().cuda().contiguous(),
                                 att0=None if att0 is None else att0.float().cuda().contiguous())
    torch.cuda.synchronize()
    return y.clone(), a.clone()


@pytest.mark.parametrize("mode", ["infer", "teacher", "sched"])
@pytest.mark.parametrize("r", [2, 5])
@pytest.mark.parametrize("B,Tx", [(1, 13), (7, 30), (32, 67)])
def test_decoder_fwd_with_initial_state_matches_oracle(mode, r, B, Tx):
    T = 6
    cfg, p, encoded, inp, dec_m, sm, h0, att0, st = _dec_case(r, B, Tx, T)
    y_ref, a_ref = SD.decoder(encoded, inp["text_length"], p, cfg, mode, T, h0, att0, mel=inp["mel"],
                              drop_masks=None if mode == "infer" else dec_m, sample_mask=sm if mode == "sched" else None)
    y, a = _run(st, r, T, mode, encoded, inp, dec_m, sm, h0, att0)
    assert_close(y, y_ref, 1e-4, f"decoder y {mode} r={r} B={B}")
    assert_close(a, a_ref, 1e-4, f"decoder align {mode} r={r} B={B}")
    y0, _ = _run(st, r, T, mode, encoded, inp, dec_m, sm, None, None)     # the state reaches the output
    assert (y0 - y).abs().max().item() > 1e-3


@pytest.mark.parametrize("mode", ["infer", "sched"])
def test_zero_state_is_bit_identical_to_null(mode):
    r, B, Tx, T = 5, 11, 40, 8
    cfg, p, encoded, inp, dec_m, sm, h0, att0, st = _dec_case(r, B, Tx, T, seed=1)
    y0, a0 = _run(st, r, T, mode, encoded, inp, dec_m, sm, None, None)
    yz, az = _run(st, r, T, mode, encoded, inp, dec_m, sm, torch.zeros_like(h0), torch.zeros_like(att0))
    assert torch.equal(y0, yz) and torch.equal(a0, az)


@pytest.mark.parametrize("max_ctas", [32, 64])
def test_cta_budget_is_bit_identical_with_states(max_ctas):
    r, B, Tx, T = 2, 32, 67, 7
    cfg, p, encoded, inp, dec_m, sm, h0, att0, st = _dec_case(r, B, Tx, T, seed=2)
    y, a = _run(st, r, T, "sched", encoded, inp, dec_m, sm, h0, att0)
    yb, ab = _run(st, r, T, "sched", encoded, inp, dec_m, sm, h0, att0, max_ctas=max_ctas)
    assert torch.equal(y, yb) and torch.equal(a, ab)


@pytest.mark.parametrize("r", [2, 5])
def test_decoder_bwd_with_h0_matches_mirror(r):
    B, Tx, T = 32, 10, 5
    cfg = SD.SpkDecOracleConfig(r=r, vocab_size=20, num_speakers=NSPK)
    p = SD.init_params(cfg, seed=1, trained_like=True, dtype=torch.float64)
    inp = O.synthetic_inputs(cfg, B, Tx, T, seed=0, ragged=True)
    inp = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in inp.items()}
    inp["speaker"] = torch.arange(B, dtype=torch.int32) % NSPK
    enc_m, dec_m = O.dropout_masks(cfg, B, Tx, T, seed=2)
    sm = O.sched_mask(cfg, B, T, seed=3)
    S, _, _ = SD.saving_forward(p, inp, cfg, enc_m, dec_m, sm)
    S["_capture"] = {}
    dY = torch.randn(B, T, 80 * r, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    grad.decoder_bwd(MK, p, {k: torch.zeros_like(v) for k, v in p.items()}, S, cfg, dY)
    ref = S["_capture"]["decoder_bwd"]
    dev = lambda t: t.float().cuda().contiguous() if t.dtype.is_floating_point else t.cuda().contiguous()
    a = {k: ([dev(x) for x in v] if isinstance(v, list) else dev(v) if torch.is_tensor(v) else v)
         for k, v in ref.items() if not k.startswith("_")}
    outs = ("DATT", "DY", "DPQ", "DSCORE", "DCTX", "DZ", "DPN2", "DPN1", "DX", "DH0")
    for k in outs:
        a[k].fill_(float("nan"))
    for i in range(3):
        a["DG"][i].fill_(float("nan")); a["DC"][i].fill_(float("nan"))
    K.decoder_bwd(a)
    torch.cuda.synchronize()
    for k in outs:
        assert_close(a[k], ref[k], 2e-4, f"{k} r={r}")
    for i in range(3):
        assert_close(a["DG"][i], ref["DG"][i], 2e-4, f"DG{i} r={r}")
        assert_close(a["DC"][i], ref["DC"][i], 2e-4, f"DC{i} r={r}")


def _model(r, T, p, precision, cuda_graph=False):
    from tacotron_b200 import Tacotron
    m = Tacotron(_config(r, max_decode_iter=T, precision=precision, cuda_graph=cuda_graph), None, train=False)
    m.load_params(p)
    return m


def _case(r=2, B=3, Tx=16, T=10, seed=0):
    cfg = SD.SpkDecOracleConfig(r=r, max_decode_iter=T, vocab_size=20, num_speakers=NSPK)
    p = SD.init_params(cfg, seed=1, trained_like=True)
    inp = O.synthetic_inputs(cfg, B, Tx, T, seed=seed, ragged=True, with_targets=False)
    inp["speaker"] = torch.tensor([3, 0, 2, 1, 3, 2, 0, 1][:B], dtype=torch.int32)
    return cfg, p, inp


@pytest.mark.parametrize("precision", ["fp32", "fp32x3", "tf32"])
@pytest.mark.parametrize("r", [2, 5])
def test_inference_matches_oracle(precision, r):
    cfg, p, inp = _case(r)
    y_ref, out_ref, a_ref = SD.inference(p, inp, cfg, train=False)
    m = _model(r, cfg.max_decode_iter, p, precision)
    y, out = m.inference(_cuda(inp), train=False)
    torch.cuda.synchronize()
    assert_close(y, y_ref, TOL[precision], "y")
    assert_close(m.alignments, a_ref, TOL[precision], "align")
    assert_close(out, out_ref, TOL[precision], "out")


def test_graph_replay_with_new_speakers_equals_eager():
    cfg, p, inp = _case(B=4)
    m = _model(2, 10, p, "fp32x3")
    mg = _model(2, 10, p, "fp32x3", cuda_graph=True)
    ci = _cuda(inp)
    y0 = mg.inference(ci, train=False)[0].clone()
    ni = dict(ci)
    ni["speaker"] = torch.tensor([1, 1, 0, 2], dtype=torch.int32, device="cuda")
    yg, outg = [t.clone() for t in mg.inference(ni, train=False)]
    ye, oute = [t.clone() for t in m.inference(ni, train=False)]
    torch.cuda.synchronize()
    assert torch.equal(yg, ye) and torch.equal(outg, oute)
    assert not torch.equal(yg, y0)


@pytest.mark.parametrize("precision", ["fp32", "fp32x3", "tf32"])
def test_training_gradients_match_autograd(precision):
    r, B, Tx, T = 5, 2, 8, 5
    cfg = SD.SpkDecOracleConfig(r=r, vocab_size=20, num_speakers=NSPK, scheduled_sample=0.0)
    p = SD.init_params(cfg, seed=1, trained_like=True)
    inp = O.synthetic_inputs(cfg, B, Tx, T, seed=0, ragged=True)
    inp["speaker"] = torch.tensor([3, 1], dtype=torch.int32)
    enc_m, dec_m = O.dropout_masks(cfg, B, Tx, T, seed=2)
    _, g_ref = SD.loss_and_grads(p, inp, cfg, enc_drop_masks=enc_m, dec_drop_masks=dec_m)
    from tacotron_b200 import Tacotron
    m = Tacotron(_config(r, precision=precision, scheduled_sample=0.0), None, train=True)
    m.load_params(p)
    gi = _cuda(inp)
    S = {}
    with ops.saving(S):
        m.seq2seq_output, m.output = m.inference(gi, True, enc_drop_masks=tuple(t.cuda() for t in enc_m),
                                                 dec_drop_masks=tuple(t.cuda() for t in dec_m))
    S.update(text=gi["text"], text_length=gi["text_length"], mel=gi["mel"], stft=gi["stft"], speaker=gi["speaker"])
    S["post/out"] = m.output
    G = m.backward(S)
    torch.cuda.synchronize()
    res = {k: ((G[k].float().cpu() - g.float()).abs().max().item(), g.abs().max().item()) for k, g in g_ref.items()}
    assert all(f"dec/spk/{n}/W" in res for n in ("attn", "h1", "h2", "h3"))
    a = torch.cat([G[k].float().cpu().reshape(-1) for k in g_ref])
    b = torch.cat([g_ref[k].float().reshape(-1) for k in g_ref])
    if precision == "tf32":                    # single-pass TF32 products in the forward and the data gradients
        assert ((a - b).norm() / b.norm()).item() <= 2e-2
        assert torch.nn.functional.cosine_similarity(a, b, dim=0).item() >= 0.999
        return
    _bar(res, 2e-3, 1e-3)
    assert ((a - b).norm() / b.norm()).item() <= 1e-4
    assert torch.nn.functional.cosine_similarity(a, b, dim=0).item() >= 0.9999


def test_drivers_speaker_decoder(tmp_path, monkeypatch):
    from tacotron_b200 import checkpoint, test as synth, train as trainer
    from tacotron_b200.models.tacotron import Config, Tacotron
    _dataset(str(tmp_path))
    monkeypatch.chdir(tmp_path)
    cfg = Config(); cfg.data_path, cfg.save_path, cfg.restore = "data/toyspk/", "toyspk/tacotron", False
    cfg.speaker_decoder = True
    m = trainer.train(Tacotron, cfg, num_steps=4, log=lambda *a: None, save_every=4)
    ck = "weights/toyspk/tacotron-4.npz"
    assert m.global_step == 4 and os.path.exists(ck) and checkpoint.speaker_decoder(ck)
    assert float(m.store["dec/spk/h1/W"].abs().max()) > 0
    waves = []
    for spk, max_ctas in ((0, None), (2, None), (2, 64)):
        c = Config(); c.data_path, c.save_path, c.max_ctas = cfg.data_path, cfg.save_path, max_ctas
        w = synth.test(Tacotron, c, ["abc de\n"], log=lambda *a: None, speaker=spk)
        assert c.speaker_decoder and len(w) == 1 and torch.isfinite(w[0]).all()
        waves.append(w[0].cpu())
    assert waves[0].shape != waves[1].shape or not torch.equal(waves[0], waves[1])     # two speakers, two outputs
    # a model without the setting refuses the checkpoint, naming the variables
    with pytest.raises(ValueError, match="dec/spk/"):
        checkpoint.restore(Tacotron(Config(r=2, vocab_size=20, num_speakers=3), None, train=False), ck)
