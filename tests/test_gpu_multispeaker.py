"""-m gpu: the multi-speaker model (models/tacotron.py:116-124, models/ops.py:101-115) on the H100: the new entry points
against their mirrors, inference against the oracle, batch permutation and CUDA-graph replay with new speaker ids, the
training gradients against torch.autograd, and the two drivers on a tiny multi-speaker data set."""
import ctypes as C
import os
import pickle

import numpy as np
import pytest
import torch

from oracle import tacotron_oracle as O
from tacotron_b200 import _lib as L
from tacotron_b200 import kernels as K
from tacotron_b200.models import ops
from tacotron_b200.params import ParamStore
from tests import mirror_kernels_spk as MK, speaker_oracle as SO
from tests.util import assert_close

pytestmark = pytest.mark.gpu
TOL = {"fp32": 2e-4, "fp32x3": 2e-4, "tf32": 5e-3}
LIN_TOL = {"fp32": 1e-5, "fp32x3": 1e-5, "tf32": 5e-3}


def _rt(precision):
    store = ParamStore([("dummy", (4,), "zeros")], "cuda")
    return ops.Runtime(store, precision)


# ---------------------------------------------------------------------------------------------------------------------
# taco_linear_fwd with a per-utterance bias
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "fp32x3", "tf32"])
@pytest.mark.parametrize("B,T,Cin,N,ldbu,act", [
    (2, 300, 128, 128, 128, L.ACT_NONE),      # several 128-row tiles per utterance
    (33, 17, 128, 128, 160, L.ACT_RELU),      # B = 33, ldbu != N
    (3, 40, 64, 130, 130, L.ACT_NONE),        # N % 4 != 0: the transposing epilogue
    (1, 5, 16, 640, 640, L.ACT_RELU),         # the speaker-dense shape (one row per utterance)
])
def test_linear_bias_utt(precision, B, T, Cin, N, ldbu, act):
    g = torch.Generator().manual_seed(B * 1000 + T)
    X = torch.randn(B, T, Cin, generator=g)
    W = torch.randn(Cin, N, generator=g) / Cin ** 0.5
    bias = torch.randn(N, generator=g)
    bu_full = torch.randn(B, ldbu, generator=g)
    ref = MK.linear_bias_utt(X.double(), W.double(), bias.double(), bu_full[:, :N].double(), act)
    rt = _rt(precision)
    Xd, Wd, bd, bud = X.cuda(), W.cuda().contiguous(), bias.cuda(), bu_full.cuda()
    Wp = ops._pack(rt, None, Wd, 1, Cin, N) if precision != "fp32" else None
    out = torch.full((B, T, N), float("nan"), device="cuda")
    ops.linear(rt, Xd, Wd, Wp, N, bias=bd, act=act, bias_utt=bud, out=out)
    torch.cuda.synchronize()
    assert_close(out, ref, LIN_TOL[precision], f"linear bias_utt {precision}")
    # without bias_utt the result is the plain linear, unchanged
    out0 = torch.empty(B, T, N, device="cuda")
    ops.linear(rt, Xd, Wd, Wp, N, bias=bd, act=act, out=out0)
    out1 = torch.empty(B, T, N, device="cuda")
    ops.linear(rt, Xd, Wd, Wp, N, bias=bd, act=act, bias_utt=torch.zeros(B, N, device="cuda"), out=out1)
    torch.cuda.synchronize()
    assert torch.equal(out0, out1)


def test_linear_bias_utt_rejects_highway():
    rt = _rt("fp32x3")
    X = torch.randn(2, 8, 128, device="cuda")
    W = torch.randn(128, 256, device="cuda")
    Wp = ops._pack(rt, None, W, 1, 128, 256)
    with pytest.raises(L.TacoError):
        ops.linear(rt, X, W, Wp, 256, highway_x=X, bias_utt=torch.zeros(2, 256, device="cuda"))


# ---------------------------------------------------------------------------------------------------------------------
# bi-GRU with initial states, per-segment column sums
# ---------------------------------------------------------------------------------------------------------------------
def _gru_case(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    xp = torch.randn(B, T, 768, generator=g)
    W = [torch.randn(128, 256, generator=g) * 0.1, torch.randn(128, 128, generator=g) * 0.1,
         torch.randn(128, 256, generator=g) * 0.1, torch.randn(128, 128, generator=g) * 0.1]
    h0 = [torch.randn(B, 128, generator=g), torch.randn(B, 128, generator=g)]
    return xp, W, h0


@pytest.mark.parametrize("B,T", [(3, 9), (33, 40), (2, 1)])
def test_bigru_fwd_h0(B, T):
    xp, W, h0 = _gru_case(B, T, B + T)
    ref = torch.zeros(B, T, 256, dtype=torch.float64)
    MK.bigru_fwd_h0(ref, xp.double(), *[w.double() for w in W], h0[0].double(), h0[1].double())
    xd, Wd, h0d = xp.cuda(), [w.cuda().contiguous() for w in W], [h.cuda() for h in h0]
    out = torch.empty(B, T, 256, device="cuda")
    K.bigru_fwd_h0(out, xd, *Wd, *h0d)
    # NULL initial states: bit-identical to the zero-state entry point
    a = torch.empty(B, T, 256, device="cuda")
    b = torch.empty(B, T, 256, device="cuda")
    K.bigru_fwd_h0(a, xd, *Wd, None, None)
    L.check(L.lib().taco_bigru_fwd(L.ptr(xd), *[L.ptr(w) for w in Wd], L.ptr(b), B, T, L.current_stream()), "taco_bigru_fwd")
    torch.cuda.synchronize()
    assert (out.double().cpu() - ref).abs().max().item() <= 2e-5
    assert torch.equal(a, b)


@pytest.mark.parametrize("B,T", [(3, 9), (32, 40), (2, 1)])
def test_bigru_bwd_h0(B, T):
    g = torch.Generator().manual_seed(10 + T)
    out = torch.tanh(torch.randn(B, T, 256, generator=g))
    ACT = torch.rand(B, T, 768, generator=g)
    ACT[:, :, 256:384] = ACT[:, :, 256:384] * 2 - 1
    ACT[:, :, 640:768] = ACT[:, :, 640:768] * 2 - 1
    dOut = torch.randn(B, T, 256, generator=g)
    _, W, h0 = _gru_case(B, T, 20 + T)
    ref, dref = torch.zeros(B, T, 768, dtype=torch.float64), torch.zeros(B, 2, 128, dtype=torch.float64)
    MK.bigru_bwd_h0(ref, dOut.double(), out.double(), ACT.double(), *[w.double() for w in W], h0[0].double(), h0[1].double(), dref)
    cu = lambda t: t.cuda().contiguous()
    dxp, dh0 = torch.empty(B, T, 768, device="cuda"), torch.empty(B, 2, 128, device="cuda")
    K.bigru_bwd_h0(dxp, cu(dOut), cu(out), cu(ACT), *map(cu, W), cu(h0[0]), cu(h0[1]), dh0)
    torch.cuda.synchronize()
    assert (dxp.double().cpu() - ref).abs().max().item() <= 1e-4 * ref.abs().max().item()
    assert (dh0.double().cpu() - dref).abs().max().item() <= 1e-4 * dref.abs().max().item()


@pytest.mark.parametrize("M,N,period", [(32 * 128, 128, 128), (33 * 7, 45, 7), (64, 128, 2)])
def test_colsum_seg(M, N, period):
    g = torch.Generator().manual_seed(M)
    A = torch.randn(M, N + 8, generator=g)[:, 4:4 + N]
    out = torch.randn(M // period, N, generator=g)
    ref = out.double().clone()
    MK.colsum_seg(ref, A.double(), period)
    od = out.cuda()
    K.colsum_seg(od, A.cuda(), period)
    o2 = out.cuda()
    K.colsum_seg(o2, A.cuda(), period)
    torch.cuda.synchronize()
    assert (od.double().cpu() - ref).abs().max().item() <= 1e-5 * (1 + ref.abs().max().item())
    assert torch.equal(od, o2)                               # deterministic


# ---------------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------------
NSPK = 4


def _model(cfg_o, p, precision, cuda_graph=False):
    from tacotron_b200 import Config, Tacotron
    cfg = Config(r=cfg_o.r, vocab_size=cfg_o.vocab_size, max_decode_iter=cfg_o.max_decode_iter, precision=precision,
                 num_speakers=getattr(cfg_o, "num_speakers", 1), cuda_graph=cuda_graph)
    m = Tacotron(cfg, None, train=False)
    m.load_params(p)
    return m


def _case(r=2, B=3, Tx=16, T=10, seed=0):
    cfg = SO.SpkOracleConfig(r=r, max_decode_iter=T, vocab_size=20, num_speakers=NSPK)
    p = SO.init_params(cfg, seed=1, trained_like=True)
    inp = O.synthetic_inputs(cfg, B, Tx, T, seed=seed, ragged=True, with_targets=False)
    inp["speaker"] = torch.tensor([3, 0, 2, 1, 3, 2, 0, 1][:B], dtype=torch.int32)
    return cfg, p, inp


def _cuda(inp):
    return {k: v.cuda().contiguous() for k, v in inp.items()}


@pytest.mark.parametrize("precision", ["fp32", "fp32x3", "tf32"])
@pytest.mark.parametrize("r", [2, 5])
def test_inference_matches_oracle(precision, r):
    cfg, p, inp = _case(r)
    y_ref, out_ref, a_ref = SO.inference(p, inp, cfg, train=False)
    m = _model(cfg, p, precision)
    y, out = m.inference(_cuda(inp), train=False)
    torch.cuda.synchronize()
    assert_close(y, y_ref, TOL[precision], "y")
    assert_close(m.alignments, a_ref, TOL[precision], "align")
    assert_close(out, out_ref, TOL[precision], "out")


def test_missing_speaker_raises_and_single_speaker_ignores_it():
    cfg, p, inp = _case()
    m = _model(cfg, p, "fp32x3")
    bad = _cuda({k: v for k, v in inp.items() if k != "speaker"})
    with pytest.raises(ValueError):
        m.inference(bad, train=False)
    cfg1 = O.OracleConfig(r=2, max_decode_iter=10, vocab_size=20)
    p1 = O.init_params(cfg1, seed=1, trained_like=True)
    m1 = _model(cfg1, p1, "fp32x3")
    y_a, _ = m1.inference(bad, train=False)
    y_a = y_a.clone()
    y_b, _ = m1.inference(_cuda(inp), train=False)
    torch.cuda.synchronize()
    assert torch.equal(y_a, y_b)


def test_batch_permutation_and_graph_replay():
    cfg, p, inp = _case(B=4)
    m = _model(cfg, p, "fp32x3")
    ci = _cuda(inp)
    y0, out0 = [t.clone() for t in m.inference(ci, train=False)]
    perm = torch.tensor([2, 0, 3, 1])
    pi = {k: v[perm.to(v.device)].contiguous() for k, v in ci.items()}
    y1, out1 = [t.clone() for t in m.inference(pi, train=False)]
    torch.cuda.synchronize()
    assert_close(y1, y0[perm.cuda()], 1e-5, "permuted y")
    assert_close(out1, out0[perm.cuda()], 1e-5, "permuted out")
    # CUDA graphs: capture with one set of speaker ids, replay with another -> equal to eager execution
    mg = _model(cfg, p, "fp32x3", cuda_graph=True)
    mg.inference(ci, train=False)
    ni = dict(ci)
    ni["speaker"] = torch.tensor([1, 1, 0, 2], dtype=torch.int32, device="cuda")
    yg, outg = [t.clone() for t in mg.inference(ni, train=False)]
    ye, oute = [t.clone() for t in m.inference(ni, train=False)]
    torch.cuda.synchronize()
    assert torch.equal(yg, ye) and torch.equal(outg, oute)
    assert not torch.equal(yg, y0)


def _bar(res, tol, floor):
    bad = {k: v for k, v in res.items() if v[0] > tol * (v[1] + floor) + 1e-7}
    assert not bad, bad


@pytest.mark.parametrize("precision", ["fp32", "fp32x3"])
def test_training_gradients_match_autograd(precision):
    r, B, Tx, T = 5, 2, 8, 5
    cfg = SO.SpkOracleConfig(r=r, vocab_size=20, num_speakers=NSPK, scheduled_sample=0.0)
    p = SO.init_params(cfg, seed=1, trained_like=True)
    inp = O.synthetic_inputs(cfg, B, Tx, T, seed=0, ragged=True)
    inp["speaker"] = torch.tensor([3, 1], dtype=torch.int32)
    enc_m, dec_m = O.dropout_masks(cfg, B, Tx, T, seed=2)
    _, g_ref = SO.loss_and_grads(p, inp, cfg, enc_drop_masks=enc_m, dec_drop_masks=dec_m)
    from tacotron_b200 import Config, Tacotron
    m = Tacotron(Config(r=r, vocab_size=20, precision=precision, num_speakers=NSPK, scheduled_sample=0.0), None, train=True)
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
    assert any(k.startswith("speaker/") for k in res) and "enc/cbhg/gru_init/Ws" in res
    _bar(res, 2e-3, 1e-3)
    a = torch.cat([G[k].float().cpu().reshape(-1) for k in g_ref])
    b = torch.cat([g_ref[k].float().reshape(-1) for k in g_ref])
    assert ((a - b).norm() / b.norm()).item() <= 1e-4
    assert torch.nn.functional.cosine_similarity(a, b, dim=0).item() >= 0.9999


def _dataset(root, N=40, Tx=12, T=8, r=2, nspk=3, seed=0):
    rng = np.random.RandomState(seed)
    d = os.path.join(root, "data", "toyspk") + "/"
    os.makedirs(d, exist_ok=True)
    np.save(d + "texts.npy", rng.randint(1, 20, size=(N, Tx)))
    np.save(d + "text_lens.npy", rng.randint(4, Tx + 1, size=N))
    np.save(d + "stfts.npy", (rng.randn(N, T, 1025 * r) * 2 - 3).astype(np.float16))
    np.save(d + "mels.npy", (rng.randn(N, T, 80 * r) * 2 - 3).astype(np.float16))
    np.save(d + "speech_lens.npy", rng.randint(3, T + 1, size=N))
    np.save(d + "speakers.npy", np.arange(N) % nspk)
    with open(d + "meta.pkl", "wb") as f:
        pickle.dump({"r": r, "vocab": {i: chr(96 + i) for i in range(20)}}, f)
    return d


def test_drivers_multispeaker(tmp_path, monkeypatch):
    from tacotron_b200 import test as synth, train as trainer
    from tacotron_b200.models.tacotron import Config, Tacotron
    _dataset(str(tmp_path))
    monkeypatch.chdir(tmp_path)
    cfg = Config(); cfg.data_path, cfg.save_path, cfg.restore = "data/toyspk/", "toyspk/tacotron", False
    m = trainer.train(Tacotron, cfg, num_steps=4, log=lambda *a: None, save_every=4)
    assert m.config.num_speakers == 3 and m.global_step == 4 and os.path.exists("weights/toyspk/tacotron-4.npz")
    assert tuple(m.store["speaker/embed"].shape) == (3, 16)
    cfg2 = Config(); cfg2.data_path, cfg2.save_path = cfg.data_path, cfg.save_path
    waves = synth.test(Tacotron, cfg2, ["abc de\n"], log=lambda *a: None, speaker=1)
    assert cfg2.num_speakers == 3 and len(waves) == 1 and torch.isfinite(waves[0]).all()
    cfg3 = Config(); cfg3.data_path, cfg3.save_path = cfg.data_path, cfg.save_path
    with pytest.raises(ValueError):
        synth.test(Tacotron, cfg3, ["abc\n"], log=lambda *a: None, speaker=3)
