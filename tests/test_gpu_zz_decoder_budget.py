"""-m gpu: the decoder kernels under a CTA budget (Config.max_ctas / the max_ctas fields of the ABI).

Forward: the row groups of a launch are independent 32-CTA machines, so any budget gives y, alignments and the saved GRU
states bit-identical to the default launch.  Backward: every output column of every stage is computed by one CTA with the
same K split over its 8 warps whatever the grid, and each utterance's attention by one CTA, so each column's arithmetic
does not depend on G: every budget is bit-identical to G = 128 (and within the float64 mirror's bar).  A budget on this
132-SM card reproduces the launch plan of a smaller part (an H100 PCIe has 114 SMs), not its clocks or memory."""
import pytest
import torch

from tests import mirror_kernels as MK
from tests.test_gpu_decoder_envelope import DEC_OUTS, _setup
from tests.util import assert_close

pytestmark = pytest.mark.gpu

_stores = {}


def _store(r, p):
    from tacotron_b200 import Config
    from tacotron_b200.models import ops
    from tacotron_b200.params import ParamStore, model_shapes
    if r not in _stores:
        st = ParamStore(model_shapes(Config(r=r, vocab_size=20)), "cuda")
        st.load(p)
        ops.runtime(st, "fp32")
        _stores[r] = st
    return _stores[r]


def _forward(r, B, Tx, T, mode, budgets):
    """{budget: (y, align, h_save or None, decoder launches)} through ops.attention_decoder on the same inputs"""
    from tacotron_b200 import _lib as L
    from tacotron_b200.models import ops
    cfg, p, encoded, mel, tl, dec_m, sm = _setup(r, B, Tx, T)
    st = _store(r, p)
    lmode = {"infer": L.DEC_INFER, "teacher": L.DEC_TEACHER, "sched": L.DEC_SCHED}[mode]
    enc, tlc, melc = encoded.cuda(), tl.cuda(), mel.cuda()
    drop = None if mode == "infer" else (dec_m[0].cuda(), dec_m[1].cuda())
    smask = sm.cuda() if mode == "sched" else None
    save = mode != "infer" and B <= 32                       # train-mode saving (h_save) holds at most 32 utterances
    ops.attention_decoder(enc, tlc, r, T, mode=lmode, mel=None if mode == "infer" else melc, sample_mask=smask, drop_masks=drop,
                          scope=ops.Scope(st, "dec"))                 # first call: packs the weights, allocates the buffers
    out = {}
    for m in budgets:
        S = {}
        n0 = L.lib().taco_launch_count()
        if save:
            with ops.saving(S):
                y, a = ops.attention_decoder(enc, tlc, r, T, mode=lmode, mel=None if mode == "infer" else melc, sample_mask=smask,
                                             drop_masks=drop, scope=ops.Scope(st, "dec"), max_ctas=m)
        else:
            y, a = ops.attention_decoder(enc, tlc, r, T, mode=lmode, mel=None if mode == "infer" else melc, sample_mask=smask,
                                         drop_masks=drop, scope=ops.Scope(st, "dec"), max_ctas=m)
        torch.cuda.synchronize()
        out[m] = (y.clone(), a.clone(), S["dec/H"].clone() if save else None, int(L.lib().taco_launch_count() - n0))
    return out


@pytest.mark.parametrize("Tx", [67, 128])
@pytest.mark.parametrize("r", [2, 5])
@pytest.mark.parametrize("B", [1, 8, 9, 24, 25, 32, 33, 64])
@pytest.mark.parametrize("mode", ["infer", "teacher", "sched"])
def test_forward_budgets_bit_identical(mode, B, r, Tx):
    from tacotron_b200 import kernels as K
    from tacotron_b200.models import ops
    cap = K.decoder_capacity()[0]
    budgets = [None, 96, 64, 32]                              # 96 = the plan a 114-SM part gets
    out = _forward(r, B, Tx, 6, mode, budgets)
    y0, a0, h0, n0 = out[None]
    assert not torch.isnan(y0).any() and not torch.isnan(a0).any()
    for m in budgets[1:]:
        y, a, h, n = out[m]
        assert torch.equal(y, y0), f"budget {m}: y"
        assert torch.equal(a, a0), f"budget {m}: align"
        if h0 is not None:
            assert torch.equal(h, h0), f"budget {m}: h_save"
        plan = ops.decoder_plan(B, cap, m)
        assert len(plan) == -(-B // (8 * (m // 32)))
        assert all(c == 32 * (m // 32) and nb <= 8 * (m // 32) for _, nb, c in plan)
        # the decoder launches are the only difference in the number of kernels launched
        assert n - n0 == len(plan) - len(ops.decoder_plan(B, cap)), (m, n, n0)


def test_capacity():
    from tacotron_b200 import kernels as K
    f, b = K.decoder_capacity()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert f == sms and b == sms                              # one CTA of either kernel per SM


# ---------------------------------------------------------------------------------------------------------------------
# backward
# ---------------------------------------------------------------------------------------------------------------------
def test_backward_budgets():
    """taco_decoder_bwd at G = 128, 114, 96, 78, 64 and 32 CTAs: each within the float64 mirror's bar (2e-4, as in
    test_gpu_decoder_envelope.py) and bit-identical to G = 128.  The weight-row cache is on from 128 down to 64 CTAs (48 to
    98 KB per CTA) and does not fit at 32 (197 KB + the partial sums > 200 KB), so both paths run."""
    from tacotron_b200 import kernels as K
    from tacotron_b200.models import grad
    from tests import grad_util
    r, B, Tx, T = 5, 32, 67, 60
    cfg, p, encoded, mel, tl, dec_m, sm = _setup(r, B, Tx, T)
    S = {"mel": mel, "text_length": tl, "dec/keep1": dec_m[0], "dec/keep2": dec_m[1], "_capture": {}, "dec/sample_mask": sm}
    grad_util.decoder_saving(encoded, tl, p, cfg, T, mel, dec_m, sm, S)
    G = {k: torch.zeros_like(v) for k, v in p.items()}
    dY = torch.randn(B, T, 80 * r, generator=torch.Generator().manual_seed(5))
    grad.decoder_bwd(MK, p, G, S, cfg, dY)
    args = {k: v for k, v in S["_capture"]["decoder_bwd"].items() if not k.startswith("_")}
    ref = {k: ([t.double() for t in v] if isinstance(v, list) else v.double() if torch.is_tensor(v) and v.is_floating_point() else v)
           for k, v in args.items()}
    MK.decoder_bwd(ref)
    outs = {}
    for m in (128, 114, 96, 78, 64, 32):
        gpu = {k: ([t.cuda() for t in v] if isinstance(v, list) else v.cuda() if torch.is_tensor(v) else v) for k, v in args.items()}
        for t in [gpu[k] for k in DEC_OUTS] + gpu["DG"] + gpu["DC"]:
            t.fill_(float("nan"))
        gpu["max_ctas"] = m
        K.decoder_bwd(gpu)
        torch.cuda.synchronize()
        what = f"decoder_bwd G={m}"
        for k in DEC_OUTS:
            assert not torch.isnan(gpu[k]).any(), f"{what} {k}: cells left unwritten"
            assert_close(gpu[k], ref[k], 2e-4, f"{what} {k}")
        for i in range(3):
            assert_close(gpu["DG"][i], ref["DG"][i], 2e-4, f"{what} DG{i}")
            assert_close(gpu["DC"][i], ref["DC"][i], 2e-4, f"{what} DC{i}")
        outs[m] = [gpu[k] for k in DEC_OUTS] + gpu["DG"] + gpu["DC"]
    for m in outs:
        for i, (x, x0) in enumerate(zip(outs[m], outs[128])):
            assert torch.equal(x, x0), f"G={m}: output {i} differs from G=128"


# ---------------------------------------------------------------------------------------------------------------------
# model: C2 inference and a C2 training step at max_ctas = 96
# ---------------------------------------------------------------------------------------------------------------------
def _c2():
    from oracle import tacotron_oracle as O
    cfg = O.OracleConfig(r=5, vocab_size=64)
    p = O.init_params(cfg, seed=1, trained_like=True)
    inp = O.synthetic_inputs(cfg, 32, 128, 200, seed=0, ragged=True)
    enc_m, dec_m = O.dropout_masks(cfg, 32, 128, 200, seed=2)
    sm = O.sched_mask(cfg, 32, 200, seed=3)
    return cfg, p, inp, enc_m, dec_m, sm


def test_c2_inference_budget():
    from tacotron_b200 import Config, Tacotron
    cfg, p, inp, *_ = _c2()
    res = {}
    for m in (None, 96):
        mod = Tacotron(Config(r=5, vocab_size=64, max_decode_iter=200, max_ctas=m), None, train=False)
        mod.load_params(p)
        y, out = mod.inference({k: v.cuda() for k, v in inp.items() if k in ("text", "text_length")}, train=False)
        torch.cuda.synchronize()
        res[m] = (y.clone(), out.clone(), mod.alignments.clone())
    for a, b in zip(res[96], res[None]):
        assert torch.equal(a, b)


def test_c2_train_step_budget():
    from tacotron_b200 import Config, Tacotron
    from tacotron_b200.models import ops
    from tests.test_gpu_train_fullsize import _log_rel_l2
    cfg, p, inp, enc_m, dec_m, sm = _c2()
    res = {}
    for m in (None, 96):
        mod = Tacotron(Config(r=5, vocab_size=64, max_ctas=m), None, train=True)
        mod.load_params(p)
        gi = {k: v.cuda().contiguous() for k, v in inp.items()}
        S = {}
        with ops.saving(S):
            y, out = mod.inference(gi, True, enc_drop_masks=tuple(x.cuda() for x in enc_m),
                                   dec_drop_masks=tuple(x.cuda() for x in dec_m), sample_mask=sm.cuda())
        loss = mod.add_loss_op(y, out, gi["mel"], gi["stft"])
        S.update(text=gi["text"], text_length=gi["text_length"], mel=gi["mel"], stft=gi["stft"])
        S["post/out"] = out
        G = mod.backward(S)
        torch.cuda.synchronize()
        names = mod.store.trainable()
        res[m] = (y.clone(), out.clone(), S["dec/H"].clone(), loss.clone(), {n: G[n].clone() for n in names})
    y, out, h, loss, g = res[96]
    y0, out0, h0, loss0, g0 = res[None]
    assert torch.equal(y, y0) and torch.equal(out, out0) and torch.equal(h, h0) and torch.equal(loss, loss0)
    # gradients: the split-K weight gradients add with float atomics, so two runs agree to that rounding; held to the bars of
    # test_gpu_train_fullsize.py (2e-4 per tensor, 3e-5 on the whole vector)
    for n in g:
        assert_close(g[n], g0[n], 2e-4, f"C2 grad max_ctas=96 {n}")
    a = torch.cat([g[n].double().reshape(-1) for n in g])
    b = torch.cat([g0[n].double().reshape(-1) for n in g])
    assert _log_rel_l2("C2 grad max_ctas=96 whole-gradient rel L2", a, b, 3e-5) <= 3e-5


# ---------------------------------------------------------------------------------------------------------------------
# drivers and errors
# ---------------------------------------------------------------------------------------------------------------------
def test_drivers_with_budget(tmp_path, monkeypatch):
    import os
    from tacotron_b200 import test as synth, train as trainer
    from tacotron_b200.models.tacotron import Config, Tacotron
    from tests.test_gpu_z_data import _dataset
    root = str(tmp_path)
    _dataset(root)
    monkeypatch.chdir(root)
    torch.manual_seed(0)
    cfg = Config()
    cfg.data_path, cfg.save_path, cfg.restore, cfg.max_ctas = "data/toy/", "toy/tacotron", False, 64
    m = trainer.train(Tacotron, cfg, num_steps=2, log=lambda *a: None, save_every=2)
    torch.cuda.synchronize()
    assert m.config.max_ctas == 64 and torch.isfinite(m.loss).all()
    cfg = Config()
    cfg.data_path, cfg.save_path, cfg.max_ctas = "data/toy/", "toy/tacotron", 64
    waves = synth.test(Tacotron, cfg, ["abc de\n", "hello, you\n"], log=lambda *a: None)
    assert len(waves) == 2 and all(torch.isfinite(w).all() for w in waves)
    assert os.path.isdir("weights")


def test_budget_below_32_raises_before_any_launch():
    import ctypes as C
    from tacotron_b200 import Config, Tacotron, _lib as L
    from tacotron_b200.models import ops
    lib = L.lib()
    n0 = lib.taco_launch_count()
    with pytest.raises(L.TacoError, match="max_ctas=31"):
        Tacotron(Config(r=2, vocab_size=20, max_ctas=31), None, train=False)
    with pytest.raises(L.TacoError, match="max_ctas=31"):
        ops.attention_decoder(torch.zeros(1, 4, 256, device="cuda"), torch.ones(1, dtype=torch.int32, device="cuda"), 2, 3,
                              scope=ops.Scope(_store(2, _setup(2, 1, 4, 3)[1]), "dec"), max_ctas=31)
    a = L.DecoderArgs()
    a.B, a.T, a.Tx, a.r, a.max_ctas = 1, 3, 4, 2, 31
    a.weights = C.pointer(L.DecoderWeights())
    assert lib.taco_decoder_fwd(C.byref(a), None) != 0 and b"max_ctas=31" in lib.taco_last_error()
    d = L.DecoderBwdArgs()
    d.B, d.T, d.Tx, d.r, d.max_ctas = 1, 3, 4, 2, 31
    assert lib.taco_decoder_bwd(C.byref(d), None) != 0 and b"max_ctas=31" in lib.taco_last_error()
    torch.cuda.synchronize()
    assert lib.taco_launch_count() == n0
