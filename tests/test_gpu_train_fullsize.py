"""-m gpu: the training path at the shape the benchmark trains at (C2: B=32, Tx=128 with ragged lengths, T=200, r=5,
scheduled sampling 0.5, dropout), in all three precision modes.

At this size the backward takes the routes that only engage above a row threshold (kernels.DW_TC_MIN_ROWS,
kernels.GEMM_TC_MIN_ROWS): weight gradients on taco_conv_dw, recomputation and data-gradient products on taco_linear_fwd.
The toy-sized gradient tests of test_gpu_train.py stay below both thresholds, so only this module checks the host wiring
of those routes end to end.

  * backward parity: the GPU backward against the SAME host code (models/grad.py) run over the float64 mirror kernels
    (tests/mirror_kernels.py) on float64 copies of the GPU's own saved activations and parameters.  Both sides see
    identical forward values -- relu masks come from the saved outputs and the saved fp32 batch-norm affine, max-pool
    argmax from the saved input, the L1 sign from the saved output -- so every difference is backward arithmetic;
  * route accounting: which of the three tensor-core routes the backward takes in each precision mode;
  * localisation: the serial decoder-backward and bi-GRU-backward kernels against their mirrors on the inputs the GPU
    captured during that backward (outputs NaN-poisoned first, so a cell the kernel never writes shows up);
  * the train-mode forward (every saved activation and the loss) against the float64 oracle.
"""
import collections

import pytest
import torch

from oracle import tacotron_oracle as O
from tests import grad_util, mirror_kernels as MK, mirror_kernels_spk as MKS, speaker_oracle as SO
from tests.util import PARITY_LOG, assert_close, relerr

pytestmark = pytest.mark.gpu

B, TX, T, R = 32, 128, 200, 5
NSPK = 109                      # VCTK-sized speaker table


def _case(num_speakers=1):
    if num_speakers > 1:
        cfg = SO.SpkOracleConfig(r=R, vocab_size=64, num_speakers=num_speakers)
        p = SO.init_params(cfg, seed=1, trained_like=True)
    else:
        cfg = O.OracleConfig(r=R, vocab_size=64)
        p = O.init_params(cfg, seed=1, trained_like=True)
    inp = O.synthetic_inputs(cfg, B, TX, T, seed=0, ragged=True)
    if num_speakers > 1:
        inp["speaker"] = torch.randint(0, num_speakers, (B,), generator=torch.Generator().manual_seed(7), dtype=torch.int32)
    enc_m, dec_m = O.dropout_masks(cfg, B, TX, T, seed=2)
    sm = O.sched_mask(cfg, B, T, seed=3)
    return cfg, p, inp, enc_m, dec_m, sm


def _cuda(x):
    if isinstance(x, torch.Tensor):
        return x.cuda().contiguous()
    return type(x)(_cuda(v) for v in x)


def _f64(x):
    """CPU copy: floating tensors cast up to float64 (exact), integer / uint8 tensors unchanged; tuples / lists kept"""
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu()
        return (x.double() if x.dtype.is_floating_point else x).contiguous()
    if isinstance(x, (tuple, list)):
        return type(x)(_f64(v) for v in x)
    return x


def _forward(cfg, p, inp, enc_m, dec_m, sm, precision):
    """train-mode forward on the GPU with the activations saved; returns (model, S, inputs on the GPU)"""
    from tacotron_b200 import Config, Tacotron
    from tacotron_b200.models import ops
    m = Tacotron(Config(r=cfg.r, vocab_size=cfg.vocab_size, precision=precision, num_speakers=getattr(cfg, "num_speakers", 1),
                        scheduled_sample=cfg.scheduled_sample), None, train=True)
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
    return m, S, gi


def _log_rel_l2(what, a, b, tol):
    e = ((a - b).norm() / b.norm()).item()
    PARITY_LOG.append((what, e, e, tol))
    return e


# ---------------------------------------------------------------------------------------------------------------------
# A1 / A5: the whole backward against the float64 mirror of the same host code, on the GPU's own forward values
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision,nspk", [("fp32x3", 1), ("fp32", 1), ("tf32", 1), ("fp32x3", NSPK)])
def test_backward_matches_fp64_mirror(precision, nspk):
    from tacotron_b200.models import grad
    cfg, p, inp, enc_m, dec_m, sm = _case(nspk)
    m, S, _ = _forward(cfg, p, inp, enc_m, dec_m, sm, precision)
    G = m.backward(S)
    torch.cuda.synchronize()
    S64 = {k: _f64(v) for k, v in S.items()}
    P64 = {n: _f64(m.store[n]) for n in m.store.names()}
    G64 = {n: torch.zeros_like(v) for n, v in P64.items()}
    grad.model_bwd(MKS if nspk > 1 else MK, P64, G64, S64, cfg)
    names = m.store.trainable()
    if nspk > 1:
        assert "speaker/embed" in names and G64["speaker/embed"].abs().max() > 0
    tag = f"fullsize bwd {precision} nspk={nspk}"
    a = torch.cat([G[n].detach().double().cpu().reshape(-1) for n in names])
    b = torch.cat([G64[n].reshape(-1) for n in names])
    if precision == "tf32":
        # single-pass TF32 data-gradient / recomputation products (10-bit mantissa): only the whole vector is held
        assert _log_rel_l2(f"{tag} whole-gradient rel L2", a, b, 1e-2) <= 1e-2
        return
    bad = []
    for n in names:
        try:
            assert_close(G[n], G64[n], 2e-4, f"{tag} {n}")
        except AssertionError as ex:
            bad.append(str(ex))
    assert not bad, "\n".join(bad)
    # Whole-vector bars.  fp32 (exact-product FFMA): measured 5.2e-7.  fp32x3: measured 1.4e-5 (1.3e-5 with 109 speakers)
    # on an H100 80GB HBM3 (400 W power limit).  Moving the products back to the exact FFMA GEMM one route after the other, on the same saved
    # activations, attributes it:
    #   * ~3e-6 from the wgmma 3xTF32 products (recomputation and data gradients, taco_linear_fwd);
    #   * ~2e-6 more from the wgmma weight gradients (taco_conv_dw), which sum up to 32000 rows (post-net);
    #   * ~9e-6 more from the 3xTF32 mma.sync taco_gemm, in the decoder and encoder gradients only (the post-net's error
    #     does not change).  taco_decoder_bwd forms its weight-only products and its dy / dx tails with that GEMM.  It
    #     splits by truncation, and its own kernel bar is 2e-5 (test_gpu_z_gemm_mma.py).
    # So fp32x3 is held to 3e-5.  The mutation this module is built to catch (one tap offset off by one in the
    # taco_conv_dw route) moves 69 of the 150 tensors by 1.6e-3 to 1.3 relative.
    bar = 1e-5 if precision == "fp32" else 3e-5
    assert _log_rel_l2(f"{tag} whole-gradient rel L2", a, b, bar) <= bar
    for n in m.store.names():
        if n.endswith(("bn_mean", "bn_var")):
            assert G[n].abs().max().item() == 0.0, n


# ---------------------------------------------------------------------------------------------------------------------
# A2: which tensor-core routes the backward takes
# ---------------------------------------------------------------------------------------------------------------------
def _route_counts(monkeypatch, case, precision):
    from tacotron_b200 import _lib as L
    from tacotron_b200 import kernels as K
    m, S, _ = _forward(*case, precision)
    torch.cuda.synchronize()
    n = collections.Counter()

    def accepted(tag, fn):
        def f(*a, **kw):
            ok = fn(*a, **kw)
            n[tag] += bool(ok)
            return ok
        return f

    check = L.check

    def counting_check(rc, what):
        n["launch " + what] += 1
        return check(rc, what)

    with monkeypatch.context() as mp:
        mp.setattr(K, "_dw_tc_ok", accepted("dw_tc", K._dw_tc_ok))
        mp.setattr(K, "_gemm_tc_ok", accepted("gemm_tc", K._gemm_tc_ok))
        mp.setattr(L, "check", counting_check)
        m.backward(S)
        torch.cuda.synchronize()
    # an accepted route is a launch of its kernel, and the data-gradient branch of conv_dx is the only taco_linear_fwd[conv_dx]
    assert n["launch taco_conv_dw"] == n["dw_tc"] and n["launch taco_linear_fwd[gemm]"] == n["gemm_tc"], dict(n)
    return n["dw_tc"], n["gemm_tc"], n["launch taco_linear_fwd[conv_dx]"]


@pytest.mark.parametrize("precision", ["fp32x3", "tf32", "fp32"])
def test_backward_routes(monkeypatch, precision):
    dw, gm, dx = _route_counts(monkeypatch, _case(), precision)
    if precision == "fp32":
        assert (dw, gm, dx) == (0, 0, 0)
    else:
        assert dw > 0 and gm > 0 and dx > 0, (dw, gm, dx)


def test_small_case_stays_below_the_row_thresholds(monkeypatch):
    """why this module exists: at the size of test_gpu_train.py's gradient tests the row-threshold routes never run"""
    cfg = O.OracleConfig(r=2, vocab_size=20)
    p = O.init_params(cfg, seed=1, trained_like=True)
    inp = O.synthetic_inputs(cfg, 2, 8, 5, seed=0, ragged=True)
    enc_m, dec_m = O.dropout_masks(cfg, 2, 8, 5, seed=2)
    dw, gm, dx = _route_counts(monkeypatch, (cfg, p, inp, enc_m, dec_m, O.sched_mask(cfg, 2, 5, seed=3)), "fp32x3")
    assert dw == 0 and gm == 0 and dx > 0


# ---------------------------------------------------------------------------------------------------------------------
# A3: the serial backward kernels at full size, on the inputs the GPU captured during the model backward
# ---------------------------------------------------------------------------------------------------------------------
DEC_OUTS = ("DATT", "DY", "DPQ", "DSCORE", "DCTX", "DZ", "DPN2", "DPN1", "DX")


def _poisoned_copy(v):
    return [t.clone() for t in v] if isinstance(v, list) else (v.clone() if isinstance(v, torch.Tensor) else v)


@pytest.mark.parametrize("precision", ["fp32x3", "fp32"])
def test_serial_backward_kernels_at_size(precision):
    from tacotron_b200 import kernels as K
    cfg, p, inp, enc_m, dec_m, sm = _case()
    m, S, _ = _forward(cfg, p, inp, enc_m, dec_m, sm, precision)
    S["_capture"] = {}
    m.backward(S)
    torch.cuda.synchronize()
    cap = S["_capture"]
    # decoder backward: T=200 steps, Tx=128, B=32, r=5
    a = {k: _poisoned_copy(v) for k, v in cap["decoder_bwd"].items() if not k.startswith("_")}
    for k in DEC_OUTS:
        a[k].fill_(float("nan"))
    for i in range(3):
        a["DG"][i].fill_(float("nan")); a["DC"][i].fill_(float("nan"))
    # the kernel forms its weight-only products with taco_gemm: rerun it with the GEMM the model's backward selected
    prev = K.set_gemm_impl(0 if precision == "fp32" else 1)
    try:
        K.decoder_bwd(a)
        torch.cuda.synchronize()
    finally:
        K.set_gemm_impl(prev)
    a64 = {k: _f64(v) for k, v in cap["decoder_bwd"].items() if not k.startswith("_")}
    for t in [a64[k] for k in DEC_OUTS] + a64["DG"] + a64["DC"]:
        t.fill_(float("nan"))
    MK.decoder_bwd(a64)
    tag = f"fullsize decoder_bwd {precision}"
    for k in DEC_OUTS:
        assert not torch.isnan(a[k]).any(), f"{k}: cells left unwritten"
        assert_close(a[k], a64[k], 2e-4, f"{tag} {k}")
    for i in range(3):
        assert not (torch.isnan(a["DG"][i]).any() or torch.isnan(a["DC"][i]).any()), f"DG{i}/DC{i}: cells left unwritten"
        assert_close(a["DG"][i], a64["DG"][i], 2e-4, f"{tag} DG{i}")
        assert_close(a["DC"][i], a64["DC"][i], 2e-4, f"{tag} DC{i}")
    # the model's own call wrote the same values as the rerun (same inputs, deterministic kernel)
    for k in DEC_OUTS:
        assert torch.equal(a[k], cap["decoder_bwd"][k]), k
    # bi-GRU backward: encoder (T=128) and post-net (T=1000) sequences
    for pre in ("enc/cbhg", "post/cbhg"):
        c = cap[f"{pre}/bigru_bwd"]
        W = [m.store[f"{pre}/{d}/{w}"][128:].contiguous() for d in ("gru_fw", "gru_bw") for w in ("Wg", "Wc")]
        dxp = torch.full_like(c["dxp"], float("nan"))
        K.bigru_bwd(dxp, c["dOut"], c["out"], c["ACT"], *W)
        torch.cuda.synchronize()
        ref = torch.zeros(c["dxp"].shape, dtype=torch.float64)
        MK.bigru_bwd(ref, _f64(c["dOut"]), _f64(c["out"]), _f64(c["ACT"]), *[_f64(w) for w in W])
        assert not torch.isnan(dxp).any(), f"{pre}: dxp cells left unwritten"
        assert_close(dxp, ref, 1e-4, f"fullsize {pre} bigru_bwd dxp {precision}")


# ---------------------------------------------------------------------------------------------------------------------
# A4: the train-mode forward at size against the float64 oracle
# ---------------------------------------------------------------------------------------------------------------------
_REF = {}


def _fp64_forward():
    if "fwd" not in _REF:
        cfg, p, inp, enc_m, dec_m, sm = _case()
        p64 = {k: v.double() for k, v in p.items()}
        inp64 = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in inp.items()}
        Sref, y, out = grad_util.saving_forward(p64, inp64, cfg, enc_m, dec_m, sm)
        loss = O.loss(y, out, inp64["mel"], inp64["stft"])[0]
        _REF["fwd"] = ({k: v for k, v in Sref.items() if isinstance(v, torch.Tensor) and v.dtype.is_floating_point}, y, out, loss)
    return _REF["fwd"]


@pytest.mark.parametrize("precision,tol", [("fp32x3", 5e-4), ("fp32", 5e-4), ("tf32", 5e-3)])
def test_train_forward_at_size(precision, tol):
    Sref, y_ref, out_ref, loss_ref = _fp64_forward()
    cfg, p, inp, enc_m, dec_m, sm = _case()
    m, S, gi = _forward(cfg, p, inp, enc_m, dec_m, sm, precision)
    loss = m.add_loss_op(m.seq2seq_output, m.output, gi["mel"], gi["stft"])
    torch.cuda.synchronize()
    missing = [k for k in Sref if k not in S and k not in ("mel", "stft", "post/out")]
    assert not missing, missing
    tag = f"fullsize train forward {precision}"
    assert_close(m.seq2seq_output, y_ref, tol, f"{tag} y")
    assert_close(m.output, out_ref, tol, f"{tag} out")
    for k, v in Sref.items():
        if k in S and k not in ("mel", "stft"):
            assert_close(S[k].reshape(v.shape), v, tol, f"{tag} {k}")
    e = relerr(loss.reshape(1), loss_ref.reshape(1))[0]
    PARITY_LOG.append((f"{tag} loss", e, e, tol))
    assert e <= tol, (float(loss), float(loss_ref))
