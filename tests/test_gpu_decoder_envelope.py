"""-m gpu: the persistent decoder kernels (taco_decoder_fwd, taco_decoder_bwd) across the shape range their ABI accepts:
Tx in [1, 256], any r with 80r <= 512 (r = 1..6), B up to 32 per launch.

Where the kernels change behaviour with the shape:
  * r: the output projection is split into NCY = ceil(80r / 32) column slices, so for r = 1 and r = 3 whole slices of the
    last stage have no columns;
  * Tx: as Tx grows the forward kernel's keys / values take more shared memory and weight segments move to L2 (read from
    the packed buffer instead).  Every residency set of decoder.cu's host logic is run once: Tx = 1-128 (none),
    129-144 (P2), 145-160 (Y), 161-176 (Y, P2), 177-192 (QP, Y), 193-208 (QP, Y, P2), 209-224 (C_RH2, QP, Y, P2),
    225-240 (G_X2, QP, Y, P2), 241-256 (G_X2, C_RH2, QP, Y, P2); from Tx = 209 an on-chain GRU stage reads its weights
    from L2;
  * text_length: the attention runs in four quarters of ceil(Tx/4) positions; a quarter past text_length is fully
    masked (its max is -inf), which random lengths in [Tx/2, Tx] never produce;
  * the backward kernel's attention loops have tails for Tx % 8 != 0 and Tx % 32 != 0.

References are float64: inputs and weights are drawn once in fp32, the GPU gets those values and the reference their
exact float64 copies.  Bars: 1e-4 of the tensor's max magnitude (max and mean), the decoder bar for T <= 20; 2e-4 for
the backward kernel, its bar in test_gpu_train.py.
"""
import pytest
import torch

from oracle import tacotron_oracle as O
from tests import grad_util, mirror_kernels as MK
from tests.util import assert_close, make_model, ocfg, to_cuda

pytestmark = pytest.mark.gpu


def short_lengths(Tx, B):
    """text lengths {1, Tq, Tq+1, 2Tq, 3Tq+1, Tx} (Tq = ceil(Tx/4), clipped to Tx) over the batch: whole attention
    quarters masked, and lengths on either side of a quarter boundary"""
    Tq = (Tx + 3) // 4
    L = [min(v, Tx) for v in (1, Tq, Tq + 1, 2 * Tq, 3 * Tq + 1, Tx)]
    return torch.tensor([L[i % len(L)] for i in range(B)], dtype=torch.int32)


def _setup(r, B, Tx, T, lengths=None, seed=0):
    cfg = ocfg(r=r, T=T, vocab=20)
    p = O.init_params(cfg, seed=1, trained_like=True)
    encoded = torch.randn(B, Tx, 256, generator=torch.Generator().manual_seed(seed)) * 0.5
    inp = O.synthetic_inputs(cfg, B, Tx, T, seed=seed, ragged=True)
    tl = inp["text_length"] if lengths is None else lengths
    _, dec_m = O.dropout_masks(cfg, B, Tx, T, seed=2)
    sm = O.sched_mask(cfg, B, T, seed=3)
    return cfg, p, encoded, inp["mel"], tl, dec_m, sm


def _run_forward(r, B, Tx, T, mode, lengths=None, seed=0):
    """taco_decoder_fwd through ops.attention_decoder, and O.decoder in float64 on the same values"""
    from tacotron_b200 import Config, _lib as L
    from tacotron_b200.models import ops
    from tacotron_b200.params import ParamStore, model_shapes
    cfg, p, encoded, mel, tl, dec_m, sm = _setup(r, B, Tx, T, lengths, seed)
    drop = None if mode == "infer" else dec_m
    smask = sm if mode == "sched" else None
    y_ref, a_ref = O.decoder(encoded.double(), tl, {k: v.double() for k, v in p.items()}, cfg, mode, T, mel=mel.double(),
                             drop_masks=drop, sample_mask=smask)
    st = ParamStore(model_shapes(Config(r=r, vocab_size=20)), "cuda")
    st.load(p)
    ops.runtime(st, "fp32")
    lmode = {"infer": L.DEC_INFER, "teacher": L.DEC_TEACHER, "sched": L.DEC_SCHED}[mode]
    y, a = ops.attention_decoder(encoded.cuda(), tl.cuda(), r, T, mode=lmode, mel=None if mode == "infer" else mel.cuda(),
                                 sample_mask=None if smask is None else smask.cuda(),
                                 drop_masks=None if drop is None else (drop[0].cuda(), drop[1].cuda()), scope=ops.Scope(st, "dec"))
    torch.cuda.synchronize()
    return y.clone(), a.clone(), y_ref, a_ref, tl


def _check_forward(y, a, y_ref, a_ref, tl, what):
    assert not torch.isnan(y).any() and not torch.isnan(a).any(), f"{what}: NaN in the output"
    assert_close(y, y_ref, 1e-4, f"{what} y")
    assert_close(a, a_ref, 1e-4, f"{what} align")
    a = a.cpu()
    s = a.sum(-1)
    assert torch.allclose(s, torch.ones_like(s), atol=1e-5), f"{what}: alignment rows do not sum to 1"
    past = torch.arange(a.shape[2])[None, None, :] >= tl[:, None, None].to(torch.int64)
    assert (a[past.expand_as(a)] == 0).all(), f"{what}: alignment weight at or past text_length"


# ---------------------------------------------------------------------------------------------------------------------
# forward: r, Tx (weight residency), B
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["infer", "teacher", "sched"])
@pytest.mark.parametrize("r", [1, 3, 4, 6])
def test_decoder_fwd_r(r, mode):
    y, a, y_ref, a_ref, tl = _run_forward(r, 9, 37, 7, mode)
    _check_forward(y, a, y_ref, a_ref, tl, f"decoder r={r} {mode}")


@pytest.mark.parametrize("r", [3, 6])
def test_inference_end_to_end_r(r):
    """Tacotron.inference in the default precision mode against the float64 oracle (bar of test_gpu_model.py)"""
    cfg = ocfg(r=r, T=7, vocab=20)
    p = O.init_params(cfg, seed=1, trained_like=True)
    inp = O.synthetic_inputs(cfg, 9, 37, 7, seed=0, ragged=True, with_targets=False)
    y_ref, out_ref, a_ref = O.inference({k: v.double() for k, v in p.items()}, inp, cfg, train=False)
    m = make_model(cfg, p, "fp32x3")
    y, out = m.inference(to_cuda(inp), train=False)
    torch.cuda.synchronize()
    assert y.shape == (9, 7, 80 * r) and out.shape == (9, 7, 1025 * r)
    assert_close(y, y_ref, 2e-4, f"e2e r={r} y")
    assert_close(m.alignments, a_ref, 2e-4, f"e2e r={r} align")
    assert_close(out, out_ref, 2e-4, f"e2e r={r} out")


@pytest.mark.parametrize("mode", ["infer", "teacher"])
@pytest.mark.parametrize("Tx", [150, 170, 185, 215, 230, 256])
def test_decoder_fwd_tx_residency(Tx, mode):
    y, a, y_ref, a_ref, tl = _run_forward(5, 32, Tx, 8, mode, lengths=short_lengths(Tx, 32))
    _check_forward(y, a, y_ref, a_ref, tl, f"decoder Tx={Tx} {mode}")


@pytest.mark.parametrize("mode", ["infer", "sched"])
@pytest.mark.parametrize("B", [8, 31])
def test_decoder_fwd_batch(B, mode):
    y, a, y_ref, a_ref, tl = _run_forward(5, B, 64, 7, mode)
    _check_forward(y, a, y_ref, a_ref, tl, f"decoder B={B} {mode}")


# ---------------------------------------------------------------------------------------------------------------------
# backward kernel
# ---------------------------------------------------------------------------------------------------------------------
DEC_OUTS = ("DATT", "DY", "DPQ", "DSCORE", "DCTX", "DZ", "DPN2", "DPN1", "DX")


def check_decoder_bwd(r, B, Tx, T, lengths=None, sched=True, seed=0):
    """taco_decoder_bwd against mirror_kernels.decoder_bwd in float64 on the same fp32 arguments.  The arguments are those
    grad.decoder_bwd builds from an fp32 decoder forward (grad_util.decoder_saving) with text lengths `lengths`."""
    from tacotron_b200 import kernels as K
    from tacotron_b200.models import grad
    cfg, p, encoded, mel, tl, dec_m, sm = _setup(r, B, Tx, T, lengths, seed)
    S = {"mel": mel, "text_length": tl, "dec/keep1": dec_m[0], "dec/keep2": dec_m[1], "_capture": {}}
    if sched:
        S["dec/sample_mask"] = sm
    grad_util.decoder_saving(encoded, tl, p, cfg, T, mel, dec_m, sm if sched else None, S)
    G = {k: torch.zeros_like(v) for k, v in p.items()}
    dY = torch.randn(B, T, 80 * r, generator=torch.Generator().manual_seed(5))
    grad.decoder_bwd(MK, p, G, S, cfg, dY)
    args = {k: v for k, v in S["_capture"]["decoder_bwd"].items() if not k.startswith("_")}
    ref = {k: ([t.double() for t in v] if isinstance(v, list) else v.double() if torch.is_tensor(v) and v.is_floating_point() else v)
           for k, v in args.items()}
    gpu = {k: ([t.cuda() for t in v] if isinstance(v, list) else v.cuda() if torch.is_tensor(v) else v) for k, v in args.items()}
    for t in [ref[k] for k in DEC_OUTS] + ref["DG"] + ref["DC"] + [gpu[k] for k in DEC_OUTS] + gpu["DG"] + gpu["DC"]:
        t.fill_(float("nan"))                                   # poisoned: a cell nobody writes shows up
    MK.decoder_bwd(ref)
    K.decoder_bwd(gpu)
    torch.cuda.synchronize()
    what = f"decoder_bwd r={r} B={B} Tx={Tx} T={T}"
    for k in DEC_OUTS:
        assert not torch.isnan(gpu[k]).any(), f"{what} {k}: cells left unwritten"
        assert_close(gpu[k], ref[k], 2e-4, f"{what} {k}")
    for i in range(3):
        assert not (torch.isnan(gpu["DG"][i]).any() or torch.isnan(gpu["DC"][i]).any()), f"{what} DG{i}/DC{i}: cells left unwritten"
        assert_close(gpu["DG"][i], ref["DG"][i], 2e-4, f"{what} DG{i}")
        assert_close(gpu["DC"][i], ref["DC"][i], 2e-4, f"{what} DC{i}")


@pytest.mark.parametrize("Tx,r,B,T,short", [
    (1, 1, 1, 1, False),
    (1, 6, 32, 200, False),
    (7, 3, 31, 200, True),          # Tx % 8 != 0, quarters of 2
    (7, 1, 32, 1, True),
    (67, 6, 31, 200, True),         # Tx % 32 != 0
    (67, 1, 1, 200, False),
    (129, 3, 32, 200, True),
    (129, 6, 1, 1, False),
    (256, 3, 32, 200, True),        # the largest width at the C2 batch and length
    (256, 1, 31, 200, True),
    (256, 6, 32, 1, False),
])
def test_decoder_bwd_envelope(Tx, r, B, T, short):
    check_decoder_bwd(r, B, Tx, T, lengths=short_lengths(Tx, B) if short else None)
