"""Host-logic pin of the hand-written backward (tacotron_b200/models/grad.py): run it over the torch-CPU mirror
of the training kernels (tests/mirror_kernels.py) and compare every parameter gradient with torch.autograd over
the oracle (oracle.tacotron_oracle.loss_and_grads).  fp64, so the comparison is tight."""
import pytest
import torch

from oracle import tacotron_oracle as O
from tacotron_b200.models import grad
from tests import grad_util, mirror_kernels as MK


def _setup(r, sched, B=2, Tx=8, T=5, seed=0, dtype=torch.float64, ragged=True):
    cfg = O.OracleConfig(r=r, vocab_size=20)
    p = O.init_params(cfg, seed=1, trained_like=True, dtype=dtype)
    inp = O.synthetic_inputs(cfg, B, Tx, T, seed=seed, ragged=ragged)
    inp = {k: (v.to(dtype) if v.dtype.is_floating_point else v) for k, v in inp.items()}
    enc_m, dec_m = O.dropout_masks(cfg, B, Tx, T, seed=2)
    sm = O.sched_mask(cfg, B, T, seed=3) if sched else None
    return cfg, p, inp, enc_m, dec_m, sm


@pytest.mark.parametrize("r,sched", [(2, True), (5, False), (5, True)])
def test_saving_forward_matches_oracle(r, sched):
    cfg, p, inp, enc_m, dec_m, sm = _setup(r, sched)
    S, y, out = grad_util.saving_forward(p, inp, cfg, enc_m, dec_m, sm)
    y0, out0, al0 = O.inference(p, inp, cfg, train=True, enc_drop_masks=enc_m, dec_drop_masks=dec_m, sample_mask=sm)
    assert torch.allclose(y, y0, atol=1e-12) and torch.allclose(out, out0, atol=1e-11)
    assert torch.allclose(S["dec/align"], al0, atol=1e-12)


@pytest.mark.parametrize("r,sched", [(2, True), (5, False), (5, True)])
def test_backward_matches_autograd(r, sched):
    _check_backward_against_autograd(*_setup(r, sched))


def test_backward_matches_autograd_batch_sized():
    """a batch of 32 ragged utterances, Tx = 67 (not a multiple of 4, 8 or 32), T = 64, scheduled sampling: the float64
    mirror backward is the reference of tests/test_gpu_train_fullsize.py, so it is pinned here beyond the toy shape"""
    _check_backward_against_autograd(*_setup(5, True, B=32, Tx=67, T=64))


def _check_backward_against_autograd(cfg, p, inp, enc_m, dec_m, sm):
    loss, g_ref = O.loss_and_grads(p, inp, cfg, enc_drop_masks=enc_m, dec_drop_masks=dec_m, sample_mask=sm)
    S, y, out = grad_util.saving_forward(p, inp, cfg, enc_m, dec_m, sm)
    G = {k: torch.zeros_like(v) for k, v in p.items()}
    grad.model_bwd(MK, p, G, S, cfg)
    worst = 0.0
    for k, g in g_ref.items():
        err = (G[k] - g).abs().max().item()
        ref = g.abs().max().item()
        worst = max(worst, err / (ref + 1e-9))
        assert err <= 1e-8 * (1.0 + ref), f"{k}: max err {err:.3e} (ref max {ref:.3e})"
    for k in p:
        if k.endswith(("bn_mean", "bn_var")):
            assert G[k].abs().max().item() == 0.0


def test_recomputed_gates_reproduce_saved_states():
    """decoder_recompute's batched gates must regenerate the saved GRU state sequences: h = u*hprev + (1-u)*c."""
    cfg, p, inp, enc_m, dec_m, sm = _setup(2, True)
    S, y, out = grad_util.saving_forward(p, inp, cfg, enc_m, dec_m, sm)
    R = grad.decoder_recompute(MK, p, S, cfg)
    T, B = R["T"], R["B"]
    for i in range(3):
        Hi = R["H"][i]
        hprev = MK._shift_rows(Hi, -B, 0)
        u = R["RU"][i][:, 256:]
        assert torch.allclose(u * hprev + (1 - u) * R["C"][i], Hi, atol=1e-12)


def test_adam_and_clip_match_oracle():
    cfg, p, inp, enc_m, dec_m, sm = _setup(2, True)
    kw = dict(enc_drop_masks=enc_m, dec_drop_masks=dec_m, sample_mask=sm)
    p_ref = {k: v.clone() for k, v in p.items()}
    m_ref = {k: torch.zeros_like(v) for k, v in p.items()}
    v_ref = {k: torch.zeros_like(v) for k, v in p.items()}
    _, gn_ref = O.train_step(p_ref, m_ref, v_ref, inp, cfg, lr=1e-3, step=1, **kw)
    # ours: flat buffers
    names = list(p)
    sizes = [p[k].numel() for k in names]
    flat = torch.cat([p[k].reshape(-1) for k in names]).clone()
    views = dict(zip(names, [t.view(p[k].shape) for t, k in zip(flat.split(sizes), names)]))
    gflat = torch.zeros_like(flat)
    G = dict(zip(names, [t.view(p[k].shape) for t, k in zip(gflat.split(sizes), names)]))
    S, _, _ = grad_util.saving_forward(views, inp, cfg, enc_m, dec_m, sm)
    grad.model_bwd(MK, views, G, S, cfg)
    ss = torch.zeros(1, dtype=flat.dtype)
    MK.sumsq(ss, gflat)
    assert abs(ss.sqrt().item() - float(gn_ref)) <= 1e-9 * float(gn_ref)
    m = torch.zeros_like(flat); v = torch.zeros_like(flat)
    import math
    lr_t = 1e-3 * math.sqrt(1 - 0.999) / (1 - 0.9)
    MK.adam_step(flat, gflat, m, v, lr_t, 0.9, 0.999, 1e-8, float(cfg.cap_grads), ss)
    for k in names:
        if k.endswith(("bn_mean", "bn_var")):
            assert torch.equal(views[k], p[k])
        else:
            assert torch.allclose(views[k], p_ref[k], atol=1e-10), k
