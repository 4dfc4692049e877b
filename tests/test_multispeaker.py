"""Multi-speaker model (models/tacotron.py:116-124, models/ops.py:101-115) without a GPU: the oracle's speaker path
against the reference's own model code, the TF name map, the hand-written backward of the speaker path over the kernel
mirrors against torch.autograd, and the input pipeline's speaker ids."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import tacotron_oracle as O
from tacotron_b200 import params as PR
from tacotron_b200.models import grad
from tacotron_b200.models.tacotron import Config
from tacotron_b200.tf_names import tf_name_to_param
from tests import grad_util_spk, mirror_kernels_spk as MK, speaker_oracle as SO
from tests.emulator import emu  # noqa: F401  (the emulated library, built once per process)

HERE = os.path.dirname(os.path.abspath(__file__))
NSPK = 3


def _speakers(B, seed=4, n=NSPK):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, n, (B,), generator=g, dtype=torch.int32)


def _setup(r, sched, B=2, Tx=8, T=5, dtype=torch.float64):
    cfg = SO.SpkOracleConfig(r=r, vocab_size=20, num_speakers=NSPK)
    p = SO.init_params(cfg, seed=1, trained_like=True, dtype=dtype)
    inp = O.synthetic_inputs(cfg, B, Tx, T, seed=0, ragged=True)
    inp = {k: (v.to(dtype) if v.dtype.is_floating_point else v) for k, v in inp.items()}
    inp["speaker"] = _speakers(B)
    enc_m, dec_m = O.dropout_masks(cfg, B, Tx, T, seed=2)
    sm = O.sched_mask(cfg, B, T, seed=3) if sched else None
    return cfg, p, inp, enc_m, dec_m, sm


@pytest.mark.parametrize("r", [2, 5])
def test_oracle_matches_reference_wiring(r):
    z = np.load(os.path.join(HERE, "golden", f"reference_wiring_spk_r{r}.npz"))
    B, Tx, T = 2, 12, 6
    cfg = SO.SpkOracleConfig(r=r, max_decode_iter=T, vocab_size=20, num_speakers=NSPK)
    p = SO.init_params(cfg, seed=1, trained_like=True)
    inp = O.synthetic_inputs(cfg, B, Tx, T, seed=0, ragged=True)
    inp["speaker"] = torch.from_numpy(z["speaker"])
    enc_m, dec_m = O.dropout_masks(cfg, B, Tx, T, seed=2)
    sm = O.sched_mask(cfg, B, T, seed=3)
    for mode in ("infer", "teacher", "sched"):
        kw = {} if mode == "infer" else dict(enc_drop_masks=enc_m, dec_drop_masks=dec_m,
                                            sample_mask=sm if mode == "sched" else None)
        y, out, al = SO.inference(p, inp, cfg, train=mode != "infer", **kw)
        np.testing.assert_allclose(y.numpy(), z[f"y_{mode}"], rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(out.numpy(), z[f"out_{mode}"], rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(al.numpy(), z[f"align_{mode}"], rtol=1e-4, atol=1e-6)


def test_speaker_changes_the_output():
    """the fixture is not degenerate: another speaker id gives another output"""
    cfg, p, inp, _, _, _ = _setup(2, False, dtype=torch.float32)
    y0, _, _ = SO.inference(p, inp, cfg, train=False, T=3)
    inp["speaker"] = (inp["speaker"] + 1) % NSPK
    y1, _, _ = SO.inference(p, inp, cfg, train=False, T=3)
    assert (y0 - y1).abs().max() > 1e-4


@pytest.mark.parametrize("r", [2, 5])
def test_tf_names_map_one_to_one(r):
    z = np.load(os.path.join(HERE, "golden", f"reference_wiring_spk_r{r}.npz"))
    names = [str(n) for n in z["tf_variable_names"]]
    cfg = Config(r=r, vocab_size=20, num_speakers=NSPK)
    shapes = {n: s for n, s, _ in PR.model_shapes(cfg)}
    mapped = [tf_name_to_param(n, multi_speaker=True) for n in names]
    assert len(set(mapped)) == len(mapped) and set(mapped) == set(shapes)


@pytest.mark.parametrize("r", [2, 5])
def test_single_speaker_map_unchanged(r):
    z = np.load(os.path.join(HERE, "golden", f"reference_wiring_r{r}.npz"))
    for n in z["tf_variable_names"]:
        assert tf_name_to_param(str(n)) == tf_name_to_param(str(n), multi_speaker=False)
    shapes = PR.model_shapes(Config(r=r, vocab_size=20))
    assert not any(n.startswith("speaker/") or "/Ws" in n for n, _, _ in shapes)


def test_param_shapes_match_oracle():
    cfg = Config(r=2, vocab_size=20, num_speakers=NSPK)
    mine = {n: tuple(s) for n, s, _ in PR.model_shapes(cfg)}
    theirs = {n: tuple(s) for n, s, _ in SO.param_shapes(SO.SpkOracleConfig(r=2, vocab_size=20, num_speakers=NSPK))}
    assert mine == theirs
    single = [n for n, _, _ in PR.model_shapes(Config(r=2, vocab_size=20))]
    assert [n for n, _, _ in PR.model_shapes(cfg)][:len(single)] == single


@pytest.mark.parametrize("r,sched", [(2, True), (5, False)])
def test_saving_forward_matches_oracle(r, sched):
    cfg, p, inp, enc_m, dec_m, sm = _setup(r, sched)
    S, y, out = grad_util_spk.saving_forward_spk(p, inp, cfg, enc_m, dec_m, sm)
    y0, out0, _ = SO.inference(p, inp, cfg, train=True, enc_drop_masks=enc_m, dec_drop_masks=dec_m, sample_mask=sm)
    assert torch.allclose(y, y0, atol=1e-12) and torch.allclose(out, out0, atol=1e-11)


@pytest.mark.parametrize("r,sched", [(2, True), (5, False)])
def test_backward_matches_autograd(r, sched):
    cfg, p, inp, enc_m, dec_m, sm = _setup(r, sched)
    loss, g_ref = SO.loss_and_grads(p, inp, cfg, enc_drop_masks=enc_m, dec_drop_masks=dec_m, sample_mask=sm)
    S, y, out = grad_util_spk.saving_forward_spk(p, inp, cfg, enc_m, dec_m, sm)
    G = {k: torch.zeros_like(v) for k, v in p.items()}
    grad.model_bwd(MK, p, G, S, cfg)
    spk_names = [n for n, _, _ in SO.speaker_param_shapes(cfg)]
    assert set(spk_names) <= set(g_ref)
    for k, g in g_ref.items():
        err = (G[k] - g).abs().max().item()
        ref = g.abs().max().item()
        assert err <= 1e-8 * (1.0 + ref), f"{k}: max err {err:.3e} (ref max {ref:.3e})"
    for k in spk_names:                                      # the speaker path is exercised, not trivially zero
        if k == "speaker/embed" or k.endswith("/Ws") or k.endswith("/Wd"):
            assert G[k].abs().max().item() > 0, k


def test_colsum_seg_and_bigru_mirrors():
    g = torch.Generator().manual_seed(5)
    A = torch.randn(12, 7, generator=g, dtype=torch.float64)
    out = torch.ones(3, 7, dtype=torch.float64)
    MK.colsum_seg(out, A, 4)
    assert torch.allclose(out, 1 + A.view(3, 4, 7).sum(1))
    # bigru_fwd_h0 with h0 = None is the zero-state GRU of the oracle; with h0 it matches the oracle's initial-state GRU
    B, T = 2, 5
    W = [torch.randn(256, 256, generator=g, dtype=torch.float64) * 0.1 for _ in range(2)]
    Wc = [torch.randn(256, 128, generator=g, dtype=torch.float64) * 0.1 for _ in range(2)]
    bg = [torch.randn(256, generator=g, dtype=torch.float64) for _ in range(2)]
    bc = [torch.randn(128, generator=g, dtype=torch.float64) for _ in range(2)]
    x = torch.randn(B, T, 128, generator=g, dtype=torch.float64)
    h0 = torch.randn(B, 128, generator=g, dtype=torch.float64)
    xp = x @ torch.cat([W[0][:128], Wc[0][:128], W[1][:128], Wc[1][:128]], 1) + torch.cat([bg[0], bc[0], bg[1], bc[1]])
    fw, bw = (W[0], bg[0], Wc[0], bc[0]), (W[1], bg[1], Wc[1], bc[1])
    for hh in (None, h0):
        out = torch.empty(B, T, 256, dtype=torch.float64)
        MK.bigru_fwd_h0(out, xp, W[0][128:], Wc[0][128:], W[1][128:], Wc[1][128:], hh, hh)
        ref = SO.bidirectional_gru_h0(x, fw, bw, hh if hh is not None else torch.zeros(B, 128, dtype=torch.float64))
        assert torch.allclose(out, ref, atol=1e-12)


def test_device_batches_stage_speaker_ids():
    from tacotron_b200 import data_input as DI
    N, Tx, T = 10, 6, 4
    rng = np.random.RandomState(0)
    spk = rng.randint(0, 5, size=N).astype(np.int64)
    arrays = {"text": rng.randint(1, 20, size=(N, Tx)).astype(np.int32), "text_length": np.full(N, Tx, np.int32),
              "speech_length": np.full(N, T, np.int32), "stft": rng.randn(N, T, 1025 * 2).astype(np.float16),
              "mel": rng.randn(N, T, 80 * 2).astype(np.float16), "speaker": spk,
              "_stats": {k: v for k, v in (("stft_mean", np.zeros(2050, np.float16)), ("stft_std", np.ones(2050, np.float32)),
                                           ("mel_mean", np.zeros(160, np.float16)), ("mel_std", np.ones(160, np.float32)))}}
    it = DI.DeviceBatches(arrays, batch_size=4, buffer_size=8, seed=1, device="cpu", K=MK)
    for _ in range(3):
        b = next(it)
        assert b["speaker"].dtype == torch.int32 and b["speaker"].shape == (4,)
        # the ids travel with their utterances: text rows identify the utterance
        for i in range(4):
            row = b["text"][i].numpy()
            idx = [j for j in range(N) if np.array_equal(arrays["text"][j], row)]
            assert int(b["speaker"][i]) in {int(spk[j]) for j in idx}
    it.pending.join()


# ---- the new CUDA paths under the host emulation (tests/cuda_emu/emu.h): index algebra without a GPU ----
def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _gru_weights(g):
    return [torch.randn(128, 256, generator=g) * 0.1, torch.randn(128, 128, generator=g) * 0.1,
            torch.randn(128, 256, generator=g) * 0.1, torch.randn(128, 128, generator=g) * 0.1]


def test_bigru_fwd_h0_under_emulation(emu):
    g = torch.Generator().manual_seed(6)
    B, T = 2, 5
    xp = torch.randn(B, T, 768, generator=g)
    W = _gru_weights(g)
    h0f, h0b = torch.randn(B, 128, generator=g), torch.randn(B, 128, generator=g)
    for hf, hb in ((h0f, h0b), (None, None)):
        ref = torch.zeros(B, T, 256)
        MK.bigru_fwd_h0(ref, xp, *W, hf, hb)
        got = torch.full((B, T, 256), float("nan"))
        assert emu.taco_bigru_fwd_h0(_p(xp), *[_p(w) for w in W], _p(hf), _p(hb), _p(got), B, T, None) == 0
        assert (torch.nan_to_num(got, nan=1e30) - ref).abs().max().item() <= 2e-5
    plain = torch.full((B, T, 256), float("nan"))
    assert emu.taco_bigru_fwd(_p(xp), *[_p(w) for w in W], _p(plain), B, T, None) == 0
    assert torch.equal(plain, got)                          # NULL initial states = the zero-state entry point


def test_bigru_bwd_h0_under_emulation(emu):
    g = torch.Generator().manual_seed(7)
    B, T = 2, 4
    out = torch.tanh(torch.randn(B, T, 256, generator=g))
    ACT = torch.rand(B, T, 768, generator=g)
    ACT[:, :, 256:384] = ACT[:, :, 256:384] * 2 - 1
    ACT[:, :, 640:768] = ACT[:, :, 640:768] * 2 - 1
    dOut = torch.randn(B, T, 256, generator=g)
    W = _gru_weights(g)
    h0f, h0b = torch.randn(B, 128, generator=g), torch.randn(B, 128, generator=g)
    ref, dref = torch.zeros(B, T, 768), torch.zeros(B, 2, 128)
    MK.bigru_bwd_h0(ref, dOut, out, ACT, *W, h0f, h0b, dref)
    got, dgot = torch.full((B, T, 768), float("nan")), torch.full((B, 2, 128), float("nan"))
    assert emu.taco_bigru_bwd_h0(_p(got), _p(dOut), _p(out), _p(ACT), *[_p(w) for w in W], _p(h0f), _p(h0b), _p(dgot), B, T, None) == 0
    assert (torch.nan_to_num(got, nan=1e30) - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()
    assert (torch.nan_to_num(dgot, nan=1e30) - dref).abs().max().item() <= 2e-5 * dref.abs().max().item()
    dz = torch.full((B, 2, 128), float("nan"))                # T = 0: the initial state does not reach the loss
    assert emu.taco_bigru_bwd_h0(_p(got), _p(dOut), _p(out), _p(ACT), *[_p(w) for w in W], _p(h0f), _p(h0b), _p(dz), B, 0, None) == 0
    assert torch.equal(dz, torch.zeros(B, 2, 128))


def test_colsum_seg_under_emulation(emu):
    g = torch.Generator().manual_seed(8)
    M, N, period = 3 * 37, 45, 37
    A = torch.randn(M, 2 * N, generator=g)[:, 3:3 + N]         # strided rows
    out = torch.randn(3, 64, generator=g)
    ref = out.clone()
    MK.colsum_seg(ref[:, :N], A, period)
    assert emu.taco_colsum_seg(_p(out), 64, _p(A), A.stride(0), M, N, period, None) == 0
    assert torch.allclose(out, ref, atol=1e-5)
    assert emu.taco_colsum_seg(_p(out), 64, _p(A), A.stride(0), M, N, 36, None) != 0    # M % period != 0 is rejected
