"""Speaker-conditioned decoder (Config.speaker_decoder) without a GPU: the float64 oracle against the encoder-only model and
the step-0 formulas, parameter shapes and TF names, the hand-written backward over the kernel mirrors against
torch.autograd, the backward kernel's initial-state path under the host emulation, and checkpoints."""
import copy
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import tacotron_oracle as O
from oracle import tf12
from tacotron_b200 import _lib as L
from tacotron_b200 import params as PR
from tacotron_b200.models import grad
from tacotron_b200.models.tacotron import Config
from tacotron_b200.tf_names import tf_name_to_param
from tests import mirror_kernels_spkdec as MK, speaker_decoder_oracle as SD, speaker_oracle as SO
from tests.emulator import emu  # noqa: F401  (the emulated library, built once per process)

HERE = os.path.dirname(os.path.abspath(__file__))
NSPK = 3
NEW_TF_NAMES = ["decoder/dense/kernel", "decoder/dense/bias"] + [
    f"decoder/speaker_state_{i}/dense/{k}" for i in (1, 2, 3) for k in ("kernel", "bias")]


def _setup(r, sched, B=2, Tx=8, T=5, dtype=torch.float64, zero=False):
    cfg = SD.SpkDecOracleConfig(r=r, vocab_size=20, num_speakers=NSPK)
    p = SD.init_params(cfg, seed=1, trained_like=True, dtype=dtype, zero=zero)
    inp = O.synthetic_inputs(cfg, B, Tx, T, seed=0, ragged=True)
    inp = {k: (v.to(dtype) if v.dtype.is_floating_point else v) for k, v in inp.items()}
    inp["speaker"] = torch.tensor([0, 2, 1, 2][:B], dtype=torch.int32)
    enc_m, dec_m = O.dropout_masks(cfg, B, Tx, T, seed=2)
    sm = O.sched_mask(cfg, B, T, seed=3) if sched else None
    return cfg, p, inp, enc_m, dec_m, sm


@pytest.mark.parametrize("mode", ["infer", "teacher", "sched"])
def test_zero_decoder_speaker_params_give_the_encoder_only_model(mode):
    cfg, p, inp, enc_m, dec_m, sm = _setup(2, mode == "sched", zero=True)
    kw = {} if mode == "infer" else dict(enc_drop_masks=enc_m, dec_drop_masks=dec_m, sample_mask=sm)
    got = SD.inference(p, inp, cfg, train=mode != "infer", T=5, **kw)
    ref = SO.inference(p, inp, cfg, train=mode != "infer", T=5, **kw)
    for a, b in zip(got, ref):
        assert torch.equal(a, b)


def test_step0_follows_the_formulas():
    cfg, p, inp, enc_m, dec_m, _ = _setup(5, False)
    tr = {}
    SD.inference(p, inp, cfg, train=True, enc_drop_masks=enc_m, dec_drop_masks=dec_m, trace=tr)
    e = p["speaker/embed"][inp["speaker"].to(torch.int64)]
    att0 = e @ p["dec/spk/attn/W"] + p["dec/spk/attn/b"]
    h0 = [torch.relu(e @ p[f"dec/spk/h{i}/W"] + p[f"dec/spk/h{i}/b"]) for i in (1, 2, 3)]
    pn = O.pre_net(inp["mel"][:, 0, 4 * 80:], p, "dec/prenet", cfg.audio_dropout_prob, (dec_m[0][0], dec_m[1][0]))
    z0 = torch.cat([pn, att0], -1) @ p["dec/in_proj/W"] + p["dec/in_proj/b"]
    assert torch.allclose(tr["dec/z0"], z0, rtol=0, atol=1e-13)
    x = z0
    for i in range(3):
        h = tf12.gru_cell(x, h0[i], p[f"dec/gru{i+1}/Wg"], p[f"dec/gru{i+1}/bg"], p[f"dec/gru{i+1}/Wc"], p[f"dec/gru{i+1}/bc"])
        assert torch.allclose(tr["dec/H"][i, 0], h, rtol=0, atol=1e-13)
        x = h
    assert (att0.abs().max() > 0.1) and min(float(h.abs().max()) for h in h0) > 0.1      # the initial state is not trivial
    # and it reaches the output: another speaker gives another output
    y0, _, _ = SD.inference(p, inp, cfg, train=False, T=3)
    inp["speaker"] = (inp["speaker"] + 1) % NSPK
    y1, _, _ = SD.inference(p, inp, cfg, train=False, T=3)
    assert (y0 - y1).abs().max() > 1e-4


def test_param_shapes_match_oracle_and_old_lists_are_unchanged():
    cfg = Config(r=2, vocab_size=20, num_speakers=NSPK, speaker_decoder=True)
    mine = {n: tuple(s) for n, s, _ in PR.model_shapes(cfg)}
    theirs = {n: tuple(s) for n, s, _ in SD.param_shapes(SD.SpkDecOracleConfig(r=2, vocab_size=20, num_speakers=NSPK))}
    assert mine == theirs
    enc_only = [x for x in PR.model_shapes(Config(r=2, vocab_size=20, num_speakers=NSPK))]
    assert PR.model_shapes(cfg)[:len(enc_only)] == enc_only
    assert [n for n, _, _ in PR.model_shapes(cfg)[len(enc_only):]] == [n for n, _, _ in SD.decoder_speaker_param_shapes(cfg)]
    assert not any(n.startswith("dec/spk/") for n, _, _ in enc_only)
    assert not any(n.startswith("dec/spk/") or n.startswith("speaker/") for n, _, _ in PR.model_shapes(Config(r=2, vocab_size=20)))
    with pytest.raises(ValueError, match="speaker_decoder"):
        PR.model_shapes(Config(r=2, vocab_size=20, speaker_decoder=True))


@pytest.mark.parametrize("r", [2, 5])
def test_tf_names_map_one_to_one(r):
    z = np.load(os.path.join(HERE, "golden", f"reference_wiring_spk_r{r}.npz"))
    names = [str(n) for n in z["tf_variable_names"]] + NEW_TF_NAMES
    shapes = {n for n, _, _ in PR.model_shapes(Config(r=r, vocab_size=20, num_speakers=NSPK, speaker_decoder=True))}
    mapped = [tf_name_to_param(n, multi_speaker=True, speaker_decoder=True) for n in names]
    assert len(set(mapped)) == len(mapped) and set(mapped) == shapes
    assert tf_name_to_param("decoder/dense/kernel", multi_speaker=True, speaker_decoder=True) == "dec/spk/attn/W"
    assert tf_name_to_param("decoder/speaker_state_2/dense/bias", multi_speaker=True, speaker_decoder=True) == "dec/spk/h2/b"
    # the encoder-only and single-speaker maps do not know the new names and are otherwise the same
    for n in NEW_TF_NAMES:
        with pytest.raises(KeyError):
            tf_name_to_param(n, multi_speaker=True)
    for n in z["tf_variable_names"]:
        assert tf_name_to_param(str(n), multi_speaker=True) == tf_name_to_param(str(n), multi_speaker=True, speaker_decoder=True)
    z1 = np.load(os.path.join(HERE, "golden", f"reference_wiring_r{r}.npz"))
    for n in z1["tf_variable_names"]:
        assert tf_name_to_param(str(n)) == tf_name_to_param(str(n), speaker_decoder=True)


@pytest.mark.parametrize("r,sched", [(2, False), (2, True), (5, False), (5, True)])
def test_saving_forward_matches_oracle(r, sched):
    cfg, p, inp, enc_m, dec_m, sm = _setup(r, sched)
    S, y, out = SD.saving_forward(p, inp, cfg, enc_m, dec_m, sm)
    y0, out0, _ = SD.inference(p, inp, cfg, train=True, enc_drop_masks=enc_m, dec_drop_masks=dec_m, sample_mask=sm)
    assert torch.allclose(y, y0, atol=1e-12) and torch.allclose(out, out0, atol=1e-11)   # (the encoder re-associates)


@pytest.mark.parametrize("r,sched", [(2, False), (2, True), (5, False), (5, True)])
def test_backward_matches_autograd(r, sched):
    cfg, p, inp, enc_m, dec_m, sm = _setup(r, sched)
    loss, g_ref = SD.loss_and_grads(p, inp, cfg, enc_drop_masks=enc_m, dec_drop_masks=dec_m, sample_mask=sm)
    S, y, out = SD.saving_forward(p, inp, cfg, enc_m, dec_m, sm)
    G = {k: torch.zeros_like(v) for k, v in p.items()}
    grad.model_bwd(MK, p, G, S, cfg)
    assert set(g_ref) == {n for n, _, _ in SD.param_shapes(cfg) if not n.endswith(O.NON_TRAINABLE_SUFFIXES)}
    for k, g in g_ref.items():
        err = (G[k] - g).abs().max().item()
        ref = g.abs().max().item()
        assert err <= 1e-8 * (1.0 + ref), f"{k}: max err {err:.3e} (ref max {ref:.3e})"
    for k, _, _ in SD.decoder_speaker_param_shapes(cfg):       # the new path is exercised, not trivially zero
        assert G[k].abs().max().item() > 0, k
    assert G["speaker/embed"].abs().max().item() > 0


# ---- the backward kernel's initial-state path under the host emulation (tests/cuda_emu/emu.h) ----
@pytest.mark.parametrize("r,sched", [(2, True), (5, False)])
def test_decoder_bwd_kernel_with_h0_under_emulation(emu, r, sched):
    B, Tx, T = 2, 8, 4
    cfg, p, inp, enc_m, dec_m, sm = _setup(r, sched, B=B, Tx=Tx, T=T, dtype=torch.float32)
    S, _, _ = SD.saving_forward(p, inp, cfg, enc_m, dec_m, sm)
    S["_capture"] = {}
    G = {k: torch.zeros_like(v) for k, v in p.items()}
    dY = torch.randn(B, T, 80 * r, generator=torch.Generator().manual_seed(5))
    grad.decoder_bwd(MK, p, G, S, cfg, dY)
    a = S["_capture"]["decoder_bwd"]                           # inputs + the mirror's outputs, DH0 included
    assert a["DH0"].abs().max().item() > 0
    outs = ("DATT", "DY", "DPQ", "DSCORE", "DCTX", "DZ", "DPN2", "DPN1", "DX", "DH0")
    e = {k: copy.deepcopy(v) for k, v in a.items() if not k.startswith("_")}
    for k in outs:
        e[k].fill_(float("nan"))
    for i in range(3):
        e["DG"][i].fill_(float("nan")); e["DC"][i].fill_(float("nan"))
    d = L.DecoderBwdArgs()
    d.B, d.T, d.Tx, d.r, d.keep_scale = B, T, Tx, r, float(a["keep_scale"])
    for k in ("W_a", "W_q", "W_out", "W_in", "W1", "W2", "v", "dy_ext", "align", "values", "keys", "PQ", "PN1", "PN2", "sel", *outs):
        e[k] = e[k].contiguous()
        setattr(d, k, e[k].data_ptr())
    for k in ("Wg", "Wc", "RU", "C", "H", "DG", "DC", "H0"):
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
    # without H0 the kernel is today's: its step-0 outputs differ from the initial-state run
    e2 = {k: v.clone() for k, v in e.items() if torch.is_tensor(v)}
    d.H0[0] = d.H0[1] = d.H0[2] = None
    d.DH0 = None
    for k in ("DZ",):
        setattr(d, k, e2[k].data_ptr())
    assert emu.taco_decoder_bwd(C.byref(d), None) == 0, emu.taco_last_error().decode()
    assert not torch.allclose(e2["DZ"][0], e["DZ"][0])


# ---- checkpoints ----
class _Model:
    def __init__(self, cfg):
        self.config = cfg
        self.store = PR.ParamStore(PR.model_shapes(cfg), "cpu")
        self.store.init_tf_default(3)
        self.global_step = 7

    def load_params(self, p):
        self.store.load(p)

    def add_train_op(self):
        pass


def test_checkpoint_round_trip_and_mismatch(tmp_path):
    from tacotron_b200 import checkpoint
    on = Config(r=2, vocab_size=20, num_speakers=NSPK, speaker_decoder=True)
    off = Config(r=2, vocab_size=20, num_speakers=NSPK)
    m = _Model(on)
    fn = checkpoint.save(m, str(tmp_path / "spk" / "tacotron"))
    assert checkpoint.speaker_decoder(fn) and checkpoint.num_speakers(fn) == NSPK
    m2 = _Model(Config(r=2, vocab_size=20, num_speakers=NSPK, speaker_decoder=True))
    m2.store.flat.zero_()
    checkpoint.restore(m2, fn)
    assert torch.equal(m2.store.flat, m.store.flat) and m2.global_step == 7
    with pytest.raises(ValueError, match="dec/spk/attn/W"):           # extra variables
        checkpoint.restore(_Model(off), fn)
    fn_off = checkpoint.save(_Model(off), str(tmp_path / "enc" / "tacotron"))
    assert not checkpoint.speaker_decoder(fn_off)
    with pytest.raises(ValueError, match="missing variables.*dec/spk/h1/W"):
        checkpoint.restore(_Model(on), fn_off)
    # TF-named import: the decoder's speaker denses travel under their TF names
    from tacotron_b200 import tf_names
    z = np.load(os.path.join(HERE, "golden", "reference_wiring_spk_r2.npz"))
    tf_vars = {}
    for n in [str(x) for x in z["tf_variable_names"]] + NEW_TF_NAMES:
        tf_vars[n] = m.store[tf_names.tf_name_to_param(n, multi_speaker=True, speaker_decoder=True)].numpy()
    m3 = _Model(on)
    m3.store.flat.zero_()
    checkpoint.import_tf_variables(m3, tf_vars)
    assert torch.equal(m3.store.flat, m.store.flat)
    with pytest.raises(ValueError, match="dec/spk/"):
        checkpoint.import_tf_variables(_Model(off), tf_vars)
