"""-m gpu: the attention window of free-running decoding (taco_decoder_args win_back / win_ahead / peak,
Config.attention_window, python -m tacotron_b200.test --attention-window) on the H100.

  1. a window that covers every position, and no window, give the default call's bits;
  2. the kernel is consistent with itself: alpha is exactly 0 outside the window built from its own p(t-1), p(t) lies in
     it and holds the row's largest weight, rows sum to 1 -- over r, the widths that hit every weight-residency set of the
     synthesis width, the batch, and ragged lengths that put windows across attention-quarter boundaries;
  3. against the float64 oracle forced with the kernel's peaks (1e-4 of the max magnitude, the decoder bar for T <= 20),
     and the oracle's own peak of every step equals the kernel's wherever its top two windowed scores are > 1e-4 apart;
  4. it constrains: a memory with one dominating key pulls the unwindowed attention there at once, the windowed one not;
  5. split launch plans and CUDA graphs give the same bits, and a changed window is never served from an old graph;
  6. a window in teacher-forced / scheduled-sampling mode, or with ahead = 0, is refused with nothing launched;
  7. Tacotron.inference against the float64 oracle, and the synthesis driver with --attention-window (plain, long-form)."""
import io
import os
import shutil

import numpy as np
import pytest
import torch

from oracle import tacotron_oracle as O
from tacotron_b200 import _lib as L
from tacotron_b200.models import ops
from tests import attention_window_oracle as AW
from tests.test_gpu_decoder_envelope import _setup, short_lengths
from tests.test_gpu_speaker_decoder import _dec_case
from tests.util import assert_close, make_model, ocfg, to_cuda

pytestmark = pytest.mark.gpu
WINDOWS = [(2, 5), (0, 3)]


def _store(p, r):
    from tacotron_b200 import Config
    from tacotron_b200.params import ParamStore, model_shapes
    st = ParamStore(model_shapes(Config(r=r, vocab_size=20)), "cuda")
    st.load(p)
    ops.runtime(st, "fp32")
    return st


def _dec(st, r, T, encoded, tl, window=None, max_ctas=None, h0=None, att0=None):
    """ops.attention_decoder in free-running mode -> (y, alpha, peaks or None), cloned"""
    res = ops.attention_decoder(encoded.float().cuda(), tl.cuda(), r, T, mode=L.DEC_INFER, scope=ops.Scope(st, "dec"),
                                max_ctas=max_ctas, window=window,
                                h0=None if h0 is None else h0.float().cuda().contiguous(),
                                att0=None if att0 is None else att0.float().cuda().contiguous())
    torch.cuda.synchronize()
    out = [x.clone() for x in res]
    return out[0], out[1], (out[2] if len(out) > 2 else None)


def check_window(a, pk, tl, window, what):
    """alpha [B,T,Tx] exactly 0 outside W_t built from pk(t-1) (p(-1) = 0), pk(t) in W_t, alpha[t, pk(t)] the row's
    largest weight up to 1e-6, rows summing to 1"""
    a, pk = a.cpu(), pk.cpu().to(torch.int64)
    B, T, Tx = a.shape
    back, ahead = window
    N = tl.to(torch.int64).clamp(max=Tx)
    prev = torch.zeros(B, dtype=torch.int64)
    for t in range(T):
        allowed = AW.window_mask(prev, N, Tx, back, ahead)
        assert (a[:, t][~allowed] == 0).all(), f"{what}: weight outside the window at step {t}"
        assert allowed.gather(1, pk[:, t:t + 1]).all(), f"{what}: peak outside the window at step {t}"
        at_p = a[:, t].gather(1, pk[:, t:t + 1])[:, 0]
        assert (at_p >= a[:, t].max(1).values * (1 - 1e-6)).all(), f"{what}: the peak is not the largest weight at step {t}"
        prev = pk[:, t]
    s = a.sum(-1)
    assert torch.allclose(s, torch.ones_like(s), atol=1e-5), f"{what}: alignment rows do not sum to 1"


# ---------------------------------------------------------------------------------------------------------------------
# 1. no window / a window covering everything: the default call's bits
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("state", [False, True])
def test_off_and_covering_windows_change_nothing(state):
    r, B, Tx, T = 5, 32, 128, 200                     # the C2 inference step
    cfg, p, encoded, inp, dec_m, sm, h0, att0, st = _dec_case(r, B, Tx, T)
    if not state:
        h0 = att0 = None
    tl = inp["text_length"]
    y0, a0, pk0 = _dec(st, r, T, encoded, tl, h0=h0, att0=att0)
    assert pk0 is None
    for window in (None, (Tx - 1, Tx - 1), (Tx, 10 ** 6), (2 ** 31 - 1, 2 ** 31 - 1)):
        y, a, pk = _dec(st, r, T, encoded, tl, window=window, h0=h0, att0=att0)
        assert torch.equal(y, y0) and torch.equal(a, a0), window
        if window is not None:
            check_window(a, pk, tl, window, f"covering window {window}")


# ---------------------------------------------------------------------------------------------------------------------
# 2. self-consistency
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("window", WINDOWS)
@pytest.mark.parametrize("B", [1, 9, 32])
@pytest.mark.parametrize("Tx", [37, 140, 256])
@pytest.mark.parametrize("r", [2, 5])
def test_window_self_consistency(r, Tx, B, window):
    T = 60
    lengths = short_lengths(Tx, B) if B > 1 else torch.tensor([Tx], dtype=torch.int32)
    cfg, p, encoded, mel, tl, dec_m, sm = _setup(r, B, Tx, T, lengths)
    st = _store(p, r)
    y, a, pk = _dec(st, r, T, encoded, tl, window=window)
    assert not torch.isnan(y).any() and not torch.isnan(a).any()
    check_window(a, pk, tl, window, f"r={r} Tx={Tx} B={B} window={window}")


# ---------------------------------------------------------------------------------------------------------------------
# 3. against float64
# ---------------------------------------------------------------------------------------------------------------------
def _against_oracle(r, B, Tx, T, window, lengths=None, state=False):
    if state:
        cfg, p, encoded, inp, dec_m, sm, h0, att0, st = _dec_case(r, B, Tx, T)
        tl = inp["text_length"]
    else:
        cfg, p, encoded, mel, tl, dec_m, sm = _setup(r, B, Tx, T, lengths)
        st, h0, att0 = _store(p, r), None, None
    y, a, pk = _dec(st, r, T, encoded, tl, window=window, h0=h0, att0=att0)
    pd = {k: v.double() for k, v in p.items()}
    tr = {}
    y_ref, a_ref, p_ref = AW.decoder(encoded.double(), tl, pd, cfg, T, window, peaks=pk.cpu(), trace=tr,
                                     h0=None if h0 is None else h0.double(), att0=None if att0 is None else att0.double())
    what = f"r={r} B={B} Tx={Tx} T={T} window={window}{' state' if state else ''}"
    assert_close(y, y_ref, 1e-4, f"{what} y")
    assert_close(a, a_ref, 1e-4, f"{what} align")
    gap = AW.top_two_gap(tr["score"])
    clear = gap > 1e-4
    pk = pk.cpu().to(torch.int64)
    assert torch.equal(pk[clear], p_ref[clear]), f"{what}: peaks differ at steps with a clear maximum"
    near = int((~clear).sum())
    print(f"{what}: {near} of {clear.numel()} steps near a tie (top-two windowed scores within 1e-4)")
    return near


@pytest.mark.parametrize("window", WINDOWS)
@pytest.mark.parametrize("r,B,Tx,T", [(2, 9, 37, 20), (5, 1, 140, 20), (2, 32, 256, 16)])
def test_matches_float64_oracle(r, B, Tx, T, window):
    _against_oracle(r, B, Tx, T, window, lengths=short_lengths(Tx, B) if B > 1 else None)


@pytest.mark.parametrize("state", [False, True])
def test_c2_free_running_matches_oracle(state):
    _against_oracle(5, 32, 128, 12, (2, 5), state=state)


# ---------------------------------------------------------------------------------------------------------------------
# 4. it constrains
# ---------------------------------------------------------------------------------------------------------------------
def test_window_keeps_attention_from_jumping_to_a_dominating_key():
    r, B, Tx, T, J = 2, 9, 64, 24, 40
    window = (2, 5)
    cfg, p, encoded, mel, tl, dec_m, sm = _setup(r, B, Tx, T, torch.full((B,), Tx, dtype=torch.int32))
    # memory row J whose key is 20 sign(v): tanh saturates to sign(v_d) on every unit, the largest score there is
    Wm, v = p["dec/attn/W_mem"].double(), p["dec/attn/v"].double()
    encoded = encoded.clone()
    encoded[:, J] = (torch.linalg.solve(Wm.t(), 20 * torch.sign(v))).float()
    st = _store(p, r)
    yu, au, _ = _dec(st, r, T, encoded, tl)
    yw, aw, pk = _dec(st, r, T, encoded, tl, window=window)
    assert (au[:, 0, J] > 0.5).all(), "the unwindowed attention should jump to the dominating key at step 0"
    check_window(aw, pk, tl, window, "dominating key")
    pk = pk.cpu().to(torch.int64)
    step = torch.diff(torch.cat([torch.zeros(B, 1, dtype=torch.int64), pk], 1), dim=1)
    assert (step <= window[1]).all() and (step >= -window[0]).all()
    reach = (torch.arange(T) + 1) * window[1]                 # furthest position step t can attend
    before = reach < J
    assert (aw.cpu()[:, before, J] == 0).all(), "windowed attention reached the key before the window could"
    assert (yw - yu).abs().max().item() > 1e-3


# ---------------------------------------------------------------------------------------------------------------------
# 5. launch plans and graphs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("max_ctas", [32, 64])
def test_split_launches_are_bit_identical(max_ctas):
    r, B, Tx, T = 2, 32, 140, 50
    cfg, p, encoded, mel, tl, dec_m, sm = _setup(r, B, Tx, T, short_lengths(Tx, B))
    st = _store(p, r)
    y, a, pk = _dec(st, r, T, encoded, tl, window=(2, 5))
    ys, as_, pks = _dec(st, r, T, encoded, tl, window=(2, 5), max_ctas=max_ctas)
    assert torch.equal(y, ys) and torch.equal(a, as_) and torch.equal(pk, pks)


def test_cuda_graph_equals_eager_and_follows_the_window():
    cfg_o = ocfg(r=2, T=30, vocab=20)
    p = O.init_params(cfg_o, seed=1, trained_like=True)
    inp = to_cuda(O.synthetic_inputs(cfg_o, 9, 37, 30, seed=0, ragged=True, with_targets=False))
    m = make_model(cfg_o, p, "fp32x3")
    eager = {}
    for w in ((2, 5), (0, 3), None):
        m.config.attention_window = w
        y, out = m.inference(inp, train=False)
        eager[w] = (y.clone(), out.clone(), m.alignments.clone(), None if w is None else m.attention_peaks.clone())
        assert (m.attention_peaks is None) == (w is None)
    assert not torch.equal(eager[(2, 5)][0], eager[(0, 3)][0])
    m.config.cuda_graph = True
    for w in ((2, 5), (0, 3), (2, 5), None, (0, 3)):              # each change of window is a graph of its own
        m.config.attention_window = w
        y, out = m.inference(inp, train=False)
        torch.cuda.synchronize()
        ey, eo, ea, ep = eager[w]
        assert torch.equal(y, ey) and torch.equal(out, eo) and torch.equal(m.alignments, ea), w
        assert (m.attention_peaks is None) if w is None else torch.equal(m.attention_peaks, ep), w


# ---------------------------------------------------------------------------------------------------------------------
# 6. errors
# ---------------------------------------------------------------------------------------------------------------------
def _raw_call(mode, back, ahead, peak=False):
    """taco_decoder_fwd on valid zero buffers (B = 2, Tx = 8, T = 3, r = 2) with the given window"""
    r, B, Tx, T = 2, 2, 8, 3
    cfg, p, *_ = _setup(r, B, Tx, T)
    st = _store(p, r)
    lib = L.lib()
    w = ops._decoder_weights(ops.Scope(st, "dec"))
    z = lambda *s: torch.zeros(*s, device="cuda")
    t = {"packed": z(lib.taco_decoder_packed_bytes(r) // 4), "keys": z(B, Tx, 256), "values": z(B, Tx, 256),
         "text_length": torch.full((B,), Tx, dtype=torch.int32, device="cuda"), "y": z(B, T, 80 * r), "align": z(B, T, Tx),
         "workspace": z(lib.taco_decoder_workspace_bytes(32, Tx, T, r) // 4), "mel": z(B, T, 80 * r),
         "sample_mask": torch.ones(T, B, dtype=torch.uint8, device="cuda")}
    if peak:
        t["peak"] = torch.zeros(B, T, dtype=torch.int32, device="cuda")
    n0 = lib.taco_launch_count()
    try:
        ops.decoder_fwd_launches(lib, ops.decoder_plan(B, 132), w, t, mode, T, r, 1.0, None, L.current_stream(),
                                 None if (back, ahead) == (0, 0) else (back, ahead))
    finally:
        torch.cuda.synchronize()
        assert lib.taco_launch_count() == n0, "something was launched"


@pytest.mark.parametrize("mode", [L.DEC_TEACHER, L.DEC_SCHED])
def test_window_in_training_modes_is_refused(mode):
    with pytest.raises(L.TacoError, match="win_ahead=5.*TACO_DEC_INFER"):
        _raw_call(mode, 2, 5)


@pytest.mark.parametrize("back,ahead,peak,word", [(2, 0, False, "win_ahead=0"), (-1, 5, False, "win_back=-1"),
                                                  (0, 0, True, "peak")])
def test_bad_window_is_refused(back, ahead, peak, word):
    with pytest.raises(L.TacoError, match=word):
        _raw_call(L.DEC_INFER, back, ahead, peak)


def test_python_refuses_before_launching():
    r, B, Tx, T = 2, 2, 8, 3
    cfg, p, encoded, mel, tl, dec_m, sm = _setup(r, B, Tx, T)
    st = _store(p, r)
    n0 = L.lib().taco_launch_count()
    with pytest.raises(L.TacoError, match="ahead"):
        _dec(st, r, T, encoded, tl, window=(2, 0))
    with pytest.raises(L.TacoError, match="window"):
        ops.attention_decoder(encoded.cuda(), tl.cuda(), r, T, mode=L.DEC_TEACHER, mel=mel.cuda(), scope=ops.Scope(st, "dec"),
                              window=(2, 5))
    assert L.lib().taco_launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------------
# 7. end to end
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("window", WINDOWS)
def test_inference_end_to_end(window):
    cfg = ocfg(r=2, T=7, vocab=20)
    p = O.init_params(cfg, seed=1, trained_like=True)
    inp = O.synthetic_inputs(cfg, 9, 37, 7, seed=0, ragged=True, with_targets=False)
    m = make_model(cfg, p, "fp32x3")
    m.config.attention_window = window
    y, out = m.inference(to_cuda(inp), train=False)
    torch.cuda.synchronize()
    pk = m.attention_peaks.cpu()
    assert pk.shape == (9, 7) and pk.dtype == torch.int32
    y_ref, out_ref, a_ref, _ = AW.inference({k: v.double() for k, v in p.items()}, inp, cfg, 7, window, peaks=pk)
    assert_close(y, y_ref, 2e-4, f"e2e window={window} y")
    assert_close(m.alignments, a_ref, 2e-4, f"e2e window={window} align")
    assert_close(out, out_ref, 2e-4, f"e2e window={window} out")
    check_window(m.alignments, pk, inp["text_length"], window, "e2e")


def _drive(monkeypatch, argv, prompts):
    """python -m tacotron_b200.test argv on the toy checkpoint; records each inference call's alignments, peaks and lengths"""
    from tacotron_b200 import test as synth
    from tacotron_b200.models.tacotron import Tacotron
    seen = []
    real = Tacotron.inference

    def spy(self, inputs, *a, **k):
        res = real(self, inputs, *a, **k)
        seen.append((self.alignments.clone(), None if self.attention_peaks is None else self.attention_peaks.clone(),
                     inputs["text_length"].cpu(), self.config.attention_window))
        return res
    monkeypatch.setattr(Tacotron, "inference", spy)
    monkeypatch.setattr("sys.stdin", io.StringIO("".join(prompts)))
    torch.manual_seed(0)
    synth.main(argv)
    torch.cuda.synchronize()
    monkeypatch.setattr(Tacotron, "inference", real)
    return seen


def test_synthesis_driver_attention_window(tmp_path, monkeypatch):
    from scipy.io import wavfile
    from tests.test_gpu_z_summary import _files, _train
    _train(str(tmp_path), monkeypatch, False)
    out = "log/toy/tacotron/test"
    prompts = ["abc de\n", "hello, you\n", "abc de\n"]
    plain = _drive(monkeypatch, ["-t", "toy"], prompts)
    assert all(s[1] is None and s[3] is None for s in plain)
    shutil.rmtree(out)
    for argv, window in ((["--attention-window"], (2, 5)), (["--attention-window", "0,3", "--trim-tail", "--summaries"], (0, 3)),
                         (["--attention-window", "--long-form"], (2, 5))):
        seen = _drive(monkeypatch, ["-t", "toy", *argv], prompts)
        assert seen and all(s[3] == window for s in seen)
        for a, pk, tl, _ in seen:
            check_window(a, pk, tl, window, f"driver {argv}")
        files = _files(out)
        for b in range(3):
            rate, samples = wavfile.read(f"{out}/{b}.wav")
            assert rate == 16000 and samples.size > 0
            al = np.load(f"{out}/{b}_attention.npy")
            assert al.ndim == 2 and al.shape[0] > 0
            assert f"{b}.txt" in files
        if "--long-form" in argv:
            assert os.path.exists(f"{out}/0_chunks.txt")
        if "--summaries" in argv:
            assert any(k.startswith("events.out.tfevents") for k in files)
        shutil.rmtree(out)
