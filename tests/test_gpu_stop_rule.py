"""-m gpu: the end-of-text stop rule of free-running decoding (taco_decoder_args stop_at / stop_hold / end_step,
Config.stop_at_end, python -m tacotron_b200.test --stop-at-end) on the H100.

  1. the rule off (the default call, and stop_at = NULL) gives the default call's bits;
  2. a stopped decode against the unstopped decode of the same inputs: every row's end_step is the host rule applied to
     the unstopped decode's own peaks, exactly; every row group g decodes D_g steps with max end_step <= D_g <= max
     end_step + TACO_DECODER_STOP_LAG, bit-identical to the unstopped decode before D_g and 0 / 0 / -1 from D_g on --
     over r, the batch (one row, one group, four groups, two launches), ragged lengths and the hold, with rows of a
     group ending at different steps and one group whose rule never fires;
  3. the same with the attention window and under split launch plans, whose bits equal the full grid's;
  4. a stop rule in teacher-forced or scheduled-sampling mode, a hold of 0 and a half-set argument pair are refused
     with nothing launched and the outputs untouched;
  5. Tacotron.inference: outputs of the kept length T', the post-net of the returned seq2seq_output, the CUDA-graph
     path equal to the eager one, and a changed hold never served from an old graph;
  6. the synthesis driver with --stop-at-end (plain, --trim-tail, --long-form)."""
import io
import os
import shutil

import numpy as np
import pytest
import torch

from oracle import tacotron_oracle as O
from tacotron_b200 import _lib as L
from tacotron_b200 import audio
from tacotron_b200.models import ops
from tests.test_gpu_decoder_envelope import _setup, short_lengths
from tests.util import make_model, ocfg, to_cuda

pytestmark = pytest.mark.gpu
LAG = L.DECODER_STOP_LAG


def _store(p, r):
    from tacotron_b200 import Config
    from tacotron_b200.params import ParamStore, model_shapes
    st = ParamStore(model_shapes(Config(r=r, vocab_size=20)), "cuda")
    st.load(p)
    ops.runtime(st, "fp32")
    return st


def _dec(st, r, T, encoded, tl, window=None, hold=None, stop_at=None, max_ctas=None):
    """ops.attention_decoder in free-running mode -> [y, alpha, peaks, end_step] (the last two None when not returned),
    cloned"""
    res = ops.attention_decoder(encoded.float().cuda(), tl.cuda(), r, T, mode=L.DEC_INFER, scope=ops.Scope(st, "dec"),
                                max_ctas=max_ctas, window=window, stop_hold=hold,
                                stop_at=None if stop_at is None else stop_at.cuda())
    torch.cuda.synchronize()
    out = [x.clone() for x in res]
    return out + [None] * (4 - len(out))


def _stop_positions(pk, Tx, T, hold, seed):
    """stop_at per row from the unstopped peaks pk [B, T]: rows of a group aim at different steps t (the lowest peak of
    steps t .. t + hold - 1, so the row ends by t + hold), row 8g ends at `hold` (stop_at = 0), and the whole second
    group never fires (stop_at = Tx)"""
    B = pk.shape[0]
    g = torch.Generator().manual_seed(seed)
    at = torch.empty(B, dtype=torch.int32)
    for b in range(B):
        k = b % 8
        if B > 8 and b // 8 == 1:
            at[b] = Tx
        elif k == 0 and B > 1:
            at[b] = 0
        else:
            t = int(T * (0.1 + 0.1 * k)) + int(torch.randint(0, 3, (1,), generator=g))
            t = min(t, T - hold)
            at[b] = int(pk[b, t:t + hold].min())
    return at


def check_stopped(ref, got, stop_at, hold, what):
    """ref = the unstopped decode [y, alpha, peaks, _], got = the stopped one; returns the per-group D_g"""
    y0, a0, p0 = (x.cpu() for x in ref[:3])
    y, a, p, end = (x.cpu() for x in got)
    B, T = p0.shape
    want = ops.stop_rule_end_steps(p0.numpy(), stop_at.numpy(), hold)
    assert end.dtype == torch.int32 and end.tolist() == want.tolist(), f"{what}: end_step {end.tolist()} != {want.tolist()}"
    D = []
    for g0 in range(0, B, 8):
        rows = slice(g0, min(g0 + 8, B))
        E = int(want[rows].max())
        stopped = (p[rows] == -1).all(0)
        Dg = int(stopped.to(torch.int64).argmax()) if stopped.any() else T
        assert E <= Dg <= min(T, E + LAG), f"{what}: group {g0 // 8} decoded {Dg} steps, last end_step {E}"
        assert not (p[rows, :Dg] == -1).any() and stopped[Dg:].all(), f"{what}: group {g0 // 8} peaks"
        assert torch.equal(y[rows, :Dg], y0[rows, :Dg]), f"{what}: group {g0 // 8} y before the stop"
        assert torch.equal(a[rows, :Dg], a0[rows, :Dg]), f"{what}: group {g0 // 8} align before the stop"
        assert torch.equal(p[rows, :Dg], p0[rows, :Dg]), f"{what}: group {g0 // 8} peaks before the stop"
        assert (y[rows, Dg:] == 0).all() and (a[rows, Dg:] == 0).all(), f"{what}: group {g0 // 8} after the stop"
        D.append((Dg, E))
    print(f"{what}: (D_g, max end_step) per group {D}")
    return D


def _pair(r, B, Tx, T, hold, window=None, max_ctas=None, seed=0):
    lengths = short_lengths(Tx, B) if B > 1 else torch.tensor([Tx - 3], dtype=torch.int32)
    cfg, p, encoded, mel, tl, dec_m, sm = _setup(r, B, Tx, T, lengths, seed=seed)
    st = _store(p, r)
    ref = _dec(st, r, T, encoded, tl, window=window if window is not None else (Tx, Tx))
    stop_at = _stop_positions(ref[2].cpu(), Tx, T, hold, seed)
    got = _dec(st, r, T, encoded, tl, window=window, hold=hold, stop_at=stop_at, max_ctas=max_ctas)
    return st, encoded, tl, ref, got, stop_at


# ---------------------------------------------------------------------------------------------------------------------
# 1. off
# ---------------------------------------------------------------------------------------------------------------------
def test_off_changes_nothing():
    r, B, Tx, T = 2, 32, 140, 60
    cfg, p, encoded, mel, tl, dec_m, sm = _setup(r, B, Tx, T, short_lengths(Tx, B))
    st = _store(p, r)
    y0, a0, pk0, e0 = _dec(st, r, T, encoded, tl)
    assert pk0 is None and e0 is None
    y1, a1, _, _ = _dec(st, r, T, encoded, tl, hold=None, stop_at=None)
    assert torch.equal(y0, y1) and torch.equal(a0, a1)
    # covering window: the peaks come with the unwindowed bits (the stop rule's reference below)
    y2, a2, pk2, _ = _dec(st, r, T, encoded, tl, window=(Tx, Tx))
    assert torch.equal(y0, y2) and torch.equal(a0, a2)
    # a rule that never fires decodes every step, with the same bits
    y3, a3, pk3, e3 = _dec(st, r, T, encoded, tl, hold=1, stop_at=torch.full((B,), Tx, dtype=torch.int32))
    assert torch.equal(y0, y3) and torch.equal(a0, a3) and torch.equal(pk2, pk3)
    assert e3.tolist() == [T] * B


# ---------------------------------------------------------------------------------------------------------------------
# 2. stopped against unstopped
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hold", [1, 3])
@pytest.mark.parametrize("B", [1, 8, 32, 33])
@pytest.mark.parametrize("r,Tx", [(2, 140), (5, 37)])
def test_stopped_decode_matches_the_unstopped_one(r, Tx, B, hold):
    T = 60
    st, encoded, tl, ref, got, stop_at = _pair(r, B, Tx, T, hold)
    D = check_stopped(ref, got, stop_at, hold, f"r={r} Tx={Tx} B={B} hold={hold}")
    if B > 8:
        assert D[1][0] == T, "the group whose rule never fires must decode every step"
    assert any(d < T for d, _ in D), "no group stopped"


def test_stop_at_zero_ends_every_row_at_hold():
    r, B, Tx, T = 2, 32, 140, 60
    cfg, p, encoded, mel, tl, dec_m, sm = _setup(r, B, Tx, T, short_lengths(Tx, B))
    st = _store(p, r)
    ref = _dec(st, r, T, encoded, tl, window=(Tx, Tx))
    for hold in (1, 5, 20):
        zero = torch.zeros(B, dtype=torch.int32)
        got = _dec(st, r, T, encoded, tl, hold=hold, stop_at=zero)
        assert got[3].tolist() == [hold] * B
        D = check_stopped(ref, got, zero, hold, f"stop_at=0 hold={hold}")
        assert all(d == min(T, hold + LAG) for d, _ in D)


# ---------------------------------------------------------------------------------------------------------------------
# 3. window and split launch plans
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [9, 32])
def test_stopped_decode_with_window(B):
    r, Tx, T, hold = 2, 140, 60, 2
    st, encoded, tl, ref, got, stop_at = _pair(r, B, Tx, T, hold, window=(2, 5))
    check_stopped(ref, got, stop_at, hold, f"window B={B}")


@pytest.mark.parametrize("window", [None, (2, 5)])
@pytest.mark.parametrize("max_ctas", [32, 64])
def test_split_launches_are_bit_identical(max_ctas, window):
    r, B, Tx, T, hold = 2, 32, 140, 60, 3
    st, encoded, tl, ref, got, stop_at = _pair(r, B, Tx, T, hold, window=window)
    split = _dec(st, r, T, encoded, tl, window=window, hold=hold, stop_at=stop_at, max_ctas=max_ctas)
    for x, s in zip(got, split):
        assert torch.equal(x, s)
    check_stopped(ref, split, stop_at, hold, f"max_ctas={max_ctas} window={window}")


# ---------------------------------------------------------------------------------------------------------------------
# 4. refusals
# ---------------------------------------------------------------------------------------------------------------------
def _raw_call(mode, hold, stop_at, end_step):
    """taco_decoder_fwd on valid buffers (B = 2, Tx = 8, T = 3, r = 2) with the given stop fields; the outputs hold a
    sentinel that must survive"""
    r, B, Tx, T = 2, 2, 8, 3
    cfg, p, *_ = _setup(r, B, Tx, T)
    st = _store(p, r)
    lib = L.lib()
    w = ops._decoder_weights(ops.Scope(st, "dec"))
    z = lambda *s: torch.zeros(*s, device="cuda")
    t = {"packed": z(lib.taco_decoder_packed_bytes(r) // 4), "keys": z(B, Tx, 256), "values": z(B, Tx, 256),
         "text_length": torch.full((B,), Tx, dtype=torch.int32, device="cuda"),
         "y": torch.full((B, T, 80 * r), 7.0, device="cuda"), "align": torch.full((B, T, Tx), 7.0, device="cuda"),
         "workspace": z(lib.taco_decoder_workspace_bytes(32, Tx, T, r) // 4), "mel": z(B, T, 80 * r),
         "sample_mask": torch.ones(T, B, dtype=torch.uint8, device="cuda"),
         "peak": torch.full((B, T), 7, dtype=torch.int32, device="cuda")}
    if stop_at:
        t["stop_at"] = torch.zeros(B, dtype=torch.int32, device="cuda")
    else:
        del t["peak"]                                  # (peak without a window or a stop rule is refused too)
    if end_step:
        t["end_step"] = torch.full((B,), 7, dtype=torch.int32, device="cuda")
    n0 = lib.taco_launch_count()
    try:
        ops.decoder_fwd_launches(lib, ops.decoder_plan(B, 132), w, t, mode, T, r, 1.0, None, L.current_stream(), None, hold)
    finally:
        torch.cuda.synchronize()
        assert lib.taco_launch_count() == n0, "something was launched"
        assert (t["y"] == 7).all() and (t["align"] == 7).all() and (t.get("peak", t["y"]) == 7).all()
        if end_step:
            assert (t["end_step"] == 7).all()


@pytest.mark.parametrize("mode", [L.DEC_TEACHER, L.DEC_SCHED])
def test_stop_rule_in_training_modes_is_refused(mode):
    with pytest.raises(L.TacoError, match="stop rule applies to free-running"):
        _raw_call(mode, 2, True, True)


@pytest.mark.parametrize("hold,stop_at,end_step,word", [(0, True, True, "stop_hold=0"), (-1, True, True, "stop_hold=-1"),
                                                        (2, True, False, "needs both"), (2, False, True, "needs both"),
                                                        (2, False, False, "without stop_at")])
def test_bad_stop_rule_is_refused(hold, stop_at, end_step, word):
    with pytest.raises(L.TacoError, match=word):
        _raw_call(L.DEC_INFER, hold, stop_at, end_step)


# ---------------------------------------------------------------------------------------------------------------------
# 5. Tacotron.inference
# ---------------------------------------------------------------------------------------------------------------------
def test_inference_keeps_the_needed_steps_and_graphs_follow_the_hold(monkeypatch):
    cfg_o = ocfg(r=2, T=30, vocab=20)
    p = O.init_params(cfg_o, seed=1, trained_like=True)
    inp = to_cuda(O.synthetic_inputs(cfg_o, 9, 37, 30, seed=0, ragged=True, with_targets=False))
    m = make_model(cfg_o, p, "fp32x3")
    T = m.config.max_decode_iter
    y_full, _ = m.inference(inp, train=False)
    y_full, a_full = y_full.clone(), m.alignments.clone()
    assert m.end_steps is None
    # stop_at = 0: every row ends after exactly `hold` steps, so the hold chooses T'
    monkeypatch.setattr(ops, "stop_positions", lambda text, n: torch.zeros(text.shape[0], dtype=torch.int32,
                                                                            device=text.device))
    eager = {}
    for hold in (3, 6, 1):
        m.config.stop_at_end = hold
        y, out = m.inference(inp, train=False)
        torch.cuda.synchronize()
        Tp = min(T, 4 * ((hold + 3) // 4))
        assert y.shape == (9, Tp, 160) and out.shape[:2] == (9, Tp), (hold, y.shape, out.shape)
        assert m.alignments.shape[:2] == (9, Tp) and m.attention_peaks.shape == (9, Tp)
        assert m.end_steps.tolist() == [hold] * 9
        out = out.clone()                          # (_postnet below writes the same scratch buffer)
        assert torch.equal(out, m._postnet(y, None)), hold
        D = min(T, hold + LAG)
        assert torch.equal(y[:, :min(D, Tp)], y_full[:, :min(D, Tp)])
        assert torch.equal(m.alignments[:, :min(D, Tp)], a_full[:, :min(D, Tp)])
        eager[hold] = (y.clone(), out.clone(), m.alignments.clone(), m.attention_peaks.clone(), m.end_steps.clone())
    m.config.cuda_graph = True
    for hold in (3, 6, 3, 1, None, 6):
        m.config.stop_at_end = hold
        y, out = m.inference(inp, train=False)
        torch.cuda.synchronize()
        if hold is None:
            assert m.end_steps is None and y.shape[1] == T and torch.equal(y, y_full)
            continue
        ey, eo, ea, ep, ee = eager[hold]
        assert torch.equal(y, ey) and torch.equal(out, eo), hold
        assert torch.equal(m.alignments, ea) and torch.equal(m.attention_peaks, ep) and torch.equal(m.end_steps, ee), hold


def test_inference_stop_positions_from_the_text():
    """the real stop_at (no stand-in): end_step is the host rule on the returned peaks"""
    cfg_o = ocfg(r=2, T=40, vocab=20)
    p = O.init_params(cfg_o, seed=1, trained_like=True)
    inp = to_cuda(O.synthetic_inputs(cfg_o, 9, 37, 40, seed=0, ragged=True, with_targets=False))
    m = make_model(cfg_o, p, "fp32x3")
    m.config.stop_at_end = 1
    y, out = m.inference(inp, train=False)
    torch.cuda.synchronize()
    at = ops.stop_positions(inp["text"], inp["text_length"]).cpu()
    pk = m.attention_peaks.cpu()
    want = ops.stop_rule_end_steps(pk.numpy(), at.numpy(), 1)
    end = m.end_steps.cpu()
    # the kept steps hold every row's end (T' >= max end_step), and -1 peaks never extend a run, so the rule on the
    # kept peaks finds each row's end_step; a row that never ends gives T' = T
    assert end.tolist() == want.tolist()
    assert y.shape[1] == ops.stopped_steps(end, m.config.max_decode_iter)
    assert torch.equal(out.clone(), m._postnet(y, None))


# ---------------------------------------------------------------------------------------------------------------------
# 6. the synthesis driver
# ---------------------------------------------------------------------------------------------------------------------
def _drive(monkeypatch, argv, prompts):
    """python -m tacotron_b200.test argv on the toy checkpoint; records each inference call's end_steps and kept steps"""
    from tacotron_b200 import test as synth
    from tacotron_b200.models.tacotron import Tacotron
    seen = []
    real = Tacotron.inference

    def spy(self, inputs, *a, **k):
        res = real(self, inputs, *a, **k)
        seen.append((None if self.end_steps is None else self.end_steps.clone(), res[1].shape[1], self.config.r))
        return res
    monkeypatch.setattr(Tacotron, "inference", spy)
    monkeypatch.setattr("sys.stdin", io.StringIO("".join(prompts)))
    torch.manual_seed(0)
    synth.main(argv)
    torch.cuda.synchronize()
    monkeypatch.setattr(Tacotron, "inference", real)
    return seen


def test_synthesis_driver_stop_at_end(tmp_path, monkeypatch):
    from scipy.io import wavfile
    from tests.test_gpu_z_summary import _files, _train
    _train(str(tmp_path), monkeypatch, False)
    out = "log/toy/tacotron/test"
    prompts = ["abc de\n", "hello, you\n", "abc de\n"]
    monkeypatch.setattr(ops, "stop_positions", lambda text, n: torch.zeros(text.shape[0], dtype=torch.int32,
                                                                            device=text.device))
    hop = audio.hop_length
    for argv, hold in ((["--stop-at-end", "5"], 5), (["--stop-at-end", "--trim-tail", "--summaries"], 4),
                       (["--stop-at-end", "2", "--long-form"], 2)):
        seen = _drive(monkeypatch, ["-t", "toy", *argv], prompts)
        assert seen and all(s[0] is not None and s[0].tolist() == [hold] * len(s[0]) for s in seen)
        end, Tp, r = seen[0]
        frames = audio.stop_frames(end, r, Tp).tolist()
        files = _files(out)
        for b in range(3):
            rate, samples = wavfile.read(f"{out}/{b}.wav")
            al = np.load(f"{out}/{b}_attention.npy")
            assert rate == 16000 and f"{b}.txt" in files
            if "--long-form" in argv:
                assert 0 < al.shape[0] * r <= frames[0] and samples.size > 0
            elif "--trim-tail" in argv:
                assert 0 < al.shape[0] * r <= frames[b] and samples.size == hop * (al.shape[0] * r - 1)
            else:
                assert al.shape[0] == frames[b] // r and samples.size == hop * (frames[b] - 1), (b, al.shape, samples.size)
        if "--summaries" in argv:
            assert any(k.startswith("events.out.tfevents") for k in files)
        shutil.rmtree(out)
