"""The end-of-text stop rule of free-running decoding (Config.stop_at_end), without a GPU: the rule on hand-made peak
arrays, stop_at from load_prompts batches (the dropped out-of-vocabulary character and the counted newline), the kept
steps T' and the frames each utterance inverts, the new taco_decoder_args fields against the header, the launch loop
over a fake library, and the Config / CLI parsing and its refusals."""
import argparse
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from tacotron_b200 import _lib as L
from tacotron_b200 import audio, data_input
from tacotron_b200.models import ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------------------------------
# the rule
# ---------------------------------------------------------------------------------------------------------------------
def test_hold_one_ends_at_the_first_peak_at_or_past_stop_at():
    peaks = np.array([[0, 1, 2, 3, 4, 5], [0, 0, 1, 1, 2, 2], [3, 0, 0, 0, 0, 0]])
    assert ops.stop_rule_end_steps(peaks, [3, 5, 3], 1).tolist() == [4, 6, 1]


def test_larger_hold_needs_consecutive_peaks():
    peaks = np.array([[0, 5, 0, 5, 5, 0, 5, 5, 5, 0], [0, 5, 5, 5, 5, 5, 5, 5, 5, 5]])
    assert ops.stop_rule_end_steps(peaks, [5, 5], 2).tolist() == [5, 3]
    assert ops.stop_rule_end_steps(peaks, [5, 5], 3).tolist() == [9, 4]
    assert ops.stop_rule_end_steps(peaks, [5, 5], 4).tolist() == [10, 5]      # never for row 0: T
    assert ops.stop_rule_end_steps(peaks, [5, 5], 11).tolist() == [10, 10]    # a hold longer than the decode


def test_stop_at_zero_ends_every_row_after_hold_steps():
    peaks = np.random.default_rng(0).integers(0, 50, size=(5, 40))
    for hold in (1, 3, 17):
        assert ops.stop_rule_end_steps(peaks, np.zeros(5, np.int64), hold).tolist() == [hold] * 5


def test_stop_at_past_the_text_never_fires():
    peaks = np.random.default_rng(1).integers(0, 50, size=(4, 30))
    assert ops.stop_rule_end_steps(peaks, np.full(4, 50), 1).tolist() == [30] * 4


def test_peaks_of_a_stopped_group_never_extend_a_run():
    """steps a row group did not decode carry p = -1, below any stop_at"""
    peaks = np.array([[0, 2, 2, -1, -1, -1]])
    assert ops.stop_rule_end_steps(peaks, [0], 3).tolist() == [3]
    assert ops.stop_rule_end_steps(peaks, [0], 4).tolist() == [6]
    assert ops.stop_rule_end_steps(peaks, [1], 3).tolist() == [6]


# ---------------------------------------------------------------------------------------------------------------------
# stop_at from load_prompts batches
# ---------------------------------------------------------------------------------------------------------------------
IVOCAB = {0: "<pad>", 1: "a", 2: "b", 3: "c", 4: " ", 5: "."}


def _batch(prompts):
    return next(data_input.load_prompts(prompts, IVOCAB, device="cpu"))


def test_stop_at_is_the_last_real_character():
    inp = _batch(["abc\n", "ab c.\n"])
    assert inp["text_length"].tolist() == [4, 6]                     # the raw line, newline included
    assert ops.stop_positions(inp["text"], inp["text_length"]).tolist() == [2, 4]


def test_stop_at_skips_a_dropped_out_of_vocabulary_character():
    inp = _batch(["ab!c\n", "?\n"])                                   # '!' and '?' are not in the vocabulary
    assert inp["text_length"].tolist() == [5, 2]
    assert inp["text"][0, :4].tolist() == [1, 2, 3, 0]
    assert ops.stop_positions(inp["text"], inp["text_length"]).tolist() == [2, 0]      # nothing left: 0


def test_stop_at_is_capped_by_text_length_and_width():
    text = torch.tensor([[1, 2, 3, 1, 2], [1, 2, 3, 1, 2], [0, 0, 0, 0, 0]], dtype=torch.int32)
    n = torch.tensor([2, 9, 0], dtype=torch.int32)
    got = ops.stop_positions(text, n)
    assert got.dtype == torch.int32 and got.tolist() == [1, 4, 0]


# ---------------------------------------------------------------------------------------------------------------------
# T' and the frames to invert
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ends,T,want", [([5, 9, 2], 180, 12), ([4, 4], 180, 4), ([180, 3], 180, 180), ([178], 180, 180),
                                         ([177], 180, 180), ([176], 180, 176), ([1], 3, 3), ([97], 100, 100)])
def test_kept_steps(ends, T, want):
    assert ops.stopped_steps(torch.tensor(ends, dtype=torch.int32), T) == want
    assert ops.stopped_steps(ends, T) == want


def test_stop_frames_round_up_to_blocks_and_stop_at_the_kept_steps():
    r, Tp = 2, 12
    got = audio.stop_frames(torch.tensor([5, 9, 2, 12], dtype=torch.int32), r, Tp)
    assert got.dtype == torch.int32 and got.tolist() == [16, 24, 8, 24]           # 4r ceil(e/4), at most 4r (T'//4)
    got = audio.stop_frames(torch.tensor([100, 37], dtype=torch.int32), 5, 98)
    assert got.tolist() == [4 * 5 * 24, 4 * 5 * 10]


def test_stop_frames_take_the_minimum_with_speech_frames():
    speech = torch.tensor([8, 40, 16], dtype=torch.int32)
    got = audio.stop_frames(torch.tensor([9, 9, 2], dtype=torch.int32), 2, 12, speech)
    assert got.tolist() == [8, 24, 8]


def test_stop_frames_are_what_invert_speech_accepts():
    for r in (1, 2, 5):
        for T in (4, 8, 100):
            n = 4 * r * (T // 4)
            if n < 5:                                  # (r = 1, T = 4: no length invert_speech accepts)
                continue
            f = audio.stop_frames(torch.arange(1, T + 1, dtype=torch.int32), r, T)
            assert ((f % (4 * r) == 0) & (f >= 5) & (f <= n)).all(), (r, T, f)


# ---------------------------------------------------------------------------------------------------------------------
# ABI
# ---------------------------------------------------------------------------------------------------------------------
def test_stop_fields_match_header():
    probe = r'''
#include <stdio.h>
#include <stddef.h>
#include "taco_b200.h"
int main(void){ printf("%zu %zu %zu %zu %zu %d\n", sizeof(taco_decoder_args), offsetof(taco_decoder_args, peak),
                       offsetof(taco_decoder_args, stop_at), offsetof(taco_decoder_args, stop_hold),
                       offsetof(taco_decoder_args, end_step), TACO_DECODER_STOP_LAG); return 0; }
'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c"); exe = os.path.join(d, "p")
        open(c, "w").write(probe)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = list(map(int, subprocess.check_output([exe]).split()))
    A = L.DecoderArgs
    assert got == [C.sizeof(A), A.peak.offset, A.stop_at.offset, A.stop_hold.offset, A.end_step.offset,
                   L.DECODER_STOP_LAG]
    assert A.stop_at.offset > A.peak.offset                    # appended: the existing fields keep their offsets
    a = A()
    assert (a.stop_at, a.stop_hold, a.end_step) == (None, 0, None)


def test_workspace_grows_by_the_status_words():
    lib = L.lib()
    off = lib.taco_decoder_trace_offset()
    T = 180
    base = (off + 16 * T + 16 + 4 * 20 * 8 + 16 + 2 * 3 * 20 * 64) * 8 + 5 * 32 * 512 * 4
    assert lib.taco_decoder_workspace_bytes(32, 140, T, 2) == base + 32 * 2 * 8


# ---------------------------------------------------------------------------------------------------------------------
# the launch loop over a fake library
# ---------------------------------------------------------------------------------------------------------------------
class _FakeLib:
    def __init__(self):
        self.calls = []

    def taco_decoder_fwd(self, aref, stream):
        a = aref._obj
        self.calls.append((a.row0, a.B, a.stop_at, a.stop_hold, a.end_step, a.peak))
        return 0


@pytest.mark.parametrize("B,max_ctas", [(27, 32), (33, None), (9, 64)])
def test_launches_pass_stop_rows(B, max_ctas):
    T, Tx = 7, 13
    t = {"packed": torch.zeros(16), "keys": torch.zeros(B, Tx, 256), "values": torch.zeros(B, Tx, 256),
         "text_length": torch.full((B,), Tx, dtype=torch.int32), "workspace": torch.zeros(16),
         "y": torch.zeros(B, T, 160), "align": torch.zeros(B, T, Tx), "peak": torch.zeros(B, T, dtype=torch.int32),
         "stop_at": torch.zeros(B, dtype=torch.int32), "end_step": torch.zeros(B, dtype=torch.int32)}
    lib = _FakeLib()
    plan = ops.decoder_plan(B, 132, max_ctas)
    ops.decoder_fwd_launches(lib, plan, L.DecoderWeights(), t, L.DEC_INFER, T, 2, 1.0, max_ctas, None, None, 3)
    assert len(lib.calls) == len(plan)
    for (b0, nb, _), (row0, n, stop_at, hold, end_step, peak) in zip(plan, lib.calls):
        assert (row0, n, hold) == (b0, nb, 3)
        assert stop_at == t["stop_at"].data_ptr() + 4 * b0
        assert end_step == t["end_step"].data_ptr() + 4 * b0
        assert peak == t["peak"].data_ptr() + 4 * T * b0


def test_no_stop_rule_leaves_the_fields_zero():
    B, T, Tx = 9, 5, 9
    t = {"packed": torch.zeros(16), "keys": torch.zeros(B, Tx, 256), "values": torch.zeros(B, Tx, 256),
         "text_length": torch.full((B,), Tx, dtype=torch.int32), "workspace": torch.zeros(16),
         "y": torch.zeros(B, T, 160), "align": torch.zeros(B, T, Tx)}
    lib = _FakeLib()
    ops.decoder_fwd_launches(lib, ops.decoder_plan(B, 132), L.DecoderWeights(), t, L.DEC_INFER, T, 2, 1.0, None, None)
    assert lib.calls and all(c[2:5] == (None, 0, None) for c in lib.calls)


# ---------------------------------------------------------------------------------------------------------------------
# Config / CLI
# ---------------------------------------------------------------------------------------------------------------------
def test_config_default_is_off():
    from tacotron_b200 import Config
    assert Config().stop_at_end is None
    assert ops.stop_rule_hold(Config().stop_at_end) is None
    assert ops.stop_rule_hold(Config(stop_at_end=4).stop_at_end) == 4


@pytest.mark.parametrize("hold", [1, 4, np.int64(3), 2 ** 31 - 1])
def test_hold_accepted(hold):
    got = ops.stop_rule_hold(hold)
    assert got == int(hold) and type(got) is int


@pytest.mark.parametrize("hold,word", [(0, "must be in"), (-2, "must be in"), (2 ** 31, "must be in"), (True, "integer"),
                                       (2.0, "integer"), ("4", "integer"), ((4,), "integer")])
def test_hold_rejected(hold, word):
    with pytest.raises(L.TacoError, match=word):
        ops.stop_rule_hold(hold)


def test_attention_decoder_refuses_before_anything_runs():
    """a half-set pair, a bad hold and a stop rule in teacher-forced or scheduled mode are refused before the decoder
    touches the device (the checks come before any buffer or launch)"""
    enc = torch.zeros(2, 5, 256)
    n = torch.full((2,), 5, dtype=torch.int32)
    at = torch.zeros(2, dtype=torch.int32)
    with pytest.raises(L.TacoError, match="give both or neither"):
        ops.attention_decoder(enc, n, 2, 4, stop_hold=4)
    with pytest.raises(L.TacoError, match="give both or neither"):
        ops.attention_decoder(enc, n, 2, 4, stop_at=at)
    with pytest.raises(L.TacoError, match="must be in"):
        ops.attention_decoder(enc, n, 2, 4, stop_hold=0, stop_at=at)
    for mode in (L.DEC_TEACHER, L.DEC_SCHED):
        with pytest.raises(L.TacoError, match="free-running"):
            ops.attention_decoder(enc, n, 2, 4, mode=mode, stop_hold=2, stop_at=at)
    with pytest.raises(L.TacoError, match="stop_at must be"):
        ops.attention_decoder(enc, n, 2, 4, stop_hold=2, stop_at=at.to(torch.int64))


def test_cli_parsing():
    from tacotron_b200.test import parse_stop_hold
    assert parse_stop_hold("4") == 4 and parse_stop_hold("1") == 1
    for bad in ("0", "-1", "a", "2.5", ""):
        with pytest.raises(argparse.ArgumentTypeError):
            parse_stop_hold(bad)


def test_cli_flag_forms(monkeypatch):
    """a bare flag means hold 4; no flag leaves the rule off; a bad value exits with a usage error before any model"""
    from tacotron_b200 import test as drv
    seen = []
    monkeypatch.setattr(drv, "test", lambda cls, config, prompts, **kw: seen.append(
        (config.stop_at_end, config.attention_window, kw["trim_tail"], kw["long_form"])))
    monkeypatch.setattr("sys.stdin", __import__("io").StringIO("hello\n"))
    drv.main(["-t", "x", "--stop-at-end"])
    drv.main(["-t", "x", "--stop-at-end", "2", "--long-form", "--trim-tail", "--attention-window", "--max-ctas", "32"])
    drv.main(["-t", "x", "--trim-tail", "--stop-at-end", "-s", "1"])
    drv.main(["-t", "x"])
    assert seen == [(4, None, False, False), (2, (2, 5), True, True), (4, None, True, False), (None, None, False, False)]
    with pytest.raises(SystemExit):
        drv.main(["-t", "x", "--stop-at-end", "0"])
    assert len(seen) == 4
