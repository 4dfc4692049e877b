"""The attention window of free-running decoding (Config.attention_window), without a GPU: the float64 oracle on
hand-checked cases, the new taco_decoder_args fields against the header, ops.decoder_fwd_launches over a fake library
(the window and peak + b0 reach every launch of a split plan), and the Config / CLI parsing and its refusals."""
import argparse
import ctypes as C
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from oracle import tacotron_oracle as O
from tacotron_b200 import _lib as L
from tacotron_b200.models import ops
from tests import attention_window_oracle as AW
from tests.util import ocfg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INF = math.inf


# ---------------------------------------------------------------------------------------------------------------------
# the oracle
# ---------------------------------------------------------------------------------------------------------------------
def test_window_mask_is_clipped_at_zero_and_at_the_text_length():
    N = torch.tensor([10, 10, 4, 10])
    p_prev = torch.tensor([0, 1, 3, 7])
    m = AW.window_mask(p_prev, N, 12, 2, 3)
    want = [[0, 1, 2, 3],                   # p = 0: clipped at 0
            [0, 1, 2, 3, 4],                # p = 1: 1 - 2 < 0, clipped
            [1, 2, 3],                      # p = 3, N = 4: clipped at N - 1 = 3
            [5, 6, 7, 8, 9]]                # p = 7: 10 past N = 10, clipped at 9
    for b, w in enumerate(want):
        assert torch.nonzero(m[b]).flatten().tolist() == w, b


def test_window_step_picks_the_lowest_index_of_a_tie_and_masks_outside():
    score = torch.tensor([[5.0, 1.0, 3.0, 3.0, 9.0, 3.0],          # 9 at j = 4 lies outside the window around p = 1
                          [0.0, 2.0, 2.0, 1.0, 2.0, 0.0]], dtype=torch.float64)
    N = torch.tensor([6, 6])
    a, p, e = AW.window_step(score, N, torch.tensor([1, 2]), 0, 2)   # W = {1, 2, 3}, {2, 3, 4}
    assert p.tolist() == [2, 2]                                      # ties 3 = 3 at j = 2, 3 / 2 = 2 at j = 2, 4
    assert torch.equal(e[0], torch.tensor([-INF, 1.0, 3.0, 3.0, -INF, -INF], dtype=torch.float64))
    assert (a[0, [0, 4, 5]] == 0).all() and (a[1, [0, 1, 5]] == 0).all()
    assert torch.allclose(a.sum(1), torch.ones(2, dtype=torch.float64))
    ref = torch.softmax(torch.tensor([1.0, 3.0, 3.0], dtype=torch.float64), 0)
    assert torch.allclose(a[0, 1:4], ref, rtol=0, atol=1e-15)


def test_window_step_keeps_p_for_an_empty_row():
    a, p, _ = AW.window_step(torch.randn(2, 5, dtype=torch.float64), torch.tensor([0, 5]), torch.tensor([0, 0]), 1, 1)
    assert p[0].item() == 0 and (a[0] == 0).all()
    assert a[1, 2:].eq(0).all() and p[1].item() in (0, 1)


def _small_case(r=2, B=5, Tx=11, T=6, seed=0):
    cfg = ocfg(r=r, T=T, vocab=20)
    p = {k: v.double() for k, v in O.init_params(cfg, seed=1, trained_like=True).items()}
    encoded = (torch.randn(B, Tx, 256, generator=torch.Generator().manual_seed(seed)) * 0.5).double()
    tl = torch.tensor([Tx, 1, 3, Tx - 2, 7][:B], dtype=torch.int32)
    return cfg, p, encoded, tl


def test_first_step_starts_at_position_zero_and_peaks_move_within_the_window():
    cfg, p, encoded, tl = _small_case()
    back, ahead = 1, 2
    tr = {}
    y, a, pk = AW.decoder(encoded, tl, p, cfg, 6, (back, ahead), trace=tr)
    N = tl.to(torch.int64)
    assert (a[:, 0, ahead + 1:] == 0).all()                          # p(-1) = 0: step 0 sees positions 0..ahead only
    prev = torch.zeros(len(tl), dtype=torch.int64)
    for t in range(6):
        allowed = AW.window_mask(prev, N, encoded.shape[1], back, ahead)
        assert (a[:, t][~allowed] == 0).all()
        assert allowed.gather(1, pk[:, t:t + 1]).all()
        assert torch.equal(pk[:, t], torch.argmax(tr["score"][:, t], 1))
        prev = pk[:, t]
    assert torch.allclose(a.sum(-1), torch.ones_like(a.sum(-1)))


@pytest.mark.parametrize("window", [(10, 10), (50, 300)])
def test_window_covering_everything_is_the_plain_decoder(window):
    cfg, p, encoded, tl = _small_case()
    y, a, _ = AW.decoder(encoded, tl, p, cfg, 6, window)
    y0, a0 = O.decoder(encoded, tl, p, cfg, "infer", 6)
    assert torch.equal(y, y0) and torch.equal(a, a0)


def test_forced_peaks_build_the_window_around_them():
    cfg, p, encoded, tl = _small_case()
    forced = torch.tensor([[4] * 6] * len(tl))
    _, a, _ = AW.decoder(encoded, tl, p, cfg, 6, (0, 1), peaks=forced)
    N = tl.to(torch.int64)
    for t in range(1, 6):
        allowed = AW.window_mask(forced[:, t - 1], N, encoded.shape[1], 0, 1)
        assert (a[:, t][~allowed] == 0).all(), t


def test_top_two_gap():
    s = torch.tensor([[1.0, -INF, 0.5], [2.0, -INF, -INF]], dtype=torch.float64)
    assert AW.top_two_gap(s).tolist() == [0.5, INF]


# ---------------------------------------------------------------------------------------------------------------------
# ABI
# ---------------------------------------------------------------------------------------------------------------------
def test_window_fields_match_header():
    probe = r'''
#include <stdio.h>
#include <stddef.h>
#include "taco_b200.h"
int main(void){ printf("%zu %zu %zu %zu %zu\n", sizeof(taco_decoder_args), offsetof(taco_decoder_args, att0),
                       offsetof(taco_decoder_args, win_back), offsetof(taco_decoder_args, win_ahead),
                       offsetof(taco_decoder_args, peak)); return 0; }
'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c"); exe = os.path.join(d, "p")
        open(c, "w").write(probe)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = list(map(int, subprocess.check_output([exe]).split()))
    A = L.DecoderArgs
    assert got == [C.sizeof(A), A.att0.offset, A.win_back.offset, A.win_ahead.offset, A.peak.offset]
    assert A.win_back.offset > A.att0.offset                   # appended: the existing fields keep their offsets


def test_trace_offset_follows_the_workspace_layout():
    """the per-stage trace starts after the exchange buffers, the attention exchange and the window's peak words
    (decoder.cu build_ws_layout), inside the workspace the library sizes"""
    lib = L.lib()
    off = lib.taco_decoder_trace_offset()
    assert off == (10 * 32 + 48) * 4 * 64 + 32 * 2 * 4 * (2 + 256) + 32 * 2 * 4
    for T in (1, 200):
        assert (off + 16 * T + 16 + 4 * 20 * 8) * 8 <= lib.taco_decoder_workspace_bytes(32, 128, T, 5)


# ---------------------------------------------------------------------------------------------------------------------
# the launch loop over a fake library
# ---------------------------------------------------------------------------------------------------------------------
class _FakeLib:
    """records the window fields and the peak pointer of each taco_decoder_fwd call"""

    def __init__(self):
        self.calls = []

    def taco_decoder_fwd(self, aref, stream):
        a = aref._obj
        self.calls.append((a.row0, a.B, a.win_back, a.win_ahead, a.peak, a.align))
        return 0


def _launch(B, T, Tx, window, peak, max_ctas=None, capacity=132):
    t = {"packed": torch.zeros(16), "keys": torch.zeros(B, Tx, 256), "values": torch.zeros(B, Tx, 256),
         "text_length": torch.full((B,), Tx, dtype=torch.int32), "workspace": torch.zeros(16),
         "y": torch.zeros(B, T, 160), "align": torch.zeros(B, T, Tx)}
    if peak:
        t["peak"] = torch.zeros(B, T, dtype=torch.int32)
    lib = _FakeLib()
    plan = ops.decoder_plan(B, capacity, max_ctas)
    ops.decoder_fwd_launches(lib, plan, L.DecoderWeights(), t, L.DEC_INFER, T, 2, 1.0, max_ctas, None, window)
    return t, plan, lib.calls


@pytest.mark.parametrize("B,max_ctas", [(27, 32), (32, 64), (9, None)])
def test_launches_pass_window_and_peak_rows(B, max_ctas):
    T, Tx = 7, 13
    t, plan, calls = _launch(B, T, Tx, (2, 5), True, max_ctas)
    assert len(calls) == len(plan)
    base, esz = t["peak"].data_ptr(), t["peak"].element_size()
    for (b0, nb, _), (row0, n, back, ahead, peak, align) in zip(plan, calls):
        assert (row0, n, back, ahead) == (b0, nb, 2, 5)
        assert peak == base + b0 * T * esz                       # peak + b0, like align
        assert align == t["align"].data_ptr() + b0 * T * Tx * 4


def test_no_window_leaves_the_fields_zero():
    _, _, calls = _launch(27, 5, 9, None, False, 32)
    assert calls and all(c[2:5] == (0, 0, None) for c in calls)
    a = L.DecoderArgs()
    assert (a.win_back, a.win_ahead, a.peak) == (0, 0, None)


# ---------------------------------------------------------------------------------------------------------------------
# Config / CLI
# ---------------------------------------------------------------------------------------------------------------------
def test_config_default_is_off():
    from tacotron_b200 import Config
    assert Config().attention_window is None
    assert ops.attention_window(Config().attention_window) is None
    assert ops.attention_window(Config(attention_window=(2, 5)).attention_window) == (2, 5)


@pytest.mark.parametrize("window,ok", [((2, 5), (2, 5)), ([0, 1], (0, 1)), ((np.int64(3), 4), (3, 4)), ((300, 300), (300, 300)),
                                       ((2 ** 31 - 1, 2 ** 31 - 1), (2 ** 31 - 1, 2 ** 31 - 1))])
def test_window_accepted(window, ok):
    got = ops.attention_window(window)
    assert got == ok and all(type(v) is int for v in got)


@pytest.mark.parametrize("window,word", [((2, 0), "ahead"), ((-1, 5), "back"), ((2.0, 5), "back"), ((2, 5.5), "ahead"),
                                         ((True, 5), "back"), ((2, "5"), "ahead"), ((1, 2, 3), "expected"), (4, "expected"),
                                         ((2 ** 32 + 2, 5), "back must be <= 2147483647"),
                                         ((2, 2 ** 31), "ahead must be <= 2147483647")])
def test_window_rejected(window, word):
    with pytest.raises(L.TacoError, match=word):
        ops.attention_window(window)


def test_cli_parsing():
    from tacotron_b200.test import parse_attention_window
    assert parse_attention_window("2,5") == (2, 5)
    assert parse_attention_window("0,1") == (0, 1)
    for bad in ("2,0", "-1,5", "2", "a,b", "2.5,3", "1,2,3", ""):
        with pytest.raises(argparse.ArgumentTypeError):
            parse_attention_window(bad)


def test_cli_flag_forms(monkeypatch):
    """a bare flag means 2,5; no flag leaves the window off; a bad value exits with a usage error before any model"""
    from tacotron_b200 import test as drv
    seen = []
    monkeypatch.setattr(drv, "test", lambda cls, config, prompts, **kw: seen.append(config.attention_window))
    monkeypatch.setattr("sys.stdin", __import__("io").StringIO("hello\n"))
    drv.main(["-t", "x", "--attention-window"])
    drv.main(["-t", "x", "--attention-window", "1,3", "--long-form", "--trim-tail"])
    drv.main(["-t", "x"])
    assert seen == [(2, 5), (1, 3), None]
    with pytest.raises(SystemExit):
        drv.main(["-t", "x", "--attention-window", "3,0"])
    assert len(seen) == 3
