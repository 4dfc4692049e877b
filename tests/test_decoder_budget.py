"""Decoder launches under a CTA budget (no GPU): the launch plan of ops.decoder_plan for the capacities of the Hopper parts
and budgets a user may set, the refusals below one 32-CTA row group, the new ABI fields against the header, and
ops.decoder_fwd_launches over a host mirror of the kernel's row indexing (strided [T][B] masks and h_save rows land where
a single launch puts them)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from tacotron_b200 import _lib as L
from tacotron_b200.models import ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAPACITIES = [132, 128, 114, 96, 78, 64, 32]     # H100 SXM, a full-launch budget, H100 PCIe, and smaller budgets / slices


@pytest.mark.parametrize("cap", CAPACITIES)
def test_plan(cap):
    groups = min(4, cap // 32)
    for B in range(1, 65):
        plan = ops.decoder_plan(B, cap)
        rows = 8 * groups
        assert len(plan) == -(-B // rows), (cap, B)
        b = 0
        for b0, nb, ctas in plan:
            assert b0 == b and 1 <= nb <= rows
            assert ctas == 32 * groups and ctas <= min(cap, 128) and ctas >= 32 * -(-nb // 8)   # within the budget, covers nb
            b += nb
        assert b == B
        assert all(nb == rows for _, nb, _ in plan[:-1])
    # the launches of today's full H100 at the C2 batch: one launch of 128 CTAs
    assert ops.decoder_plan(32, 132) == [(0, 32, 128)]
    assert ops.decoder_plan(64, 132) == [(0, 32, 128), (32, 32, 128)]


def test_plan_examples():
    assert ops.decoder_plan(1, 132) == [(0, 1, 128)]                        # C5: the full grid, as before budgets existed
    assert ops.decoder_plan(25, 132) == [(0, 25, 128)]
    assert ops.decoder_plan(1, 114) == [(0, 1, 96)]
    assert ops.decoder_plan(32, 114) == [(0, 24, 96), (24, 8, 96)]          # H100 PCIe
    assert ops.decoder_plan(32, 78) == [(0, 16, 64), (16, 16, 64)]
    assert ops.decoder_plan(9, 32) == [(0, 8, 32), (8, 1, 32)]
    # a budget caps the capacity; None and 0 mean the capacity; a budget above it changes nothing
    assert ops.decoder_plan(32, 132, 96) == ops.decoder_plan(32, 114)
    assert ops.decoder_plan(32, 132, 64) == ops.decoder_plan(32, 64)
    assert ops.decoder_plan(32, 132, None) == ops.decoder_plan(32, 132, 0) == ops.decoder_plan(32, 132, 1000)
    assert ops.decoder_plan(32, 64, 132) == ops.decoder_plan(32, 64)


def test_budget_below_one_row_group_is_refused():
    with pytest.raises(L.TacoError, match="max_ctas=31"):
        ops.decoder_plan(1, 132, 31)
    with pytest.raises(L.TacoError, match="only 31"):
        ops.decoder_plan(1, 31)
    with pytest.raises(L.TacoError):
        ops.decoder_budget(132, 1)
    assert ops.decoder_budget(132, 32) == 32 and ops.decoder_budget(114) == 114


def test_struct_fields_match_header():
    """offsets of the new fields (and the sizes) of both decoder argument structs, from gcc against the header"""
    probe = r'''
#include <stdio.h>
#include <stddef.h>
#include "taco_b200.h"
int main(void){ printf("%zu %zu %zu %zu %zu %zu %zu\n", sizeof(taco_decoder_args), offsetof(taco_decoder_args, row0),
                       offsetof(taco_decoder_args, row_stride), offsetof(taco_decoder_args, max_ctas),
                       sizeof(taco_decoder_bwd_args), offsetof(taco_decoder_bwd_args, max_ctas),
                       offsetof(taco_decoder_bwd_args, workspace)); return 0; }
'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c"); exe = os.path.join(d, "p")
        open(c, "w").write(probe)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = list(map(int, subprocess.check_output([exe]).split()))
    A, Bw = L.DecoderArgs, L.DecoderBwdArgs
    assert got == [C.sizeof(A), A.row0.offset, A.row_stride.offset, A.max_ctas.offset, C.sizeof(Bw), Bw.max_ctas.offset,
                   Bw.workspace.offset]


def test_capacity_is_exported():
    assert "taco_decoder_capacity" in L.EXPORTS
    assert hasattr(L.lib(), "taco_decoder_capacity")


# ---------------------------------------------------------------------------------------------------------------------
# the launch loop over a host mirror of the kernel's indexing
# ---------------------------------------------------------------------------------------------------------------------
class _MirrorLib:
    """taco_decoder_fwd on host memory with the kernel's row indexing: launch row b is full-batch row row0 + b of the
    [T][B]-major tensors (row_stride rows per step) and row b of the [B]-major ones.  Writes, for every (b, t):
    y[b,t,:4] = (sample_mask, keep1[.., 5], keep2[.., 7], keys[b,0,0]) as read, y[b,t,4:] = b (the launch's row), align[b,t,:] = values[b,0,0],
    h_save[i,t,row0+b,:] = keys[b,0,0] + i.  Applies the host checks of taco_decoder_fwd (rows inside the stride, B within
    8 x (budget // 32)) and records each launch's grid."""

    def __init__(self, capacity):
        self.capacity = capacity
        self.grids = []

    def taco_decoder_fwd(self, aref, stream):
        a = aref._obj
        B, T, Tx, RS, R0 = a.B, a.T, a.Tx, a.row_stride, a.row0
        out = 80 * a.r
        assert 0 <= R0 and R0 + B <= RS
        budget = min(a.max_ctas, self.capacity) if a.max_ctas else self.capacity
        groups = min(4, budget // 32)
        assert budget >= 32 and B <= 8 * groups
        self.grids.append(32 * groups)
        arr = lambda addr, n, ct: np.ctypeslib.as_array((ct * n).from_address(addr))
        keys = arr(a.keys, B * Tx * 256, C.c_float).reshape(B, Tx, 256)
        values = arr(a.values, B * Tx * 256, C.c_float).reshape(B, Tx, 256)
        y = arr(a.y, B * T * out, C.c_float).reshape(B, T, out)
        align = arr(a.align, B * T * Tx, C.c_float).reshape(B, T, Tx)
        sm = arr(a.sample_mask, T * RS, C.c_uint8) if a.sample_mask else None
        k1 = arr(a.keep1, T * RS * 256, C.c_uint8) if a.keep1 else None
        k2 = arr(a.keep2, T * RS * 128, C.c_uint8) if a.keep2 else None
        hs = arr(a.h_save, 3 * T * RS * 256, C.c_float) if a.h_save else None
        for b in range(B):
            for t in range(T):
                o = t * RS + R0 + b
                y[b, t, 0] = sm[o] if sm is not None else -1
                y[b, t, 1] = k1[o * 256 + 5] if k1 is not None else -1
                y[b, t, 2] = k2[o * 128 + 7] if k2 is not None else -1
                y[b, t, 3] = keys[b, 0, 0]
                y[b, t, 4:] = b
                align[b, t, :] = values[b, 0, 0]
                if hs is not None:
                    for i in range(3):
                        base = ((i * T + t) * RS + R0 + b) * 256
                        hs[base:base + 256] = keys[b, 0, 0] + i
        return 0


def _run_mirror(B, T, Tx, capacity, max_ctas, sched=True, save=True):
    g = torch.Generator().manual_seed(B)
    t = {"packed": torch.zeros(16), "keys": torch.randn(B, Tx, 256, generator=g), "text_length": torch.full((B,), Tx, dtype=torch.int32),
         "workspace": torch.zeros(16), "y": torch.full((B, T, 160), float("nan")), "align": torch.full((B, T, Tx), float("nan")),
         "mel": torch.zeros(B, T, 160), "keep1": (torch.rand(T, B, 256, generator=g) < 0.5).to(torch.uint8),
         "keep2": (torch.rand(T, B, 128, generator=g) < 0.5).to(torch.uint8)}
    t["values"] = t["keys"] * 2
    if sched:
        t["sample_mask"] = (torch.rand(T, B, generator=g) < 0.5).to(torch.uint8)
    if save:
        t["h_save"] = torch.full((3, T, B, 256), float("nan"))
    lib = _MirrorLib(capacity)
    plan = ops.decoder_plan(B, capacity, max_ctas)
    ops.decoder_fwd_launches(lib, plan, L.DecoderWeights(), t, L.DEC_SCHED if sched else L.DEC_TEACHER, T, 2, 2.0, max_ctas, None)
    assert lib.grids == [c for _, _, c in plan]
    return t


@pytest.mark.parametrize("B,capacity,max_ctas", [(27, 132, 64), (27, 132, 32), (32, 114, None), (9, 132, 32), (25, 78, None),
                                                 (64, 132, 96)])
def test_launch_slicing_over_mirror(B, capacity, max_ctas):
    T, Tx = 5, 7
    save = B <= 32
    t = _run_mirror(B, T, Tx, capacity, max_ctas, save=save)
    one = _run_mirror(B, T, Tx, 10 ** 6 if B <= 32 else capacity, None, save=save)      # one launch (B <= 32)
    for k in ("y", "align") + (("h_save",) if save else ()):
        assert not torch.isnan(t[k]).any(), k
        assert torch.equal(t[k][..., :4] if k == "y" else t[k], one[k][..., :4] if k == "y" else one[k]), k
    # and what each row read is that row's mask entry
    y = t["y"]
    assert torch.equal(y[:, :, 0], t["sample_mask"].t().float())
    assert torch.equal(y[:, :, 1], t["keep1"][:, :, 5].t().float())
    assert torch.equal(y[:, :, 2], t["keep2"][:, :, 7].t().float())
    assert torch.equal(y[:, :, 3], t["keys"][:, 0, 0][:, None].expand(B, T))
    rows = torch.cat([torch.arange(nb, dtype=torch.float32) for _, nb, _ in ops.decoder_plan(B, capacity, max_ctas)])
    assert torch.equal(y[:, :, 4:], rows[:, None, None].expand(B, T, 156))         # the launches' rows cover the batch once
    if save:
        want = t["keys"][:, 0, 0][None, None, :, None] + torch.arange(3.0)[:, None, None, None]
        assert torch.equal(t["h_save"], want.expand(3, T, B, 256))
