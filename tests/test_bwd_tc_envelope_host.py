"""The backward's wgmma routes on CPU (csrc/gemm_tc.cu is not emulated): which forms models/grad.py sends them, the
launch plan of taco_conv_dw, and whether the bars of tests/bwd_tc_envelope_checks.py can tell 3xTF32 from what a broken
kernel would compute.

* Route accounting: grad.py runs over the float64 mirror with a recorder (single-speaker, speaker and speaker-decoder
  models, r = 2 and 5, scheduled sampling on and off).  Each recorded gemm / conv_dx call is replayed on float32
  stand-ins with the same strides and offsets through kernels._dw_tc_ok, kernels._gemm_tc_ok and conv_dx's TMA test
  (row thresholds 1); every form that would take a wgmma route must have a case in tests/bwd_tc_envelope_cases.py.
* Launch plan: bwd_tc_envelope_cases.dw_plan against hand-worked plans, and the case list reaches every split-plan and
  dW-reduction edge.
* Bar sensitivity: a CPU model of the products (rn_tf32 restated with bit operations, fp32 accumulation per k8 step,
  chains added in fp32) passes the bar at every rand case at an 8 x 8 output; single-pass TF32, a model that drops one
  cross term and one that shifts X by one row fail it at every case.
* Layouts: guard layouts are disjoint from the operands.
"""
from contextlib import ExitStack
from dataclasses import replace
from unittest import mock

import pytest
import torch

from tacotron_b200 import kernels
from tests import bwd_tc_envelope_cases as BC
from tests import bwd_tc_envelope_checks as CH
from tests import mirror_kernels as MK
from tests import mirror_kernels_spkdec as MKD
from tests.test_train_envelope_host import _backward


# ------------------------------------------------------------------------------------------------------------------
# route accounting
# ------------------------------------------------------------------------------------------------------------------
def _f32(t):
    """a float32 tensor with t's shape, strides and storage offset (torch's CPU allocations are 64-byte aligned)"""
    n = t.untyped_storage().nbytes() // t.element_size()
    return torch.as_strided(torch.empty(n, dtype=torch.float32), t.shape, t.stride(), t.storage_offset())


def _slice(t):
    return t.shape[0] > 0 and t.stride(0) > 0 and t.storage_offset() % t.stride(0) != 0


def dw_form(batch, beta, period, shift, x_slice, z_slice):
    return ("dw", batch > 1, float(beta), period > 0, shift != 0, bool(x_slice), bool(z_slice))


def gemm_form(tb, beta, shift, period, a_slice, c_slice):
    return ("gemm", bool(tb), float(beta), shift != 0, period > 0, bool(a_slice), bool(c_slice))


def dx_form(taps, beta, z_slice):
    return ("dx", taps > 1, taps % 2 == 0, float(beta), bool(z_slice))


def case_forms():
    f = set()
    for c in BC.DW_CASES:
        if c.via == "gemm":
            f.add(dw_form(c.taps, c.beta, c.T if c.period else 0, c.t0, c.x_col0, c.z_col0))
    for c in BC.GEMM_CASES:
        f.add(gemm_form(c.tb, c.beta, c.shift, c.period, c.a_col0, c.c_col0))
    for c in BC.CONV_DX_CASES:
        if c.bank:
            f |= {dx_form(k, c.beta, True) for k in range(1, 9)}
        else:
            f.add(dx_form(c.taps, c.beta, False))
    return f


class _TcRecorder:
    """the mirror namespace; each gemm / conv_dx call that a wgmma route would take is reduced to its form"""

    def __init__(self, K):
        self.K, self.forms = K, {}

    def __getattr__(self, name):
        return getattr(self.K, name)

    def padded_rows(self, rows, cols, like):                   # kernels.padded_rows: pitch rounded up to 4 floats
        return torch.empty((rows, BC.up4(cols)), dtype=like.dtype)[:, :cols]

    def gemm(self, Cm, A, B, **kw):
        k = dict(ta=False, tb=False, beta=0.0, shift=0, period=0, taps=1, dshift=0, kper=0, batch=1, a_bstride=0,
                 b_bstride=0, c_bstride=0, bshift=0)
        k.update(kw)
        Cf, Af, Bf = _f32(Cm), _f32(A), _f32(B)
        if k["ta"]:
            if kernels._dw_tc_ok(Cf, Af, Bf, k["tb"], k["beta"], k["period"], k["taps"], k["dshift"], k["kper"], k["batch"],
                                 k["a_bstride"], k["b_bstride"], k["c_bstride"], k["bshift"]):
                f = dw_form(k["batch"], k["beta"], k["period"], k["shift"], _slice(A), _slice(B))
                self.forms.setdefault(f, (tuple(Cm.shape), tuple(A.shape), tuple(B.shape), kw))
        elif kernels._gemm_tc_ok(Cf, Af, Bf, k["beta"], k["period"], k["taps"], k["dshift"], k["kper"], k["batch"]):
            f = gemm_form(k["tb"], k["beta"], k["shift"], k["period"], _slice(A), _slice(Cm))
            self.forms.setdefault(f, (tuple(Cm.shape), tuple(A.shape), tuple(B.shape), kw))
        return self.K.gemm(Cm, A, B, **kw)

    def conv_dx(self, dX, dZ, W, T, beta=0.0):
        Zf = _f32(dZ)
        if (Zf.stride(0) * 4) % 16 == 0 and Zf.data_ptr() % 16 == 0 and dZ.shape[0] % T == 0:     # kernels.conv_dx's tma_ok
            self.forms.setdefault(dx_form(W.shape[0], beta, _slice(dZ)), (tuple(dX.shape), tuple(dZ.shape), tuple(W.shape)))
        return self.K.conv_dx(dX, dZ, W, T, beta=beta)


def test_every_wgmma_form_of_the_backward_has_a_case():
    rec = _TcRecorder(MKD)
    with ExitStack() as st:
        st.enter_context(mock.patch.object(kernels, "DW_TC_MIN_ROWS", 1))
        st.enter_context(mock.patch.object(kernels, "GEMM_TC_MIN_ROWS", 1))
        for kind in ("single", "speaker", "speaker_decoder"):
            for r in (2, 5):
                for sched in (True, False):
                    _backward(rec, kind, r, sched, B=2, Tx=8, T=8)
    kinds = {f[0] for f in rec.forms}
    assert kinds == {"dw", "gemm", "dx"} and len(rec.forms) >= 10, sorted(rec.forms)
    covered = case_forms()
    missing = {f: ex for f, ex in rec.forms.items() if f not in covered}
    assert not missing, "wgmma-routed forms without a case (form: shapes, arguments):\n" + \
        "\n".join(f"{f}: {ex}" for f, ex in missing.items())


# ------------------------------------------------------------------------------------------------------------------
# launch plan
# ------------------------------------------------------------------------------------------------------------------
def test_dw_plan_hand_worked():
    p = BC.dw_plan(32, 1000, 1024, 256, 3)            # post-net projection at C2: 8 x 2 x 3 tiles, 132 // 48 = 2 splits
    assert (p.tiles, p.splits, p.per_split, p.total_blocks) == (48, 2, 512, 1024)
    assert len(p.chains()) == 32 and p.chains()[16] == (512, 544)
    p = BC.dw_plan(3, 200, 80, 80, 1)                 # 1 tile, 3 x 7 blocks: one block per split
    assert (p.splits, p.per_split, p.total_blocks) == (21, 1, 21)
    p = BC.dw_plan(32, 200, 80, 128, 3)               # 44 splits asked, 6 blocks each -> 38 splits, the last of 2
    assert (p.tiles, p.splits, p.per_split, p.n_iters[-1]) == (3, 38, 6, 2)
    p = BC.dw_plan(1, 1025, 1024, 1028, 1)            # 72 tiles: one split of 33 blocks, chains 32 + 1
    assert (p.tiles, p.splits, p.chains()) == (72, 1, [(0, 32), (32, 33)])
    lay = BC.DwLayout(BC.DwCase("x", 1, 1, 80, 128, taps=3, dw_off=1))
    assert lay.vec2 == 0 and BC.DwLayout(BC.DwCase("x", 1, 1, 80, 128, taps=3)).vec2 == 1


def test_cases_reach_every_plan_edge():
    plans = [(c, BC.plan_of(c), BC.DwLayout(c)) for c in BC.DW_CASES]
    assert any(p.splits == 1 for _, p, _ in plans)
    assert any(p.splits == p.total_blocks > 1 for _, p, _ in plans)
    assert any(p.n_iters[-1] < p.per_split for _, p, _ in plans), "no short last split"
    one = {p.per_split for _, p, _ in plans if p.splits == 1}
    assert {31, 32, 33} <= one and max(p.per_split for _, p, _ in plans) > 64
    assert any(len(p.chains()) > p.splits for _, p, _ in plans), "no CTA with several drains"
    assert any(c.N % 2 and lay.vec2 for c, _, lay in plans), "odd N on the vec2 path"
    assert any(lay.ldw % 2 and not lay.vec2 for c, _, lay in plans)
    assert any(c.taps > 1 and lay.tap_stride % 2 and not lay.vec2 for c, _, lay in plans)
    for via in ("direct", "gemm"):
        assert any(c.via == via and lay.W.off % 2 and not lay.vec2 for c, _, lay in plans), via
    assert {c.C % 128 for c in BC.DW_CASES} >= {0, 1, 127} and {c.N % 128 for c in BC.DW_CASES} >= {0, 1, 127}
    assert {c.T % 32 for c in BC.DW_CASES} >= {0, 1, 31} and {c.B for c in BC.DW_CASES} >= {1, 3, 32}
    assert {c.taps for c in BC.DW_CASES} >= {1, 2, 3, 4, 7, 8, 16}
    assert {c.M for c in BC.GEMM_CASES} >= {2047, 2048, 2049, 32000}
    assert {c.taps for c in BC.CONV_DX_CASES} >= set(range(1, 9)) | {16}
    assert {c.impl for c in BC.CONV_DX_CASES} == {"fp32x3", "tf32"}


def test_layouts_are_disjoint_and_guarded():
    ops = []
    for c in BC.DW_CASES:
        lay = BC.DwLayout(c)
        ops += [lay.X, lay.Z, lay.W]
        assert lay.X.ld % 4 == 0 and lay.Z.ld % 4 == 0 and lay.X.col0 % 4 == 0 and lay.Z.col0 % 4 == 0, c.name
    for c in BC.GEMM_CASES:
        lay = BC.GemmLayout(c)
        ops += [lay.A, lay.B, lay.C]
        assert lay.A.ld % 4 == 0 and lay.C.ld % 4 == 0 and lay.A.col0 % 4 == 0 and lay.C.col0 % 4 == 0, c.name
    for c in BC.CONV_DX_CASES:
        lay = BC.ConvDxLayout(c)
        ops += [lay.Z, lay.X]
        assert lay.Z.ld % 4 == 0 and (lay.X.ld % 4 != 0) == c.ldy_odd, c.name
    for op in ops:
        m = op.mask()
        assert int(m.sum()) == op.nb * op.rows * op.cols                       # entries do not overlap
        assert not bool(m[:op.off - op.col0].any()) and not bool(m[-BC.GUARD * op.ld:].any())
        assert op.ld > op.col0 + op.cols or op.nb > 1                          # a padding column after every row


# ------------------------------------------------------------------------------------------------------------------
# the sequences restate the mirror, and the bar's sensitivity on a CPU model of the products
# ------------------------------------------------------------------------------------------------------------------
def test_sequences_restate_the_mirror():
    g = CH.gen(5)
    for c in [BC.DwCase("a", 3, 37, 5, 4, taps=4), BC.DwCase("b", 1, 70, 5, 4, tap0=-3, period=False)]:
        X, Z = torch.randn(c.rows, c.C, generator=g).double(), torch.randn(c.rows, c.N, generator=g).double()
        ref = torch.zeros(c.taps * c.C, c.N, dtype=torch.float64)
        MK.gemm(ref[:c.C], X, Z, ta=True, beta=1.0, shift=c.t0, period=c.T if c.period else 0, batch=c.taps, bshift=1,
                c_bstride=c.C * c.N)
        for j in range(c.taps):
            out = CH.contraction(*CH.dw_sequences(c, X, Z, j), torch.zeros(c.C, c.N, dtype=torch.float64))[0]
            torch.testing.assert_close(out, ref[j * c.C:(j + 1) * c.C], rtol=1e-12, atol=1e-12)
    for c in [BC.GemmCase("g", 40, 37, 8, tb=True, shift=-1, period=10), BC.GemmCase("h", 40, 33, 8, shift=-4)]:
        A = torch.randn(c.M, c.Kc, generator=g).double()
        Bm = torch.randn(*((c.N, c.Kc) if c.tb else (c.Kc, c.N)), generator=g).double()
        ref = torch.zeros(c.M, c.N, dtype=torch.float64)
        MK.gemm(ref, A, Bm, tb=c.tb, shift=c.shift, period=c.period)
        out = CH.contraction(*CH.gemm_sequences(c, A, Bm), torch.zeros(c.M, c.N, dtype=torch.float64))[0]
        torch.testing.assert_close(out, ref, rtol=1e-12, atol=1e-12)
    for taps in (1, 2, 3, 4, 5, 16):
        T, B, Cin, Cout = 9, 2, 5, 40
        dZ = torch.randn(B * T, Cout, generator=g).double()
        W = torch.randn(taps, Cin, Cout, generator=g).double()
        ref = torch.zeros(B * T, Cin, dtype=torch.float64)
        MK.conv_dx(ref, dZ, W, T)
        out = CH.contraction(*CH.conv_dx_sequences(T, dZ, W), torch.zeros(B * T, Cin, dtype=torch.float64))[0]
        torch.testing.assert_close(out, ref, rtol=1e-12, atol=1e-12)


def test_rn_tf32_bits():
    x = torch.tensor([1.0, 1.0 + 2 ** -11, 1.0 + 2 ** -11 - 2 ** -23, -(1.0 + 2 ** -11), 3.0e-39, 0.0])
    got = CH.rn_tf32(x)
    assert got.tolist() == [1.0, 1.0 + 2 ** -10, 1.0, -(1.0 + 2 ** -10), CH.rn_tf32(torch.tensor([3.0e-39])).item(), 0.0]
    assert (got.view(torch.int32) & 0x1FFF == 0).all()


def _model(As, Bs, chains, init, kind):
    """fp32 result of a route modelled on the CPU: 3xTF32 products ("x3"), single-pass TF32 ("single"), or 3xTF32 without
    the hi.lo term ("drop"); each k8 step's products summed exactly, added into an fp32 accumulator; chains added in fp32"""
    ah, bh = CH.rn_tf32(As.float()), CH.rn_tf32(Bs.float())
    al, bl = CH.rn_tf32(As.float() - ah), CH.rn_tf32(Bs.float() - bh)
    terms = {"x3": [(al, bh), (ah, bl), (ah, bh)], "single": [(ah, bh)], "drop": [(al, bh), (ah, bh)]}[kind]
    terms = [(a.double(), b.double()) for a, b in terms]
    out = init.float()
    for k0, k1 in chains:
        acc = torch.zeros_like(out)
        for s in range(k0, k1, 8):
            p = sum(a[s:s + 8].t() @ b[s:s + 8] for a, b in terms)
            acc = (acc.double() + p).float()
        out = (out.double() + acc.double()).float()
    return out.double()


W8 = 8          # output columns / rows of the model: the bar is per element, the plan comes from the full case


def _sens_inputs(c, g):
    """(As, Bs, chains, init, As shifted by one row) of a random-class case at an 8 x 8 (dw) or 8-column output"""
    if isinstance(c, BC.DwCase):
        X, Z = torch.randn(c.rows, W8, generator=g), torch.randn(c.rows, W8, generator=g)
        j = min(c.taps - 1, max(0, -c.t0))                    # the tap with no shift (T = 1 leaves no other row)
        As, Bs, ch = CH.dw_sequences(c, X.double(), Z.double(), j)
        As1 = CH.dw_sequences(c, X.double(), Z.double(), j, extra_shift=1)[0]
        init = torch.randn(W8, W8, generator=g).double()
    elif isinstance(c, BC.GemmCase):
        A = torch.randn(c.M, c.Kc, generator=g)
        Bm = torch.randn(*((W8, c.Kc) if c.tb else (c.Kc, W8)), generator=g)
        cc = replace(c, N=W8)
        As, Bs, ch = CH.gemm_sequences(cc, A.double(), Bm.double())
        As1 = CH.gemm_sequences(cc, A.double(), Bm.double(), extra_shift=1)[0]
        sel = torch.arange(0, c.M, max(1, c.M // 64))[:64]
        As, As1 = As[:, sel], As1[:, sel]
        init = torch.randn(len(sel), W8, generator=g).double() * float(c.beta)
    else:
        lay = BC.ConvDxLayout(c)
        Z = torch.randn(lay.Z.rows, c.Cout if not c.bank else 128, generator=g).double()
        taps = 8 if c.bank else c.taps
        W = torch.randn(taps, W8, Z.shape[1], generator=g).double()
        As, Bs, ch = CH.conv_dx_sequences(c.T, Z, W)
        As1 = CH.conv_dx_sequences(c.T, Z, W, extra_shift=1)[0]
        sel = torch.arange(0, As.shape[1], max(1, As.shape[1] // 64))[:64]
        As, As1 = As[:, sel], As1[:, sel]
        init = torch.randn(len(sel), W8, generator=g).double() * float(c.beta)
    f32 = lambda t: t.float().double()
    return f32(As), f32(Bs), ch, f32(init), f32(As1)


SENS_CASES = BC.DW_CASES + BC.GEMM_CASES + [c for c in BC.CONV_DX_CASES if c.impl == "fp32x3"]


@pytest.mark.parametrize("case", SENS_CASES, ids=[f"{type(c).__name__}-{c.name}" for c in SENS_CASES])
def test_bar_sensitivity(case):
    As, Bs, chains, init, As1 = _sens_inputs(case, CH.gen(11))
    ref, rss, A, S = CH.contraction(As, Bs, chains, init)
    ratio = lambda got: CH.unit_ratio(got, ref, rss, A)
    w = ratio(_model(As, Bs, chains, init, "x3"))
    assert w <= CH.C_BAR / 4, f"3xTF32 model at {w:.3f} of the unit bar (C_BAR {CH.C_BAR})"
    for kind in ("single", "drop"):
        w = ratio(_model(As, Bs, chains, init, kind))
        assert w > CH.C_BAR, f"{kind} passes the bar: {w:.2f} <= {CH.C_BAR}"
    w = ratio(_model(As1, Bs, chains, init, "x3"))
    assert w > CH.C_BAR, f"X shifted by one row passes the bar: {w:.2f}"
