"""The case list of the taco_gemm envelope (tests/test_gpu_train_envelope.py on the device, tests/test_train_envelope_host.py
under the host emulation) and the operand layout each case runs with.

A case is one taco_gemm descriptor: sizes, transposes, beta, the row shift and its period, the K segments of a conv data
gradient, the batch strides, plus which operands are column slices of a wider buffer and how batched operands are packed.
Every row-major operand sits inside a larger buffer: GUARD rows before and after it, padding columns up to its row stride
and, for batched operands, a gap row between blocks.  Inputs are NaN there, so that a read outside the operand poisons the
result; the output is a sentinel bit pattern there, so that a write outside the view is seen.  The layout is a pure
function of the case, so the device test and the emulation build the same buffers.

`form()` reduces a descriptor to the addressing form the kernels see; tests/test_train_envelope_host.py records the forms
models/grad.py issues and asserts that each has a case here.  `split_k()` restates the split computation of taco_gemm."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field, replace

import torch

from tacotron_b200 import _lib as L

GUARD = 2
SENTINEL = 0x7FA5A5A5               # a quiet-NaN payload no kernel produces: every bit must survive
GBM, GBN, GBK = 64, 64, 16          # taco_gemm tile sizes (csrc/train.cu)


@dataclass(frozen=True)
class Case:
    name: str
    M: int
    N: int
    K: int                           # total K (taps * kper for the K-segmented form)
    ta: bool = False
    tb: bool = False
    beta: float = 0.0
    shift: int = 0
    period: int = 0
    taps: int = 1
    batch: int = 1
    a_pack: str = ""                 # batched operand packing: "" = shared by every batch entry (bstride 0),
    b_pack: str = ""                 # "block" = blocks one after the other, "inter" = time-major rows, entry z at
    c_pack: str = ""                 #   columns [z*width, (z+1)*width) of each row (DCTX[:, b])
    bshift: int = 0
    view: str = ""                   # operands ("C", "A", "B") that are column slices of a wider buffer
    pad: dict = field(default_factory=dict, compare=False, hash=False)   # extra padding columns per operand
    emu: dict = field(default_factory=dict, compare=False, hash=False)   # smaller sizes for the host emulation

    @property
    def kper(self):
        return self.K // self.taps if self.taps > 1 else 0

    @property
    def dshift(self):
        return -1 if self.taps > 1 else 0

    def for_emulation(self):
        return replace(self, **self.emu) if self.emu else self

    def form(self):
        return form(self.ta, self.tb, self.beta, self.shift, self.period, self.taps, self.batch, self.a_pack != "",
                    self.b_pack != "", self.c_pack != "", self.bshift, "C" in self.view, "A" in self.view, "B" in self.view)


def form(ta, tb, beta, shift, period, taps, batch, a_bs, b_bs, c_bs, bshift, c_view, a_view, b_view):
    return (bool(ta), bool(tb), float(beta), shift != 0, period > 0, taps > 1, batch > 1, bool(a_bs), bool(b_bs), bool(c_bs),
            bshift != 0, bool(c_view), bool(a_view), bool(b_view))


def split_k(M, N, K, batch, beta):
    """(splits, kchunk) as taco_gemm computes them: split-K only when accumulating (beta = 1) over K > 512"""
    tiles = -(-M // GBM) * -(-N // GBN) * batch
    s = 1
    if beta == 1.0 and K > 512:
        s = min(max(-(-444 // tiles), 1), -(-K // 256))
    kchunk = max(-(-(-(-K // s)) // GBK) * GBK, GBK)
    s = -(-K // kchunk) if K > 0 else 1
    return s, kchunk


def boundaries(c: Case):
    s, kchunk = split_k(c.M, c.N, c.K, c.batch, c.beta)
    return [j * kchunk for j in range(1, s)]


@dataclass
class Op:
    """one row-major operand: `rows` x `cols` at column col0 of rows `ld` apart, `nb` entries `bstride` apart"""
    rows: int
    cols: int
    ld: int
    col0: int = 0
    nb: int = 1
    bstride: int = 0

    @property
    def off(self):
        return GUARD * self.ld + self.col0

    @property
    def size(self):
        return self.off + max(self.nb - 1, 0) * self.bstride + self.rows * self.ld + GUARD * self.ld

    def view(self, buf, z=0):
        return torch.as_strided(buf, (self.rows, self.cols), (self.ld, 1), self.off + z * self.bstride)

    def mask(self, device=None):
        """bool [size]: the elements that belong to the operand (every batch entry)"""
        m = torch.zeros(self.size, dtype=torch.bool, device=device)
        for z in range(self.nb):
            self.view(m, z).fill_(True)
        return m


def _op(rows, cols, c: Case, name, pack, nb):
    pad = c.pad.get(name, 0) + (3 if name in c.view else 1)
    col0 = 2 if name in c.view else 0
    if nb > 1 and pack == "inter":
        return Op(rows, cols, nb * cols + col0 + pad, col0, nb, cols)
    ld = cols + col0 + pad
    if nb > 1:                                                  # "block" (and the taps of B): one gap row between entries
        return Op(rows, cols, ld, col0, nb, (rows + 1) * ld)
    return Op(rows, cols, ld, col0)


class Layout:
    def __init__(self, c: Case):
        kseg = c.kper if c.taps > 1 else c.K
        self.A = _op(c.K, c.M, c, "A", c.a_pack, c.batch if c.a_pack else 1) if c.ta else \
            _op(c.M, kseg, c, "A", c.a_pack, c.batch if c.a_pack else 1)
        if c.tb:
            nb = c.taps if c.taps > 1 else (c.batch if c.b_pack else 1)
            self.B = _op(c.N, kseg, c, "B", c.b_pack or "block", nb)
        else:
            self.B = _op(c.K, c.N, c, "B", c.b_pack, c.batch if c.b_pack else 1)
        self.C = _op(c.M, c.N, c, "C", c.c_pack, c.batch if c.c_pack else 1)

    def kwargs(self, c: Case):
        """keyword arguments of kernels.gemm / mirror_kernels.gemm for the views of entry 0"""
        kw = dict(ta=c.ta, tb=c.tb, beta=c.beta, shift=c.shift, period=c.period, taps=c.taps, dshift=c.dshift, kper=c.kper,
                  batch=c.batch, bshift=c.bshift, a_bstride=self.A.bstride if c.a_pack else 0,
                  b_bstride=self.B.bstride if c.b_pack else 0, c_bstride=self.C.bstride if c.c_pack else 0)
        kw["b_tap_stride"] = self.B.bstride if c.taps > 1 else 0
        return kw

    def desc(self, c: Case, a, b, cc):
        """GemmDesc for buffers at addresses a, b, cc (ints)"""
        d = L.GemmDesc()
        kw = self.kwargs(c)
        d.A = a + 4 * self.A.off; d.lda = self.A.ld
        d.B = b + 4 * self.B.off; d.ldb = self.B.ld
        d.C = cc + 4 * self.C.off; d.ldc = self.C.ld
        d.M, d.N, d.K = c.M, c.N, c.K
        d.ta, d.tb, d.beta = int(c.ta), int(c.tb), float(c.beta)
        d.shift, d.period, d.taps, d.dshift, d.kper = c.shift, c.period, c.taps, c.dshift, c.kper
        d.b_tap_stride = kw["b_tap_stride"]
        d.batch, d.a_bstride, d.b_bstride, d.c_bstride, d.bshift = c.batch, kw["a_bstride"], kw["b_bstride"], kw["c_bstride"], c.bshift
        return d


def call_gemm(lib, d, stream=None):
    rc = lib.taco_gemm(C.byref(d), stream)
    assert rc == 0, lib.taco_last_error().decode()


# ------------------------------------------------------------------------------------------------------------------
# the cases.  C2 training shape: B = 32 utterances, Tx = 128 characters (encoder rows 4096), T = 200 decoder steps
# (time-major rows 6400), r = 5 (post-net rows 32000, 1000 frames per utterance).
# ------------------------------------------------------------------------------------------------------------------
def _conv_dx(name, M, T, Cin, taps, kper, beta=0.0, view="", **kw):
    """data gradient of a conv1d('same'): dX[M, Cin] = sum_j dZ[m - tap0 - j] . W[j]^T (kernels.conv_dx)"""
    return Case(name, M, Cin, taps * kper, tb=True, beta=beta, shift=(taps - 1) // 2, period=T, taps=taps, view=view, **kw)


def _conv_dw(name, Cin, Cout, taps, T, rows, view="", **kw):
    """weight gradient of a conv1d('same') on the plain route: one batch entry per tap (grad.conv_bwd)"""
    return Case(name, Cin, Cout, rows, ta=True, beta=1.0, shift=-((taps - 1) // 2), period=T, batch=taps, c_pack="block",
                bshift=1, view=view, **kw)


def cases():
    out = []
    add = out.append
    # plain forms, edges, views
    add(Case("plain", 70, 45, 37))
    add(Case("beta1", 70, 45, 37, beta=1.0))
    add(Case("tb", 70, 45, 37, tb=True))
    add(Case("tb-beta1", 129, 65, 17, tb=True, beta=1.0))
    add(Case("ta", 70, 45, 37, ta=True))
    add(Case("ta-beta1", 65, 129, 300, ta=True, beta=1.0))
    add(Case("ta-tb", 70, 45, 37, ta=True, tb=True))
    add(Case("ta-tb-beta1", 70, 45, 37, ta=True, tb=True, beta=1.0))
    add(Case("K5", 70, 45, 5))
    add(Case("K0", 70, 45, 0))
    add(Case("K0-beta1", 70, 45, 0, beta=1.0))
    add(Case("M1", 1, 77, 33, beta=1.0))
    add(Case("N1", 67, 1, 33))
    add(Case("M1-N1-ta", 1, 1, 600, ta=True, beta=1.0))
    add(Case("view-C", 70, 45, 37, beta=1.0, view="C"))
    add(Case("view-CA", 70, 45, 37, beta=1.0, view="CA"))
    add(Case("view-AB-tb", 70, 45, 37, tb=True, view="AB"))                     # highway dX = dH . W_H^T
    add(Case("view-B-tb", 70, 45, 37, tb=True, beta=1.0, view="B"))
    add(Case("view-A-tb-beta1", 70, 45, 37, tb=True, beta=1.0, view="A"))       # dHin += dc . Wc^T
    add(Case("view-C-tb", 70, 45, 37, tb=True, view="C"))                       # d a(-1) = dz(0) . W_in^T
    add(Case("view-C-tb-beta1", 2, 128, 128, tb=True, beta=1.0, view="C"))      # ds_l += du . Wd^T
    add(Case("view-A-tb", 70, 45, 37, tb=True, view="A"))                       # dHin = dg . Wg^T
    add(Case("view-A-ta", 128, 128, 2, ta=True, beta=1.0, view="A"))            # dW += s_l^T . du
    add(Case("view-B-ta", 70, 45, 37, ta=True, beta=1.0, view="B"))             # dW from a [gates | cand] slice
    add(Case("view-AB-ta", 70, 45, 37, ta=True, beta=1.0, view="AB"))
    add(Case("view-B-ta-firststep", 128, 256, 32, ta=True, beta=1.0, view="B", pad={"B": 700}))   # dxp[:, first] rows
    # h(t-1) products: shift +-1 inside period blocks (bi-GRU), time-major shift = -B (decoder), first-step rows [:B]
    for sh in (-1, 1):
        add(Case(f"gru-gate-shift{sh:+d}", 130, 256, 128, beta=1.0, shift=sh, period=13, view="CA"))
        add(Case(f"gru-dWh-shift{sh:+d}", 128, 256, 130, ta=True, beta=1.0, shift=sh, period=13, view="AB"))
        add(Case(f"gru-dWh-shift{sh:+d}-Bview", 128, 256, 130, ta=True, beta=1.0, shift=sh, period=13, view="B"))
        add(Case(f"gru-gate-shift{sh:+d}-C2", 32000, 256, 128, beta=1.0, shift=sh, period=1000, view="CA",
                 emu=dict(M=250, period=125)))
    add(Case("dec-shift-B", 40, 512, 256, beta=1.0, shift=-4))
    add(Case("dec-shift-B-C2", 6400, 512, 256, beta=1.0, shift=-32, emu=dict(M=96, N=128)))
    add(Case("dec-dW-shift-B", 256, 512, 40, ta=True, beta=1.0, shift=-4))
    add(Case("dec-dW-shift-B-C2", 256, 512, 6400, ta=True, beta=1.0, shift=-32, emu=dict(M=64, N=64, K=1300)))
    add(Case("dec-firststep", 32, 512, 256, beta=1.0))
    add(Case("dec-firststep-ta", 256, 512, 32, ta=True, beta=1.0))
    # K-segmented conv data gradient: taps 1, 2, 3, 4, 7, 16 (even taps: tap0 = -(taps-1)//2 is not centred)
    for taps, kper, T in ((1, 128, 9), (2, 128, 9), (3, 24, 7), (4, 16, 9), (7, 80, 10), (16, 128, 9)):
        add(_conv_dx(f"conv-dx-k{taps}", 4 * T, 37, T, taps, kper))
        add(_conv_dx(f"conv-dx-k{taps}-beta1-bank", 4 * T, 37, T, taps, kper, beta=1.0, view="A"))
    add(_conv_dx("conv-dx-k3-beta1-viewC", 36, 9, 40, 3, 24, beta=1.0, view="C"))
    add(_conv_dx("conv-dx-k1-beta1", 20, 20, 256, 1, 256, beta=1.0))            # dense data gradient, accumulated
    add(_conv_dx("conv-dx-k5-T1", 3, 1, 8, 5, 16))                               # taps > T: every shifted row but one leaves
    add(_conv_dx("conv-dx-k3-enc-C2", 4096, 128, 256, 3, 128, beta=1.0, emu=dict(M=64, N=64, period=32)))
    add(_conv_dx("conv-dx-k3-post-C2", 32000, 1000, 256, 3, 256, beta=1.0, emu=dict(M=64, N=64, period=100)))
    # batched: attention context (per-utterance products), dvalues (time-major DCTX), conv dW (bshift = 1)
    add(Case("ctx-batched", 7, 256, 9, batch=3, a_pack="block", b_pack="block", c_pack="block"))
    add(Case("ctx-batched-C2", 200, 256, 128, batch=32, a_pack="block", b_pack="block", c_pack="block",
             emu=dict(M=20, K=16, batch=3)))
    add(Case("dvalues", 9, 256, 7, ta=True, batch=3, a_pack="block", b_pack="inter", c_pack="block", view="B"))
    add(Case("dvalues-C2", 128, 256, 200, ta=True, batch=32, a_pack="block", b_pack="inter", c_pack="block", view="B",
             emu=dict(M=16, K=20, batch=3)))
    for taps in (1, 2, 3, 4, 5):
        add(_conv_dw(f"conv-dw-k{taps}", 24, 16, taps, 40, 640))
    for taps in (1, 2, 3):
        add(_conv_dw(f"conv-dw-k{taps}-Bview", 24, 16, taps, 40, 640, view="B"))
    add(_conv_dw("conv-dw-k3-enc-C2", 128, 128, 3, 128, 4096, emu=dict(K=640, period=40)))
    # split-K: 1, 2 and >= 8 splits; chunk boundaries inside a period block and inside a tap segment
    add(Case("split2-bigtiles", 1024, 1024, 768, beta=1.0, emu=dict(M=64, N=64)))
    add(_conv_dx("split2-conv-dx-k3x256", 7100, 100, 128, 3, 256, beta=1.0, emu=dict(M=64, N=64)))
    add(_conv_dx("split3-conv-dx-k7x80", 64, 8, 64, 7, 80, beta=1.0))
    add(_conv_dx("split9-conv-dx-k16x130", 60, 6, 40, 16, 130, beta=1.0, view="A"))
    add(Case("split16-gru-dWh", 16, 64, 4000, ta=True, beta=1.0, shift=-1, period=125, view="AB"))
    add(Case("split56-gru-dWh-post-C2", 128, 256, 32000, ta=True, beta=1.0, shift=-1, period=1000, view="AB",
             emu=dict(M=16, N=64, K=4000, period=125)))
    add(Case("split56-gru-dWh-post-C2-bw", 128, 256, 32000, ta=True, beta=1.0, shift=1, period=1000, view="B",
             emu=dict(M=16, N=64, K=4000, period=125)))
    add(Case("split-dW-enc-C2", 128, 256, 4096, ta=True, beta=1.0, view="B", emu=dict(M=16, N=64, K=1000)))
    add(Case("split-ta-tb", 64, 64, 1000, ta=True, tb=True, beta=1.0))
    add(Case("split-tb-highway-dX", 64, 64, 1000, tb=True, beta=1.0, view="AB"))
    return out


CASES = cases()
