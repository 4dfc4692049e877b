"""The case list of the backward's wgmma routes (tests/test_gpu_zz_bwd_tc_envelope.py on the device,
tests/test_bwd_tc_envelope_host.py on CPU) and the operand layout each case runs with.

Three routes, each reached the way models/grad.py reaches it in 'fp32x3' / 'tf32' mode:
  DwCase      taco_conv_dw (dw_tc_kernel), called directly or through kernels.gemm(..., ta=True):
              dW[j][c][n] += sum_{b,t} X[b, t+tap0+j, c] dZ[b, t, n]
  GemmCase    kernels._gemm_tc (kernels.gemm, ta=False): Y (+)= shift(X) . W (tb: W^T) on taco_linear_fwd, the
              accumulation being the kernel's residual input with residual = Y
  ConvDxCase  kernels.conv_dx on taco_linear_fwd: dZ convolved with the taps reversed and the weights transposed
Every input sits in a NaN guard buffer (GUARD rows before and after, NaN padding columns between the operand's width and
its row pitch, and NaN columns before a column slice); row pitches of the TMA operands are multiples of 4 floats.  Every
output sits in sentinel bits (train_envelope_cases.SENTINEL) that must survive.

`dw_plan()` restates taco_conv_dw_tc_impl's launch plan (csrc/gemm_tc.cu): tiles, splits, rows per split, the 1024-row
chains of each split and the vec2 reduction switch."""
from __future__ import annotations

from dataclasses import dataclass

from tacotron_b200 import _lib as L
from tests.train_envelope_cases import GUARD, SENTINEL, Op  # noqa: F401  (SENTINEL: re-exported for the checks)

TACO_SMS = 132                  # csrc/common.cuh
KB = 32                         # rows (dw) / channels (linear) per k-block
DW_DRAIN = 32                   # k-blocks per chain of dw_tc_kernel


def up4(n):
    return (n + 3) // 4 * 4


def tf_tap0(taps):
    return -((taps - 1) // 2)


# ------------------------------------------------------------------------------------------------------------------
# taco_conv_dw
# ------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class DwCase:
    name: str
    B: int
    T: int
    C: int
    N: int
    taps: int = 1
    tap0: int | None = None      # None: TF's -((taps-1)//2)
    beta: float = 1.0            # 0: kernels.gemm zeroes dW first (the direct call always accumulates)
    via: str = "gemm"            # "gemm" = kernels.gemm(..., ta=True), "direct" = lib.taco_conv_dw
    period: bool = True          # False: kernels.gemm gets period = 0 (the decoder's time-major rows: B must be 1)
    x_col0: int = 0              # X / dZ as column slices of a wider buffer (multiples of 4: 16-byte aligned)
    z_col0: int = 0
    ldw_odd: bool = False
    ts_odd: bool = False
    dw_off: int = 0              # dW's first element this many floats past an 8-byte boundary

    @property
    def t0(self):
        return tf_tap0(self.taps) if self.tap0 is None else self.tap0

    @property
    def rows(self):
        return self.B * self.T


class DwLayout:
    def __init__(self, c: DwCase):
        self.X = Op(c.rows, c.C, up4(c.x_col0 + c.C + 1 + (3 if c.x_col0 else 0)), c.x_col0)
        self.Z = Op(c.rows, c.N, up4(c.z_col0 + c.N + 1 + (3 if c.z_col0 else 0)), c.z_col0)
        ldw = c.N + 1
        if ldw % 2 != int(c.ldw_odd):
            ldw += 1
        ts = (c.C + 1) * ldw
        if ts % 2 != int(c.ts_odd):
            ts += 1
        self.ldw, self.tap_stride = ldw, ts
        self.W = Op(c.C, c.N, ldw, c.dw_off, c.taps, ts)        # col0 = dw_off: off = GUARD*ldw + dw_off (GUARD even)
        assert GUARD % 2 == 0

    @property
    def vec2(self):
        return int(self.W.off % 2 == 0 and self.ldw % 2 == 0 and self.tap_stride % 2 == 0)


@dataclass(frozen=True)
class DwPlan:
    tiles: int
    splits: int
    per_split: int
    total_blocks: int
    blocks_per_seq: int

    def split_blocks(self):
        """[(g0, g1)) of every split (grid.y)"""
        return [(s * self.per_split, min(self.total_blocks, (s + 1) * self.per_split)) for s in range(self.splits)]

    def chains(self):
        """[(g0, g1)) of every chain: DW_DRAIN k-blocks from the start of its split, then a drain into dW"""
        return [(a, min(g1, a + DW_DRAIN)) for g0, g1 in self.split_blocks() for a in range(g0, g1, DW_DRAIN)]

    @property
    def n_iters(self):
        return [g1 - g0 for g0, g1 in self.split_blocks()]


def dw_plan(B, T, C, N, taps):
    """taco_conv_dw_tc_impl's plan"""
    tiles = -(-C // 128) * -(-N // 128) * taps
    bps = -(-T // KB)
    total = B * bps
    splits = min(max(TACO_SMS // tiles, 1), total)
    per = -(-total // splits)
    splits = -(-total // per)
    return DwPlan(tiles, splits, per, total, bps)


def plan_of(c: DwCase):
    return dw_plan(c.B, c.T, c.C, c.N, c.taps)


def dw_deterministic(c: DwCase):
    """one split of at most DW_DRAIN k-blocks: one reduction into each dW element, so the result is a pure function of the
    inputs.  Otherwise the order of the atomics decides the last bits (not a law)."""
    p = plan_of(c)
    return p.splits == 1 and p.total_blocks <= DW_DRAIN


def dw_cases():
    out = []
    add = lambda name, *a, **kw: out.append(DwCase(name, *a, **kw))
    # C and N through the tile edges, both entry points
    for C, N in ((1, 1), (3, 2), (80, 3), (127, 80), (128, 127), (129, 128), (256, 129), (1024, 768), (80, 1028)):
        for via in ("direct", "gemm"):
            add(f"CN-{C}x{N}-{via}", 3, 200, C, N, taps=1, via=via)
    # T through the k-block edges, B in {1, 3, 32}
    for T in (1, 31, 32, 33, 200, 1000, 1025):
        add(f"T{T}-B3", 3, T, 80, 128, taps=3)
    add("T33-B1", 1, 33, 128, 80, taps=3)
    add("T200-B32", 32, 200, 128, 128, taps=1, beta=0.0)
    # taps (TF tap0) and beta 0 through kernels.gemm
    for taps in (1, 2, 3, 4, 7, 8, 16):
        add(f"taps{taps}", 2, 70, 128, 128, taps=taps, beta=0.0)
        add(f"taps{taps}-beta1-C80", 3, 33, 80, 128, taps=taps)
    # bi-GRU h(t-1) products: shift +-1 inside periods; the decoder's shift = -B over the time-major rows
    for sh in (-1, 1):
        add(f"gru-shift{sh:+d}", 32, 200, 128, 256, tap0=sh, x_col0=0, z_col0=256)
        add(f"gru-shift{sh:+d}-T1000", 4, 1000, 128, 256, tap0=sh, z_col0=256)
    add("dec-shift-B32", 1, 6400, 256, 512, tap0=-32, period=False, x_col0=256)
    add("dec-shift-B3", 1, 600, 256, 128, tap0=-3, period=False, x_col0=128, z_col0=256)
    # split plan edges
    add("splits1-iters31", 1, 992, 1024, 1028, via="direct")      # 72 tiles: one split of 31 k-blocks
    add("splits1-iters32", 1, 1024, 1024, 1028, via="direct")
    add("splits1-iters33", 1, 1025, 1024, 1028, via="direct")
    add("splits1-iters99", 3, 1025, 1024, 1028)                   # 3 chains in one CTA
    add("splits-all", 3, 200, 80, 80)                             # 1 tile, 21 blocks: a split per block
    add("split-short-last", 32, 200, 80, 128, taps=3)             # 3 tiles: 38 splits of 6 blocks, the last of 2
    # vec2 both ways
    add("vec2-oddN", 3, 200, 80, 129)
    add("vec2-odd-ldw", 3, 200, 80, 128, ldw_odd=True)
    add("vec2-odd-tapstride", 3, 200, 80, 128, taps=3, ts_odd=True)
    add("vec2-dw-off1", 3, 200, 80, 128, taps=3, dw_off=1, via="direct")
    add("vec2-dw-off1-gemm", 3, 200, 80, 128, taps=3, dw_off=1)
    # column slices (bank gradient dZ[:, k*128:(k+1)*128], GRU [gates | cand])
    add("bank-slice", 3, 200, 80, 128, taps=4, z_col0=384)
    add("gru-gates-cand-slice", 4, 250, 128, 256, tap0=-1, x_col0=128, z_col0=512)
    # dense weight gradients over flat rows (period 0), plain and as slices
    add("dense", 1, 600, 256, 128, period=False)
    add("dense-zslice", 1, 600, 128, 128, period=False, z_col0=128)
    add("dense-xslice", 1, 600, 128, 128, period=False, x_col0=128)
    add("dense-xzslice", 1, 600, 128, 128, period=False, x_col0=128, z_col0=256)
    add("dec-shift-B2", 1, 600, 256, 512, tap0=-2, period=False)
    for sh in (-1, 1):
        add(f"gru-shift{sh:+d}-noslice", 4, 150, 128, 256, tap0=sh)
    add("bank-slice-k2", 3, 200, 80, 128, taps=2, z_col0=128)
    # the C2 post-net projection gradient: 3 x 1024 -> 256 over 32 x 1000 rows (48 tiles, 2 splits of 512 blocks)
    add("post-proj-C2", 32, 1000, 1024, 256, taps=3)
    return out


# ------------------------------------------------------------------------------------------------------------------
# kernels._gemm_tc and kernels.conv_dx on taco_linear_fwd
# ------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class GemmCase:
    name: str
    M: int
    Kc: int
    N: int
    tb: bool = False
    beta: float = 0.0
    shift: int = 0
    period: int = 0
    impl: str = "fp32x3"         # DX_TC_IMPL: "fp32x3" (TACO_IMPL_TC3) or "tf32" (TACO_IMPL_TC)
    a_col0: int = 0
    c_col0: int = 0


class GemmLayout:
    def __init__(self, c: GemmCase):
        self.A = Op(c.M, c.Kc, up4(c.a_col0 + c.Kc + 1), c.a_col0)
        self.B = Op(c.N, c.Kc, c.Kc + 1) if c.tb else Op(c.Kc, c.N, c.N + 1)
        self.C = Op(c.M, c.N, c.c_col0 + c.N + 4, c.c_col0)


def gemm_cases():
    out = []
    add = lambda *a, **kw: out.append(GemmCase(*a, **kw))
    for M in (2047, 2048, 2049):
        add(f"M{M}", M, 128, 128)
        add(f"M{M}-tb-beta1", M, 256, 80, tb=True, beta=1.0)
    add("gru-gate-shift-1", 32000, 128, 768, beta=1.0, shift=-1, period=1000)
    add("gru-gate-shift+1", 32000, 128, 768, beta=1.0, shift=1, period=1000)
    add("gru-dh-shift-1-tb", 4000, 256, 128, tb=True, beta=1.0, shift=-1, period=125, a_col0=256)
    add("dec-shift-32", 6400, 256, 512, beta=1.0, shift=-32, c_col0=512)
    add("dec-shift-32-tb", 6400, 512, 256, tb=True, shift=-32, a_col0=128)
    add("highway-dx", 32000, 128, 128, tb=True, beta=1.0, a_col0=128, c_col0=128)
    add("recompute-wide", 4096, 1024, 256, tb=False)
    add("plain-beta1", 2048, 256, 256, beta=1.0)
    add("plain-beta1-cslice", 2048, 128, 128, beta=1.0, c_col0=128)
    add("plain-beta1-acslice", 2048, 128, 128, beta=1.0, a_col0=128, c_col0=256)
    add("shift-period-acslice", 2048, 128, 256, beta=1.0, shift=1, period=16, a_col0=128, c_col0=256)
    add("shift-2-beta1", 2048, 256, 256, beta=1.0, shift=-2)
    add("tb-beta0", 2048, 256, 128, tb=True)
    add("tb-beta1-aslice", 2048, 128, 128, tb=True, beta=1.0, a_col0=128)
    add("tb-beta1-cslice", 2048, 128, 128, tb=True, beta=1.0, c_col0=128)
    add("tf32-shift+1", 4000, 256, 128, beta=1.0, shift=1, period=200, impl="tf32")
    return out


@dataclass(frozen=True)
class ConvDxCase:
    name: str
    B: int
    T: int
    Cin: int
    Cout: int
    taps: int = 3
    beta: float = 0.0
    impl: str = "fp32x3"
    bank: bool = False           # dZ = slices of the 8 x 128 bank gradient, accumulated over k = 1..8 (taps ignored)
    ldy_odd: bool = False        # dX row pitch not a multiple of 4: the transposing epilogue


class ConvDxLayout:
    def __init__(self, c: ConvDxCase):
        M = c.B * c.T
        self.Z = Op(M, 8 * 128, 8 * 128 + 4) if c.bank else Op(M, c.Cout, up4(c.Cout + 1))
        self.X = Op(M, c.Cin, up4(c.Cin) + 4 + (1 if c.ldy_odd else 0))

    def z_slices(self, c: ConvDxCase):
        """(taps, column of the slice) per conv_dx call"""
        return [(k, (k - 1) * 128) for k in range(1, 9)] if c.bank else [(c.taps, 0)]


def conv_dx_cases():
    out = []
    add = lambda *a, **kw: out.append(ConvDxCase(*a, **kw))
    for impl in ("fp32x3", "tf32"):
        for taps in (1, 2, 3, 4, 5, 6, 7, 8, 16):
            add(f"k{taps}-{impl}", 3, 129, 128, 128, taps=taps, beta=float(taps % 2), impl=impl)
        add(f"bank-{impl}", 2, 300, 80, 128, bank=True, beta=1.0, impl=impl)
        add(f"ldy-odd-{impl}", 3, 130, 80, 256, taps=3, ldy_odd=True, impl=impl)
    add("enc-proj-C2", 32, 128, 128, 256, taps=3, beta=1.0)
    add("post-proj-C2", 32, 1000, 256, 256, taps=3)
    add("T1-k5", 3, 1, 80, 128, taps=5)
    add("dense-1025-beta0", 3, 257, 256, 1025, taps=1)
    add("Cout1028-k1", 3, 257, 128, 1028, taps=1, beta=1.0)
    return out


DW_CASES = dw_cases()
GEMM_CASES = gemm_cases()
CONV_DX_CASES = conv_dx_cases()
IMPL = {"fp32x3": L.IMPL_TC3, "tf32": L.IMPL_TC}
