"""The case list of tests/test_gpu_linear_envelope.py and the operand layout each case runs with.

A case is one taco_linear_fwd descriptor shape: sizes, taps / bank / highway, the epilogue fields, and which epilogue
(register-direct or transposing) its strides and alignment select.  Every row-major operand sits inside a larger buffer:
GUARD rows before and after it and padding columns up to its row stride, so that a read outside the operand meets NaN
and a write outside the output changes a sentinel.  The layout is a pure function of the case, so the route the
library picks for it (taco_linear_route) is the same for the device buffers of the GPU test and for the stand-in
addresses of the CPU test (tests/test_linear_routes.py)."""
from __future__ import annotations

from dataclasses import dataclass, field, replace

from tacotron_b200 import _lib as L

GUARD = 2                                  # NaN / sentinel rows before and after every row-major operand
IMPL = {"fp32": L.IMPL_SIMT, "tf32": L.IMPL_TC, "fp32x3": L.IMPL_TC3}
TC_IMPLS = ("tf32", "fp32x3")
FEATURES = ("plain", "keep", "residual", "pool", "bias_utt")


def _up4(n):
    return (n + 3) // 4 * 4


def cpad(c):
    return (c + 31) // 32 * 32


@dataclass
class Case:
    name: str
    B: int
    T: int
    C: int
    N: int                       # output channels of the contraction (highway: 2U)
    taps: int = 1
    tap0: str = "tf"             # "tf" = -(taps-1)//2 (TF 'same'), "zero" = 0, "left" = -(taps-1)
    bank_K: int = 0              # > 0: conv bank, N = 128 bank_K
    highway: bool = False
    act: int = L.ACT_RELU
    bias: bool = True
    bn: bool = False             # batch-norm affine (scale, shift)
    keep: bool = False
    residual: bool = False
    bias_utt: bool = False
    pool: bool = False
    transposing: str = ""        # "" = register-direct layout; else what forces the transposing epilogue:
                                 # "ldy" (ldy % 4 != 0), "y_align" (Y 4 bytes off 16), "ldr", "ldhx", "n4" (N % 4 != 0),
                                 # "keep16" (keep with N % 16 != 0)
    impls: tuple = ("fp32", "tf32", "fp32x3")
    tc: dict = field(default_factory=dict)   # expected (bn, stages) per tensor-core impl, where the case pins it

    @property
    def classes(self):
        # sigmoid, tanh and the highway gate are not exact in fp32: those cases run the float class only
        exact_ok = not self.highway and self.act in (L.ACT_NONE, L.ACT_RELU)
        return ("exact", "float") if exact_ok else ("float",)

    @property
    def tap0_value(self):
        return {"tf": -((self.taps - 1) // 2), "zero": 0, "left": -(self.taps - 1)}[self.tap0]

    @property
    def nout(self):
        return self.N // 2 if self.highway else self.N

    def features(self):
        f = {n for n in FEATURES[1:] if getattr(self, n)}
        return f or {"plain"}


class Layout:
    """Row strides, buffer sizes and operand offsets (in elements) of a case."""

    def __init__(self, c: Case):
        M = c.B * c.T
        self.M = M
        self.ldx = _up4(c.C + 1)                                   # >= 1 NaN column, 16-byte rows
        self.ldy = _up4(c.nout) + 4 + (1 if c.transposing == "ldy" else 0)
        self.y_off = GUARD * self.ldy + (1 if c.transposing == "y_align" else 0)
        self.y_size = (M + 2 * GUARD) * self.ldy + 4
        self.ldr = _up4(c.N) + 4 + (2 if c.transposing == "ldr" else 0)
        self.ldhx = 128 + 8 + (1 if c.transposing == "ldhx" else 0)
        self.ldbu = c.N + 3
        self.max_taps = c.bank_K if c.bank_K else c.taps
        self.ldwp = self.max_taps * cpad(c.C)
        # (rows, row stride, offset of row 0) of every padded operand
        self.shapes = {
            "X": (M, self.ldx, GUARD * self.ldx),
            "residual": (M, self.ldr, GUARD * self.ldr),
            "hx": (M, self.ldhx, GUARD * self.ldhx),
            "bias_utt": (c.B, self.ldbu, self.ldbu),
        }

    def size(self, name):
        rows, ld, _ = self.shapes[name]
        return (rows + 2 * GUARD) * ld


def desc(c: Case, impl: str, addr: dict, lay: Layout | None = None, keep_scale: float = 2.0):
    """LinearDesc of case c for impl, from the addresses (ints, operand row 0) in addr."""
    lay = lay or Layout(c)
    d = L.LinearDesc()
    d.X = addr["X"]; d.ldx = lay.ldx; d.B = c.B; d.T = c.T; d.C = c.C
    d.taps = c.taps; d.tap0 = c.tap0_value; d.N = c.N
    d.bank_K = c.bank_K; d.bank_cout = 128 if c.bank_K else 0
    d.W = addr.get("W"); d.Wp = addr.get("Wp"); d.ldwp = lay.ldwp
    d.Y = addr["Y"]; d.ldy = lay.ldy
    d.bias = addr.get("bias") if c.bias else None
    d.act = L.ACT_NONE if c.highway else c.act
    if c.bn:
        d.scale = addr["scale"]; d.shift = addr["shift"]
    if c.keep:
        d.keep = addr["keep"]
    d.keep_scale = keep_scale
    if c.residual:
        d.residual = addr["residual"]; d.ldr = lay.ldr
    if c.highway:
        d.epilogue = L.EPI_HIGHWAY; d.hx = addr["hx"]; d.ldhx = lay.ldhx
    d.pool = 1 if c.pool else 0
    if c.bias_utt:
        d.bias_utt = addr["bias_utt"]; d.ldbu = lay.ldbu
    d.impl = IMPL[impl]
    return d


def stand_in_addresses(c: Case, lay: Layout | None = None):
    """Addresses with the alignment the GPU test's buffers have (each buffer 4 KB aligned, operands at their offsets):
    enough for taco_linear_route, which only looks at pointer alignment."""
    lay = lay or Layout(c)
    base = iter(range(1 << 40, 1 << 41, 1 << 32))
    a = {name: next(base) + 4 * off for name, (_, _, off) in lay.shapes.items()}
    a.update(Y=next(base) + 4 * lay.y_off, W=next(base), Wp=next(base), bias=next(base), scale=next(base),
             shift=next(base), keep=next(base))
    return a


def route(c: Case, impl: str):
    """(bn, stages, mode, direct, tile_stride) that taco_linear_route reports for case c."""
    return L.linear_route(desc(c, impl, stand_in_addresses(c)))


def check_route(c: Case, impl: str, r):
    bn, stages, mode, direct, tile_stride = r
    assert mode == (1 if c.highway else 0), (c.name, impl, r)
    assert direct == (0 if (c.transposing or impl == "fp32") else 1), (c.name, impl, r)
    if impl != "fp32":
        assert tile_stride == (127 if c.pool else 128), (c.name, impl, r)
        if c.highway:
            assert (bn, stages) == (256, 2), (c.name, impl, r)
        if impl in c.tc:
            assert (bn, stages) == c.tc[impl], (c.name, impl, r, c.tc[impl])


def instantiation(impl, r):
    bn, stages, mode, _, _ = r
    return (impl, bn, stages, mode)


# ------------------------------------------------------------------------------------------------------------------
# the grid
# ------------------------------------------------------------------------------------------------------------------
S, TH, R, NO = L.ACT_SIGMOID, L.ACT_TANH, L.ACT_RELU, L.ACT_NONE

# epilogue field combinations: each field alone, and the combinations the model uses (pre-net: relu + dropout; conv
# projections: relu + BN (+ residual); speaker conditioning: bias_utt with any of them)
COMBOS = [
    ("none", dict(act=NO)), ("nobias", dict(act=R, bias=False)), ("relu", dict(act=R)), ("sigmoid", dict(act=S)),
    ("tanh", dict(act=TH)), ("keep", dict(act=NO, keep=True)), ("relu_keep", dict(keep=True)),
    ("res", dict(act=NO, residual=True)), ("bn", dict(act=NO, bn=True)), ("relu_bn_res", dict(bn=True, residual=True)),
    ("bu", dict(act=NO, bias_utt=True)), ("bu_relu_bn", dict(bias_utt=True, bn=True)), ("bu_keep", dict(bias_utt=True, keep=True)),
    ("bu_res", dict(act=NO, bias_utt=True, residual=True)), ("sig_bn_bu", dict(act=S, bn=True, bias_utt=True)),
    ("tanh_keep", dict(act=TH, keep=True)), ("tanh_bn_res", dict(act=TH, bn=True, residual=True)),
    ("relu_all", dict(bn=True, keep=True, residual=True, bias_utt=True)),
    ("sig_all", dict(act=S, bn=True, keep=True, residual=True, bias_utt=True)),
]
POOL_COMBOS = [
    ("pool", dict(act=NO, pool=True)), ("pool_relu_bn", dict(bn=True, pool=True)),
    ("pool_bu_relu_bn", dict(bias_utt=True, bn=True, pool=True)), ("pool_tanh_bn", dict(act=TH, bn=True, pool=True)),
]

# two shape families that between them reach every normal-epilogue instantiation:
#   A: conv 7 taps, C = 33 (2 k-chunks, 14 k-iterations), N = 80 (N % 32 = 16), 6 m-tiles: fp32x3 takes the 32-column
#      n-tiles (3 with the fused pool, which they do not serve), tf32 the 3-stage ring
#   B: dense C = 256 (8 k-iterations), N = 128, 96 m-tiles: 128-column tiles with the 2-stage ring in both modes
FAMILIES = {
    "A": (dict(B=3, T=129, C=33, N=80, taps=7), {"tf32": (128, 3), "fp32x3": (32, 6)}, {"tf32": (128, 3), "fp32x3": (128, 2)}),
    "B": (dict(B=32, T=257, C=256, N=128, taps=1), {"tf32": (128, 2), "fp32x3": (128, 2)}, {"tf32": (128, 2), "fp32x3": (128, 2)}),
}


def cases():
    out = []

    def add(name, **kw):
        c = Case(name=name, **kw)
        if c.pool:                                       # the fused max-pool is a tensor-core feature
            c = replace(c, impls=tuple(i for i in c.impls if i != "fp32"))
        out.append(c)

    # 1. every epilogue field and combination on both families, register-direct and transposing
    for fam, (shape, tc, tc_pool) in FAMILIES.items():
        for cname, fields in COMBOS + POOL_COMBOS:
            pool = fields.get("pool", False)
            for tr in ("", "ldy"):
                add(f"{fam}-{cname}-{tr or 'direct'}", **shape, **fields, transposing=tr, tc=tc_pool if pool else tc)
        add(f"{fam}-relu-y_align", **shape, transposing="y_align", tc=tc)
        add(f"{fam}-relu_bn_res-ldr", **shape, bn=True, residual=True, transposing="ldr", tc=tc)
        add(f"{fam}-pool_relu_bn-y_align", **shape, bn=True, pool=True, transposing="y_align", tc=tc_pool)

    # 2. dropout keep mask at N % 32 = 16 (the last 16-column half of a row) and N % 16 != 0 (transposing only)
    add("keep-N48-direct", B=3, T=129, C=32, N=48, keep=True, bias_utt=True)
    add("keep-N48-ldy", B=3, T=129, C=32, N=48, keep=True, transposing="ldy")
    add("keep-N8", B=3, T=2, C=8, N=8, keep=True, transposing="keep16")
    add("keep-N1025", B=1, T=257, C=256, N=1025, keep=True, residual=True, transposing="n4")
    add("keep-bank-K8", B=3, T=130, C=80, N=8 * 128, bank_K=8, keep=True, bn=True)    # bank without pool

    # 3. shapes: channels, widths, lengths, batch, taps (also > T) and tap offsets
    for i, (B, T, C, N, taps, tap0) in enumerate([
            (3, 1, 1, 48, 1, "tf"), (3, 2, 8, 80, 3, "tf"), (32, 2, 8, 128, 5, "zero"), (3, 1, 31, 8, 4, "left"),
            (1, 127, 31, 8, 2, "tf"), (3, 128, 32, 128, 4, "left"), (3, 129, 33, 80, 7, "zero"), (1, 255, 80, 256, 5, "tf"),
            (3, 256, 128, 768, 1, "tf"), (1, 257, 256, 1025, 1, "tf"), (32, 128, 1024, 128, 3, "tf"),
            (32, 128, 2048, 128, 3, "tf"), (3, 257, 2048, 256, 3, "left"), (3, 257, 1024, 256, 3, "zero"),
            (32, 1000, 80, 256, 1, "tf"), (32, 1000, 128, 768, 1, "tf"), (8, 1000, 256, 1025, 1, "tf"),
            (3, 1000, 256, 128, 2, "left"), (1, 2, 33, 48, 7, "left"), (32, 1, 80, 80, 5, "tf")]):
        tr = "n4" if N % 4 else ""
        add(f"shape{i}-{B}x{T}x{C}->{N}-k{taps}{tap0}", B=B, T=T, C=C, N=N, taps=taps, tap0=tap0, bn=(i % 2 == 0),
            transposing=tr)
        if i % 3 == 0 and not tr:
            add(f"shape{i}-{B}x{T}x{C}->{N}-k{taps}{tap0}-ldy", B=B, T=T, C=C, N=N, taps=taps, tap0=tap0, act=NO,
                residual=True, transposing="ldy")

    # 4. fused max-pool over t on a plain conv: tiles advance by 127 rows; row 127 of a tile only at the sequence end
    for T in (1, 2, 126, 127, 128, 129, 253, 254, 255, 256, 381):
        N = 80 if T % 2 else 128
        add(f"pool-conv-T{T}", B=3, T=T, C=80, N=N, taps=3, bn=True, pool=True)
        if T in (2, 127, 254, 381):
            add(f"pool-conv-T{T}-ldy", B=3, T=T, C=80, N=N, taps=3, bn=True, pool=True, bias_utt=True, transposing="ldy")

    # 5. conv banks (filter k: k taps, tap0 = -(k-1)//2), fused pool, at the pooled tile edges
    for K, C, T, B, tr in ((1, 80, 1, 3, ""), (2, 128, 2, 3, "ldy"), (4, 80, 126, 3, ""), (8, 80, 127, 1, ""),
                           (16, 128, 128, 3, ""), (8, 128, 129, 3, "ldy"), (4, 32, 253, 1, ""), (2, 33, 254, 3, ""),
                           (16, 80, 255, 1, "y_align"), (8, 31, 256, 3, ""), (16, 128, 381, 3, ""), (1, 8, 129, 32, "")):
        add(f"bank-K{K}-C{C}-T{T}-B{B}-{tr or 'direct'}", B=B, T=T, C=C, N=128 * K, bank_K=K, bn=True, pool=True,
            bias_utt=(K == 4), transposing=tr)
    add("bank-K8-nopool", B=2, T=300, C=80, N=8 * 128, bank_K=8, bn=True)
    add("bank-K16-nopool-ldy", B=3, T=129, C=128, N=16 * 128, bank_K=16, bn=True, bias_utt=True, transposing="ldy")

    # 6. highway (float class): U = 128, ldhx and ldy > 128
    for M in (1, 127, 128, 129, 40000):
        add(f"highway-M{M}", B=1, T=M, C=128, N=256, highway=True)
    add("highway-M129-ldy", B=1, T=129, C=128, N=256, highway=True, transposing="ldy")
    add("highway-M40000-ldhx", B=1, T=40000, C=128, N=256, highway=True, transposing="ldhx")
    add("highway-B3-ldhx", B=3, T=129, C=128, N=256, highway=True, transposing="ldhx", bias=False)
    return out


CASES = cases()
