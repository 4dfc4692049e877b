"""The case list of the fused CBHG highway stack (taco_highway_stack_fwd, csrc/gemm_tc.cu highway_stack_kernel), run on
the device by tests/test_gpu_highway_stack_envelope.py and on a CPU mirror by tests/test_highway_stack_envelope_host.py.

A case is one descriptor: rows M, input width C (1..128; C != 128 adds the width-fixing dense), highway layers L (1..4)
and the five row strides.  A stride of 0 means its minimum (ldx: round_up(C, 4), ldy: 768, ldwd: round_up(C, 32),
ldhw / ldxp: 128).  The list covers:
  * every C residue mod 32, with the layer-0 k-blocks kin = ceil(C / 32) crossed with every L (the producer cursor's
    ring phase depends on both);
  * M around the 128-row tile and the tile counts either side of each xp split boundary of taco_highway_stack_split
    (6 / 3 / 2 / 1 CTAs per tile), the last tile partial;
  * each stride at its minimum, minimum + 4 and a larger value;
  * the model's shapes (C2 encoder 32 x 128 rows, C2 post-net 32 x 1000, C5 500 / 140) and one case whose output
    passes 2^31 elements (checked on its first and last tiles)."""
from __future__ import annotations

from dataclasses import dataclass

BM = 128                # rows per tile (HS_BM)
XP_N = 768              # bi-GRU input products per row
SMS = 132               # TACO_SMS
GUARD = 2               # guard rows before and after every buffer
BIG_M = 2_796_203       # M * 768 > 2^31


def split_of(M):
    """xp column splits per tile, as taco_highway_stack_split computes them: the most of 6, 3, 2 that keep every CTA on
    its own SM, else 1"""
    tiles = -(-M // BM)
    for s in (6, 3, 2):
        if tiles * s <= SMS:
            return s
    return 1


def _r(n, m):
    return -(-n // m) * m


@dataclass(frozen=True)
class Case:
    name: str
    M: int
    C: int
    L: int = 4
    ldx: int = 0
    ldy: int = 0
    ldwd: int = 0
    ldhw: int = 0
    ldxp: int = 0

    @property
    def dense(self):
        return self.C != 128

    @property
    def Cpad(self):
        return _r(self.C, 32)

    @property
    def kin(self):
        return self.Cpad // 32

    @property
    def lds(self):
        """(ldx, ldy, ldwd, ldhw, ldxp) with the minimum for every 0"""
        return (self.ldx or _r(self.C, 4), self.ldy or XP_N, self.ldwd or self.Cpad, self.ldhw or 128, self.ldxp or 128)

    @property
    def split(self):
        return split_of(self.M)

    @property
    def big(self):
        """checked on its first and last tiles only"""
        return self.M >= BIG_M

    def check_rows(self):
        """the rows the float64 check covers"""
        if not self.big:
            return [(0, self.M)]
        last = (self.M - 1) // BM * BM
        return [(0, BM), (last, self.M)]


def _cases():
    out = []
    # C sweep at 257 rows (3 tiles, the last one row long), every L for C = 80 and C = 128
    for C in (1, 4, 31, 32, 33, 64, 80, 95, 96, 97, 127, 128):
        out.append(Case(f"C{C}_M257", 257, C))
    for C in (80, 128):
        for L in (1, 2, 3):
            out.append(Case(f"C{C}_L{L}", 300, C, L))
    # every residue r of C mod 32; kin = r % 4 + 1 and L = (r // 4) % 4 + 1 cross every (kin, L) pair
    for r in range(32):
        C = (r or 32) + 32 * (r % 4)
        out.append(Case(f"res{r}_C{C}_L{(r // 4) % 4 + 1}", 129 + 2 * r, C, (r // 4) % 4 + 1))
    # rows around the tile
    for M in (0, 1, 15, 16, 17, 127, 128, 129, 257):
        out.append(Case(f"M{M}_C80", M, 80))
        out.append(Case(f"M{M}_C128", M, 128))
    # tile counts either side of each split boundary (22 / 23, 44 / 45, 66 / 67 tiles), the last tile partial, with and
    # without the width-fixing dense
    for i, tiles in enumerate((22, 23, 44, 45, 66, 67)):
        C, L = (80, 33, 97)[i % 3], i % 3 + 1
        out.append(Case(f"tiles{tiles}_C128", tiles * BM - 37, 128))
        out.append(Case(f"tiles{tiles}_C{C}_L{L}", tiles * BM - 37, C, L))
    # the model's shapes
    out += [Case("C2_encoder", 32 * 128, 128), Case("C2_postnet", 32 * 1000, 80),
            Case("C5_postnet", 500, 80), Case("C5_encoder", 140, 128)]
    # strides: minimum + 4 and a larger value, each alone
    for field, vals in (("ldx", (84, 200)), ("ldy", (772, 1024)), ("ldwd", (100, 160)), ("ldhw", (132, 256)),
                        ("ldxp", (132, 200))):
        for v in vals:
            out.append(Case(f"{field}{v}_C80", 300, 80, **{field: v}))
    out += [Case("ldx8_C1", 300, 1, ldx=8), Case("ldx40_C33", 300, 33, ldx=40),
            Case("all_lds_C97", 700, 97, 3, ldx=104, ldy=800, ldwd=132, ldhw=160, ldxp=136)]
    out.append(Case("big_C4", BIG_M, 4))
    return out


CASES = _cases()


def host_cases():
    """the cases the CPU mirror runs: every case up to 700 rows"""
    return [c for c in CASES if 0 < c.M <= 700]
