"""-m gpu: the fused CBHG highway stack (taco_highway_stack_fwd) over its whole envelope (tests/highway_stack_envelope_cases.py)
against float64 (tests/highway_stack_envelope_checks.py for the reference, the classes and the bar).  For every case:
  * the exact class equals float64 rounded once, bit for bit; the float class stays within the bar;
  * the result equals the unfused route (taco_linear_fwd: dense, each highway layer, the xp products) bit for bit, the
    same packed weights at the same strides;
  * a second run gives the same bits; NaN rows of X give all-NaN xp rows on both routes and leave the other rows' bits;
  * X sits in NaN bands (guard rows, and columns [C, ldx)), the packed weights have NaN in their columns past the ones
    the kernel reads, and Y sits in sentinel bits: rows past M, columns [768, ldy) and the guard rows must survive;
  * one launch per call, none for M = 0.
Descriptors the kernel cannot run are refused with a message, no launch and Y untouched.

The case past 2^31 output elements (M = 2 796 203) is checked on its first and last tiles and needs about 9 GB free."""
import ctypes as C
import json
import os
from types import SimpleNamespace

import pytest
import torch

from tacotron_b200 import _lib as L
from tests import highway_stack_envelope_cases as HC
from tests import highway_stack_envelope_checks as CH
from tests.train_envelope_cases import SENTINEL

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(WORST):
        print(f"HIGHWAY_STACK {k}: {WORST[k]:.4f}")
    path = os.environ.get("TACO_ENVELOPE_LOG")
    if path and WORST:
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        with open(path, "w") as f:
            json.dump({"worst": WORST, "c_hw": CH.C_HW}, f, indent=1)


def _sentinel(n):
    return torch.full((n,), SENTINEL, dtype=torch.int32, device=DEV).view(torch.float32)


class Run:
    """the device buffers of one case and class: X in NaN bands, packed weights with NaN past the columns the kernel
    reads, biases, and a sentinel Y of round_up(M, 128) rows between guard rows"""

    def __init__(self, c: HC.Case, X, p):
        self.c = c
        ldx, ldy, ldwd, ldhw, ldxp = c.lds
        self.ldx, self.ldy = ldx, ldy
        self.Xbuf = torch.full(((c.M + 2 * HC.GUARD) * ldx,), NAN, device=DEV)
        self.xview().copy_(X.to(DEV))
        self.p = {k: ([t.to(DEV) for t in v] if isinstance(v, list) else v.to(DEV)) for k, v in p.items()}
        self.Wd_p = self._pack(self.p["Wd"], ldwd) if c.dense else None
        self.hw_p = [self._pack(W, ldhw) for W in self.p["Whw"]]
        self.xp_p = self._pack(self.p["Wx"], ldxp)
        self.Yrows = HC._r(max(c.M, 1), HC.BM) + 2 * HC.GUARD

    def _pack(self, W, ld):
        K, N = W.shape
        buf = torch.full((2 * N, ld), NAN, device=DEV)
        L.check(L.lib().taco_pack_weight_x3(L.ptr(W), 1, K, N, L.ptr(buf), C.c_void_p(buf.data_ptr() + N * ld * 4), ld,
                                            L.current_stream()), "taco_pack_weight_x3")
        return buf

    def xview(self, buf=None):
        buf = self.Xbuf if buf is None else buf
        return torch.as_strided(buf, (self.c.M, self.c.C), (self.ldx, 1), HC.GUARD * self.ldx)

    def new_y(self):
        return _sentinel(self.Yrows * self.ldy)

    def yview(self, Y, r0=0, r1=None):
        r1 = self.c.M if r1 is None else r1
        return torch.as_strided(Y, (r1 - r0, HC.XP_N), (self.ldy, 1), (HC.GUARD + r0) * self.ldy)

    def desc(self, Y, X=None):
        c = self.c
        d = L.HighwayStackDesc()
        d.X = (self.Xbuf if X is None else X).data_ptr() + 4 * HC.GUARD * self.ldx
        d.ldx = self.ldx; d.M = c.M; d.C = c.C
        if c.dense:
            d.Wd_p = self.Wd_p.data_ptr(); d.ldwd = self.Wd_p.stride(0); d.bd = self.p["bd"].data_ptr()
        d.L = c.L
        for l in range(c.L):
            d.hw_p[l] = self.hw_p[l].data_ptr(); d.hw_b[l] = self.p["bhw"][l].data_ptr()
        d.ldhw = self.hw_p[0].stride(0)
        d.xp_p = self.xp_p.data_ptr(); d.ldxp = self.xp_p.stride(0); d.xp_b = self.p["bx"].data_ptr()
        d.Y = Y.data_ptr() + 4 * HC.GUARD * self.ldy; d.ldy = self.ldy
        d.impl = L.IMPL_TC3
        return d

    def fused(self, X=None):
        """one call into a fresh sentinel Y: (Y, launches)"""
        Y = self.new_y()
        n0 = L.lib().taco_launch_count()
        rc = L.lib().taco_highway_stack_fwd(C.byref(self.desc(Y, X)), L.current_stream())
        assert rc == 0, L.lib().taco_last_error().decode()
        torch.cuda.synchronize()
        return Y, L.lib().taco_launch_count() - n0

    def unfused(self, r0, r1, X=None):
        """rows [r0, r1) of X (default: the case's X buffer) through taco_linear_fwd layer by layer (models/ops.py highway +
        the xp products)"""
        from tacotron_b200.models import ops
        c, n = self.c, r1 - r0
        rt = SimpleNamespace(impl=L.IMPL_TC3)
        h = torch.as_strided(self.Xbuf if X is None else X, (1, n, c.C), (n * self.ldx, self.ldx, 1), (HC.GUARD + r0) * self.ldx)
        new = lambda w: torch.empty(1, n, w, device=DEV)
        if c.dense:
            h = ops.linear(rt, h, self.p["Wd"], self.Wd_p, 128, bias=self.p["bd"], out=new(128))
        for l in range(c.L):
            h = ops.linear(rt, h, self.p["Whw"][l], self.hw_p[l], 256, bias=self.p["bhw"][l], highway_x=h, out=new(128))
        out = ops.linear(rt, h, self.p["Wx"], self.xp_p, HC.XP_N, bias=self.p["bx"], out=new(HC.XP_N))
        torch.cuda.synchronize()
        return out[0]

    def guards_intact(self, Y):
        """every element of Y outside its [M, 768] view still holds the sentinel (for the big case: in the guard rows and
        the rows of the first and last tiles)"""
        c, ldy = self.c, self.ldy
        Yi = Y.view(torch.int32).view(self.Yrows, ldy)
        rows = torch.arange(self.Yrows, device=DEV)
        if c.big:
            rows = torch.cat([rows[:HC.GUARD + HC.BM], rows[HC.GUARD + c.M - HC.BM:]])
            Yi = Yi[rows]
        inside = ((rows >= HC.GUARD) & (rows < HC.GUARD + c.M))[:, None] & (torch.arange(ldy, device=DEV) < HC.XP_N)[None]
        return bool((Yi[~inside] == SENTINEL).all())


def _bits(t):
    return t.contiguous().view(torch.int32)


def _free_gb():
    free, _ = torch.cuda.mem_get_info()
    return free / 2 ** 30


@pytest.mark.parametrize("case", HC.CASES, ids=[c.name for c in HC.CASES])
def test_highway_stack_envelope(case):
    if case.big:
        torch.cuda.empty_cache()
        if _free_gb() < 9.0:
            pytest.skip(f"M = {case.M} needs about 9 GB of free device memory, {_free_gb():.1f} GB free")
    for seed, klass in enumerate(CH.CLASSES):
        name = f"{case.name} [{klass}]"
        X, p = CH.inputs(case, klass, seed), CH.params(case, klass, seed + 10)
        run = Run(case, X, p)
        Y, launches = run.fused()
        assert launches == (1 if case.M > 0 else 0), f"{name}: {launches} launches"
        assert run.guards_intact(Y), f"{name}: a write outside Y's [M, 768] view"
        if case.M == 0:
            continue
        pd = CH.to(p, DEV)
        for r0, r1 in case.check_rows():
            ref, P, Q = CH.reference(X[r0:r1].to(DEV, torch.float64), pd, case.L, exact=klass == "exact")
            got = run.yview(Y, r0, r1)
            if klass == "exact":
                CH.check_exact(got, ref, f"{name} rows {r0}:{r1}")
            else:
                w = CH.check_float(got, ref, P, Q, f"{name} rows {r0}:{r1}")
                WORST["float"] = max(WORST.get("float", 0.0), w)
            unf = run.unfused(r0, r1)
            diff = int((_bits(got) != _bits(unf)).sum())
            assert diff == 0, f"{name} rows {r0}:{r1}: {diff} elements differ from the unfused route"
        del ref, P, Q, got, unf
        if case.big:
            del Y, run
            torch.cuda.empty_cache()
            continue
        again, _ = run.fused()
        assert torch.equal(_bits(run.yview(again)), _bits(run.yview(Y))), f"{name}: a second run differs"
        # NaN rows of X (the quiet NaN 0x7fc00000, its negation, and the canonical NaN 0x7fffffff GPU arithmetic produces)
        # give all-NaN xp rows on the fused and on the layered route, and every other row keeps its bits
        nan_rows = {case.M // 2: 0x7FC00000, 0: 0x7FFFFFFF, case.M - 1: -0x400000}
        Xn = run.Xbuf.clone()
        for j, bits in nan_rows.items():
            run.xview(Xn)[j].view(torch.int32).fill_(bits)
        Yn, _ = run.fused(Xn)
        got, bad = run.yview(Y), run.yview(Yn)
        layered = run.unfused(0, case.M, Xn)
        rows = torch.ones(case.M, dtype=torch.bool, device=DEV)
        for j in nan_rows:
            rows[j] = False
            assert bool(torch.isnan(bad[j]).all()), f"{name}: NaN row {j} of X gave a finite xp element"
            assert bool(torch.isnan(layered[j]).all()), f"{name}: NaN row {j} of X gave a finite xp element (layered)"
        assert torch.equal(_bits(bad[rows]), _bits(got[rows])), f"{name}: a NaN row leaked into other rows"
        assert run.guards_intact(Yn)


# ------------------------------------------------------------------------------------------------------------------
# refused descriptors: a message, no launch, Y untouched
# ------------------------------------------------------------------------------------------------------------------
def _ldx_small(d, run): d.ldx = 76
def _ldx_mod4(d, run): d.ldx = 82
def _ldwd_small(d, run): d.ldwd = 92
def _ldhw_small(d, run): d.ldhw = 124
def _hw_null(d, run): d.hw_p[run.c.L - 1] = None
def _y_misaligned(d, run): d.Y = d.Y + 4


@pytest.mark.parametrize("mutate,msg", [
    (_ldx_small, "ldx"), (_ldx_mod4, "ldx"), (_ldwd_small, "ldwd"), (_ldhw_small, "ldhw"),
    (_hw_null, "highway layer 3: NULL"), (_y_misaligned, "16-byte aligned"),
], ids=["ldx<C", "ldx%4", "ldwd<Cpad", "ldhw<128", "hw_p NULL", "Y misaligned"])
def test_refused(mutate, msg):
    case = HC.Case("refuse", 300, 80, ldx=84)
    run = Run(case, CH.inputs(case, "float", 0), CH.params(case, "float", 1))
    Y = run.new_y()
    d = run.desc(Y)
    mutate(d, run)
    torch.cuda.synchronize()
    n0 = L.lib().taco_launch_count()
    rc = L.lib().taco_highway_stack_fwd(C.byref(d), L.current_stream())
    torch.cuda.synchronize()
    assert rc != 0
    assert msg in L.lib().taco_last_error().decode()
    assert L.lib().taco_launch_count() == n0
    assert bool((Y.view(torch.int32) == SENTINEL).all())
