"""The highway stack envelope without a GPU: the case list reaches what the kernel's indexing depends on, and the float64
checks of tests/highway_stack_envelope_checks.py pass a CPU mirror of the kernel's arithmetic and fail it under each
injected fault (the index faults are tested here, not on the device)."""
import pytest
import torch

from tests import highway_stack_envelope_cases as HC
from tests import highway_stack_envelope_checks as CH
from tests.bwd_tc_envelope_checks import rn_tf32

FAULTS = ("tf32", "no_lohi", "swap_T", "next_bias", "row_shift", "pad")
INDEX_FAULTS = ("swap_T", "next_bias", "row_shift", "pad")


def test_reach():
    cs = HC.CASES
    splits = {c.split for c in cs if c.M > 0}
    assert splits == {1, 2, 3, 6}
    # each split boundary from both sides, the last tile partial
    for t in (22, 44, 66):
        for tiles in (t, t + 1):
            assert any(-(-c.M // HC.BM) == tiles and c.M % HC.BM for c in cs), f"no case with {tiles} tiles, last partial"
    assert [HC.split_of(t * HC.BM) for t in (22, 23, 44, 45, 66, 67)] == [6, 3, 3, 2, 2, 1]
    assert {c.L for c in cs} == {1, 2, 3, 4}
    assert {c.C % 32 for c in cs} == set(range(32))
    assert {(c.kin, c.L) for c in cs if c.dense} == {(k, l) for k in (1, 2, 3, 4) for l in (1, 2, 3, 4)}
    assert {(c.L, c.split) for c in cs if not c.dense and c.M > 0} >= {(4, s) for s in (1, 2, 3, 6)}
    mins = lambda c: (HC._r(c.C, 4), HC.XP_N, c.Cpad, 128, 128)
    for i, name in enumerate(("ldx", "ldy", "ldwd", "ldhw", "ldxp")):
        extra = {c.lds[i] - mins(c)[i] for c in cs if c.dense or name != "ldwd"}
        assert 0 in extra and 4 in extra and max(extra) > 4, f"{name}: {sorted(extra)}"
    assert {0, 1, 15, 16, 17, 127, 128, 129, 257} <= {c.M for c in cs}
    assert {4096, 32000, 500} <= {c.M for c in cs}
    assert any(c.M * HC.XP_N > 2 ** 31 for c in cs)
    assert len({c.name for c in cs}) == len(cs)


# ------------------------------------------------------------------------------------------------------------------
# CPU mirror of highway_stack_kernel: A and W split into rn_tf32 hi / lo, per k8 step lo.hi + hi.lo + hi.hi into an fp32
# accumulator, k in order, fp32 epilogues with the kernel's expressions
# ------------------------------------------------------------------------------------------------------------------
def _split(x):
    hi = rn_tf32(x)
    return hi, rn_tf32(x - hi)


def _mm(A, W, fault):
    """A [M, K] . W [K, N], K a multiple of 8"""
    ah, al = _split(A)
    wh, wl = _split(W)
    M, K = A.shape
    parts = lambda a, w: torch.bmm(a.reshape(M, K // 8, 8).transpose(0, 1), w.reshape(K // 8, 8, -1))
    hh, hl, lh = parts(ah, wh), parts(ah, wl), parts(al, wh)
    d = torch.zeros(M, W.shape[1])
    for k in range(K // 8):
        if fault != "tf32":
            if fault != "no_lohi":
                d = d + lh[k]
            d = d + hl[k]
        d = d + hh[k]
    return d


def mirror(c: HC.Case, X, p, fault=None):
    h = X.clone()
    if fault == "row_shift":                     # row r of a tile reads row r + 1 of the same tile
        r = torch.arange(c.M)
        src = torch.where((r % HC.BM != HC.BM - 1) & (r + 1 < c.M), r + 1, r)
        h = h[src]
    pad = 0.5 if fault == "pad" else 0.0
    if c.dense:
        A = torch.full((c.M, c.Cpad), pad)
        A[:, :c.C] = h
        W = torch.full((c.Cpad, 128), pad)
        W[:c.C] = p["Wd"]
        h = _mm(A, W, fault) + p["bd"]
    for l in range(c.L):
        b = p["bhw"][(l + 1) % c.L if fault == "next_bias" else l]
        W = p["Whw"][l]
        H = (_mm(h, W[:, :128], fault) + b[:128]).clamp_min(0.0)
        T = torch.sigmoid(_mm(h, W[:, 128:], fault) + b[128:])
        h = H * (1 - T) + h * T if fault == "swap_T" else H * T + h * (1 - T)
    return _mm(h, p["Wx"], fault) + p["bx"]


def _check(c, klass, got, X, p):
    ref, P, Q = CH.reference(X.double(), CH.to(p, "cpu"), c.L, exact=klass == "exact")
    if klass == "exact":
        CH.check_exact(got, ref, c.name)
        return 0.0
    return CH.check_float(got, ref, P, Q, c.name)


def _applies(c, fault):
    if fault == "next_bias":
        return c.L >= 2
    if fault == "row_shift":
        return c.M >= 2
    if fault == "pad":
        return c.C % 32 != 0
    return True


CASES = HC.host_cases()
WORST = {}


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_mirror_passes(case):
    for klass in CH.CLASSES:
        X, p = CH.inputs(case, klass, 3), CH.params(case, klass, 4)
        w = _check(case, klass, mirror(case, X, p), X, p)
        WORST[klass] = max(WORST.get(klass, 0.0), w)


@pytest.mark.parametrize("fault", FAULTS)
def test_mirror_faults_fail(fault):
    cases = [c for c in CASES if _applies(c, fault)]
    assert len(cases) >= 10
    for c in cases:
        for klass in CH.CLASSES:
            if klass == "exact" and fault not in INDEX_FAULTS:
                continue                          # exact inputs have no lo halves: the float class must catch these
            X, p = CH.inputs(c, klass, 3), CH.params(c, klass, 4)
            with pytest.raises(AssertionError):
                _check(c, klass, mirror(c, X, p, fault), X, p)
