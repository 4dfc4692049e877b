"""-m gpu: the backward's wgmma routes over every form training sends them, against float64 (tests/bwd_tc_envelope_checks.py
for the references, classes and bars; tests/bwd_tc_envelope_cases.py for the cases and layouts):
  * taco_conv_dw (weight gradients), directly and through kernels.gemm(..., ta=True): C / N tile edges, T around the
    32-row k-block, taps 1-16, row shifts +-1 with a period and -B without, the split plan's edges, both dW reductions
    (vec2 and scalar), column slices, the C2 post-net projection gradient;
  * kernels._gemm_tc (recomputation and data-gradient products): tb, in-place accumulate, shifts, M around 2048
    (GEMM_TC_MIN_ROWS: 2047 must take taco_gemm), both n-tile widths;
  * kernels.conv_dx on taco_linear_fwd: taps 1-8 and 16, the bank-gradient slices, both epilogues, 3xTF32 and TF32.
Each case runs the int, offset and rand classes; NaN guards around every input, sentinels around every output.

Measured on an NVIDIA H100 80GB HBM3 (power limit 700 W), worst (err - 2u|ref|) / (2^-22 rss + u A), i.e. the 3xTF32
bar with C_BAR = 1 (the bar uses C_BAR = 16):
  taco_conv_dw   rand 6.11   offset 1.10
  _gemm_tc       rand 6.25   offset 1.58    (tf32 mode: 0.11 of 2^-9 S; M = 2047 on taco_gemm: 0.03 of 2^-16 S)
  conv_dx        rand 6.43   offset 1.42    (tf32 mode: 0.14 of 2^-9 S)
  module wall time: 28 s (126 tests)
"""
import ctypes as C
import json
import os

import pytest
import torch

from tacotron_b200 import _lib as L
from tacotron_b200 import kernels as K
from tests import bwd_tc_envelope_cases as BC
from tests import bwd_tc_envelope_checks as CH

pytestmark = pytest.mark.gpu
DEV = "cuda"
WORST = {}
ROUTES = set()


def _note(key, w):
    WORST[key] = max(WORST.get(key, 0.0), w)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(WORST):
        print(f"BWD_TC {k}: {WORST[k]:.4f}")
    path = os.environ.get("TACO_ENVELOPE_LOG")
    if path and WORST:
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        with open(path, "w") as f:
            json.dump({"worst": WORST, "c_bar": CH.C_BAR, "routes": sorted(map(list, ROUTES))}, f, indent=1)


@pytest.mark.parametrize("case", BC.DW_CASES, ids=[c.name for c in BC.DW_CASES])
def test_conv_dw(case):
    for i, klass in enumerate(CH.CLASSES):
        w = CH.check_dw(K, case, klass, DEV, seed=i)
        if klass != "int":
            _note(f"conv_dw {klass}", w)


@pytest.mark.parametrize("case", BC.GEMM_CASES, ids=[c.name for c in BC.GEMM_CASES])
def test_gemm_tc(case):
    for i, klass in enumerate(CH.CLASSES):
        w, route, mode = CH.check_gemm_tc(K, case, klass, DEV, seed=i)
        if route is not None:
            ROUTES.add(("gemm",) + tuple(route))
        if mode is not None:
            _note(f"gemm_tc {mode} {klass}", w)


@pytest.mark.parametrize("case", BC.CONV_DX_CASES, ids=[c.name for c in BC.CONV_DX_CASES])
def test_conv_dx(case):
    for i, klass in enumerate(CH.CLASSES):
        w, routes, mode = CH.check_conv_dx(K, case, klass, DEV, seed=i)
        ROUTES.update(("conv_dx",) + tuple(r) for r in routes)
        if mode is not None:
            _note(f"conv_dx {mode} {klass}", w)


def test_zz_routes_reached():
    """both n-tile widths and both epilogues of taco_linear_fwd, as taco_linear_route reports them"""
    if not ROUTES:
        pytest.skip("run with the route tests")
    bns = {r[1] for r in ROUTES}
    directs = {r[4] for r in ROUTES}
    assert {32, 128} <= bns and directs == {0, 1}, sorted(ROUTES)
    assert all(r[4] == 1 for r in ROUTES if r[0] == "gemm"), "_gemm_tc_ok admits only register-direct layouts"


# ------------------------------------------------------------------------------------------------------------------
# refusals: an error and no launch
# ------------------------------------------------------------------------------------------------------------------
def test_conv_dw_refusals():
    lib = L.lib()
    X = torch.zeros(64 * 132 + 16, device=DEV)
    Z = torch.zeros(64 * 132 + 16, device=DEV)
    W = torch.zeros(3 * 128 * 132, device=DEV)
    P = lambda t, off=0: C.c_void_p(t.data_ptr() + 4 * off)
    ok = dict(X=P(X), ldx=128, Z=P(Z), ldz=128, B=2, T=32, C=128, N=128, taps=3)
    bad = [dict(X=P(X, 1)), dict(Z=P(Z, 2)), dict(ldx=130), dict(ldz=129), dict(B=0), dict(T=0), dict(C=0), dict(N=0),
           dict(taps=0)]
    for b in bad:
        a = {**ok, **b}
        n0 = lib.taco_launch_count()
        rc = lib.taco_conv_dw(P(W), 128, 128 * 128, a["X"], a["ldx"], a["Z"], a["ldz"], a["B"], a["T"], a["C"], a["N"],
                              a["taps"], -1, L.current_stream())
        assert rc != 0 and "taco_conv_dw" in lib.taco_last_error().decode(), b
        assert lib.taco_launch_count() == n0, f"{b}: launched"
    torch.cuda.synchronize()
    assert torch.count_nonzero(W) == 0


@pytest.mark.parametrize("form", ["aligned", "x-misaligned", "ldx-odd", "z-misaligned", "tb", "rows-511"])
def test_dw_fallback_exactly_when_refused(form):
    """kernels.gemm(ta=True) calls taco_conv_dw exactly when _dw_tc_ok accepts, taco_gemm otherwise; both correct"""
    from tests import mirror_kernels as MK
    g = CH.gen(3)
    R, Cc, N = 511 if form == "rows-511" else 640, 80, 128
    wide = torch.full((R, 132), float("nan"))
    ldx_cols = 81 if form == "ldx-odd" else 132
    wideX = torch.full((R, ldx_cols), float("nan"))
    x0 = 1 if form == "x-misaligned" else 0
    z0 = 2 if form == "z-misaligned" else 0
    X = torch.randn(R, Cc, generator=g)
    Z = torch.randn(R, N, generator=g)
    wideX[:, x0:x0 + Cc] = X
    wide[:, z0:z0 + N] = Z
    tb = form == "tb"
    beta = 1.0
    W0 = torch.randn(Cc, N, generator=g)
    Xg, Zg = wideX.to(DEV)[:, x0:x0 + Cc], wide.to(DEV)[:, z0:z0 + N]
    got = W0.to(DEV)
    if tb:                                        # C[M=Cc, N] = X^T . (Z^T)^T: B stored [N, K] = Z^T
        Bg, Bc = Zg.t().contiguous(), Z.t().contiguous()
    else:
        Bg, Bc = Zg, Z
    with CH.recording(K, DW_TC=True) as rec:
        ok = K._dw_tc_ok(got, Xg, Bg, tb, beta, 0, 1, 0, 0, 1, 0, 0, 0, 0)
        K.gemm(got, Xg, Bg, ta=True, tb=tb, beta=beta)
    torch.cuda.synchronize()
    assert rec.calls == (["taco_conv_dw"] if ok else ["taco_gemm"]), (form, ok, rec.calls)
    assert ok == (form == "aligned"), form
    ref = W0.double().clone()
    MK.gemm(ref, X.double(), Bc.double(), ta=True, tb=tb, beta=beta)
    S = X.double().abs().t() @ Z.double().abs() + W0.double().abs()
    assert bool(((got.cpu().double() - ref).abs() <= CH.TOL_FALLBACK * S).all()), form
