"""The checks of the training-kernel envelope, written once for both places they run: on the device through
tacotron_b200.kernels (tests/test_gpu_train_envelope.py) and on CPU through the same marshalling over the host emulation
of csrc/train.cu (tests/test_train_envelope_host.py).

Every reference is float64, from the functions of tests/mirror_kernels.py on float64 copies of the operands; none calls
the library.  Two classes of inputs:
  exact  small integers (and gains of 2^k, masks, selects, signs): every product and partial sum is an integer below
         2^24, or the kernel performs a single rounding, so the result must equal float64 (rounded once to fp32) bit
         for bit -- a wrong row, tap, batch entry, split or column is off by at least one;
  float  random fp32 values with some large rows: each element must lie within a bar derived from the kernel's
         arithmetic (`tol * S`, S the float64 sum of the magnitudes the element is formed from).
Every operand sits in a guard buffer: NaN around inputs, a sentinel bit pattern around outputs that must survive."""
from __future__ import annotations

import math

import torch

from tests import mirror_kernels as MK
from tests.train_envelope_cases import GUARD, SENTINEL, Case, Layout, Op, call_gemm

U = 2.0 ** -24                       # fp32 unit roundoff
GEMM_TOL = {0: 2.0 ** -19, 1: 2.0 ** -16}      # FFMA, truncating 3xTF32 (per element, times S; see test_gpu_train_envelope.py)
GEMM_GLOBAL = {0: 1e-4, 1: 2e-5}                 # the bars of tests/train_checks.check_gemm (times max|ref|)
NAN = float("nan")


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def sentinel(n, device):
    return torch.full((n,), SENTINEL, dtype=torch.int32, device=device).view(torch.float32)


def guards_intact(buf, mask):
    return bool((buf.view(torch.int32)[~mask] == SENTINEL).all())


def _fill(op: Op, vals, base):
    """copy vals (one [rows, cols] tensor per entry, on CPU) into a flat buffer `base` at op's views"""
    for z, v in enumerate(vals):
        op.view(base, z).copy_(v)
    return base


# ------------------------------------------------------------------------------------------------------------------
# taco_gemm
# ------------------------------------------------------------------------------------------------------------------
def gemm_operands(c: Case, lay: Layout, klass: str, seed: int):
    """CPU fp32 values of A, B and the input C per entry"""
    g = _gen(seed)

    def rnd(op, scale=1.0, big_rows=False):
        out = []
        for _ in range(op.nb):
            if klass == "exact":
                v = torch.randint(-4, 5, (op.rows, op.cols), generator=g).float()
            else:
                v = torch.randn(op.rows, op.cols, generator=g) * scale
                if big_rows and op.rows > 1:
                    v[3::7] *= 64.0                             # some large rows: S is dominated by few terms
            out.append(v)
        return out
    A = rnd(lay.A, big_rows=True)
    B = rnd(lay.B)
    Cin = [v * 4 for v in rnd(lay.C)] if c.beta == 1.0 else None
    return A, B, Cin


def run_gemm(lib, c: Case, impl: int, klass: str, device, stream=None, seed=0):
    """one case through taco_gemm (impl already selected); returns (worst err / bar, worst err / global bar)"""
    lay = Layout(c)
    A, B, Cin = gemm_operands(c, lay, klass, seed)
    dev = torch.device(device)
    bufA = _fill(lay.A, A, torch.full((lay.A.size,), NAN)).to(dev)
    bufB = _fill(lay.B, B, torch.full((lay.B.size,), NAN)).to(dev)
    cmask = lay.C.mask()
    bufC = sentinel(lay.C.size, "cpu")
    _fill(lay.C, Cin if Cin is not None else [torch.full((c.M, c.N), NAN)] * lay.C.nb, bufC)   # beta = 0: C is not read
    bufC = bufC.to(dev)
    call_gemm(lib, lay.desc(c, bufA.data_ptr(), bufB.data_ptr(), bufC.data_ptr()), stream)
    if dev.type == "cuda":
        torch.cuda.synchronize()
    # float64 references: the result and S = sum |a||b| (+ |C|)
    kw = lay.kwargs(c)
    ref = _fill(lay.C, Cin if Cin is not None else [torch.zeros(c.M, c.N)] * lay.C.nb, torch.zeros(lay.C.size)).double().to(dev)
    S = ref.abs()
    MK.gemm(lay.C.view(ref), lay.A.view(bufA.double()), lay.B.view(bufB.double()), **kw)
    MK.gemm(lay.C.view(S), lay.A.view(bufA.double().abs()), lay.B.view(bufB.double().abs()), **kw)
    cmask = cmask.to(dev)
    assert guards_intact(bufC, cmask), f"{c.name}: write outside C's view"
    got = bufC.double()[cmask]
    r, s = ref[cmask], S[cmask]
    assert bool(torch.isfinite(got).all()), f"{c.name}: non-finite result (a NaN guard or an unwritten beta=0 C was read)"
    err = (got - r).abs()
    if klass == "exact":
        bad = int((err != 0).sum())
        assert bad == 0, f"{c.name} impl {impl}: {bad} elements differ from float64, max {err.max().item():g}"
        return 0.0, 0.0
    bar = GEMM_TOL[impl] * s
    ratio = torch.where(bar > 0, err / bar, torch.where(err > 0, torch.inf, 0.0))
    worst = ratio.max().item() if ratio.numel() else 0.0
    assert worst <= 1.0, f"{c.name} impl {impl}: worst element at {worst:.3f} of tol*S"
    rmax = r.abs().max().item() if r.numel() else 0.0
    gworst = err.max().item() / (GEMM_GLOBAL[impl] * rmax) if rmax > 0 else 0.0
    return worst, gworst


# ------------------------------------------------------------------------------------------------------------------
# element-wise, reduction and optimizer kernels.  `K` is tacotron_b200.kernels (or its emulated twin); sizes:
#   "tiny"  one row / T = 1 or 2;   "wrap"  not a multiple of 256, > 3 grid-stride passes (> 3 * 132*16*256 elements);
#   "c2"    the C2 training call site (B = 32, Tx = 128, T = 200 decoder steps, r = 5: post-net rows 32000).
# ------------------------------------------------------------------------------------------------------------------
WRAP = 3 * 132 * 16 * 256 + 1000


def gmat(rows, cols, device, fill=NAN, col0=1, pad=3):
    """([rows, cols] view, flat buffer, Op) inside a guard buffer: GUARD rows around it, col0 + pad extra columns"""
    op = Op(rows, cols, cols + col0 + pad, col0)
    buf = sentinel(op.size, device) if fill == "sentinel" else torch.full((op.size,), fill, device=device)
    return op.view(buf), buf, op


def gvec(n, device, fill=NAN, g=16):
    buf = sentinel(n + 2 * g, device) if fill == "sentinel" else torch.full((n + 2 * g,), fill, device=device)
    return buf[g:g + n], buf


def vmask(buf, n, g=16):
    m = torch.zeros(buf.numel(), dtype=torch.bool, device=buf.device)
    m[g:g + n] = True
    return m


def _sync(device):
    if torch.device(device).type == "cuda":
        torch.cuda.synchronize()


def _ratio(err, bar):
    r = torch.where(bar > 0, err / bar, torch.where(err > 0, torch.inf, 0.0))
    return r.max().item() if r.numel() else 0.0


def _check(name, got, ref, bar=None):
    """exact (bar None): got == fp32(ref) bit for bit; else per element |got - ref| <= bar.  Returns the worst ratio."""
    got = got.detach().cpu().double()
    ref = ref.detach().cpu().double()
    assert bool(torch.isfinite(got).all()), f"{name}: non-finite output (a NaN guard was read)"
    if bar is None:
        bad = (got != ref.float().double())
        assert not bool(bad.any()), f"{name}: {int(bad.sum())} elements differ, max {(got - ref).abs().max().item():g}"
        return 0.0
    w = _ratio((got - ref).abs(), bar.detach().cpu().double())
    assert w <= 1.0, f"{name}: worst element at {w:.3f} of its bar"
    return w


def _ints(shape, g, lo=-8, hi=9):
    return torch.randint(lo, hi, shape, generator=g).float()


def _rows(size, tiny, wrap_cols, c2):
    return {"tiny": tiny, "wrap": (-(-WRAP // wrap_cols), wrap_cols), "c2": c2}[size]


def check_bias_act(K, device, size, act, klass):
    g = _gen(1)
    M, N = _rows(size, (1, 37), 257, (32000, 256))
    Cv, buf, op = gmat(M, N, device, fill="sentinel")
    x = _ints((M, N), g) if klass == "exact" else torch.randn(M, N, generator=g) * 4
    if klass == "float":
        x[::97] = torch.linspace(-30, 30, N)                    # saturated inputs around +-30
    bias = (_ints((N,), g) if klass == "exact" else torch.randn(N, generator=g))
    bias_v, bias_b = gvec(N, device)
    bias_v.copy_(bias.to(device))
    Cv.copy_(x.to(device))
    K.bias_act_(Cv, bias_v, act)
    _sync(device)
    assert guards_intact(buf, op.mask(buf.device)), "bias_act: write outside C"
    v = (x + bias).double() if klass == "exact" else (x + bias).double()     # fp32 add, then the activation
    ref = v.clone()
    MK.bias_act_(ref, None, act)
    if klass == "exact":
        return _check(f"bias_act[{act}]", Cv, ref)
    d = {MK.ACT_SIGMOID: ref * (1 - ref), MK.ACT_TANH: 1 - ref * ref}.get(act, torch.ones_like(ref))
    return _check(f"bias_act[{act}]", Cv, ref, 8 * U * ref.abs() + 2 * U * (v.abs() * d.abs()) + 1e-45)


def check_mul_shift(K, device, size, shift, period):
    g = _gen(2)
    M, N = _rows(size, (2, 128), 128, (32000, 128))
    out, ob, oop = gmat(M, N, device, fill="sentinel")
    X, _, _ = gmat(M, N, device, col0=3)
    H, _, _ = gmat(M, N, device, col0=0, pad=5)
    x, h = torch.randn(M, N, generator=g), torch.randn(M, N, generator=g)
    X.copy_(x.to(device)); H.copy_(h.to(device))
    K.mul_shift(out, X, H, shift, period)
    _sync(device)
    assert guards_intact(ob, oop.mask(ob.device)), "mul_shift: write outside out"
    ref = torch.empty(M, N, dtype=torch.float64)
    MK.mul_shift(ref, x.double(), h.double(), shift, period)
    return _check(f"mul_shift[{shift},{period}]", out, ref)          # one rounding: exact


def check_epi_bwd(K, device, size, form):
    """form: "plain" (no relu), "relu", "relu_bn", "relu_bn_res" -- gain 2 (dropout keep 1/2) throughout"""
    g = _gen(3)
    M, N = _rows(size, (1, 80), 256, (32000, 256))
    dZ, zb, zop = gmat(M, N, device, fill="sentinel")
    dY, _, _ = gmat(M, N, device, col0=2)
    Y, _, _ = gmat(M, N, device, col0=0)
    R, _, _ = gmat(M, N, device, col0=3)
    dy, z, r = torch.randn(M, N, generator=g), torch.randn(M, N, generator=g), torch.randn(M, N, generator=g)
    y = torch.relu(z)                                            # relu outputs: exact zeros are common
    relu = form != "plain"
    bn = form.startswith("relu_bn")
    res = form == "relu_bn_res"
    scale = shift = None
    if bn:                                                       # y = relu(z)*scale + shift (+ R): dead units give y == shift (+ R)
        scale = torch.rand(N, generator=g) + 0.5
        shift = torch.randn(N, generator=g) * 0.1
        y = y * scale + shift
        if res:
            y = y + r
    dY.copy_(dy.to(device)); Y.copy_(y.to(device)); R.copy_(r.to(device))
    sc = sh = None
    if bn:
        sc, _ = gvec(N, device); sc.copy_(scale.to(device))
        sh, _ = gvec(N, device); sh.copy_(shift.to(device))
    K.epi_bwd(dZ, dY, Y if relu else None, relu, scale=sc, shift=sh, gain=2.0, R=R if res else None)
    _sync(device)
    assert guards_intact(zb, zop.mask(zb.device)), "epi_bwd: write outside dZ"
    ref = torch.empty(M, N, dtype=torch.float64)
    # the mask is a comparison of fp32 values the kernel forms, ((Y - R) - shift) * scale > 0: it is evaluated on the same
    # fp32 values, the gradient it gates in float64
    if bn:
        base = (y - r) if res else y
        mask = ((base - shift) * scale > 0).double()
        refv = dy.double() * 2.0 * scale.double() * mask
        return _check(f"epi_bwd[{form}]", dZ, refv)
    MK.epi_bwd(ref, dy.double(), y.double(), relu, gain=2.0)
    return _check(f"epi_bwd[{form}]", dZ, ref)


def check_epi_fwd_keep(K, device, size):
    g = _gen(4)
    M, N = _rows(size, (1, 48), 256, (6400, 256))
    X, xb, xop = gmat(M, N, device, fill="sentinel")
    x = torch.randn(M, N, generator=g)
    keep = (torch.rand(M, N, generator=g) < 0.5).to(torch.uint8)
    X.copy_(x.to(device))
    kb = torch.zeros(M * N + 32, dtype=torch.uint8, device=device)
    kb[16:16 + M * N] = keep.reshape(-1).to(device)
    kb[:16] = 7; kb[16 + M * N:] = 7                             # guard bytes: non-zero (would keep) outside the mask
    K.epi_fwd_keep_(X, kb[16:16 + M * N].view(M, N), 2.0)
    _sync(device)
    assert guards_intact(xb, xop.mask(xb.device)), "epi_fwd_keep: write outside X"
    ref = x.double().clone()
    MK.epi_fwd_keep_(ref, keep, 2.0)
    return _check("epi_fwd_keep", X, ref)


def check_bn_param_grad(K, device, size):
    g = _gen(5)
    N = {"tiny": 1, "wrap": 1000, "c2": 256}[size]
    vals = [torch.randn(N, generator=g) for _ in range(6)]
    vals[4] = torch.rand(N, generator=g) + 0.5                   # gamma
    bufs = []
    for i, v in enumerate(vals):
        t, b = gvec(N, device, fill="sentinel" if i < 2 else NAN)
        t.copy_(v.to(device)); bufs.append((t, b))
    (dgm, dgb), (dbt, dbb) = bufs[0], bufs[1]
    K.bn_param_grad(dgm, dbt, bufs[2][0], bufs[3][0], bufs[4][0], bufs[5][0])
    _sync(device)
    assert guards_intact(dgb, vmask(dgb, N)) and guards_intact(dbb, vmask(dbb, N)), "bn_param_grad: write outside"
    dg, db = vals[0].double().clone(), vals[1].double().clone()
    S1, S2, gm, bt = (v.double() for v in vals[2:])
    MK.bn_param_grad(dg, db, S1, S2, gm, bt)
    w = _check("bn_param_grad dbeta", dbt, db)
    mag = vals[0].double().abs() + (S2.abs() + (bt * S1).abs()) / gm.abs()
    return max(w, _check("bn_param_grad dgamma", dgm, dg, 4 * U * mag))


def check_maxpool_bwd(K, device, size):
    g = _gen(6)
    B, T, Cc = {"tiny": (1, 2, 128), "wrap": (3, 5 * 283 + 1, 419), "c2": (32, 128, 128)}[size]
    x = _ints((B, T, Cc), g, -2, 3)                              # integer X: equal neighbours are common (ties)
    dp = _ints((B, T, Cc), g)
    n = B * T * Cc
    X, _ = gvec(n, device); X.copy_(x.reshape(-1).to(device))
    dP, _ = gvec(n, device); dP.copy_(dp.reshape(-1).to(device))
    dX, xb = gvec(n, device, fill="sentinel")
    K.maxpool_bwd(dX.view(B, T, Cc), dP.view(B, T, Cc), X.view(B, T, Cc))
    _sync(device)
    assert guards_intact(xb, vmask(xb, n)), "maxpool_bwd: write outside dX"
    ref = torch.empty(B, T, Cc, dtype=torch.float64)
    MK.maxpool_bwd(ref, dp.double(), x.double())
    return _check("maxpool_bwd", dX.view(B, T, Cc), ref)


def _highway_inputs(M, U_, g):
    P = torch.randn(M, 2 * U_, generator=g) * 3
    P[::41, :] = torch.linspace(-30, 30, 2 * U_)                # saturated gates
    return P, torch.randn(M, U_, generator=g), torch.randn(M, U_, generator=g)


def check_highway(K, device, size):
    g = _gen(7)
    M = {"tiny": 1, "wrap": -(-WRAP // 128), "c2": 4096}[size]
    U_ = 128
    Pm, _, _ = gmat(M, 2 * U_, device, col0=2)
    X, _, _ = gmat(M, U_, device, col0=1, pad=5)
    dY, _, _ = gmat(M, U_, device, col0=0)
    p, x, dy = _highway_inputs(M, U_, g)
    Pm.copy_(p.to(device)); X.copy_(x.to(device)); dY.copy_(dy.to(device))
    Y, yb, yop = gmat(M, U_, device, fill="sentinel")
    dP, pb, pop = gmat(M, 2 * U_, device, fill="sentinel", col0=3)
    dX, db, dop = gmat(M, U_, device, fill="sentinel")
    K.highway_fwd(Y, Pm, X)
    K.highway_bwd(dP, dX, dY, Pm, X)
    _sync(device)
    for b, op, nm in ((yb, yop, "Y"), (pb, pop, "dP"), (db, dop, "dX")):
        assert guards_intact(b, op.mask(b.device)), f"highway: write outside {nm}"
    p64, x64, dy64 = p.double(), x.double(), dy.double()
    h, t = torch.relu(p64[:, :U_]), torch.sigmoid(p64[:, U_:])
    # t carries the expf error (a few ulp, relative to t and to 1 - t); every other op rounds once
    et = 8 * U * t * (1 - t) * (1 + p64[:, U_:].abs()) + 4 * U * t
    y = torch.empty(M, U_, dtype=torch.float64)
    MK.highway_fwd(y, p64, x64)
    w = _check("highway_fwd", Y, y, et * (h - x64).abs() + 4 * U * (h * t + (x64 * (1 - t)).abs()) + 1e-45)
    rp, rx = torch.empty(M, 2 * U_, dtype=torch.float64), torch.empty(M, U_, dtype=torch.float64)
    MK.highway_bwd(rp, rx, dy64, p64, x64)
    bh = (dy64 * t).abs() * 4 * U + dy64.abs() * et
    bt = 8 * U * (dy64 * (h - x64) * t * (1 - t)).abs() + (dy64 * (h - x64)).abs() * et * (1 + 2 * t) + 1e-45
    w = max(w, _check("highway_bwd dP", dP, rp, torch.cat([bh + 1e-45, bt], 1)))
    return max(w, _check("highway_bwd dX", dX, rx, 4 * U * (dy64 * (1 - t)).abs() + dy64.abs() * et + 1e-45))


def check_l1_bwd(K, device, size, beta, padded):
    g = _gen(8)
    if padded:                                                   # the [M][1025] linear-spectrogram gradient
        rows, cols = {"tiny": (2, 1025), "wrap": (-(-WRAP // 1025), 1025), "c2": (32000, 1025)}[size]
    else:                                                        # the [B*T][80 r] mel gradient, flat
        rows, cols = {"tiny": (1, 80), "wrap": (1, WRAP), "c2": (1, 32000 * 80)}[size]
    n = rows * cols
    a = torch.randn(n, generator=g)
    b = torch.randn(n, generator=g)
    b[::3] = a[::3]                                              # d = 0 exactly: sign 0
    A, _ = gvec(n, device); A.copy_(a.to(device))
    Bt, _ = gvec(n, device); Bt.copy_(b.to(device))
    d0 = _ints((rows, cols), g)
    if padded:                                                  # the [M][1025] spectrogram gradient in a 1028-float pitch
        ld = (cols + 3) // 4 * 4
        op = Op(rows, cols, ld, 0)
        buf = sentinel(op.size, device)
        dA = op.view(buf)
        mask = op.mask(buf.device)
    else:
        dA, buf = gvec(n, device, fill="sentinel")
        mask = vmask(buf, n)
    if beta:
        dA.copy_(d0.to(device).view(dA.shape))
    K.l1_bwd(dA, A.view(dA.shape), Bt.view(dA.shape), beta=beta)
    _sync(device)
    assert guards_intact(buf, mask), "l1_bwd: write outside dA"
    ref = d0.double().clone() if beta else torch.empty(rows, cols, dtype=torch.float64)
    MK.l1_bwd(ref, a.double().view(rows, cols), b.double().view(rows, cols), beta)
    return _check(f"l1_bwd[beta={beta}, padded={padded}]", dA.reshape(rows, cols), ref)


def check_scatter_add_rows(K, device, size):
    g = _gen(9)
    V, W = 70, 256
    rows = {"tiny": 1, "wrap": -(-WRAP // W), "c2": 4096}[size]
    ids = torch.randint(-3, V + 3, (rows,), generator=g, dtype=torch.int32)    # repeated and out-of-range (clamped)
    ids[:4] = torch.tensor([5, 5, -1, V + 9], dtype=torch.int32)[:min(4, rows)]
    dr = _ints((rows, W), g)
    dr[::5] = 0.0
    t0 = _ints((V, W), g)
    Tb, tb = gvec(V * W, device, fill="sentinel"); Tb.copy_(t0.reshape(-1).to(device))
    Dr, _ = gvec(rows * W, device); Dr.copy_(dr.reshape(-1).to(device))
    Ib = torch.full((rows + 32,), 1 << 30, dtype=torch.int32, device=device)
    Ib[16:16 + rows] = ids.to(device)
    K.scatter_add_rows(Tb.view(V, W), Ib[16:16 + rows], Dr.view(rows, W))
    _sync(device)
    assert guards_intact(tb, vmask(tb, V * W)), "scatter_add_rows: write outside the table"
    ref = t0.double().clone()
    MK.scatter_add_rows(ref, ids, dr.double())
    return _check("scatter_add_rows", Tb.view(V, W), ref)


def check_colsum(K, device, size, form):
    """form: "sum" (bias gradient), "dot" (sum dY*Y), "dot_res" (sum dY*(Y - R)); integer operands: exact"""
    g = _gen(10)
    M, N = _rows(size, (1, 37), 256, (32000, 256))
    A, _, _ = gmat(M, N, device, col0=2)
    Bm, _, _ = gmat(M, N, device, col0=0)
    R, _, _ = gmat(M, N, device, col0=1, pad=6)
    a, b, r = _ints((M, N), g, -3, 4), _ints((M, N), g, -3, 4), _ints((M, N), g, -3, 4)
    A.copy_(a.to(device)); Bm.copy_(b.to(device)); R.copy_(r.to(device))
    o0 = _ints((N,), g)
    out, ob = gvec(N, device, fill="sentinel"); out.copy_(o0.to(device))
    K.colsum(out, A, Bm if form != "sum" else None, R if form == "dot_res" else None)
    _sync(device)
    assert guards_intact(ob, vmask(ob, N)), "colsum: write outside out"
    ref = o0.double().clone()
    MK.colsum(ref, a.double(), b.double() if form != "sum" else None, r.double() if form == "dot_res" else None)
    return _check(f"colsum[{form}]", out, ref)


def check_colsum_seg(K, device, size, period, repeat=True):
    g = _gen(11)
    N = 128 if size != "tiny" else 37
    segs = {"tiny": 1, "wrap": -(-WRAP // (N * period)), "c2": 32}[size]
    M = segs * period
    A, _, _ = gmat(M, N, device, col0=1)
    a = _ints((M, N), g) if period != 7 else torch.randn(M, N, generator=g)
    A.copy_(a.to(device))
    o0 = _ints((segs, N), g)
    out, ob, oop = gmat(segs, N, device, fill="sentinel", col0=2)
    out.copy_(o0.to(device))
    K.colsum_seg(out, A, period)
    _sync(device)
    assert guards_intact(ob, oop.mask(ob.device)), "colsum_seg: write outside out"
    ref = o0.double() + a.double().view(segs, period, N).sum(1)
    if period == 7:                                             # float operands: 7 rows in a fixed order
        w = _check(f"colsum_seg[{period}]", out, ref, (period + 8) * U * (o0.double().abs() + a.double().abs().view(segs, period, N).sum(1)))
    else:
        w = _check(f"colsum_seg[{period}]", out, ref)
    if repeat:                                                  # deterministic: a second run is bit-identical
        first = out.clone()
        out.copy_(o0.to(device))
        K.colsum_seg(out, A, period)
        _sync(device)
        assert torch.equal(first.view(torch.int32), out.view(torch.int32)), "colsum_seg: not deterministic"
    return w


def check_dec_inputs(K, device, size, r, sched):
    g = _gen(12)
    B, T = {"tiny": (1, 1), "wrap": (33, 7 * 77), "c2": (32, 200)}[size]
    if size == "tiny" and sched:
        T = 2
    OUT = 80 * r
    mel = torch.randn(B, T, OUT, generator=g)
    y = torch.randn(B, T, OUT, generator=g)
    sm = (torch.rand(T, B, generator=g) < 0.5).to(torch.uint8)
    Mv, _ = gvec(mel.numel(), device); Mv.copy_(mel.reshape(-1).to(device))
    Yv, _ = gvec(y.numel(), device); Yv.copy_(y.reshape(-1).to(device))
    smb = torch.full((T * B + 32,), 1, dtype=torch.uint8, device=device)
    smb[16:16 + T * B] = sm.reshape(-1).to(device)
    Xin, xb = gvec(T * B * 80, device, fill="sentinel")
    selb = torch.full((T * B + 32,), 0xA5, dtype=torch.uint8, device=device)
    K.dec_inputs(Xin.view(T, B, 80), selb[16:16 + T * B].view(T, B), Mv.view(B, T, OUT), Yv.view(B, T, OUT),
                 smb[16:16 + T * B].view(T, B) if sched else None, r, sched)
    _sync(device)
    assert guards_intact(xb, vmask(xb, T * B * 80)), "dec_inputs: write outside Xin"
    selc = selb.cpu()
    assert bool((selc[:16] == 0xA5).all()) and bool((selc[16 + T * B:] == 0xA5).all()), "dec_inputs: write outside sel"
    rx, rs = torch.empty(T, B, 80, dtype=torch.float64), torch.empty(T, B, dtype=torch.uint8)
    MK.dec_inputs(rx, rs, mel.double(), y.double(), sm, r, sched)
    assert torch.equal(selc[16:16 + T * B].view(T, B), rs), "dec_inputs: sel"
    return _check(f"dec_inputs[r={r}, sched={sched}]", Xin.view(T, B, 80), rx)


def check_attn_bwd_post(K, device, size):
    g = _gen(13)
    B, T, Tx = {"tiny": (1, 1, 3), "wrap": (3, 9, 67), "c2": (32, 200, 128)}[size]
    ds = torch.randn(B, T, Tx, generator=g)
    ds[:, :, Tx - 2:] = 0.0                                      # masked positions
    keys = torch.randn(B, Tx, 256, generator=g)
    keys[:, ::5] *= 15                                           # saturated tanh
    pq = torch.randn(T, B, 256, generator=g)
    v = torch.randn(256, generator=g)
    dv0 = torch.randn(256, generator=g)
    bufs = []
    for t in (ds, keys, pq, v):
        x, _ = gvec(t.numel(), device); x.copy_(t.reshape(-1).to(device)); bufs.append(x.view(t.shape))
    dk, kb = gvec(B * Tx * 256, device, fill="sentinel")
    dv, vb = gvec(256, device, fill="sentinel"); dv.copy_(dv0.to(device))
    K.attn_bwd_post(dk.view(B, Tx, 256), dv, *bufs)
    _sync(device)
    assert guards_intact(kb, vmask(kb, B * Tx * 256)) and guards_intact(vb, vmask(vb, 256)), "attn_bwd_post: write outside"
    rk, rv = torch.empty(B, Tx, 256, dtype=torch.float64), dv0.double().clone()
    MK.attn_bwd_post(rk, rv, ds.double(), keys.double(), pq.double(), v.double())
    Sk = torch.zeros(B, Tx, 256, dtype=torch.float64)
    Sv = dv0.double().abs()
    for t in range(T):                                           # the magnitudes each output is formed from
        e = torch.tanh(keys.double() + pq.double()[t][:, None, :])
        dst = ds.double()[:, t][:, :, None]
        Sk += (dst * v.double()).abs() * (1 + e * e)
        Sv = Sv + (dst.abs() * e.abs()).sum((0, 1))
    w = _check("attn_bwd_post dkeys", dk.view(B, Tx, 256), rk, (T + 8) * 4 * U * Sk + 1e-45)
    return max(w, _check("attn_bwd_post dv", dv, rv, (T + B * Tx + 8) * 4 * U * Sv + 1e-45))


def _two_stage_bar(n, blocks, S):
    """bar of a fixed-grid two-stage sum: elements per thread in fp32, a 5-level warp tree, 8 warps in fp32, double after"""
    ept = max(1, -(-n // (blocks * 256)))
    return (ept + 5 + 8 + 1) * U * S


def check_sumsq(K, device, n, repeat=True):
    g = _gen(14)
    x = torch.randn(n, generator=g)
    if n > 7:
        x[::7919] *= 100.0
    xv, _ = gvec(n, device); xv.copy_(x.to(device))
    out, ob = gvec(1, device, fill="sentinel")
    K.sumsq(out, xv)
    _sync(device)
    assert guards_intact(ob, vmask(ob, 1)), "sumsq: write outside out"
    ref = torch.zeros(1, dtype=torch.float64)
    MK.sumsq(ref, x.double())
    w = _check(f"sumsq[n={n}]", out, ref, _two_stage_bar(n, 1184, ref.abs()) + 1e-45)
    if repeat:
        first = out.clone()
        K.sumsq(out, xv)
        _sync(device)
        assert torch.equal(first.view(torch.int32), out.view(torch.int32)), "sumsq: not deterministic"
    return w


def check_l1_loss_fwd(lib, device, n, stream=None):
    """taco_l1_loss_fwd: float4 body, n % 4 tail in block 0, fixed-grid two-stage sum; run twice (deterministic)"""
    g = _gen(15)
    a, b = torch.randn(n, generator=g), torch.randn(n, generator=g)
    av, _ = gvec(n, device); av.copy_(a.to(device))
    bv, _ = gvec(n, device); bv.copy_(b.to(device))
    nb = lib.taco_l1_partial_count()
    part = torch.full((nb,), NAN, device=device)
    out, ob = gvec(1, device, fill="sentinel")
    outs = []
    for _ in range(2):
        assert lib.taco_l1_loss_fwd(av.data_ptr(), bv.data_ptr(), n, part.data_ptr(), out.data_ptr(), stream) == 0
        _sync(device)
        outs.append(out.clone())
    assert guards_intact(ob, vmask(ob, 1)), "l1_loss_fwd: write outside out"
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), "l1_loss_fwd: not deterministic"
    ref = (a.double() - b.double()).abs().sum().reshape(1)
    return _check(f"l1_loss_fwd[n={n}]", out, ref, _two_stage_bar(-(-n // 4), nb, ref) * 4 + 1e-45)


def check_mask_rows(K, device, size):
    g = _gen(16)
    B, T, Cc = {"tiny": (3, 1, 128), "wrap": (5, 1301, 256), "c2": (32, 128, 256)}[size]
    x = torch.randn(B, T, Cc, generator=g)
    length = torch.tensor([0, T, T + 5] + [int(v) for v in torch.randint(0, T + 1, (B - 3,), generator=g)], dtype=torch.int32)
    xv, _ = gvec(x.numel(), device); xv.copy_(x.reshape(-1).to(device))
    out, ob = gvec(x.numel(), device, fill="sentinel")
    K.mask_rows(out.view(B, T, Cc), xv.view(B, T, Cc), length.to(device))
    _sync(device)
    assert guards_intact(ob, vmask(ob, x.numel())), "mask_rows: write outside dst"
    ref = torch.empty(B, T, Cc, dtype=torch.float64)
    MK.mask_rows(ref, x.double(), length)
    return _check("mask_rows", out.view(B, T, Cc), ref)


def check_adam(K, device, n, clip_mode):
    """clip_mode: "active" (norm > clip), "inactive" (norm < clip), "off" (clip <= 0)"""
    g = _gen(17)
    f32 = lambda v: float(torch.tensor(v, dtype=torch.float32))
    p0, g0 = torch.randn(n, generator=g), torch.randn(n, generator=g)
    m0, v0 = torch.randn(n, generator=g) * 0.1, torch.rand(n, generator=g) * 0.01
    ss = float((g0.double() ** 2).sum())
    norm = math.sqrt(ss)
    clip = {"active": f32(norm / 3 + 1e-3), "inactive": f32(norm * 3 + 1.0), "off": 0.0}[clip_mode]
    lr_t, b1, b2, eps = f32(1e-3), f32(0.9), f32(0.999), f32(1e-8)
    bufs = []
    for t in (p0, g0, m0, v0):
        x, b = gvec(n, device, fill="sentinel"); x.copy_(t.to(device)); bufs.append((x, b))
    sst, _ = gvec(1, device); sst.fill_(ss)
    K.adam_step(bufs[0][0], bufs[1][0], bufs[2][0], bufs[3][0], lr_t, b1, b2, eps, clip, sst)
    _sync(device)
    for x, b in bufs:
        assert guards_intact(b, vmask(b, n)), "adam: write outside"
    assert torch.equal(bufs[1][0].cpu(), g0), "adam: g changed"
    rp, rm, rv = p0.double().clone(), m0.double().clone(), v0.double().clone()
    MK.adam_step(rp, g0.double(), rm, rv, lr_t, b1, b2, eps, clip, torch.tensor([float(sst[0:1].item())], dtype=torch.float64))
    scale = (clip / max(math.sqrt(float(torch.tensor(ss, dtype=torch.float32))), clip)) if clip > 0 else 1.0
    gc = g0.double().abs() * scale
    bm = 8 * U * (b1 * m0.double().abs() + (1 - b1) * gc)
    bv = 8 * U * (b2 * v0.double() + (1 - b2) * gc * gc)
    step = lr_t * rm.abs() / (rv.sqrt() + eps)
    w = _check(f"adam m[{clip_mode}]", bufs[2][0], rm, bm + 1e-45)
    w = max(w, _check(f"adam v[{clip_mode}]", bufs[3][0], rv, bv + 1e-45))
    # the update carries the errors of m (absolute: m may cancel) and of v (relative, halved by the square root)
    bp = 2 * U * rp.abs() + 16 * U * step + lr_t * bm / (rv.sqrt() + eps) + step * bv / (2 * rv + 1e-300)
    return max(w, _check(f"adam p[{clip_mode}]", bufs[0][0], rp, bp + 1e-45))
