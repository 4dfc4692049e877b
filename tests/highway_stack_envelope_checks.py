"""The float64 reference of the fused CBHG highway stack and its bar, written once for the device module
(tests/test_gpu_highway_stack_envelope.py) and the CPU mirror (tests/test_highway_stack_envelope_host.py).

The operation (models/ops.py highway_stack, the unfused chain ops.highway x L + the bi-GRU input products):
    h = x . Wd + bd                                   (C != 128: the width-fixing dense)
    per layer l: H = relu(h . WH + bH), T = sigmoid(h . WT + bT), h = H T + h (1 - T)
    xp = h . Wx + bx                                  [M, 768]
The reference never calls the library: it runs in float64 from the kernel's own fp32 inputs.

Classes of inputs:
  exact  small-integer X, sparse +-1 weights (TF32-exact, so the lo halves are 0) and integer biases; every gate bias is
         +4096 or -4096, far enough that sigmoidf_acc is exactly 1 or 0 and a layer passes exactly H or exactly x.  The
         sparsity pattern, the gate pattern and the biases differ per column and per layer, so a swapped activation
         buffer, a wrong layer order or another layer's bias changes bits.  `reference` asserts the premise (every
         activation an integer, every |partial sum| below 2^24, every gate at least 30 from 0 on the 1 side and 100 on
         the 0 side); the kernel must then equal float64 rounded once, bit for bit;
  float  random normal values, every fifth row of X 30 times larger so that its gates saturate.
Bar of the float class, per element, first order in the errors, u = 2^-24:
    |got - ref| <= C_HW u P + Q
  every dense adds its own error C_HW u S, S = rss(operand, W) + |b| in float64 (3xTF32 products and the fp32
  accumulation, bias add included; rss(X, W) = sqrt(X^2 . W^2), independent per-term errors add in quadrature as in
  tests/decoder_step_checks.py), and passes its input's bound on through rss(bound, W).  Why not the L1 form
  |operand| . |W| + |b|: carried through four layers, |W| grows the bound by about sqrt(128) per layer.  On the CPU mirror
  that makes single-pass TF32 pass a one-row case (worst ratio 1.1).  rss keeps every injected fault above 20 times the bar.
  The device does not accumulate independently: wgmma truncates, so its errors add with a bias.  That bias is why the
  H100's worst ratio is about 6 times the mirror's, and C_HW absorbs it.  It is calibrated over every K the ABI allows
  (K <= 128, four layers).  A highway layer carries both through
  its derivatives: the relu mask (kept where the pre-activation is within its own bound of the kink), sigma'(pre_T) |H - x|
  for the gate plus 2.5e-7 for sigmoidf_acc (common.cuh), T on H's bound, (1 - T) on x's bound, and 2u (H T + |x|) for
  the fp32 combine.  P collects the terms scaled by C_HW, Q the rest.
C_HW is about twice the worst ratio (|got - ref| - Q) / (u P) measured on an H100 80GB HBM3 (700 W) over every case,
C_HW_MEASURED (DESIGN.md section 3.1).  A bar of that size still fails single-pass TF32 and a dropped lo.hi term by a
factor above 20 on every case of the CPU mirror (tests/test_highway_stack_envelope_host.py)."""
from __future__ import annotations

import torch

from tests import highway_stack_envelope_cases as HC

U = 2.0 ** -24
C_HW = 96.0
C_HW_MEASURED = 44.95         # worst (|got - ref| - Q) / (u P) of the H100 run over every case
SIG_ERR = 2.5e-7
GATE_BIAS = 4096.0
CLASSES = ("exact", "float")
XP_N = HC.XP_N


def gen(seed):
    return torch.Generator().manual_seed(seed)


def _sparse(rows, cols, nnz, g):
    """[rows, cols] with min(nnz, rows) entries +-1 per column at random rows, 0 elsewhere"""
    idx = torch.rand(rows, cols, generator=g).argsort(dim=0)[:min(nnz, rows)]
    sign = torch.randint(0, 2, idx.shape, generator=g).float() * 2 - 1
    return torch.zeros(rows, cols).scatter_(0, idx, sign)


def params(c: HC.Case, klass, seed):
    """CPU fp32 parameters in the model's layout: Wd [C,128], bd [128] (C != 128), Whw[l] = [WH | WT] [128,256],
    bhw[l] = [bH | bT] [256], Wx [128,768], bx [768]"""
    g = gen(seed)
    p = {"Whw": [], "bhw": []}
    if klass == "exact":
        if c.dense:
            p["Wd"] = _sparse(c.C, 128, 3, g)
            p["bd"] = torch.randint(-3, 4, (128,), generator=g).float()
        for _ in range(c.L):
            W = torch.cat([_sparse(128, 128, 3, g), _sparse(128, 128, 2, g)], dim=1)
            bT = torch.where(torch.rand(128, generator=g) < 0.5, GATE_BIAS, -GATE_BIAS)
            p["Whw"].append(W)
            p["bhw"].append(torch.cat([torch.randint(-4, 5, (128,), generator=g).float(), bT]))
        p["Wx"] = _sparse(128, XP_N, 3, g)
        p["bx"] = torch.randint(-8, 9, (XP_N,), generator=g).float()
        return p
    if c.dense:
        p["Wd"] = torch.randn(c.C, 128, generator=g) / c.C ** 0.5
        p["bd"] = 0.5 * torch.randn(128, generator=g)
    for _ in range(c.L):
        p["Whw"].append(torch.randn(128, 256, generator=g) / 128 ** 0.5)
        p["bhw"].append(0.5 * torch.randn(256, generator=g))
    p["Wx"] = torch.randn(128, XP_N, generator=g) / 128 ** 0.5
    p["bx"] = 0.5 * torch.randn(XP_N, generator=g)
    return p


def inputs(c: HC.Case, klass, seed):
    """CPU fp32 X [M, C]"""
    g = gen(seed + 1000)
    if klass == "exact":
        return torch.randint(-2, 3, (c.M, c.C), generator=g).float()
    X = torch.randn(c.M, c.C, generator=g)
    X[::5] *= 30.0
    return X


def to(p, dev, dtype=torch.float64):
    return {k: ([t.to(dev, dtype) for t in v] if isinstance(v, list) else v.to(dev, dtype)) for k, v in p.items()}


def rss(X, W):
    """sqrt(X^2 . W^2): the size of X . W for independent per-term errors of size X (tests/decoder_step_checks.py)"""
    return torch.sqrt((X * X) @ (W * W))


def _premise(name, h, S):
    assert bool((S < 2.0 ** 24).all()), f"{name}: exact-class premise broken: a partial sum reaches 2^24"
    assert bool((h == h.round()).all()), f"{name}: exact-class premise broken: a non-integer activation"


def reference(X, p, L, c_bar=C_HW, exact=False):
    """float64 (xp, P, Q) of rows X [n, C] (float64) under parameters p (float64, same device); exact = the exact class
    (asserts its premise, gates taken as the step they saturate to)"""
    h = X
    P = torch.zeros_like(h)
    Q = torch.zeros_like(h)

    def dense(h, P, Q, W, b, name):
        y = h @ W + b
        if exact:
            _premise(name, y, h.abs() @ W.abs() + b.abs())
        return y, rss(P, W) + rss(h, W) + b.abs(), rss(Q, W)

    if "Wd" in p:
        h, P, Q = dense(h, P, Q, p["Wd"], p["bd"], "dense")
    for l in range(L):
        W, b = p["Whw"][l], p["bhw"][l]
        a, Pa, Qa = dense(h, P, Q, W[:, :128], b[:128], f"highway{l} H")
        t, Pt, Qt = dense(h, P, Q, W[:, 128:], b[128:], f"highway{l} T")
        H = a.clamp_min(0.0)
        if exact:
            assert bool(((t >= 30) | (t <= -100)).all()), f"highway{l}: exact-class premise broken: a gate not saturated"
            T = (t > 0).double()
        else:
            T = torch.sigmoid(t)
        y = H * T + h * (1 - T)
        live = (a > -(c_bar * U * Pa + Qa)).double()
        ds = T * (1 - T)
        d = (H - h).abs()
        P, Q = (ds * Pt * d + T * live * Pa + (1 - T) * P,
                (ds * Qt + SIG_ERR) * d + T * live * Qa + (1 - T) * Q + 2 * U * (H * T + h.abs()))
        h = y
    return dense(h, P, Q, p["Wx"], p["bx"], "xp")


def check_exact(got, ref, name):
    """bit for bit the float64 result rounded once (every exact-class result is an integer below 2^24)"""
    want = ref.float()
    bad = int((got != want).sum()) + int(torch.isnan(got).sum())
    assert bad == 0, f"{name}: {bad} elements differ from float64, max |d| {(got.double() - ref).abs().max().item():g}"


def unit_ratio(got, ref, P, Q):
    """worst (|got - ref| - Q) / (u P): the bar with C_HW = 1"""
    err = ((got.double() - ref).abs() - Q).clamp_min(0)
    unit = U * P
    r = torch.where(unit > 0, err / unit, torch.where(err > 0, torch.inf, 0.0))
    return r.max().item() if r.numel() else 0.0


def check_float(got, ref, P, Q, name):
    """asserts finite output within the bar; returns the worst unit ratio"""
    assert bool(torch.isfinite(got).all()), f"{name}: non-finite output (a NaN guard or padding was read)"
    w = unit_ratio(got, ref, P, Q)
    assert w <= C_HW, f"{name}: worst element at {w:.3f} of the unit bar, C_HW = {C_HW}"
    return w
