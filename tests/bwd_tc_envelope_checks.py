"""The checks of the backward's wgmma routes (tests/bwd_tc_envelope_cases.py), written once: the device module runs them
through tacotron_b200.kernels and the library; the host module uses the same sequence builders, bars and plan.

Reference.  Every route computes out[p, q] = init + sum_k a[k, p] b[k, q] in a known k order: k-blocks of 32 rows
(taco_conv_dw: 32 rows t of one utterance, tap-shifted X, zero rows past T) or 32 channels (taco_linear_fwd: tap-major,
channels zero-padded to a multiple of 32).  `dw_sequences` / `gemm_sequences` / `conv_dx_sequences` build those operand
sequences in float64 from the kernel's own fp32 inputs, and `contraction` forms, in float64 on the same device, the
result and the two quantities the bar is made of.

Classes of inputs:
  int     small integers, every partial sum below 2^24: each route must equal float64 bit for bit.  Exact sums do not
          depend on the order of the atomics, so this holds whatever the split plan;
  offset  positive values 1 + k 2^-12 (X) and 1 + k 2^-13 (dZ, W) whose low bits lie below TF32 precision: a dropped lo
          term is then a systematic error of ~2^-12 relative, which no bar below absorbs;
  rand    random normal values.
Bar (offset and rand classes), per element, u = 2^-24:
    |got - ref| <= C_BAR (2^-22 rss + u A) + 2 u |ref|
  rss = sqrt(sum_k a^2 b^2): the 3xTF32 products (lo.lo dropped, each half rounded to nearest) err by ~2^-22 |a b| each,
        with random sign, so they add in quadrature;
  A   = the accumulation: sum over k-blocks of |running sum at the block's end| inside each chain (the tensor core adds
        12 products per k-block into an fp32 accumulator), + S = sum |a||b| (the products' own alignment inside each
        wgmma), + sum over chains of |init + chain totals so far| (each chain's fp32 result added into dW by an atomic,
        or the residual added by the epilogue).  taco_conv_dw cuts chains every 1024 rows, so A does not grow faster
        than the result with the rows.
  2u|ref|: the final rounding to fp32 and the residual add.
  Single-pass TF32 errs by ~2^-11 |a b| per product: 2^11 / C_BAR times the product term at any K, and above the
  accumulation term at every case of the list (tests/test_bwd_tc_envelope_host.py checks both on a CPU model).
  DX_TC_IMPL = TACO_IMPL_TC (tf32 mode, single pass) is held to the linear envelope's 2^-9 S; a call that falls back to
  taco_gemm to the training envelope's 2^-16 S.
C_BAR is set from the H100 run (DESIGN.md 3.5): see C_BAR_MEASURED."""
from __future__ import annotations

import ctypes as C
from contextlib import contextmanager
from unittest import mock

import torch

from tacotron_b200 import _lib as L
from tests import bwd_tc_envelope_cases as BC
from tests.train_envelope_checks import _fill, guards_intact, sentinel

U = 2.0 ** -24
C_BAR = 16.0
C_BAR_MEASURED = 6.43          # worst (err - 2u|ref|) / (2^-22 rss + u A) of the H100 run over every route (conv_dx rand)
TOL_TF32 = 2.0 ** -9
TOL_FALLBACK = 2.0 ** -16
NAN = float("nan")
CLASSES = ("int", "offset", "rand")


def gen(seed):
    return torch.Generator().manual_seed(seed)


def values(klass, shape, g, role):
    """CPU fp32 values of one operand; role "x" (X, A, dZ of conv_dx), "z" (dZ of dw, W), "init" (accumulated-into)"""
    if klass == "int":
        return torch.randint(-4, 5, shape, generator=g).float()
    if klass == "offset":
        step = 2.0 ** -12 if role == "x" else 2.0 ** -13
        return 1.0 + torch.randint(0, 8, shape, generator=g).float() * step
    return torch.randn(shape, generator=g)


def rn_tf32(x):
    """rn_tf32 of csrc/gemm_tc.cu on the bit pattern: (bits + 0x1000) & 0xffffe000"""
    b = x.float().contiguous().view(torch.int32)
    r = (b + 0x1000) & -0x2000                      # int32 wrap-around add and mask = the uint32 bit operations
    return r.view(torch.float32).view(x.shape)


# ------------------------------------------------------------------------------------------------------------------
# operand sequences in kernel k order (float64 [K, P] and [K, Q], K a multiple of 32) and the chains over them
# ------------------------------------------------------------------------------------------------------------------
def _shift_utt(X, B, T, sh):
    """[B*T, C] -> [B, T, C]: row t of utterance b = X[b, t + sh] (zero outside [0, T))"""
    X3 = X.reshape(B, T, -1)
    out = torch.zeros_like(X3)
    lo, hi = max(0, -sh), min(T, T - sh)
    if lo < hi:
        out[:, lo:hi] = X3[:, lo + sh:hi + sh]
    return out


def _pad_rows(X3, bps):
    B, T, Cc = X3.shape
    out = torch.zeros(B, bps * BC.KB, Cc, dtype=X3.dtype, device=X3.device)
    out[:, :T] = X3
    return out.reshape(B * bps * BC.KB, Cc)


def dw_sequences(c: BC.DwCase, X, Z, j, extra_shift=0):
    """(As, Bs, chains) of tap j: rows (b, t) in blocks of 32 per utterance"""
    p = BC.plan_of(c)
    As = _pad_rows(_shift_utt(X, c.B, c.T, c.t0 + j + extra_shift), p.blocks_per_seq)
    Bs = _pad_rows(Z.reshape(c.B, c.T, -1), p.blocks_per_seq)
    return As, Bs, [(a * BC.KB, b * BC.KB) for a, b in p.chains()]


def _pad_k(X, kpad):
    out = torch.zeros(kpad, X.shape[1], dtype=X.dtype, device=X.device)
    out[:X.shape[0]] = X
    return out


def gemm_sequences(c: BC.GemmCase, A, Bm, extra_shift=0):
    """Y = shift(A) . W: k = channel, in 32-channel blocks"""
    from tests import mirror_kernels as MK
    kp = -(-c.Kc // BC.KB) * BC.KB
    As = _pad_k(MK._shift_rows(A, c.shift + extra_shift, c.period).t(), kp)
    W = Bm.t() if c.tb else Bm
    return As, _pad_k(W, kp), [(0, kp)]


def conv_dx_sequences(T, dZ, W, extra_shift=0):
    """dX = dZ convolved with the taps reversed, W^T: k = (i, c) tap-major, channels padded to 32"""
    taps, Cin, Cout = W.shape
    B = dZ.shape[0] // T
    cp = -(-Cout // BC.KB) * BC.KB
    t0r = -(BC.tf_tap0(taps) + taps - 1)
    As = torch.zeros(taps * cp, B * T, dtype=dZ.dtype, device=dZ.device)
    Bs = torch.zeros(taps * cp, Cin, dtype=W.dtype, device=W.device)
    for i in range(taps):
        As[i * cp:i * cp + Cout] = _shift_utt(dZ, B, T, t0r + i + extra_shift).reshape(B * T, Cout).t()
        Bs[i * cp:i * cp + Cout] = W[taps - 1 - i].t()
    return As, Bs, [(0, taps * cp)]


def contraction(As, Bs, chains, init):
    """float64 (ref, rss, A) of out = init + As^T Bs over the chains (see the module docstring)"""
    acc = torch.zeros_like(init)
    run = init.clone()
    chain_term = torch.zeros_like(init)
    for k0, k1 in chains:
        P = torch.zeros_like(init)
        for b0 in range(k0, k1, BC.KB):
            P += As[b0:b0 + BC.KB].t() @ Bs[b0:b0 + BC.KB]
            acc += P.abs()
        run += P
        chain_term += run.abs()
    rss = torch.sqrt((As * As).t() @ (Bs * Bs))
    S = As.abs().t() @ Bs.abs()
    return run, rss, acc + S + chain_term, S


def unit_ratio(got, ref, rss, A):
    """worst (|got - ref| - 2u|ref|) / (2^-22 rss + u A): the 3xTF32 bar with C_BAR = 1 (elements whose every product is 0
    must be exact)"""
    err = ((got - ref).abs() - 2 * U * ref.abs()).clamp_min(0)
    unit = 2.0 ** -22 * rss + U * A
    r = torch.where(unit > 0, err / unit, torch.where(err > 0, torch.inf, 0.0))
    return r.max().item() if r.numel() else 0.0


def bar_ratio(got, ref, rss, A, S, mode, name):
    """worst ratio to the bar; asserts finite output and, for the int class (mode None), bit equality"""
    assert bool(torch.isfinite(got).all()), f"{name}: non-finite output (a NaN guard or an unwritten beta=0 dW was read)"
    err = (got - ref).abs()
    if mode is None:
        bad = int((err != 0).sum())
        assert bad == 0, f"{name}: {bad} elements differ from float64, max {err.max().item():g}"
        return 0.0
    if mode == "tf32":
        bar = TOL_TF32 * S + 2 * U * ref.abs()
    elif mode == "fallback":
        bar = TOL_FALLBACK * S + 2 * U * ref.abs()
    else:
        w = unit_ratio(got, ref, rss, A)
        assert w <= C_BAR, f"{name}: worst element at {w:.3f} of the unit bar, C_BAR = {C_BAR}"
        return w
    r = torch.where(bar > 0, err / bar, torch.where(err > 0, torch.inf, 0.0))
    w = r.max().item() if r.numel() else 0.0
    assert w <= 1.0, f"{name}: worst element at {w:.3f} of its bar"
    return w


# ------------------------------------------------------------------------------------------------------------------
# library call recording: which entry a kernels.* call reached, and the taco_linear_fwd route it took
# ------------------------------------------------------------------------------------------------------------------
class Recorder:
    def __init__(self, lib):
        self._lib, self.calls, self.routes = lib, [], []

    def __getattr__(self, name):
        f = getattr(self._lib, name)
        if name in ("taco_linear_route", "taco_last_error", "taco_launch_count"):      # queries, not launches
            return f

        def call(*a):
            self.calls.append(name)
            if name == "taco_linear_fwd":
                self.routes.append(L.linear_route(a[0]._obj))
            return f(*a)
        return call


@contextmanager
def recording(K, **switches):
    rec = Recorder(L.lib())
    prev = {k: getattr(K, k) for k in switches}
    for k, v in switches.items():
        setattr(K, k, v)
    try:
        with mock.patch.object(L, "lib", lambda: rec):
            yield rec
    finally:
        for k, v in prev.items():
            setattr(K, k, v)


def _sync(dev):
    if torch.device(dev).type == "cuda":
        torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------
# taco_conv_dw
# ------------------------------------------------------------------------------------------------------------------
def dw_inputs(c: BC.DwCase, klass, seed):
    g = gen(seed)
    X = values(klass, (c.rows, c.C), g, "x")
    Z = values(klass, (c.rows, c.N), g, "z")
    init = [values(klass, (c.C, c.N), g, "init") for _ in range(c.taps)]
    if c.via == "gemm" and c.beta == 0.0:
        init = [torch.zeros(c.C, c.N)] * c.taps
    return X, Z, init


def run_dw(K, c: BC.DwCase, X, Z, init, dev):
    """one call on fresh guarded buffers; returns (dW buffer, Recorder)"""
    lay = BC.DwLayout(c)
    bufX = _fill(lay.X, [X], torch.full((lay.X.size,), NAN)).to(dev)
    bufZ = _fill(lay.Z, [Z], torch.full((lay.Z.size,), NAN)).to(dev)
    w0 = [torch.full((c.C, c.N), NAN)] * c.taps if (c.via == "gemm" and c.beta == 0.0) else init
    bufW = _fill(lay.W, w0, sentinel(lay.W.size, "cpu")).to(dev)
    with recording(K, DW_TC=True, DW_TC_MIN_ROWS=1) as rec:
        if c.via == "direct":
            P = lambda buf, op: C.c_void_p(buf.data_ptr() + 4 * op.off)
            rc = L.lib().taco_conv_dw(P(bufW, lay.W), lay.ldw, lay.tap_stride, P(bufX, lay.X), lay.X.ld, P(bufZ, lay.Z),
                                      lay.Z.ld, c.B, c.T, c.C, c.N, c.taps, c.t0, L.current_stream())
            assert rc == 0, L.lib().taco_last_error().decode()
        else:
            K.gemm(lay.W.view(bufW), lay.X.view(bufX), lay.Z.view(bufZ), ta=True, beta=c.beta, shift=c.t0,
                   period=c.T if c.period else 0, batch=c.taps, bshift=1, c_bstride=lay.tap_stride if c.taps > 1 else 0)
    _sync(dev)
    assert rec.calls == ["taco_conv_dw"], f"{c.name}: expected one taco_conv_dw call, got {rec.calls}"
    assert guards_intact(bufW, lay.W.mask(dev)), f"{c.name}: write outside the dW views"
    return bufW, lay


def check_dw(K, c: BC.DwCase, klass, dev, seed=0):
    X, Z, init = dw_inputs(c, klass, seed)
    bufW, lay = run_dw(K, c, X, Z, init, dev)
    Xd, Zd = X.to(dev, torch.float64), Z.to(dev, torch.float64)
    worst = 0.0
    for j in range(c.taps):
        As, Bs, chains = dw_sequences(c, Xd, Zd, j)
        ref, rss, A, S = contraction(As, Bs, chains, init[j].to(dev, torch.float64))
        got = lay.W.view(bufW, j).double()
        worst = max(worst, bar_ratio(got, ref, rss, A, S, None if klass == "int" else "x3", f"{c.name} [{klass}] tap {j}"))
    if klass == "rand" and BC.dw_deterministic(c):
        again, _ = run_dw(K, c, X, Z, init, dev)
        assert torch.equal(again.view(torch.int32), bufW.view(torch.int32)), f"{c.name}: one-drain launch not bit-reproducible"
    return worst


# ------------------------------------------------------------------------------------------------------------------
# kernels._gemm_tc (kernels.gemm, ta = False)
# ------------------------------------------------------------------------------------------------------------------
def gemm_inputs(c: BC.GemmCase, klass, seed):
    g = gen(seed)
    A = values(klass, (c.M, c.Kc), g, "x")
    Bm = values(klass, (c.N, c.Kc) if c.tb else (c.Kc, c.N), g, "z")
    C0 = values(klass, (c.M, c.N), g, "init") if c.beta == 1.0 else torch.zeros(c.M, c.N)
    return A, Bm, C0


def run_gemm_tc(K, c: BC.GemmCase, A, Bm, C0, dev, rows=None):
    """kernels.gemm on fresh guarded buffers (rows = (r0, r1): kernels._gemm_tc on those rows alone)"""
    lay = BC.GemmLayout(c)
    bufA = _fill(lay.A, [A], torch.full((lay.A.size,), NAN)).to(dev)
    bufB = _fill(lay.B, [Bm], torch.full((lay.B.size,), NAN)).to(dev)
    bufC = _fill(lay.C, [C0 if c.beta == 1.0 else torch.full((c.M, c.N), NAN)], sentinel(lay.C.size, "cpu")).to(dev)
    Av, Bv, Cv = lay.A.view(bufA), lay.B.view(bufB), lay.C.view(bufC)
    with recording(K, GEMM_TC=True, DX_TC_IMPL=BC.IMPL[c.impl]) as rec:
        if rows is None:
            K.gemm(Cv, Av, Bv, tb=c.tb, beta=c.beta, shift=c.shift, period=c.period)
        else:
            K._gemm_tc(Cv[rows[0]:rows[1]], Av[rows[0]:rows[1]], Bv, c.tb, c.beta, c.shift, c.period)
    _sync(dev)
    assert guards_intact(bufC, lay.C.mask(dev)), f"{c.name}: write outside Y's view"
    return bufC, lay, rec


def check_gemm_tc(K, c: BC.GemmCase, klass, dev, seed=0):
    A, Bm, C0 = gemm_inputs(c, klass, seed)
    bufC, lay, rec = run_gemm_tc(K, c, A, Bm, C0, dev)
    Cv = lay.C.view(bufC)
    tc = c.M >= K.GEMM_TC_MIN_ROWS                # every case's layout passes the other conditions of _gemm_tc_ok
    expect = ["taco_pack_weight_x3" if c.impl == "fp32x3" else "taco_pack_weight", "taco_linear_fwd"] if tc else ["taco_gemm"]
    assert rec.calls == expect, f"{c.name}: expected {expect}, got {rec.calls}"
    As, Bs, chains = gemm_sequences(c, A.to(dev, torch.float64), Bm.to(dev, torch.float64))
    ref, rss, Aacc, S = contraction(As, Bs, chains, C0.to(dev, torch.float64))
    mode = None if klass == "int" else ("fallback" if not tc else ("tf32" if c.impl == "tf32" else "x3"))
    w = bar_ratio(Cv.double(), ref, rss, Aacc, S, mode, f"{c.name} [{klass}]")
    if tc and klass == "rand":
        # no atomics: bit for bit again, and rows run alone give the same bits (each row is its own dot products)
        again, _, _ = run_gemm_tc(K, c, A, Bm, C0, dev)
        assert torch.equal(again.view(torch.int32), bufC.view(torch.int32)), f"{c.name}: not bit-reproducible"
        if c.period > 0 or c.shift == 0:
            r0 = c.M - (c.period if c.period else 300)
            alone, _, _ = run_gemm_tc(K, c, A, Bm, C0, dev, rows=(r0, c.M))
            assert torch.equal(lay.C.view(alone)[r0:].contiguous().view(torch.int32),
                               Cv[r0:].contiguous().view(torch.int32)), f"{c.name}: rows {r0}: alone differ"
    return w, (rec.routes[0] if rec.routes else None), mode


# ------------------------------------------------------------------------------------------------------------------
# kernels.conv_dx on the TC route
# ------------------------------------------------------------------------------------------------------------------
def conv_dx_inputs(c: BC.ConvDxCase, klass, seed):
    g = gen(seed)
    lay = BC.ConvDxLayout(c)
    Z = values(klass, (lay.Z.rows, lay.Z.cols), g, "x")
    Ws = [values(klass, (k, c.Cin, 128 if c.bank else c.Cout), g, "z") for k, _ in lay.z_slices(c)]
    X0 = values(klass, (lay.X.rows, c.Cin), g, "init") if c.beta == 1.0 else torch.zeros(lay.X.rows, c.Cin)
    return Z, Ws, X0


def run_conv_dx(K, c: BC.ConvDxCase, Z, Ws, X0, dev):
    lay = BC.ConvDxLayout(c)
    bufZ = _fill(lay.Z, [Z], torch.full((lay.Z.size,), NAN)).to(dev)
    bufX = _fill(lay.X, [X0 if c.beta == 1.0 else torch.full(X0.shape, NAN)], sentinel(lay.X.size, "cpu")).to(dev)
    Zv, Xv = lay.Z.view(bufZ), lay.X.view(bufX)
    with recording(K, DX_TC=True, DX_TC_IMPL=BC.IMPL[c.impl]) as rec:
        for (k, col), W in zip(lay.z_slices(c), Ws):
            width = 128 if c.bank else c.Cout
            K.conv_dx(Xv, Zv[:, col:col + width], W.to(dev), c.T, beta=c.beta)
    _sync(dev)
    n = len(lay.z_slices(c))
    assert rec.calls.count("taco_linear_fwd") == n and "taco_gemm" not in rec.calls, f"{c.name}: {rec.calls}"
    assert guards_intact(bufX, lay.X.mask(dev)), f"{c.name}: write outside dX's view"
    return bufX, lay, rec


def check_conv_dx(K, c: BC.ConvDxCase, klass, dev, seed=0):
    Z, Ws, X0 = conv_dx_inputs(c, klass, seed)
    bufX, lay, rec = run_conv_dx(K, c, Z, Ws, X0, dev)
    Zd = Z.to(dev, torch.float64)
    seqs = []
    for (k, col), W in zip(lay.z_slices(c), Ws):
        width = 128 if c.bank else c.Cout
        seqs.append(conv_dx_sequences(c.T, Zd[:, col:col + width], W.to(dev, torch.float64)))
    As = torch.cat([s[0] for s in seqs])
    Bs = torch.cat([s[1] for s in seqs])
    chains, k0 = [], 0
    for s in seqs:                      # one chain per call: each call's result is added to dX by its epilogue
        chains.append((k0, k0 + s[0].shape[0]))
        k0 += s[0].shape[0]
    ref, rss, Aacc, S = contraction(As, Bs, chains, X0.to(dev, torch.float64))
    mode = None if klass == "int" else ("tf32" if c.impl == "tf32" else "x3")
    w = bar_ratio(lay.X.view(bufX).double(), ref, rss, Aacc, S, mode, f"{c.name} [{klass}]")
    if klass == "rand":
        again, _, _ = run_conv_dx(K, c, Z, Ws, X0, dev)
        assert torch.equal(again.view(torch.int32), bufX.view(torch.int32)), f"{c.name}: not bit-reproducible"
    return w, rec.routes, mode
