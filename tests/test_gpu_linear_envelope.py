"""-m gpu: taco_linear_fwd over its whole dispatch envelope against float64, in all three modes (fp32 = SIMT FFMA,
tf32 = wgmma TF32, fp32x3 = wgmma 3xTF32), with guard bands around every operand; the weight packing bit for bit.

Cases and operand layouts: tests/linear_envelope_cases.py (tests/test_linear_routes.py checks on the CPU that they
reach every route the dispatcher allows).  Each case runs two input classes:
  * exact: small integers for X, W, biases, shift and residual, +-2^k scales, keep_scale 2.  Every product and partial sum
    is an integer below 2^22, exact in fp32, in TF32 and in the 3xTF32 split (lo = 0): the result must be bit-identical
    to float64 in every mode, so a wrong tap, padding row, utterance, column or pool neighbour fails by at least 1;
  * float: random fp32 values, some rows scaled so that pre-activations reach +-100 (sigmoid / tanh saturate).  Each
    element is held to tol[mode] * S + eps_act, S = the float64 contraction of |X| |W| carried through the epilogue's
    magnitudes (|scale|, |bias|, |shift|, |residual|), eps_act = the absolute error of the device sigmoid / tanh.
Guard bands: X, residual, hx and bias_utt sit in NaN-filled buffers (GUARD rows before and after, NaN padding columns up
to the row stride), bias / scale / shift have NaN tails, and Y's buffer is filled with a sentinel bit pattern: a read
outside an operand turns the output NaN, a write outside the output changes a sentinel.
References are float64 torch on the device; they never call the library."""
import ctypes as C
import json
import os
import zlib

import numpy as np
import pytest
import torch

from tacotron_b200 import _lib as L
from tests.linear_envelope_cases import CASES, Layout, cpad, check_route, desc

pytestmark = pytest.mark.gpu

# per-element bars (times S), from the error model.  Worst float-class element of this file on an H100 80GB HBM3 (400 W
# power limit), as a fraction of the bar:
#   fp32   (FFMA chains, round-to-nearest)                                   2^-20: 0.92 (16-filter bank, K = 2048)
#   tf32   (10-bit mantissa products)                                         2^-9:  0.52
#   fp32x3 (3xTF32: the dropped lo.lo term is 2^-22; the tensor core's fp32 accumulation truncates, and each k8-step adds
#           three products into the accumulators, so K = 6144 is 2304 truncating additions whose errors do not cancel)
#                                                                             2^-16: 0.72 (C = 2048, 3 taps, K = 6144)
TOL = {"fp32": 2.0 ** -20, "fp32x3": 2.0 ** -16, "tf32": 2.0 ** -9}
# global bars of tests/test_gpu_linear.py (max |err| / max |ref| over the output), which hold as well -- except fp32x3
# beyond K = 2048: there the truncating accumulation above reaches 6.7e-5 of max |ref| (C = 2048, 3 taps), so the
# long-K contractions are held to 1e-4
GLOBAL = {"fp32": 2e-5, "fp32x3": 2e-5, "tf32": 3e-3}
GLOBAL_LONG_K = {"fp32x3": (2048, 1e-4)}
# absolute error of sigmoidf_acc / tanhf_acc (csrc/common.cuh): __expf (2 + 1.17|x| ulp relative) and __fdividef (2 ulp)
EPS_ACT = {L.ACT_SIGMOID: 2.5e-7, L.ACT_TANH: 5e-7}
SENTINEL = 0x7FC0FEED
DEV = "cuda"
WORST = {}                     # mode -> worst float-class |err| as a fraction of its per-element bound, and its case


def _seed(*parts):
    return zlib.crc32("/".join(map(str, parts)).encode())


def _weights_shapes(c):
    if c.bank_K:
        return [(k, c.C, 128) for k in range(1, c.bank_K + 1)]
    return [(c.taps, c.C, c.N)]


def _inputs(c, cls, seed):
    g = torch.Generator().manual_seed(seed)
    M, N = c.B * c.T, c.N
    if cls == "exact":
        ri = lambda shape, m: torch.randint(-m, m + 1, shape, generator=g).float()
        X = ri((M, c.C), 3)
        Ws = [ri(s, 3) for s in _weights_shapes(c)]
        scale = torch.where(torch.rand(N, generator=g) < 0.5, -1.0, 1.0) * 2.0 ** torch.randint(-2, 3, (N,), generator=g).float()
        d = dict(X=X, W=Ws, bias=ri((N,), 8), bias_utt=ri((c.B, N), 8), scale=scale, shift=ri((N,), 8),
                 residual=ri((M, N), 8), hx=ri((M, 128), 8), ks=2.0)
    else:
        rows = torch.where(torch.rand(M, 1, generator=g) < 0.1, 25.0, 1.0)
        X = torch.randn(M, c.C, generator=g) * rows
        Ws = [torch.randn(s, generator=g) / (s[0] * s[1]) ** 0.5 for s in _weights_shapes(c)]
        d = dict(X=X, W=Ws, bias=0.5 * torch.randn(N, generator=g), bias_utt=0.5 * torch.randn(c.B, N, generator=g),
                 scale=1 + 0.5 * torch.randn(N, generator=g), shift=0.5 * torch.randn(N, generator=g),
                 residual=torch.randn(M, N, generator=g), hx=torch.randn(M, 128, generator=g), ks=1.25)
    d["keep"] = (torch.rand(M, c.nout, generator=g) >= 0.5).to(torch.uint8)
    return d


def _pack(W, taps, Cin, N, dst, row0, n_total, x3):
    ld = dst.shape[1]
    st = L.current_stream()
    hi = C.c_void_p(dst.data_ptr() + row0 * ld * 4)
    if x3:
        lo = C.c_void_p(dst.data_ptr() + (n_total + row0) * ld * 4)
        L.check(L.lib().taco_pack_weight_x3(L.ptr(W), taps, Cin, N, hi, lo, ld, st), "taco_pack_weight_x3")
    else:
        L.check(L.lib().taco_pack_weight(L.ptr(W), taps, Cin, N, hi, ld, st), "taco_pack_weight")


class _Buffers:
    """The device operands of a case, each inside its guard band; .addr = address of each operand's row 0."""

    def __init__(self, c, lay, data, impl):
        dev = "cuda"
        self.keepalive = []
        self.addr = {}
        nan = lambda n: torch.full((n,), float("nan"), device=dev)

        def place(name, t):
            rows, ld, off = lay.shapes[name]
            buf = nan(lay.size(name))
            buf[off:off + rows * ld].view(rows, ld)[:, :t.shape[1]] = t.to(dev)
            self.keepalive.append(buf)
            self.addr[name] = buf.data_ptr() + 4 * off

        def vec(name, t):
            buf = nan(t.numel() + 8)
            buf[:t.numel()] = t.to(dev)
            self.keepalive.append(buf)
            self.addr[name] = buf.data_ptr()

        place("X", data["X"])
        if c.residual:
            place("residual", data["residual"])
        if c.highway:
            place("hx", data["hx"])
        if c.bias_utt:
            place("bias_utt", data["bias_utt"])
        vec("bias", data["bias"]); vec("scale", data["scale"]); vec("shift", data["shift"])
        keep = data["keep"].to(dev)
        self.keepalive.append(keep)
        self.addr["keep"] = keep.data_ptr()
        self.ybuf = torch.full((lay.y_size,), SENTINEL, dtype=torch.int32, device=dev)
        self.addr["Y"] = self.ybuf.data_ptr() + 4 * lay.y_off
        Wd = [w.to(dev).contiguous() for w in data["W"]]
        Wflat = torch.cat([w.reshape(-1) for w in Wd])          # TF layout; a bank's filters back to back
        self.keepalive += Wd + [Wflat]
        self.addr["W"] = Wflat.data_ptr()
        if impl != "fp32":
            x3 = impl == "fp32x3"
            Wp = torch.zeros(((2 if x3 else 1) * c.N, lay.ldwp), device=dev)
            if c.bank_K:
                for k, w in enumerate(Wd, start=1):
                    _pack(w, k, c.C, 128, Wp, (k - 1) * 128, c.N, x3)
            else:
                _pack(Wd[0], c.taps, c.C, c.N, Wp, 0, c.N, x3)
            self.keepalive.append(Wp)
            self.addr["Wp"] = Wp.data_ptr()


def _conv(X, W, tap0):
    """float64 conv1d with zero outside [0, T) of each utterance: X [B,T,C], W [taps,C,N]"""
    B, T, _ = X.shape
    out = torch.zeros(B, T, W.shape[2], dtype=torch.float64, device=X.device)
    for j in range(W.shape[0]):
        s = tap0 + j
        lo, hi = max(0, -s), min(T, T - s)
        if lo < hi:
            out[:, lo:hi] += X[:, lo + s:hi + s] @ W[j]
    return out


def _pool(v, c):
    """max_pooling1d(2, 1, 'same') over t within each utterance"""
    v = v.view(c.B, c.T, -1)
    out = v.clone()
    out[:, :-1] = torch.maximum(v[:, :-1], v[:, 1:])
    return out.view(c.B * c.T, -1)


def _reference(c, data, tol):
    """float64 result and per-element bound tol * S + eps_act"""
    dev = DEV
    M = c.B * c.T
    X = data["X"].to(dev, torch.float64).view(c.B, c.T, c.C)
    Ws = [w.to(dev, torch.float64) for w in data["W"]]
    if c.bank_K:
        acc = torch.cat([_conv(X, w, -((w.shape[0] - 1) // 2)) for w in Ws], -1)
        S = torch.cat([_conv(X.abs(), w.abs(), -((w.shape[0] - 1) // 2)) for w in Ws], -1)
    else:
        acc = _conv(X, Ws[0], c.tap0_value)
        S = _conv(X.abs(), Ws[0].abs(), c.tap0_value)
    acc, S = acc.view(M, -1), S.view(M, -1)
    d64 = lambda k: data[k].to(dev, torch.float64)
    bias = d64("bias") if c.bias else torch.zeros(c.N, dtype=torch.float64, device=dev)
    if c.highway:
        U = c.nout
        P, SP = acc + bias, S + bias.abs()
        H, Tg, hx = torch.relu(P[:, :U]), torch.sigmoid(P[:, U:]), d64("hx")
        A = H.abs() + hx.abs()
        y = H * Tg + hx * (1 - Tg)
        return y, tol * (SP[:, :U] + A * (SP[:, U:] + 1)) + A * EPS_ACT[L.ACT_SIGMOID]
    u, Su = acc + bias, S + bias.abs()
    if c.bias_utt:
        bu = d64("bias_utt").repeat_interleave(c.T, 0)
        u, Su = u + bu, Su + bu.abs()
    eps = EPS_ACT.get(c.act, 0.0)
    if c.act == L.ACT_RELU:
        a = torch.relu(u)
    elif c.act == L.ACT_SIGMOID:
        a, Su = torch.sigmoid(u), Su + 1
    elif c.act == L.ACT_TANH:
        a, Su = torch.tanh(u), Su + 1
    else:
        a = u
    E = torch.full_like(a, eps)
    if c.bn:
        sc, sh = d64("scale"), d64("shift")
        a, Su, E = a * sc + sh, Su * sc.abs() + sh.abs(), E * sc.abs()
    if c.pool:
        a, Su, E = _pool(a, c), _pool(Su, c), _pool(E, c)
    if c.keep:
        k = data["keep"].to(dev, torch.float64) * data["ks"]
        a, Su, E = a * k, Su * k, E * k
    if c.residual:
        r = d64("residual")
        a, Su = a + r, Su + r.abs()
    return a, tol * Su + E


RUNS = [(c, impl, cls) for c in CASES for impl in c.impls for cls in c.classes]


@pytest.mark.parametrize("c,impl,cls", RUNS, ids=[f"{c.name}-{impl}-{cls}" for c, impl, cls in RUNS])
def test_envelope(c, impl, cls):
    lay = Layout(c)
    data = _inputs(c, cls, _seed(c.name, cls))
    bufs = _Buffers(c, lay, data, impl)
    d = desc(c, impl, bufs.addr, lay, keep_scale=data["ks"])
    check_route(c, impl, L.linear_route(d))
    L.check(L.lib().taco_linear_fwd(C.byref(d), L.current_stream()), f"taco_linear_fwd[{c.name}]")
    torch.cuda.synchronize()

    M, nout = c.B * c.T, c.nout
    ybits = bufs.ybuf.clone()
    region = ybits[lay.y_off:lay.y_off + M * lay.ldy].view(M, lay.ldy)[:, :nout]
    y = region.view(torch.float32).double()
    ref, bound = _reference(c, data, TOL[impl])
    region.fill_(SENTINEL)
    bad = int((ybits != SENTINEL).sum())
    assert bad == 0, f"{c.name} {impl}: {bad} elements written outside Y (rows, padding columns or guard rows)"
    assert not torch.isnan(y).any(), f"{c.name} {impl}: NaN in Y (an operand was read outside its bounds)"
    if cls == "exact":
        diff = (y != ref).nonzero()
        assert diff.numel() == 0, (f"{c.name} {impl}: {diff.shape[0]} elements differ from float64, first (row, col) "
                                   f"{tuple(diff[0].tolist())}: {float(y[tuple(diff[0])])} vs {float(ref[tuple(diff[0])])}")
        return
    err = (y - ref).abs()
    over = err > bound
    if over.any():
        i = tuple(over.nonzero()[0].tolist())
        pytest.fail(f"{c.name} {impl}: {int(over.sum())} elements beyond tol*S + eps_act, first {i}: "
                    f"|err| {float(err[i]):.3e} > bound {float(bound[i]):.3e} (ref {float(ref[i]):.4e})")
    if c.act not in (L.ACT_SIGMOID, L.ACT_TANH) and not c.highway:
        # (not behind a sigmoid / tanh: their output is bounded whatever the scale of their input, whose rounding error
        # grows with that scale -- pre-activations of +-100 here.  The per-element bound above holds those elements.)
        bar = GLOBAL[impl]
        if impl in GLOBAL_LONG_K and (c.bank_K or c.taps) * c.C > GLOBAL_LONG_K[impl][0]:
            bar = GLOBAL_LONG_K[impl][1]
        g = float(err.max() / ref.abs().max().clamp_min(1e-30))
        assert g <= bar, f"{c.name} {impl}: max-rel err {g:.3e} > {bar:.1e}"
    ratio = float((err / bound.clamp_min(1e-300)).max())                # worst error as a fraction of its bar
    w = WORST.get(impl)
    if w is None or ratio > w[0]:
        WORST[impl] = (ratio, c.name)


def test_zz_report_worst_float_errors():
    """Record the worst float-class error of each mode as a fraction of its bar (TACO_ENVELOPE_LOG=<path>)."""
    path = os.environ.get("TACO_ENVELOPE_LOG")
    if path and WORST:
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        with open(path, "w") as f:
            json.dump({m: {"worst_fraction_of_bar": r, "case": n, "tol": TOL[m]} for m, (r, n) in WORST.items()}, f, indent=1)


# ------------------------------------------------------------------------------------------------------------------
# weight packing, bit for bit
# ------------------------------------------------------------------------------------------------------------------
def _rna(bits):
    """cvt.rna.tf32.f32 on the bit pattern: round the magnitude to 10 mantissa bits, ties away from zero"""
    return (bits.astype(np.uint64) + 0x1000 & 0xFFFFE000).astype(np.uint32)


def _special_weights(shape, seed):
    rng = np.random.default_rng(seed)
    n = int(np.prod(shape))
    mant = rng.integers(0, 1 << 23, n, dtype=np.uint64)
    expo = rng.integers(1, 253, n, dtype=np.uint64)                      # normal, |W| < 2^126
    sign = rng.integers(0, 2, n, dtype=np.uint64) << 31
    bits = (sign | expo << 23 | mant).astype(np.uint32)
    k = np.arange(n)
    tie = (bits & 0xFFFFE000) | 0x1000                                   # exactly half a TF32 ulp: ties of both signs
    bits = np.where(k % 7 == 1, tie, bits)
    bits = np.where(k % 7 == 2, tie ^ 1, bits)                           # just past the tie
    bits = np.where(k % 7 == 3, (tie - 1) & 0xFFFFFFFF, bits)            # just below the tie
    bits = np.where(k % 7 == 4, (sign | mant).astype(np.uint32), bits)   # subnormals
    bits = np.where(k % 31 == 5, (sign & 0x80000000).astype(np.uint32), bits)   # +-0
    bits = np.where(k % 29 == 6, (sign | 252 << 23 | mant).astype(np.uint32), bits)   # just below 2^126
    bits = np.where(k % 37 == 7, (sign | 0xFFF).astype(np.uint32), bits)              # subnormal tie neighbourhood
    return bits.view(np.float32).reshape(shape)


@pytest.mark.parametrize("taps,Cin,N", [(1, 1, 8), (3, 40, 24), (2, 33, 130), (5, 64, 16)])
def test_pack_weight_bits(taps, Cin, N):
    W = _special_weights((taps, Cin, N), _seed("pack", taps, Cin, N))
    Cp = cpad(Cin)
    ld = taps * Cp + 8                                                   # 8 columns the packer must not touch
    wb = W.view(np.uint32)
    hi_ref = _rna(wb)
    lo_ref = _rna((W - hi_ref.view(np.float32)).view(np.uint32))
    Wd = torch.from_numpy(W.copy()).cuda()
    for x3 in (False, True):
        dst = torch.full(((2 if x3 else 1) * N, ld), SENTINEL, dtype=torch.int32, device="cuda")
        _pack(Wd, taps, Cin, N, dst, 0, N, x3)
        torch.cuda.synchronize()
        got = dst.cpu().numpy().view(np.uint32)
        for half, ref in ((0, hi_ref),) + (((1, lo_ref),) if x3 else ()):
            g = got[half * N:(half + 1) * N]                             # [N][ld]
            for j in range(taps):
                blk = g[:, j * Cp:(j + 1) * Cp]
                np.testing.assert_array_equal(blk[:, :Cin], ref[j].T, err_msg=f"x3={x3} half={half} tap {j}")
                assert (blk[:, Cin:] == 0).all(), "padding channels must be +0"
            assert (g[:, taps * Cp:] == SENTINEL).all(), "columns past taps*Cpad were written"
        if x3:
            hi = got[:N].view(np.float32).astype(np.float64)
            lo = got[N:].view(np.float32).astype(np.float64)
            w = np.stack([W[j].T for j in range(taps)], 1).reshape(N, taps, Cin).astype(np.float64)
            hl = (hi.reshape(N, -1)[:, :taps * Cp].reshape(N, taps, Cp)[:, :, :Cin]
                  + lo.reshape(N, -1)[:, :taps * Cp].reshape(N, taps, Cp)[:, :, :Cin])
            normal = (np.abs(w) >= 2.0 ** -100) & (np.abs(w) < 2.0 ** 126)
            assert (np.abs(hl - w)[normal] <= 2.0 ** -22 * np.abs(w)[normal]).all()


def test_pack_weight_bank_layout():
    """A bank packed filter by filter (rows (k-1)*128 of the hi half and of the lo half at row K*128), as
    ops.conv1d_banks does: each filter's rows hold its k taps, the rest of the row stays zero."""
    K, Cin, cout = 3, 40, 128
    Cp = cpad(Cin)
    Ws = [_special_weights((k, Cin, cout), _seed("bank", k)) for k in range(1, K + 1)]
    for x3 in (False, True):
        dst = torch.zeros(((2 if x3 else 1) * K * cout, K * Cp), device="cuda")
        for k, w in enumerate(Ws, start=1):
            _pack(torch.from_numpy(w.copy()).cuda(), k, Cin, cout, dst, (k - 1) * cout, K * cout, x3)
        torch.cuda.synchronize()
        got = dst.cpu().numpy().view(np.uint32)
        for k, w in enumerate(Ws, start=1):
            hi_ref = _rna(w.view(np.uint32))
            lo_ref = _rna((w - hi_ref.view(np.float32)).view(np.uint32))
            for half, ref in ((0, hi_ref),) + (((1, lo_ref),) if x3 else ()):
                rows = got[half * K * cout + (k - 1) * cout:half * K * cout + k * cout]
                for j in range(k):
                    np.testing.assert_array_equal(rows[:, j * Cp:j * Cp + Cin], ref[j].T)
                    assert (rows[:, j * Cp + Cin:(j + 1) * Cp] == 0).all()
                assert (rows[:, k * Cp:] == 0).all(), f"filter {k} wrote past its {k} taps"


# ------------------------------------------------------------------------------------------------------------------
# rejected descriptors: the launch never happens, and the message names the field
# ------------------------------------------------------------------------------------------------------------------
def test_rejected_descriptors():
    B, T, Cin, N = 2, 16, 32, 128
    x = torch.zeros(B * T, Cin, device="cuda")
    W = torch.zeros(Cin, N, device="cuda")
    Wp = torch.zeros(2 * 256, Cin, device="cuda")                       # the fp32x3 hi | lo rows of the widest case
    big = torch.zeros(B * T * 2 * N + 64, device="cuda")               # large enough for any row stride tried below
    lib = L.lib()

    def base(impl):
        d = L.LinearDesc()
        d.X = x.data_ptr(); d.ldx = Cin; d.B = B; d.T = T; d.C = Cin; d.taps = 1; d.N = N
        d.W = W.data_ptr(); d.Wp = Wp.data_ptr(); d.ldwp = Cin
        d.Y = big.data_ptr(); d.ldy = N; d.keep_scale = 1.0; d.impl = impl
        return d

    def rejected(d, msg):
        rc = lib.taco_linear_fwd(C.byref(d), L.current_stream())
        assert rc != 0 and msg in lib.taco_last_error().decode(), (rc, lib.taco_last_error())

    for impl in (L.IMPL_SIMT, L.IMPL_TC, L.IMPL_TC3):
        d = base(impl); d.ldy = N - 4
        rejected(d, "ldy")
        d = base(impl); d.residual = big.data_ptr(); d.ldr = N - 4
        rejected(d, "ldr")
        d = base(impl); d.N = 256; d.epilogue = L.EPI_HIGHWAY; d.hx = big.data_ptr(); d.ldhx = 124; d.ldy = 128
        rejected(d, "ldhx")
        d = base(impl); d.N = 256; d.epilogue = L.EPI_HIGHWAY; d.hx = big.data_ptr(); d.ldhx = 128; d.ldy = 124
        rejected(d, "ldy")
    d = base(L.IMPL_SIMT); d.pool = 1
    rejected(d, "max-pool")
    torch.cuda.synchronize()
    assert torch.count_nonzero(big) == 0
