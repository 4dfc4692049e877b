"""The signal-path kernels over their envelope, against float64: the FFT pair (taco_rfft2048 / taco_irfft2048), the
Griffin-Lim kernels (gl_init, gl_ola, gl_frame, gl_phase, padded and packed) of csrc/audio.cu and the feature kernels
(feature_frames, feature_spec) of csrc/features.cu.  Written once, run on the H100 by tests/test_gpu_z_stft_envelope.py
and under the host emulation (tests/cuda_emu) by tests/test_stft_envelope_host.py.

Every check takes an `Env`: a kernel namespace `K` (tacotron_b200.kernels, over the device library or the emulated
one), the device and the stream.  Every reference is float64, computed from the kernel's own float32 operands -- in a chain, the
output of the previous kernel -- so every bar is local.  Outputs are prefilled with a sentinel bit pattern (NaN-like,
never produced by arithmetic) and sit inside PAD elements of it that must survive; operands sit inside NaN bands.

Bars, u = 2^-24 (unit roundoff), eps = 2^-23, N = 2048, SAFETY = 2 on every local bar:
* window: hann_at(j) = 0.5 - 0.5 cospif(2i/W) in float32 has an ABSOLUTE error dw: the quotient 2i/W rounded (at most
  2u, times |d cos(pi x)/dx| <= pi), cospif's (<= 2 ulp of a value <= 1, so 2u), halved, and the subtraction's
  rounding (u): dw <= (pi + 1 + 1) u; DW = 6u.  Relative to w it is large at the window's first samples (w = 7e-6 at
  i = 1 of 1200), which matters wherever a sample is covered only by window tails (hop > win/2).
* FFT forward: six levels (the post-pass, five radix-4 stages), each rounding one twiddle product and two complex
  additions, about 2u of its operand's norm.  The levels' errors are independent, so they add in quadrature:
  ||dX|| ~ sqrt(6) 2u ||X||, ||X|| = sqrt(N/2) ||x||, which is 1.7 eps sqrt(N) ||x||; C_FWD = 2, per row in norm and per
  element (no element's error exceeds the norm).  The worst-case bound (the errors aligned, about 45) would not notice
  a twiddle table one ulp off; this one does: with every cosine of the table one ulp high, the tones' worst error
  under the emulation grows from 0.49 to 1.45 eps sqrt(N) ||x||, and the Nyquist sine (a row of rounding-level
  values) crosses the bar.
* FFT inverse: the same model carried to x = IFFT / N (||dx|| ~ C_FWD eps ||X_full|| / sqrt(N)), times a peak factor of
  about 4 for the largest of 2048 elements and 2 for the pre-pass's extra twiddle product: C_INV = 16 on
  eps ||X_full||_2 / N per element.
* gl_ola: y = sum w f / sum w^2 over k frames, fma chains:
      |dy| <= SAFETY ((k + 2) u (sum |w f| + |y| sum w^2) + sum dw (|f| + 2 |y| w)) / sum w^2,  exactly 0 where no frame
  has a non-zero weight.
* gl_frame / feature_frames: |d| <= SAFETY (u |w| + DW) |y[q]|  (one product rounding, the window's error).
* gl_init: mag within SAFETY (u |v'| + 2 ulp) relative of exp(v') (v' = v scale + shift exactly; fmaf rounds it once,
  expf is within 2 ulp); |full - mag e^{2 pi i u}| <= SAFETY 4u mag from the kernel's own mag.
* gl_phase: |full - m z/|z|| <= SAFETY m (8u + 3 * 2^-149 / |z|): hypotf within 3 ulp (an absolute 3 * 2^-149 when
  |z| is subnormal), the quotient and the product rounded once each; z = +-0 gives exactly (m, +0).
* feature_spec: stft = log(|X| + 1e-8f) within SAFETY ((4u |X| + u (|X| + 1e-8)) / (|X| + 1e-8) + 2u |stft|);
  mel the same with |X| -> |M| and gamma_K sqrt(2) sum_k |basis_k| |X_k| added to the numerator (K the filter's bins,
  plus five butterfly levels).  float16 outputs must be a float16 neighbour of a value inside the float32 bar.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass

import numpy as np
import torch

N = 2048
NB = 1025
U = 2.0 ** -24
EPS = 2.0 ** -23
SAFETY = 2.0
DW = 6 * U
C_FWD = 2.0
C_INV = 16.0
PAD = 4096
SENT = 0x7FA5A5A5
NAN, INF = float("nan"), float("inf")
EPS_LOG = float(np.float32(1e-8))
SUBMIN = 2.0 ** -149


@dataclass
class Env:
    K: object                   # the kernels, with tacotron_b200.kernels' signatures
    lib: object                 # the C ABI under them (taco_rfft2048 / taco_irfft2048 with explicit row counts)
    device: str
    stream: object = None

    def sync(self):
        if self.device != "cpu":
            torch.cuda.synchronize()


def gen(seed):
    return torch.Generator().manual_seed(seed)


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


# ------------------------------------------------------------------------------------------------------------------
# guarded buffers
# ------------------------------------------------------------------------------------------------------------------
class Out:
    """an output of `shape` (float32, float16 or complex64) inside PAD words of the sentinel pattern, prefilled with it
    too, so an element never written fails every value check"""

    def __init__(self, shape, device, dtype=torch.float32):
        self.words = math.prod(shape) * (2 if dtype == torch.complex64 else 1)
        wdt = torch.int16 if dtype == torch.float16 else torch.int32
        self.buf = torch.full((self.words + 2 * PAD,), SENT if wdt == torch.int32 else 0x7DA5, dtype=wdt, device=device)
        self.sent = SENT if wdt == torch.int32 else 0x7DA5
        inner = self.buf[PAD:PAD + self.words]
        if dtype == torch.complex64:
            self.t = inner.view(torch.float32).view(torch.complex64).view(shape)
        else:
            self.t = inner.view(dtype).view(shape)

    def bands_intact(self):
        return bool((self.buf[:PAD] == self.sent).all()) and bool((self.buf[PAD + self.words:] == self.sent).all())

    def untouched(self):
        return bool((self.buf == self.sent).all())

    def written(self):
        return not bool((self.buf[PAD:PAD + self.words] == self.sent).any())


def operand(t, device):
    """a copy of t inside NaN guard bands"""
    if t is None:
        return None
    if t.dtype == torch.complex64:
        buf = torch.full((2 * t.numel() + 2 * PAD,), NAN, device=device)
        v = buf[PAD:PAD + 2 * t.numel()].view(torch.complex64).view(t.shape)
    else:
        buf = torch.full((t.numel() + 2 * PAD,), NAN if t.is_floating_point() else -(2 ** 30), dtype=t.dtype,
                         device=device)
        v = buf[PAD:PAD + t.numel()].view(t.shape)
    v.copy_(t)
    return v


def same_bits(a, b):
    if a.dtype == torch.complex64:
        a, b = torch.view_as_real(a), torch.view_as_real(b)
    w = torch.int16 if a.dtype == torch.float16 else torch.int32
    return a.shape == b.shape and torch.equal(a.contiguous().view(w), b.contiguous().view(w))


def _frac(err, bar, what):
    """worst err / bar; fails on any element above its bar (NaN included)"""
    if err.numel() == 0:
        return 0.0
    bar = torch.as_tensor(bar, dtype=err.dtype, device=err.device).expand_as(err)
    q = err / bar
    bad = ~(q <= 1.0)
    if bool(bad.any()):
        i = int(torch.nonzero(bad.flatten())[0])
        raise AssertionError(f"{what}: {int(bad.sum())} elements over the bar; first at flat index {i}: error "
                             f"{err.flatten()[i].item():.4g}, bar {bar.flatten()[i].item():.4g}")
    return float(q.max())


# ------------------------------------------------------------------------------------------------------------------
# 1. the FFT pair
# ------------------------------------------------------------------------------------------------------------------
def run_rfft(env, x):
    rows = x.numel() // N
    o = Out((rows, NB), env.device, torch.complex64)
    env.K.rfft2048(o.t, operand(x.reshape(rows, N), env.device))
    env.sync()
    assert o.bands_intact(), "rfft2048 wrote outside X"
    assert rows == 0 or o.written(), "rfft2048 left an element of X unwritten"
    return o.t


def run_irfft(env, X):
    rows = X.numel() // NB
    o = Out((rows, N), env.device)
    env.K.irfft2048(o.t, operand(X.reshape(rows, NB), env.device))
    env.sync()
    assert o.bands_intact(), "irfft2048 wrote outside x"
    assert rows == 0 or o.written(), "irfft2048 left an element of x unwritten"
    return o.t


def rfft_err(x, X):
    """(worst per-element fraction, worst normwise fraction) of rfft2048's X against float64 from x"""
    if x.numel() == 0:
        return 0.0, 0.0
    x64 = x.double().to(X.device)
    ref = torch.fft.rfft(x64, dim=-1)
    d = (X.to(torch.complex128) - ref).abs()
    nx = x64.norm(dim=-1, keepdim=True)
    scale = EPS * math.sqrt(N) * nx
    return (_frac(d, C_FWD * scale + 1e-300, "rfft2048 per element"),
            _frac(d.norm(dim=-1, keepdim=True), C_FWD * scale + 1e-300, "rfft2048 normwise"))


def irfft_ref(X):
    X64 = X.to(torch.complex128)
    im = X64.imag.clone()
    im[..., [0, NB - 1]] = 0
    X64 = torch.complex(X64.real.contiguous(), im)
    full = (X64[..., 0].abs() ** 2 + X64[..., NB - 1].abs() ** 2 + 2 * (X64[..., 1:NB - 1].abs() ** 2).sum(-1)).sqrt()
    return torch.fft.irfft(X64, n=N, dim=-1), full


def irfft_err(X, x):
    if X.numel() == 0:
        return 0.0
    ref, full = irfft_ref(X.to(x.device))
    return _frac((x.double() - ref).abs(), C_INV * EPS * full[..., None] / N + 1e-300, "irfft2048 per element")


def fft_rows(kind, rows, seed, sel=None):
    """float32 [rows, 2048] of one input class; impulses at positions sel (default 0, 1, ...), tones at bins sel"""
    g = gen(seed)
    sel = torch.arange(rows) if sel is None else torch.as_tensor(sel)
    if kind == "gauss":
        return torch.randn(rows, N, generator=g)
    if kind == "range":                         # e^+-20 inside each row
        return torch.randn(rows, N, generator=g) * torch.exp((torch.rand(rows, N, generator=g) * 2 - 1) * 20)
    if kind == "impulse":                       # a unit impulse at position i % 2048
        x = torch.zeros(len(sel), N)
        x[torch.arange(len(sel)), sel % N] = 1.0
        return x
    if kind == "tone":                          # row 2i: cos at bin sel[i], row 2i+1: sin at it
        i = torch.arange(2 * len(sel))
        k = (sel[i // 2] % NB).double()[:, None]
        ph = 2 * math.pi * k * torch.arange(N, dtype=torch.float64)[None] / N
        return torch.where((i % 2 == 0)[:, None], ph.cos(), ph.sin()).float()
    raise ValueError(kind)


def spectra(rows, seed, kind="random"):
    """complex64 [rows, 1025]: independent Gaussian bins, or Hermitian spectra (rfft of real rows, float64 rounded)"""
    g = gen(seed)
    if kind == "random":
        return torch.complex(torch.randn(rows, NB, generator=g), torch.randn(rows, NB, generator=g))
    return torch.fft.rfft(torch.randn(rows, N, generator=g).double(), dim=-1).to(torch.complex64)


def fft_forward(env, kind, rows, seed, sel=None):
    """(per-element, normwise) fractions; with more than 528 rows (the grid), rows 0, 527, 528 and the last also give
    the same bits alone"""
    x = fft_rows(kind, rows, seed, sel)
    X = run_rfft(env, x)
    e, en = rfft_err(x, X)
    fin = X[:, [0, NB - 1]].imag
    assert bool((fin == 0).all()), "rfft2048: DC / Nyquist imaginary parts not exactly 0"
    if x.shape[0] > 528:
        for i in (0, 527, 528, x.shape[0] - 1):
            assert same_bits(run_rfft(env, x[i:i + 1]), X[i:i + 1]), f"rfft2048 row {i} differs in a batch of one"
    return e, en


def fft_inverse(env, kind, rows, seed):
    X = spectra(rows, seed, kind)
    x = run_irfft(env, X)
    if rows > 528:
        for i in (0, 527, 528, rows - 1):
            assert same_bits(run_irfft(env, X[i:i + 1]), x[i:i + 1]), f"irfft2048 row {i} differs in a batch of one"
    return irfft_err(X, x)


def fft_roundtrip(env, rows, seed):
    """irfft(rfft(x)) against x: the forward's normwise error carried through the inverse (at most
    ||dX_full||_2 / sqrt(N) per sample, ||dX_full|| <= sqrt(2) ||dX||) plus the inverse's own bar"""
    x = fft_rows("gauss", rows, seed)
    X = run_rfft(env, x)
    y = run_irfft(env, X)
    nx = x.double().norm(dim=-1, keepdim=True).to(y.device)
    bar = EPS * nx * (math.sqrt(2) * C_FWD + C_INV / math.sqrt(N))
    return _frac((y.double() - x.double().to(y.device)).abs(), bar, "irfft2048(rfft2048(x))")


def fft_laws(env, rows, seed):
    """bit for bit: 2^k scaling both ways, row position independence (batch of one, reversed batch), NaN / Inf row
    isolation, the inverse ignoring DC / Nyquist imaginary parts, determinism"""
    x = fft_rows("gauss", rows, seed)
    X = run_rfft(env, x)
    assert same_bits(run_rfft(env, x), X), "rfft2048 not deterministic"
    for k in (-9, 7):
        assert same_bits(run_rfft(env, x * 2.0 ** k), (X * 2.0 ** k)), f"rfft2048 not exact under 2^{k} scaling"
    picks = sorted({0, rows - 1, rows // 2, min(rows - 1, 528), min(rows - 1, 527)})
    for i in picks:
        assert same_bits(run_rfft(env, x[i:i + 1]), X[i:i + 1]), f"rfft2048 row {i} differs in a batch of one"
    assert same_bits(run_rfft(env, x.flip(0)), X.flip(0)), "rfft2048 rows differ in reversed order"
    Xs = spectra(rows, seed + 1)
    xs = run_irfft(env, Xs)
    assert same_bits(run_irfft(env, Xs), xs), "irfft2048 not deterministic"
    for k in (-9, 7):
        assert same_bits(run_irfft(env, Xs * 2.0 ** k), xs * 2.0 ** k), f"irfft2048 not exact under 2^{k} scaling"
    for i in picks:
        assert same_bits(run_irfft(env, Xs[i:i + 1]), xs[i:i + 1]), f"irfft2048 row {i} differs in a batch of one"
    g = gen(seed + 2)
    for junk in (NAN, INF, 1e30):
        Xj = Xs.clone()
        Xj[:, 0] = torch.complex(Xj[:, 0].real, torch.full((rows,), junk))
        Xj[:, NB - 1] = torch.complex(Xj[:, NB - 1].real, torch.randn(rows, generator=g) * 1e3)
        Xz = Xs.clone()
        Xz[:, 0] = torch.complex(Xz[:, 0].real, torch.zeros(rows))
        Xz[:, NB - 1] = torch.complex(Xz[:, NB - 1].real, torch.zeros(rows))
        assert same_bits(run_irfft(env, Xj), run_irfft(env, Xz)), "irfft2048 reads the DC / Nyquist imaginary parts"
    if rows >= 3:
        i = rows // 2
        for v in (NAN, INF):
            xb = x.clone()
            xb[i, 17] = v
            Xb = run_rfft(env, xb)
            keep = torch.ones(rows, dtype=torch.bool)
            keep[i] = False
            assert same_bits(Xb[keep.to(Xb.device)], X[keep.to(X.device)]), f"rfft2048: a {v} row changed another row"
            Xsb = Xs.clone()
            Xsb[i, 33] = complex(v, 0)
            xsb = run_irfft(env, Xsb)
            assert same_bits(xsb[keep.to(xsb.device)], xs[keep.to(xs.device)]), f"irfft2048: a {v} row changed another"


def fft_empty(env):
    """rows = 0 is accepted and writes nothing (through the C ABI: an empty torch tensor has no data pointer, which the
    ABI refuses before it looks at the row count)"""
    for fwd in (True, False):
        o = Out((4, NB) if fwd else (4, N), env.device, torch.complex64 if fwd else torch.float32)
        src = operand(torch.zeros(4, N) if fwd else torch.zeros(4, NB, dtype=torch.complex64), env.device)
        fn = env.lib.taco_rfft2048 if fwd else env.lib.taco_irfft2048
        assert fn(_p(o.t), _p(src), 0, env.stream) == 0, env.lib.taco_last_error().decode()
        env.sync()
        assert o.untouched(), "rows = 0 wrote"


# ------------------------------------------------------------------------------------------------------------------
# 2. Griffin-Lim kernels
# ------------------------------------------------------------------------------------------------------------------
def hann64(n_fft, win_length, device="cpu"):
    lpad = (n_fft - win_length) // 2
    w = torch.zeros(n_fft, dtype=torch.float64, device=device)
    i = torch.arange(win_length, dtype=torch.float64, device=device)
    w[lpad:lpad + win_length] = 0.5 - 0.5 * torch.cos(2 * math.pi * i / win_length)
    return w


def frame_map(n, r):
    """(t(f), c(f)) of every frame f of gl_init's layout"""
    f = torch.arange(n)
    rem = f % (4 * r)
    return 4 * (f // (4 * r)) + (rem & 3), rem >> 2


def gl_init_ref(spec, r, n, scale=None, shift=None):
    """(v', m64): v' = v * scale + shift exactly in float64 and m64 = exp(v') of every [b, f, k]"""
    B, T, W = spec.shape
    F = W // r
    t, c = frame_map(n, r)
    t, c = t.to(spec.device), c.to(spec.device)
    v = spec.double().view(B, T, r, F)[:, t, c]
    if scale is not None:
        v = v * scale.double().view(r, F)[c] + shift.double().view(r, F)[c]
    return v, v.exp()


def gl_init_err(spec, phase_u, r, mag, full, scale=None, shift=None):
    """(mag fraction, full fraction) of one padded or single-utterance gl_init output [B, n, F]"""
    B, n, F = mag.shape
    if mag.numel() == 0:
        return 0.0, 0.0
    v, m64 = gl_init_ref(spec.to(mag.device), r, n, scale if scale is None else scale.to(mag.device),
                         shift if shift is None else shift.to(mag.device))
    em = _frac((mag.double() - m64).abs(), SAFETY * (U * v.abs() + 2 * EPS) * m64, "gl_init mag")
    m = mag.double()
    ph = 2 * math.pi * phase_u.double().to(mag.device)
    ref = torch.complex(m * ph.cos(), m * ph.sin())
    ef = _frac((full.to(torch.complex128) - ref).abs(), SAFETY * 4 * U * m + 1e-300, "gl_init full")
    return em, ef


def gl_init_inputs(B, T, r, F, seed):
    """log-magnitudes over [-18.4, 20] (and rows past 4*(T/4) NaN: never read), phases with the edge values"""
    g = gen(seed)
    spec = torch.rand(B, T, F * r, generator=g) * (20 + 18.4) - 18.4
    spec[:, 4 * (T // 4):] = NAN
    n = 4 * r * (T // 4)
    pu = torch.rand(B, n, F, generator=g)
    edge = torch.tensor([0.0, 0.25, 0.5, 0.75, 1 - 2.0 ** -24])
    sel = torch.rand(B, n, F, generator=g) < 0.05
    pu[sel] = edge[torch.randint(0, 5, (int(sel.sum()),), generator=g)]
    scale = torch.rand(F * r, generator=g) * 1.5 + 0.25
    shift = torch.randn(F * r, generator=g)
    return spec, pu, scale, shift


def run_gl_init(env, spec, pu, r, scale=None, shift=None):
    B, T, W = spec.shape
    F = W // r
    n = 4 * r * (T // 4)
    dev = env.device
    om, of = Out((B, n, F), dev), Out((B, n, F), dev, torch.complex64)
    env.K.gl_init(of.t, om.t, operand(spec, dev), operand(pu, dev), r, operand(scale, dev), operand(shift, dev))
    env.sync()
    assert om.bands_intact() and of.bands_intact(), "gl_init wrote outside its outputs"
    assert B * n * F == 0 or (om.written() and of.written()), "gl_init left outputs unwritten"
    return om.t, of.t


def gl_init_check(env, B, T, r, F, seed):
    spec, pu, scale, shift = gl_init_inputs(B, T, r, F, seed)
    worst = [0.0, 0.0]
    for sc, sh in ((None, None), (scale, shift)):
        mag, full = run_gl_init(env, spec, pu, r, sc, sh)
        em, ef = gl_init_err(spec, pu, r, mag, full, sc, sh)
        worst = [max(worst[0], em), max(worst[1], ef)]
    return worst


def gl_init_mapping(env, B, T, r, F):
    """index-coded spec: v = code * 2^-18, so round(log(mag) * 2^18) names the spec element each output read"""
    n = 4 * r * (T // 4)
    code = torch.arange(B * T * F * r, dtype=torch.float64).view(B, T, F * r)
    assert code.numel() < 2 ** 18
    spec = (code * 2.0 ** -18).float()
    spec[:, 4 * (T // 4):] = NAN
    mag, _ = run_gl_init(env, spec, torch.zeros(B, n, F), r)
    got = torch.round(mag.double().log().cpu() * 2 ** 18).long()
    t, c = frame_map(n, r)
    want = code.view(B, T, r, F)[:, t, c].long()
    assert torch.equal(got, want), "gl_init reads the wrong spec element"


def ola_terms(fr, hop, n_fft, win_length, L):
    """float64 per-sample sums over the frames covering it: (y, sum w^2, sum |w f|, sum dw |f|, sum dw w, k)"""
    B, n, _ = fr.shape
    dev = fr.device
    w = hann64(n_fft, win_length, dev)
    nz = w != 0
    f = torch.where(nz, fr.double(), torch.zeros((), dtype=torch.float64, device=dev))
    idx = (torch.arange(n, device=dev)[:, None] * hop + torch.arange(n_fft, device=dev)[None]).flatten()
    width = hop * (n - 1) + n_fft
    lo = n_fft // 2

    def acc(vals):
        out = torch.zeros(B, width, dtype=torch.float64, device=dev)
        out.index_add_(1, idx, vals.reshape(B, -1))
        return out[:, lo:lo + L]
    ww = acc((w * w).expand(B, n, n_fft))
    num = acc(w * f)
    aw = acc((w * f).abs())
    df = acc(DW * f.abs() * nz)
    dw = acc((DW * w * nz).expand(B, n, n_fft))
    k = acc(nz.double().expand(B, n, n_fft))
    y = torch.where(ww > 0, num / torch.where(ww > 0, ww, torch.ones_like(ww)), torch.zeros_like(ww))
    return y, ww, aw, df, dw, k


def gl_ola_err(fr, y, hop, win_length):
    B, n, n_fft = fr.shape
    L = hop * (n - 1)
    ref, ww, aw, df, dw, k = ola_terms(fr.to(y.device), hop, n_fft, win_length, L)
    y64 = y.double().view(B, L)
    none = ww == 0
    assert bool((y64[none] == 0).all()), "gl_ola: a sample no frame covers is not exactly 0"
    bar = SAFETY * ((k + 2) * U * (aw + ref.abs() * ww) + df + 2 * ref.abs() * dw) / torch.where(none, torch.ones_like(ww), ww)
    return _frac((y64 - ref).abs()[~none], bar[~none], "gl_ola")


def reflect_index(n, hop, n_fft, L, device="cpu"):
    q = torch.arange(n, device=device)[:, None] * hop + torch.arange(n_fft, device=device)[None] - n_fft // 2
    q = torch.where(q < 0, -q, q)
    return torch.where(q >= L, 2 * (L - 1) - q, q)


def gl_frame_err(y, frw, hop, win_length):
    B, n, n_fft = frw.shape
    L = hop * (n - 1)
    dev = frw.device
    w = hann64(n_fft, win_length, dev)
    q = reflect_index(n, hop, n_fft, L, dev)
    yq = y.double().to(dev).view(B, L)[:, q]
    ref = torch.where(w != 0, w * yq, torch.zeros((), dtype=torch.float64, device=dev))
    assert bool((frw[:, :, w == 0] == 0).all()), "gl_frame: outside the window not exactly 0"
    bar = SAFETY * (U * w + DW) * yq.abs()
    return _frac((frw.double() - ref).abs()[:, :, w != 0], bar[:, :, w != 0] + 1e-300, "gl_frame")


def run_gl_ola(env, fr, hop, win_length):
    B, n, n_fft = fr.shape
    o = Out((B, hop * (n - 1)), env.device)
    env.K.gl_ola(o.t, operand(fr, env.device), hop, win_length)
    env.sync()
    assert o.bands_intact(), "gl_ola wrote outside y"
    assert o.t.numel() == 0 or o.written(), "gl_ola left samples unwritten"
    return o.t


def run_gl_frame(env, y, n, n_fft, hop, win_length):
    B = y.shape[0]
    o = Out((B, n, n_fft), env.device)
    env.K.gl_frame(o.t, operand(y, env.device), hop, win_length)
    env.sync()
    assert o.bands_intact(), "gl_frame wrote outside frw"
    assert o.t.numel() == 0 or o.written(), "gl_frame left elements unwritten"
    return o.t


def window_of(env, n_fft, win_length):
    """the kernel's own window: gl_frame of y = 1 is w exactly; checked against float64 within DW"""
    hop = n_fft
    y = torch.ones(1, hop * 2)
    w = run_gl_frame(env, y, 3, n_fft, hop, win_length)[0, 1].double()
    e = _frac((w - hann64(n_fft, win_length, w.device)).abs(), torch.full_like(w, DW), "hann_at")
    return w, e


def gl_ola_frame_check(env, B, n, hop, n_fft, win_length, seed):
    """gl_ola on random frames (rows of very different scales), gl_frame on its output, and gl_frame's reflect index
    exactly with y[b, q] = b * L + q + 1 (decoded against the kernel's own window)"""
    g = gen(seed)
    fr = torch.randn(B, n, n_fft, generator=g) * torch.exp(torch.randn(B, n, 1, generator=g) * 3)
    y = run_gl_ola(env, fr, hop, win_length)
    eo = gl_ola_err(fr, y, hop, win_length)
    ef = 0.0
    L = hop * (n - 1)
    if L > n_fft // 2:
        frw = run_gl_frame(env, y, n, n_fft, hop, win_length)
        ef = gl_frame_err(y, frw, hop, win_length)
        if B * L < 2 ** 22:
            wk, _ = window_of(env, n_fft, win_length)
            code = torch.arange(1, B * L + 1, dtype=torch.float32).view(B, L)
            got = run_gl_frame(env, code, n, n_fft, hop, win_length).double()
            nz = wk != 0
            dec = torch.round(got[:, :, nz] / wk[nz])
            q = reflect_index(n, hop, n_fft, L, got.device)[:, nz]
            want = (torch.arange(B, device=got.device)[:, None, None] * L + q[None] + 1).double()
            assert torch.equal(dec, want), "gl_frame reads the wrong sample"
    return eo, ef


def gl_phase_inputs(count, seed):
    """|z| log-uniform over [1e-44, 3e38] at random angles, exact zeros of every sign, magnitudes over e^[-18.4, 20]"""
    g = gen(seed)
    lz = torch.rand(count, generator=g, dtype=torch.float64) * (math.log(3e38) - math.log(1e-44)) + math.log(1e-44)
    th = torch.rand(count, generator=g, dtype=torch.float64) * 2 * math.pi
    z = torch.complex((lz.exp() * th.cos()).float(), (lz.exp() * th.sin()).float())
    zs = [complex(0.0, 0.0), complex(-0.0, 0.0), complex(0.0, -0.0), complex(-0.0, -0.0)]
    for i, v in enumerate(zs):
        z[i::97] = torch.complex(torch.tensor(v.real), torch.tensor(v.imag))
    neg = torch.tensor(-0.0)
    zr = torch.view_as_real(z)
    zr[1::97, 0] = neg
    zr[3::97, 0] = neg
    zr[2::97, 1] = neg
    zr[3::97, 1] = neg
    m = torch.exp(torch.rand(count, generator=g) * 38.4 - 18.4)
    return z, m


def gl_phase_err(mag, rebuilt, full):
    z = rebuilt.to(torch.complex128).to(full.device)
    m = mag.double().to(full.device)
    a = z.abs()
    zero = a == 0
    fr = torch.view_as_real(full)
    assert bool((fr[..., 0][zero] == mag.to(full.device)[zero]).all()), "gl_phase: z = 0 does not give m"
    im = fr[..., 1][zero].contiguous().view(torch.int32)
    assert bool((im == 0).all()), "gl_phase: z = 0 does not give an imaginary part of +0"
    ref = m * z / torch.where(zero, torch.ones_like(a), a)
    bar = SAFETY * m * (8 * U + 3 * SUBMIN / torch.where(zero, torch.ones_like(a), a))
    return _frac((full.to(torch.complex128) - ref).abs()[~zero], bar[~zero], "gl_phase")


def run_gl_phase(env, mag, rebuilt):
    o = Out(tuple(mag.shape), env.device, torch.complex64)
    env.K.gl_phase(o.t, operand(mag, env.device), operand(rebuilt, env.device))
    env.sync()
    assert o.bands_intact() and (mag.numel() == 0 or o.written()), "gl_phase: guards"
    return o.t


def gl_phase_check(env, count, seed):
    z, m = gl_phase_inputs(count, seed)
    full = run_gl_phase(env, m, z)
    return gl_phase_err(m, z, full)


# ---- packed ----
def packed_off(lengths):
    off = np.zeros(len(lengths) + 1, dtype=np.int64)
    np.cumsum(lengths, out=off[1:])
    return torch.from_numpy(off)


def packed_check(env, lengths, T, r, hop, n_fft, win_length, seed, nan_utt=None, sample=None):
    """gl_init / gl_ola / gl_frame packed: every utterance (or those in `sample`) within the padded bars and
    bit-identical to the padded path on it alone; with nan_utt, a NaN in that utterance's input stays in it.  Returns
    the worst fractions."""
    B, F = len(lengths), NB
    nfull = 4 * r * (T // 4)
    off = packed_off(lengths)
    Nr = int(off[-1])
    nmax = max(lengths)
    dev = env.device
    spec, _, scale, shift = gl_init_inputs(B, T, r, F, seed)
    g = gen(seed + 1)
    pu = torch.rand(Nr, F, generator=g)
    offd = operand(off, dev)
    om, of = Out((Nr, F), dev), Out((Nr, F), dev, torch.complex64)
    env.K.gl_init_packed(of.t, om.t, operand(spec, dev), operand(pu, dev), offd, r, nmax, operand(scale, dev),
                         operand(shift, dev))
    fr = torch.randn(Nr, n_fft, generator=g) * torch.exp(torch.randn(Nr, 1, generator=g) * 3)
    if nan_utt is not None:
        fr[int(off[nan_utt]):int(off[nan_utt + 1])] = NAN
    oy = Out((hop * (Nr - B),), dev)
    env.K.gl_ola_packed(oy.t, operand(fr, dev), offd, nmax, hop, win_length)
    yin = torch.randn(hop * (Nr - B), generator=g)
    if nan_utt is not None:
        s0 = hop * (int(off[nan_utt]) - nan_utt)
        yin[s0:s0 + hop * (lengths[nan_utt] - 1)] = NAN
    ofr = Out((Nr, n_fft), dev)
    env.K.gl_frame_packed(ofr.t, operand(yin, dev), offd, nmax, hop, win_length)
    env.sync()
    for o in (om, of, oy, ofr):
        assert o.bands_intact(), "packed kernels: wrote outside their outputs"
    for o in (om, of, oy):
        assert o.written(), "packed kernels: left outputs unwritten"
    worst = {"init mag": 0.0, "init full": 0.0, "ola": 0.0, "frame": 0.0}
    for b, nb in enumerate(lengths):
        if sample is not None and b not in sample and b != nan_utt:
            continue
        r0, r1 = int(off[b]), int(off[b + 1])
        s0 = hop * (r0 - b)
        Lb = hop * (nb - 1)
        if nan_utt is not None:
            bad = b == nan_utt
            for t in (oy.t[s0:s0 + Lb], ofr.t[r0:r1]):
                assert bool(torch.isnan(t).any()) == bad or (not bad and not bool(torch.isnan(t).any())), \
                    "packed: a NaN crossed into another utterance"
            if bad:
                continue
        # alone, on the padded path: the padded gl_init takes all 4r*(T/4) frames, so the packed rows are its first nb
        magp, fullp = run_gl_init(env, spec[b:b + 1], torch.cat([pu[r0:r1], torch.zeros(nfull - nb, F)])[None], r,
                                  scale, shift)
        assert same_bits(om.t[r0:r1], magp[0, :nb]) and same_bits(of.t[r0:r1], fullp[0, :nb]), \
            f"gl_init_packed utterance {b} differs from the padded path"
        em, ef = _init_err_prefix(spec[b:b + 1], pu[r0:r1], r, nfull, om.t[r0:r1], of.t[r0:r1], scale, shift)
        worst["init mag"] = max(worst["init mag"], em)
        worst["init full"] = max(worst["init full"], ef)
        if nb >= 2:
            yp = run_gl_ola(env, fr[r0:r1][None], hop, win_length)
            assert same_bits(oy.t[s0:s0 + Lb], yp[0]), f"gl_ola_packed utterance {b} differs from the padded path"
            worst["ola"] = max(worst["ola"], gl_ola_err(fr[r0:r1][None], oy.t[s0:s0 + Lb][None], hop, win_length))
        if Lb <= n_fft // 2:                           # too short to reflect-pad: gl_frame_packed leaves its rows alone
            assert bool((ofr.t[r0:r1].contiguous().view(torch.int32) == SENT).all()), "gl_frame_packed wrote a short one"
        else:
            assert bool((ofr.t[r0:r1].contiguous().view(torch.int32) != SENT).all()), "gl_frame_packed left rows unwritten"
            fp = run_gl_frame(env, yin[s0:s0 + Lb][None], nb, n_fft, hop, win_length)
            assert same_bits(ofr.t[r0:r1], fp[0]), f"gl_frame_packed utterance {b} differs from the padded path"
            worst["frame"] = max(worst["frame"], gl_frame_err(yin[s0:s0 + Lb][None], ofr.t[r0:r1][None], hop,
                                                              win_length))
    return worst


def _init_err_prefix(spec, pu, r, nfull, mag, full, scale, shift):
    nb = mag.shape[0]
    v, m64 = gl_init_ref(spec.to(mag.device), r, nfull, None if scale is None else scale.to(mag.device),
                         None if shift is None else shift.to(mag.device))
    v, m64 = v[0, :nb], m64[0, :nb]
    em = _frac((mag.double() - m64).abs(), SAFETY * (U * v.abs() + 2 * EPS) * m64, "gl_init_packed mag")
    m = mag.double()
    ph = 2 * math.pi * pu.double().to(mag.device)
    ref = torch.complex(m * ph.cos(), m * ph.sin())
    ef = _frac((full.to(torch.complex128) - ref).abs(), SAFETY * 4 * U * m + 1e-300, "gl_init_packed full")
    return em, ef


# ------------------------------------------------------------------------------------------------------------------
# 3. every Griffin-Lim iteration from its own state
# ------------------------------------------------------------------------------------------------------------------
class CheckingK:
    """forwards every kernel call to `base` and, after each launch, checks its output against float64 from the operands
    it actually received; worst fractions per kernel in .worst, calls counted in .calls"""

    def __init__(self, env, base, hop=300, win_length=1200):
        self.env, self.base, self.hop, self.win = env, base, hop, win_length
        self.worst, self.calls = {}, {}

    def _note(self, k, w):
        self.worst[k] = max(self.worst.get(k, 0.0), w)
        self.calls[k] = self.calls.get(k, 0) + 1

    def gl_init(self, full, mag, spec, phase_u, r, scale=None, shift=None):
        self.base.gl_init(full, mag, spec, phase_u, r, scale, shift)
        self.env.sync()
        em, ef = gl_init_err(spec, phase_u, r, mag, full, scale, shift)
        self._note("gl_init mag", em)
        self._note("gl_init full", ef)

    def gl_init_packed(self, full, mag, spec, phase_u, off, r, max_frames, scale=None, shift=None):
        self.base.gl_init_packed(full, mag, spec, phase_u, off, r, max_frames, scale, shift)
        self.env.sync()
        o = off.cpu().tolist()
        nfull = 4 * r * (spec.shape[1] // 4)
        for b in range(len(o) - 1):
            em, ef = _init_err_prefix(spec[b:b + 1], phase_u[o[b]:o[b + 1]], r, nfull, mag[o[b]:o[b + 1]],
                                      full[o[b]:o[b + 1]], scale, shift)
            self._note("gl_init mag", em)
            self._note("gl_init full", ef)

    def irfft2048(self, x, X):
        self.base.irfft2048(x, X)
        self.env.sync()
        self._note("irfft2048", _chunked(lambda a, b: irfft_err(a, b), X.reshape(-1, NB), x.reshape(-1, N)))

    def rfft2048(self, X, x):
        self.base.rfft2048(X, x)
        self.env.sync()
        e = _chunked(lambda a, b: max(rfft_err(a, b)), x.reshape(-1, N), X.reshape(-1, NB))
        self._note("rfft2048", e)

    def gl_ola(self, y, fr, hop, win_length):
        self.base.gl_ola(y, fr, hop, win_length)
        self.env.sync()
        self._note("gl_ola", max(gl_ola_err(fr[b:b + 1], y[b:b + 1], hop, win_length) for b in range(fr.shape[0])))

    def gl_frame(self, frw, y, hop, win_length):
        self.base.gl_frame(frw, y, hop, win_length)
        self.env.sync()
        self._note("gl_frame", max(gl_frame_err(y[b:b + 1], frw[b:b + 1], hop, win_length) for b in range(y.shape[0])))

    def gl_ola_packed(self, y, fr, off, max_frames, hop, win_length):
        self.base.gl_ola_packed(y, fr, off, max_frames, hop, win_length)
        self.env.sync()
        o = off.cpu().tolist()
        for b in range(len(o) - 1):
            s0, Lb = hop * (o[b] - b), hop * (o[b + 1] - o[b] - 1)
            self._note("gl_ola", gl_ola_err(fr[o[b]:o[b + 1]][None], y[s0:s0 + Lb][None], hop, win_length))

    def gl_frame_packed(self, frw, y, off, max_frames, hop, win_length):
        self.base.gl_frame_packed(frw, y, off, max_frames, hop, win_length)
        self.env.sync()
        o = off.cpu().tolist()
        for b in range(len(o) - 1):
            s0, Lb = hop * (o[b] - b), hop * (o[b + 1] - o[b] - 1)
            self._note("gl_frame", gl_frame_err(y[s0:s0 + Lb][None], frw[o[b]:o[b + 1]][None], hop, win_length))

    def gl_phase(self, full, mag, rebuilt):
        self.base.gl_phase(full, mag, rebuilt)
        self.env.sync()
        self._note("gl_phase", _chunked(lambda a, b: gl_phase_err(a[0], a[1], b), (mag.reshape(-1), rebuilt.reshape(-1)),
                                        full.reshape(-1)))


def _chunked(fn, a, b, rows=4096):
    """fn over row chunks (bounds the float64 temporaries of a C2-sized launch)"""
    n = (a[0] if isinstance(a, tuple) else a).shape[0]
    step = rows if (a[0] if isinstance(a, tuple) else a).dim() > 1 else rows * NB
    w = 0.0
    for i in range(0, max(n, 1), step):
        ai = tuple(t[i:i + step] for t in a) if isinstance(a, tuple) else a[i:i + step]
        w = max(w, fn(ai, b[i:i + step]))
    return w


def gl_iterations(env, spec, r, n_iter, seed, frames=None, scale=None, shift=None):
    """Griffin-Lim (padded, or packed with `frames`) through CheckingK after checking that the proxy route gives the
    same bits as the plain one; returns the proxy's worst fractions"""
    from tacotron_b200 import audio
    g = gen(seed)
    B, T, _ = spec.shape
    n = 4 * r * (T // 4)
    dev = env.device
    spec = spec.to(dev)
    sc = None if scale is None else scale.to(dev)
    sh = None if shift is None else shift.to(dev)
    if frames is None:
        pu = torch.rand(B, n, NB, generator=g).to(dev)
        y0 = audio.griffinlim_batch(spec, r, n_iter, sc, sh, pu, K=env.K)
        ck = CheckingK(env, env.K)
        y1 = audio.griffinlim_batch(spec, r, n_iter, sc, sh, pu, K=ck)
    else:
        pu = torch.rand(int(sum(frames)), NB, generator=g).to(dev)
        y0, _ = audio.invert_speech_packed(spec, r, frames, n_iter, sh, sc, pu, K=env.K)
        ck = CheckingK(env, env.K)
        y1, _ = audio.invert_speech_packed(spec, r, frames, n_iter, sh, sc, pu, K=ck)
    env.sync()
    assert same_bits(y0, y1), "the checking proxy changed the result"
    assert ck.calls.get("gl_phase", 0) >= n_iter and ck.calls.get("irfft2048", 0) == n_iter + 1
    return ck.worst


def speech_like(B, T, r, seed):
    """log-magnitudes shaped like speech: a loud low band over quiet bins down to log(1e-8)"""
    g = gen(seed)
    k = torch.arange(NB, dtype=torch.float32)
    env_ = 2.0 - 18.0 * (k / NB) ** 0.5
    s = env_[None, None].repeat(B, T * r, 1) + torch.randn(B, T * r, NB, generator=g) * 1.5
    s = s.clamp(min=math.log(1e-8))
    return s.view(B, T, r * NB).contiguous()


# ------------------------------------------------------------------------------------------------------------------
# 4. feature kernels
# ------------------------------------------------------------------------------------------------------------------
def feature_frames_ref(y, start, length, n, max_len, hop, n_fft, win_length, preemph):
    """(frw64, |e|): pre-emphasis in numpy float32 (two roundings, as the kernel), reflect at max_len, the float64
    window"""
    B = len(start)
    w = hann64(n_fft, win_length)
    q = reflect_index(n, hop, n_fft, max_len)
    yn = y.numpy()
    out = torch.zeros(B, n, n_fft, dtype=torch.float64)
    ea = torch.zeros(B, n, n_fft, dtype=torch.float64)
    for b in range(B):
        x = np.zeros(max_len + 1, np.float32)
        L = int(length[b])
        x[:L] = yn[int(start[b]):int(start[b]) + L]
        e = np.empty(max_len, np.float32)
        e[0] = x[0]
        e[1:] = x[1:max_len] - np.float32(preemph) * x[:max_len - 1]
        et = torch.from_numpy(e.astype(np.float64))[q]
        out[b] = w * et
        ea[b] = et.abs()
    return out, ea


def feature_frames_check(env, y, start, length, max_len, hop=300, n_fft=2048, win_length=1200, preemph=0.97):
    B = len(start)
    n = 1 + max_len // hop
    dev = env.device
    o = Out((B, n, n_fft), dev)
    env.K.feature_frames(o.t, operand(y, dev), operand(start, dev), operand(length, dev), max_len, hop, win_length,
                         preemph)
    env.sync()
    assert o.bands_intact() and o.written(), "feature_frames: guards"
    ref, ea = feature_frames_ref(y, start, length, n, max_len, hop, n_fft, win_length, preemph)
    w = hann64(n_fft, win_length)
    got = o.t.double().cpu()
    assert bool((got[:, :, w == 0] == 0).all()), "feature_frames: outside the window not exactly 0"
    return _frac((got - ref).abs(), SAFETY * (U * w + DW) * ea + 1e-300, "feature_frames"), o.t


def feature_spec_ref_bars(X, basis, lo, hi):
    """float64 (stft, bar), (mel, bar) per frame [B, n, .] from the kernel's X"""
    Z = X.to(torch.complex128)
    a = Z.abs()
    st = (a + EPS_LOG).log()
    sbar = SAFETY * ((4 * U * a + U * (a + EPS_LOG)) / (a + EPS_LOG) + 2 * U * st.abs())
    bd = basis.double().to(X.device)
    M = torch.complex(Z.real @ bd.T, Z.imag @ bd.T)
    S = a @ bd.abs().T
    K = (hi - lo).double().to(X.device)
    gam = ((K / 32).ceil() + 6) * U
    am = M.abs()
    ml = (am + EPS_LOG).log()
    mbar = SAFETY * ((gam * math.sqrt(2) * S + 4 * U * am + U * (am + EPS_LOG)) / (am + EPS_LOG) + 2 * U * ml.abs())
    return st, sbar, ml, mbar


def _placed(v, r, nf_used):
    """[B, n, W] per frame -> [B, T, W r] in the reshape_frames layout (frames >= nf_used dropped)"""
    B, n, W = v.shape
    T = nf_used // r
    return v[:, :nf_used].reshape(B, nf_used // (4 * r), r, 4, W).permute(0, 1, 3, 2, 4).reshape(B, T, r * W)


def _f16_within(got, ref, bar):
    """every float16 `got` is a float16 neighbour of some value in [ref - bar, ref + bar]"""
    g = got.cpu().numpy().astype(np.float16)
    up = np.nextafter(g, np.float16(np.inf)).astype(np.float64)
    dn = np.nextafter(g, np.float16(-np.inf)).astype(np.float64)
    r_, b_ = ref.cpu().numpy(), bar.cpu().numpy()
    ok = (up > r_ - b_) & (dn < r_ + b_)
    assert ok.all(), f"feature_spec float16: {int((~ok).sum())} outputs are not a neighbour of the float32 bar"
    gv = g.astype(np.float64)
    return float(np.max(np.maximum(np.abs(gv - r_) - np.abs(up - gv), 0) / b_)) if g.size else 0.0


def run_feature_spec(env, X, basis, lo, hi, r, dtype):
    B, n, _ = X.shape
    nfu = 4 * r * (n // (4 * r))
    T = nfu // r
    n_mels = basis.shape[0]
    dev = env.device
    os_, om = Out((B, T, NB * r), dev, dtype), Out((B, T, n_mels * r), dev, dtype)
    env.K.feature_spec(os_.t, om.t, operand(X, dev), operand(basis, dev), operand(lo, dev), operand(hi, dev), r)
    env.sync()
    assert os_.bands_intact() and om.bands_intact() and os_.written() and om.written(), "feature_spec: guards"
    return os_.t, om.t


def feature_spec_check(env, X, basis, lo, hi, r, dtype):
    B, n, _ = X.shape
    nfu = 4 * r * (n // (4 * r))
    Xn = X.clone()
    Xn[:, nfu:] = complex(NAN, NAN)                     # frames at or past nf_used must not be read
    so, mo = run_feature_spec(env, Xn, basis, lo, hi, r, dtype)
    st, sbar, ml, mbar = feature_spec_ref_bars(X[:, :nfu].to(so.device), basis, lo, hi)
    st, sbar, ml, mbar = (_placed(t, r, nfu) for t in (st, sbar, ml, mbar))
    if dtype == torch.float16:
        return _f16_within(so, st, sbar), _f16_within(mo, ml, mbar)
    return (_frac((so.double() - st).abs(), sbar, "feature_spec stft"),
            _frac((mo.double() - ml).abs(), mbar, "feature_spec mel"))


def feature_spec_mapping(env, B, n, r, basis, lo, hi):
    """index-coded |X| = code: exp(stft) - 1e-8 rounds back to the code of the frame and bin each output read"""
    code = torch.arange(1, B * n * NB + 1, dtype=torch.float64).view(B, n, NB)
    assert code.numel() < 2 ** 17
    X = torch.complex(code.float(), torch.zeros(B, n, NB))
    so, _ = run_feature_spec(env, X, basis, lo, hi, r, torch.float32)
    got = torch.round(so.double().cpu().exp() - EPS_LOG)
    want = _placed(code, r, 4 * r * (n // (4 * r)))
    assert torch.equal(got, want), "feature_spec places a frame or bin in the wrong spot"
