"""The bi-GRU forward (csrc/gru.cu) and BPTT (csrc/gru_bwd.cu) kernels over their envelope, against float64: written once,
run on the H100 by tests/test_gpu_bigru_envelope.py and under the host emulation (tests/cuda_emu) by
tests/test_bigru_envelope_host.py.

Every check takes an `Env`: a kernel namespace `K` with bigru_fwd_h0 / bigru_bwd_h0 (tacotron_b200.kernels, or its twin
over the emulated library), the raw library for the ABI's refusals, the device, and the activation error bounds of the
library under test.  Every reference is float64, from tests/mirror_kernels_spk (bigru_fwd_h0 / bigru_bwd_h0) or from the
one-step restatements below, on float64 copies of the exact fp32 operands.

Three kinds of check:
* local (teacher-forced): the kernel's state after a step is exactly what it stores, so each step can be formed in
  float64 from the kernel's own previous state and compared with a bar derived from the kernel's arithmetic (`fwd_local`,
  `bwd_local_dr`, and `bwd_compose` at its split steps).  The bar does not grow with T and holds whatever the
  recurrence's conditioning.
* free running: the whole sequence against the float64 mirror, per row, to a bar measured on the H100.
* exact laws, bit for bit: time reversal, restart / composition, utterance and direction independence, NaN isolation,
  zero state = NULL, determinism, and input classes whose float64 result is fp32-representable.
Operands sit inside NaN guard bands and outputs inside a sentinel bit pattern that must survive.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass

import torch

from oracle import tacotron_oracle as O
from tests import mirror_kernels_spk as MK

H = 128
U = 2.0 ** -24                  # fp32 unit roundoff
GAMMA = 2.0 ** -20              # a 128-term fp32 dot product at most 16 roundings deep (the kernels' depth: 13 fwd, 9 bwd)
SAFETY = 2.0                    # every local bar is applied with this factor
PAD = 4096                      # guard band, floats: more than five 768-column rows on each side
SENT = 0x7FA5A5A5               # a signalling-NaN bit pattern no arithmetic produces
NAN, INF = float("nan"), float("inf")
H0_MODES = ("none", "same", "diff", "half")     # NULL/NULL, h/h (what ops passes), h_fw != h_bw, NULL/h
FREE_FWD_TOL = 1e-6             # free-running forward, absolute (states are in (-1, 1)); see test_gpu_bigru_envelope.py
FREE_BWD_TOL = 1e-5             # free-running backward, relative to each (b, direction, t) row's max |ref|


@dataclass
class Env:
    K: object                   # bigru_fwd_h0(out, xp, Wg_fw, Wc_fw, Wg_bw, Wc_bw, h0_fw, h0_bw), bigru_bwd_h0(...)
    lib: object                 # the C ABI (taco_bigru_fwd_h0 / taco_bigru_bwd_h0 / taco_last_error)
    device: str
    stream: object = None
    eps_sig: float = 2.5e-7     # absolute bounds of sigmoidf_acc / tanhf_acc (csrc/common.cuh)
    eps_tanh: float = 5e-7

    def sync(self):
        if self.device != "cpu":
            torch.cuda.synchronize()


def gen(seed):
    return torch.Generator().manual_seed(seed)


# ------------------------------------------------------------------------------------------------------------------
# guarded buffers
# ------------------------------------------------------------------------------------------------------------------
def guarded(shape, device, sentinel=False):
    """(buf, view): a contiguous view of `shape` inside PAD elements of NaN (operands) or of the sentinel bit pattern
    (outputs; the view is prefilled with it too, so an element never written fails every value check)"""
    n = math.prod(shape)
    buf = torch.empty(n + 2 * PAD, dtype=torch.float32, device=device)
    if sentinel:
        buf.view(torch.int32).fill_(SENT)
    else:
        buf.fill_(NAN)
    return buf, buf[PAD:PAD + n].view(shape)


def nan_guarded(t, device):
    """a copy of t (fp32) inside NaN guard bands, or None"""
    if t is None:
        return None
    _, v = guarded(tuple(t.shape), device)
    v.copy_(t)
    return v


def bands_intact(buf, n):
    bits = buf.view(torch.int32)
    return bool((bits[:PAD] == SENT).all()) and bool((bits[PAD + n:] == SENT).all())


def untouched(buf):
    return bool((buf.view(torch.int32) == SENT).all())


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def d64(t):
    return None if t is None else t.double()


# ------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------
_PARAMS = {}


def gru_weights(scope):
    """the recurrent rows of a CBHG GRU pair at trained-like glorot scale: (Wg_fw, Wc_fw, Wg_bw, Wc_bw), plus the input
    rows and biases that make xp"""
    if not _PARAMS:
        _PARAMS.update(O.init_params(O.OracleConfig(), seed=1, trained_like=True))
    p = lambda d, n: _PARAMS[f"{scope}/cbhg/gru_{d}/{n}"]
    W = [p("fw", "Wg")[H:], p("fw", "Wc")[H:], p("bw", "Wg")[H:], p("bw", "Wc")[H:]]
    Wx = torch.cat([p("fw", "Wg")[:H], p("fw", "Wc")[:H], p("bw", "Wg")[:H], p("bw", "Wc")[:H]], 1)
    bx = torch.cat([p("fw", "bg"), p("fw", "bc"), p("bw", "bg"), p("bw", "bc")])
    return [w.float().contiguous() for w in W], Wx.float(), bx.float()


def h0_pair(mode, B, g):
    h = lambda: torch.tanh(torch.randn(B, H, generator=g))
    if mode == "none":
        return None, None
    if mode == "same":
        x = h()
        return x, x.clone()
    if mode == "diff":
        return h(), h()
    return None, h()


def fwd_inputs(B, T, regime, h0_mode, seed, scope="post"):
    """CPU fp32 (xp, [Wg_fw, Wc_fw, Wg_bw, Wc_bw], h0_fw, h0_bw) of one input regime:
    typical    -- xp = x.Wx + b of the trained-like CBHG weights with x ~ N(0, 1) (a highway output's scale)
    expansive  -- the same with the recurrent weights x3 (free running means nothing; the local check still holds)
    saturating -- |xp| up to 90 with 2 % of it +-inf"""
    g = gen(seed)
    W, Wx, bx = gru_weights(scope)
    if regime == "expansive":
        W = [w * 3 for w in W]
    if regime == "saturating":
        xp = (torch.rand(B, T, 768, generator=g) * 2 - 1) * 90
        sel = torch.rand(B, T, 768, generator=g)
        xp[sel < 0.01] = INF
        xp[sel > 0.99] = -INF
    else:
        xp = torch.randn(B, T, H, generator=g) @ Wx + bx
    h0f, h0b = h0_pair(h0_mode, B, g)
    return xp.contiguous(), W, h0f, h0b


def run_fwd(env, xp, W, h0f, h0b):
    """one guarded forward: operands copied into NaN bands, out in sentinels; returns out (on the device) after checking
    the bands"""
    B, T, _ = xp.shape
    dev = env.device
    ops = [nan_guarded(t, dev) for t in (xp, *W, h0f, h0b)]
    obuf, out = guarded((B, T, 256), dev, sentinel=True)
    env.K.bigru_fwd_h0(out, *ops)
    env.sync()
    assert bands_intact(obuf, out.numel()), "bigru_fwd wrote outside out"
    return out


def ref_fwd(xp, W, h0f, h0b):
    """the float64 mirror on the operands' device"""
    B, T, _ = xp.shape
    ref = torch.zeros(B, T, 256, dtype=torch.float64, device=xp.device)
    if T:
        MK.bigru_fwd_h0(ref, xp.double(), *[w.double() for w in W], d64(h0f), d64(h0b))
    return ref


def _prev_state(out, h0f, h0b, t0=0, t1=None):
    """float64 [B, t1-t0, 2, 128]: the state each step of [t0, t1) starts from, per direction (the kernel's own stored
    state of the previous processed step, or h0, or 0)"""
    B, T, _ = out.shape
    t1 = T if t1 is None else t1
    dev = out.device
    z = torch.zeros(B, H, dtype=torch.float64, device=dev)
    o = out.double()
    hf = torch.cat([(z if h0f is None else h0f.double().to(dev))[:, None], o[:, :T - 1, :H]], 1)[:, t0:t1]
    hb = torch.cat([o[:, 1:, H:], (z if h0b is None else h0b.double().to(dev))[:, None]], 1)[:, t0:t1]
    return torch.stack([hf, hb], 2)


def _gate_bound(x, S):
    """gamma * S where the input is finite; 0 where it is infinite (the activation is then exact: sigmoid 0 / 1,
    tanh +-1)"""
    return torch.where(torch.isinf(x), torch.zeros_like(S), GAMMA * S)


def fwd_local(env, xp, W, h0f, h0b, out, t0=0, t1=None):
    """1a: at every step of [t0, t1), one GRU step in float64 from the kernel's own previous state against the stored
    state, |h'_kernel - h'_64| <= SAFETY * e_h (the bar of the module docstring of test_gpu_bigru_envelope.py).
    Returns the worst |error| / (SAFETY * e_h)."""
    B, T, _ = out.shape
    t1 = T if t1 is None else t1
    if B == 0 or t1 <= t0:
        return 0.0
    dev = out.device
    hp = _prev_state(out, h0f, h0b, t0, t1)                      # [B, n, 2, 128]
    x = xp[:, t0:t1].to(dev).double().view(B, t1 - t0, 2, 384)
    got = out[:, t0:t1].double().view(B, t1 - t0, 2, H)
    worst = 0.0
    for d in range(2):
        Wg, Wc = W[2 * d].to(dev).double(), W[2 * d + 1].to(dev).double()
        h, xd, gd = hp[:, :, d], x[:, :, d], got[:, :, d]
        xg, xc = xd[..., :2 * H], xd[..., 2 * H:]
        ag = xg + h @ Wg
        eg = 0.25 * _gate_bound(xg, xg.abs() + h.abs() @ Wg.abs()) + env.eps_sig
        g = torch.sigmoid(ag)
        r, u, er, eu = g[..., :H], g[..., H:], eg[..., :H], eg[..., H:]
        rh = r * h
        ac = xc + rh @ Wc
        c = torch.tanh(ac)
        ec = (1 - c * c) * (_gate_bound(xc, xc.abs() + rh.abs() @ Wc.abs()) + (h.abs() * er) @ Wc.abs()) + env.eps_tanh
        hn = u * h + (1 - u) * c
        eh = (h - c).abs() * eu + (1 - u) * ec + 4 * U * ((u * h).abs() + ((1 - u) * c).abs() + hn.abs())
        err = (gd - hn).abs()
        assert not torch.isnan(gd).any(), f"dir {d}: NaN in the stored state"
        ratio = (err / (SAFETY * eh)).max().item()
        if ratio > 1.0:
            i = torch.nonzero(err > SAFETY * eh)[0].tolist()
            raise AssertionError(f"dir {d}: step {t0 + i[1]} of utterance {i[0]}, unit {i[2]}: kernel "
                                 f"{gd[tuple(i)].item():.9g}, float64 {hn[tuple(i)].item():.9g}, bar "
                                 f"{SAFETY * eh[tuple(i)].item():.3g} ({ratio:.3g} of it)")
        worst = max(worst, ratio)
    return worst


def fwd_free(xp, W, h0f, h0b, out, tol=FREE_FWD_TOL):
    """1b: the free-running state against the float64 mirror, absolute; returns the max |error|"""
    dev = out.device
    ref = ref_fwd(xp.to(dev), [w.to(dev) for w in W], None if h0f is None else h0f.to(dev),
                  None if h0b is None else h0b.to(dev))
    err = (out.double() - ref).abs().max().item() if out.numel() else 0.0
    assert err <= tol, f"free-running forward off by {err:.3g} (bar {tol:.3g})"
    return err


# ------------------------------------------------------------------------------------------------------------------
# forward: exact laws
# ------------------------------------------------------------------------------------------------------------------
def _swap_halves(t, w):
    """swap the two w-wide direction blocks of the last axis"""
    return torch.cat([t[..., w:], t[..., :w]], -1).contiguous()


def fwd_laws(env, xp, W, h0f, h0b, out=None, restarts=True):
    """1c, bit for bit: determinism, time reversal, restart, direction and NaN isolation, zero state = NULL"""
    B, T, _ = xp.shape
    dev = env.device
    run = lambda *a: run_fwd(env, *a)
    out = run(xp, W, h0f, h0b) if out is None else out
    assert same_bits(run(xp, W, h0f, h0b), out), "two runs differ"
    if B == 0 or T == 0:
        return out
    # time reversal: flipped time, swapped direction blocks / weights / initial states
    rev = run(_swap_halves(xp.flip(1), 384), [W[2], W[3], W[0], W[1]], h0b, h0f)
    assert same_bits(_swap_halves(rev.flip(1), H), out), "time reversal"
    # restart at s: fw over [s, T) from out[:, s-1], bw over [0, s) from out[:, s]
    if restarts:
        ocpu = out.cpu()
        for s in sorted({s for s in (1, 2, 3, T // 2, T - 1) if 1 <= s < T}):
            a = run(xp[:, s:].contiguous(), W, ocpu[:, s - 1, :H].contiguous(), h0b)
            assert same_bits(a[:, :, :H], out[:, s:, :H]), f"fw restart at {s}"
            b = run(xp[:, :s].contiguous(), W, h0f, ocpu[:, s, H:].contiguous())
            assert same_bits(b[:, :, H:], out[:, :s, H:]), f"bw restart at {s}"
    # direction isolation: new weights in one direction leave the other half alone
    g = gen(7)
    a = run(xp, [W[0], W[1], W[2] * 0.5 + 0.01 * torch.randn(W[2].shape, generator=g), W[3].flip(0).contiguous()], h0f, h0b)
    assert same_bits(a[..., :H], out[..., :H]), "bw weights changed the fw half"
    a = run(xp, [W[0].flip(1).contiguous(), W[1] * 0.5, W[2], W[3]], h0f, h0b)
    assert same_bits(a[..., H:], out[..., H:]), "fw weights changed the bw half"
    # NaN isolation: a NaN in one fw gate column of utterance 1 at t0 changes only that utterance's fw half from t0 on
    if B >= 2:
        t0 = T // 2
        xn = xp.clone()
        xn[1, t0, 37] = NAN
        a = run(xn, W, h0f, h0b)
        keep = torch.ones(B, T, 256, dtype=torch.bool, device=dev)
        keep[1, t0:, :H] = False
        assert same_bits(a[keep], out[keep]), "a NaN leaked outside utterance 1's fw half from t0"
        assert torch.isnan(a[1, t0:, :H]).all(), "the NaN did not reach every fw state from t0 on"
    # zero state = NULL
    z = torch.zeros(B, H)
    null = out if h0f is None and h0b is None else run(xp, W, None, None)
    assert same_bits(run(xp, W, z, z), null), "h0 = zeros differs from NULL"
    return out


def fwd_utterances(env, xp, W, h0f, h0b, out):
    """1c utterance independence: every utterance of a batched launch equals a B = 1 launch on its rows"""
    for b in range(xp.shape[0]):
        sl = lambda t: None if t is None else t[b:b + 1].contiguous()
        assert same_bits(run_fwd(env, sl(xp), W, sl(h0f), sl(h0b)), out[b:b + 1]), f"utterance {b} of {xp.shape[0]}"


def fwd_exact(env, B, T, seed):
    """1d: gate inputs in {-inf, 0, +inf} (r, u in {0, 1/2, 1}; a finite input only on columns whose recurrent weights
    are 0), candidate inputs +-inf (c = +-1), dyadic h0; u in {0, 1} when T > 16.  The state stays exactly representable
    at any T, so the kernel must equal float64 bit for bit."""
    g = gen(seed)
    sign = lambda *s: torch.where(torch.rand(*s, generator=g) < 0.5, -INF, INF)
    W = [torch.randn(H, 256, generator=g) * 0.1, torch.randn(H, H, generator=g) * 0.1,
         torch.randn(H, 256, generator=g) * 0.1, torch.randn(H, H, generator=g) * 0.1]
    xp = torch.zeros(B, T, 768)
    for d in range(2):
        free = torch.rand(256, generator=g) < 0.5             # gate columns that may see a 0 input
        if T > 16:
            free[H:] = False                                   # u in {0, 1}: no halving of the state
        W[2 * d][:, free] = 0
        xg = sign(B, T, 256)
        zero = (torch.rand(B, T, 256, generator=g) < 0.4) & free
        xg[zero] = 0
        xp[:, :, 384 * d:384 * d + 256] = xg
        xp[:, :, 384 * d + 256:384 * d + 384] = sign(B, T, H)
    h0f = torch.randint(-8, 9, (B, H), generator=g).float() / 8
    h0b = torch.randint(-8, 9, (B, H), generator=g).float() / 8
    ref = ref_fwd(xp, W, h0f, h0b)
    assert torch.equal(ref.float().double(), ref), "the exact class left fp32"
    out = run_fwd(env, xp, W, h0f, h0b)
    assert same_bits(out.cpu(), ref.float()), "exact class: the kernel differs from float64"
    return out


# ------------------------------------------------------------------------------------------------------------------
# forward: the C ABI
# ------------------------------------------------------------------------------------------------------------------
def _vp(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def fwd_call(env, xp, W, h0f, h0b, out, B, T):
    return env.lib.taco_bigru_fwd_h0(_vp(xp), *[_vp(w) for w in W], _vp(h0f), _vp(h0b), _vp(out), B, T, env.stream)


def fwd_abi(env, refusals=True):
    """1e: T = 0 / B = 0 return 0 and leave out untouched, also with NULL operands of the empty sequence; with
    `refusals`, NULL pointers of a non-empty launch and negative sizes are refused (under the host emulation: the entry
    point's checks are the same source there, and a call they let through cannot reach a device)"""
    dev = env.device
    B, T = 3, 4
    xp, W, h0f, h0b = fwd_inputs(B, T, "typical", "diff", 5)
    xp, h0f, h0b = nan_guarded(xp, dev), nan_guarded(h0f, dev), nan_guarded(h0b, dev)
    W = [nan_guarded(w, dev) for w in W]
    obuf, out = guarded((B, T, 256), dev, sentinel=True)
    for b, t in ((1, 0), (3, 0), (0, 5), (0, 0)):
        assert fwd_call(env, xp, W, h0f, h0b, out, b, t) == 0, env.lib.taco_last_error()
        assert fwd_call(env, xp, W, None, None, out, b, t) == 0
        assert fwd_call(env, None, W, None, None, None, b, t) == 0, env.lib.taco_last_error()
    env.sync()
    assert untouched(obuf), "an empty launch wrote to out"
    for i in range(4):
        assert fwd_call(env, xp, W[:i] + [None] + W[i + 1:], h0f, h0b, out, 0, 0) != 0, f"NULL weight {i} accepted"
    if not refusals:
        return
    for i in range(6):
        args = [xp, *W, out]
        args[i] = None
        assert fwd_call(env, args[0], args[1:5], h0f, h0b, args[5], B, T) != 0, f"NULL operand {i} accepted"
    for b, t in ((-1, 4), (3, -1), (-1, -1)):
        assert fwd_call(env, xp, W, h0f, h0b, out, b, t) != 0, f"negative size ({b}, {t}) accepted"
    env.sync()
    assert untouched(obuf), "a refused call wrote to out"


LIMIT_BT = (2 ** 31 - 1) // 768       # the largest B*T the forward's 32-bit offsets admit: 2 796 202


def fwd_limit(env, tail=4096):
    """1e at the ABI's limit: B*T = LIMIT_BT (B = 2, T = 1 398 101) is accepted and locally right on the first and last
    `tail` steps of each direction; one more is refused before anything is launched.  The buffers hold LIMIT_BT + 1
    rows, so even the refused call could not reach outside them."""
    dev = env.device
    B, T = 2, LIMIT_BT // 2
    assert B * T == LIMIT_BT and (LIMIT_BT + 1) * 768 >= 2 ** 31
    W, Wx, bx = gru_weights("post")
    xbuf, xp = guarded((LIMIT_BT + 1, 768), dev)
    torch.manual_seed(0)
    for i in range(0, LIMIT_BT + 1, 1 << 18):                 # typical inputs, built in slices
        rows = xp[i:i + (1 << 18)]
        rows.copy_(torch.randn(rows.shape[0], H, device=dev) @ Wx.to(dev) + bx.to(dev))
    Wd = [nan_guarded(w, dev) for w in W]
    g = gen(3)
    h0f, h0b = nan_guarded(torch.tanh(torch.randn(B, H, generator=g)), dev), nan_guarded(torch.tanh(torch.randn(B, H, generator=g)), dev)
    obuf, out = guarded((LIMIT_BT + 1, 256), dev, sentinel=True)
    assert fwd_call(env, xp, Wd, h0f, h0b, out, 1, LIMIT_BT + 1) != 0, "B*T = 2^31 / 768 + 1 accepted"
    env.sync()
    assert untouched(obuf), "the refused call wrote to out"
    assert fwd_call(env, xp, Wd, h0f, h0b, out, B, T) == 0, env.lib.taco_last_error()
    env.sync()
    bits = obuf.view(torch.int32)
    assert bool((bits[:PAD] == SENT).all()) and bool((bits[PAD + LIMIT_BT * 256:] == SENT).all()), \
        "bigru_fwd wrote outside out at the limit"
    o = out[:LIMIT_BT].view(B, T, 256)
    x = xp[:LIMIT_BT].view(B, T, 768)
    worst = 0.0
    for t0, t1 in ((0, tail), (T - tail, T)):
        # one more step on each side inside the sequence, so that every checked step's previous state is in the window
        a0, a1 = max(t0 - 1, 0), min(t1 + 1, T)
        worst = max(worst, fwd_local(env, x[:, a0:a1], W, h0f if a0 == 0 else None, h0b if a1 == T else None,
                                     o[:, a0:a1], t0 - a0, t1 - a0))
    return worst


# ------------------------------------------------------------------------------------------------------------------
# backward
# ------------------------------------------------------------------------------------------------------------------
def act_from(xp, W, out, h0f, h0b):
    """ACT [B,T,768] = r | u | c per direction, recomputed in float64 from the kernel's forward (its stored states) and
    rounded to fp32, as models/grad.py recomputes it"""
    B, T, _ = out.shape
    dev = out.device
    hp = _prev_state(out, h0f, h0b)
    x = xp.to(dev).double().view(B, T, 2, 384)
    parts = []
    for d in range(2):
        Wg, Wc = W[2 * d].to(dev).double(), W[2 * d + 1].to(dev).double()
        h = hp[:, :, d]
        g = torch.sigmoid(x[:, :, d, :2 * H] + h @ Wg)
        c = torch.tanh(x[:, :, d, 2 * H:] + (g[..., :H] * h) @ Wc)
        parts += [g, c]
    return torch.cat(parts, -1).float().contiguous()


def bwd_inputs(env, B, T, h0_mode, seed, scope="post"):
    """a real forward's (out, ACT) on the device; dOut random with 1 row in 8 x64.  Returns CPU fp32 tensors."""
    xp, W, h0f, h0b = fwd_inputs(B, T, "typical", h0_mode, seed, scope)
    out = run_fwd(env, xp, W, h0f, h0b)
    ACT = act_from(xp, W, out, h0f, h0b)
    g = gen(seed + 1)
    dOut = torch.randn(B, T, 256, generator=g)
    dOut[torch.rand(B, T, generator=g) < 0.125] *= 64
    return dict(dOut=dOut, out=out.cpu(), ACT=ACT.cpu(), W=W, h0f=h0f, h0b=h0b)


def run_bwd(env, dOut, out, ACT, W, h0f, h0b, want_dh0=True):
    """one guarded backward: returns (dxp, dh0 or None) on the device"""
    B, T, _ = out.shape
    dev = env.device
    ops = [nan_guarded(t, dev) for t in (dOut, out, ACT, *W, h0f, h0b)]
    xbuf, dxp = guarded((B, T, 768), dev, sentinel=True)
    hbuf, dh0 = guarded((B, 2, H), dev, sentinel=True)
    env.K.bigru_bwd_h0(dxp, *ops, dh0 if want_dh0 else None)
    env.sync()
    assert bands_intact(xbuf, dxp.numel()), "bigru_bwd wrote outside dxp"
    if not want_dh0:
        assert untouched(hbuf), "bigru_bwd wrote a NULL dh0"
        return dxp, None
    assert bands_intact(hbuf, dh0.numel()), "bigru_bwd wrote outside dh0"
    return dxp, dh0


def ref_bwd(dOut, out, ACT, W, h0f, h0b, device):
    B, T, _ = out.shape
    dxp = torch.zeros(B, T, 768, dtype=torch.float64, device=device)
    dh0 = torch.zeros(B, 2, H, dtype=torch.float64, device=device)
    dv = lambda t: None if t is None else t.to(device).double()
    MK.bigru_bwd_h0(dxp, dv(dOut), dv(out), dv(ACT), *[dv(w) for w in W], dv(h0f), dv(h0b), dh0)
    return dxp, dh0


def bwd_free(env, I, dxp, dh0, tol=FREE_BWD_TOL):
    """2c: every (b, direction, t) row of dxp, and dh0 per (b, direction), against the float64 mirror, relative to that
    row's max |ref|.  Returns the worst |error| / max|ref row|."""
    B, T, _ = I["out"].shape
    if B == 0:
        return 0.0
    rx, rh = ref_bwd(I["dOut"], I["out"], I["ACT"], I["W"], I["h0f"], I["h0b"], dxp.device)
    worst = 0.0
    for got, ref in ((dxp.double().view(B, T, 2, 384), rx.view(B, T, 2, 384)), (dh0.double(), rh)):
        if ref.numel() == 0:
            continue
        ratio = _ratio((got - ref).abs(), ref.abs().amax(-1, keepdim=True))
        w = ratio.max().item()
        if not w <= tol:
            i = torch.nonzero(ratio == ratio.max())[0].tolist()
            raise AssertionError(f"free-running backward: row {i[:-1]} element {i[-1]} off by {w:.3g} of its row's max "
                                 f"(bar {tol:.3g})")
        worst = max(worst, w)
    return worst


def _hprev(I, device):
    return _prev_state(I["out"].to(device), I["h0f"], I["h0b"])          # [B, T, 2, 128] float64


def bwd_local_dr(env, I, dxp):
    """2b, every step: dr_pre from the kernel's own dc_pre of that step (phase 1 depends on nothing else):
    drh = dc.Wc^T, dr_pre = drh * hprev * r(1-r), within SAFETY * (|hprev r(1-r)| gamma S + 5u |dr_pre|)"""
    B, T, _ = dxp.shape
    if B == 0 or T == 0:
        return 0.0
    dev = dxp.device
    hp = _hprev(I, dev)
    got = dxp.double().view(B, T, 2, 384)
    A = I["ACT"].to(dev).double().view(B, T, 2, 384)
    worst = 0.0
    for d in range(2):
        Wc = I["W"][2 * d + 1].to(dev).double()
        dc = got[:, :, d, 2 * H:]
        r = A[:, :, d, :H]
        f = hp[:, :, d] * r * (1 - r)
        dr = (dc @ Wc.t()) * f
        bar = SAFETY * (f.abs() * GAMMA * (dc.abs() @ Wc.abs().t()) + 5 * U * dr.abs())
        err = (got[:, :, d, :H] - dr).abs()
        assert not torch.isnan(got[:, :, d, :H]).any()
        ratio = _ratio(err, bar).max().item()
        assert ratio <= 1.0, f"dir {d}: dr_pre off by {ratio:.3g} of its bar"
        worst = max(worst, ratio)
    return worst


def _ratio(err, bar):
    """err / bar per element (0 where err is 0, inf where only the bar is; NaN stays NaN)"""
    return torch.where(err == 0, torch.zeros_like(err), err / bar)


def _du_dc_ratio(I, dxp_row, carry, t, d, device):
    """du_pre and dc_pre of step t, direction d, from dh = fl32(dOut + carry) in float64, against the kernel's row"""
    hp = _hprev(I, device)[:, t, d]
    a = I["ACT"][:, t, 384 * d:384 * d + 384].to(device).double()
    u, c = a[:, H:2 * H], a[:, 2 * H:]
    dh = (I["dOut"][:, t, H * d:H * d + H].to(device) + carry.to(device)).double()
    du = dh * (hp - c) * u * (1 - u)
    dc = dh * (1 - u) * (1 - c * c)
    bar_du = SAFETY * 6 * U * du.abs()
    bar_dc = SAFETY * (6 * U * dc.abs() + 2 * U * (dh * (1 - u)).abs() * c * c)
    got = dxp_row.to(device).double()
    r = 0.0
    for gv, rv, bv in ((got[:, H:2 * H], du, bar_du), (got[:, 2 * H:], dc, bar_dc)):
        r = max(r, _ratio((gv - rv).abs(), bv).max().item())
    return r


def bwd_compose(env, I, dxp, dh0, splits, check_local=True):
    """2a (and 2b at the split steps).  For a split s, three runs:
      A  [s, T) with h0_fw = out[:, s-1, fw]: dxp fw[s:] bit for bit, its dh0 fw = the carry entering step s-1;
      B  [0, s) with h0_bw = out[:, s, bw] and that carry added to dOut[:, s-1, fw] (one fp32 add): dxp fw[:s] and the
         full dh0 fw; dxp bw[:s], its dh0 bw = the carry entering step s;
      C  [s, T) with that carry added to dOut[:, s, bw]: dxp bw[s:] and the full dh0 bw.
    With the carry known exactly, du_pre / dc_pre of steps s-1 (fw) and s (bw) are checked locally in float64.
    Returns the worst local ratio."""
    dOut, out, ACT, W, h0f, h0b = (I[k] for k in ("dOut", "out", "ACT", "W", "h0f", "h0b"))
    B, T, _ = out.shape
    dev = env.device
    sl = lambda t, a, b: t[:, a:b].contiguous()
    worst = 0.0
    full = dxp.cpu().view(B, T, 2, 384)
    fdh = dh0.cpu()
    for s in splits:
        hs_f = out[:, s - 1, :H].contiguous()
        hs_b = out[:, s, H:].contiguous()
        a, ah = run_bwd(env, sl(dOut, s, T), sl(out, s, T), sl(ACT, s, T), W, hs_f, h0b)
        a, ah = a.cpu().view(B, T - s, 2, 384), ah.cpu()
        assert same_bits(a[:, :, 0], full[:, s:, 0]), f"split {s}: fw suffix"
        cf = ah[:, 0]
        d2 = dOut[:, :s].clone()
        d2[:, s - 1, :H] += cf
        b, bh = run_bwd(env, d2, sl(out, 0, s), sl(ACT, 0, s), W, h0f, hs_b)
        b, bh = b.cpu().view(B, s, 2, 384), bh.cpu()
        assert same_bits(b[:, :, 0], full[:, :s, 0]), f"split {s}: fw prefix"
        assert same_bits(bh[:, 0], fdh[:, 0]), f"split {s}: fw dh0 is not the carry"
        assert same_bits(b[:, :, 1], full[:, :s, 1]), f"split {s}: bw prefix"
        cb = bh[:, 1]
        d3 = dOut[:, s:].clone()
        d3[:, 0, H:] += cb
        c, ch = run_bwd(env, d3, sl(out, s, T), sl(ACT, s, T), W, hs_f, h0b)
        c, ch = c.cpu().view(B, T - s, 2, 384), ch.cpu()
        assert same_bits(c[:, :, 1], full[:, s:, 1]), f"split {s}: bw suffix"
        assert same_bits(ch[:, 1], fdh[:, 1]), f"split {s}: bw dh0 is not the carry"
        if check_local:
            worst = max(worst, _du_dc_ratio(I, full[:, s - 1, 0], cf, s - 1, 0, dev),
                        _du_dc_ratio(I, full[:, s, 1], cb, s, 1, dev))
    if check_local and T:                                     # the first processed step of each direction: carry 0
        z = torch.zeros(B, H)
        worst = max(worst, _du_dc_ratio(I, full[:, T - 1, 0], z, T - 1, 0, dev),
                    _du_dc_ratio(I, full[:, 0, 1], z, 0, 1, dev))
    assert worst <= 1.0, f"du_pre / dc_pre off by {worst:.3g} of the bar"
    return worst


def splits_for(T, n_random=8, seed=0):
    g = gen(seed)
    s = {x for x in (1, 2, 3, T // 2, T - 1) if 1 <= x < T}
    if T > 2:
        s |= set(torch.randint(1, T, (n_random,), generator=g).tolist())
    return sorted(s)


def bwd_laws(env, I, dxp, dh0):
    """2d, bit for bit: determinism, time reversal, utterance independence, direction and NaN isolation, NULL dh0"""
    dOut, out, ACT, W, h0f, h0b = (I[k] for k in ("dOut", "out", "ACT", "W", "h0f", "h0b"))
    B, T, _ = out.shape
    a, ah = run_bwd(env, dOut, out, ACT, W, h0f, h0b)
    assert same_bits(a, dxp) and same_bits(ah, dh0), "two runs differ"
    a, _ = run_bwd(env, dOut, out, ACT, W, h0f, h0b, want_dh0=False)
    assert same_bits(a, dxp), "a NULL dh0 changed dxp"
    if B == 0 or T == 0:
        return
    fl = lambda t, w: _swap_halves(t.flip(1), w)
    a, ah = run_bwd(env, fl(dOut, H), fl(out, H), fl(ACT, 384), [W[2], W[3], W[0], W[1]], h0b, h0f)
    assert same_bits(fl(a, 384), dxp) and same_bits(ah.flip(1), dh0), "time reversal"
    g = gen(11)
    a, ah = run_bwd(env, dOut, out, ACT, [W[0], W[1], W[2] * 0.5, (W[3] + 0.01 * torch.randn(H, H, generator=g))], h0f, h0b)
    assert same_bits(a[..., :384], dxp[..., :384]) and same_bits(ah[:, 0], dh0[:, 0]), "bw weights changed the fw half"
    a, ah = run_bwd(env, dOut, out, ACT, [W[0].flip(0).contiguous(), W[1] * 0.5, W[2], W[3]], h0f, h0b)
    assert same_bits(a[..., 384:], dxp[..., 384:]) and same_bits(ah[:, 1], dh0[:, 1]), "fw weights changed the bw half"
    if B >= 2:                       # a NaN in utterance 1's fw dOut at t0 reaches only its fw rows t <= t0 and dh0 fw
        t0 = T // 2
        dn = dOut.clone()
        dn[1, t0, 5] = NAN
        a, ah = run_bwd(env, dn, out, ACT, W, h0f, h0b)
        keep = torch.ones(B, T, 768, dtype=torch.bool, device=dxp.device)
        keep[1, :t0 + 1, :384] = False
        assert same_bits(a[keep], dxp[keep]), "a NaN leaked outside utterance 1's fw rows up to t0"
        keep = torch.ones(B, 2, H, dtype=torch.bool, device=dxp.device)
        keep[1, 0] = False
        assert same_bits(ah[keep], dh0[keep]), "a NaN leaked into another dh0"
        assert torch.isnan(a[1, :t0, :384]).all() and torch.isnan(a[1, t0, :H]).all() and \
            torch.isnan(a[1, t0, [H + 5, 2 * H + 5]]).all(), "the NaN did not reach what depends on it"


def bwd_utterances(env, I, dxp, dh0):
    B = I["out"].shape[0]
    for b in range(B):
        sl = lambda t: None if t is None else t[b:b + 1].contiguous()
        a, ah = run_bwd(env, sl(I["dOut"]), sl(I["out"]), sl(I["ACT"]), I["W"], sl(I["h0f"]), sl(I["h0b"]))
        assert same_bits(a, dxp[b:b + 1]) and same_bits(ah, dh0[b:b + 1]), f"utterance {b} of {B}"


def _signed_perm(g):
    P = torch.zeros(H, H)
    P[torch.arange(H), torch.randperm(H, generator=g)] = torch.where(torch.rand(H, generator=g) < 0.5, -1.0, 1.0)
    return P


def bwd_exact_long(env, B, T, seed):
    """2d exact class: u, r in {0, 1}, c = 0, signed-permutation Wc, integer dOut in [-8, 8].  Every dh feeds one carry
    with weight +-1, so |carry| stays below 8 * 128 * T < 2^24 at T = 1000, and every product is exact."""
    g = gen(seed)
    dOut = torch.randint(-8, 9, (B, T, 256), generator=g).float()
    out = torch.randint(-4, 5, (B, T, 256), generator=g).float() / 4
    ACT = torch.zeros(B, T, 768)
    for d in range(2):
        ACT[:, :, 384 * d:384 * d + 256] = torch.randint(0, 2, (B, T, 256), generator=g).float()
    W = [torch.randint(-3, 4, (H, 256), generator=g).float(), _signed_perm(g),
         torch.randint(-3, 4, (H, 256), generator=g).float(), _signed_perm(g)]
    h0f = torch.randint(-4, 5, (B, H), generator=g).float() / 4
    return _bwd_exact(env, dict(dOut=dOut, out=out, ACT=ACT, W=W, h0f=h0f, h0b=None))


def bwd_exact_short(env, B, T, seed):
    """2d exact class exercising every formula: r = u = 1/2, hprev and c in multiples of 1/2, sparse small-integer Wg /
    Wc and integer dOut.  Each step adds about four fraction bits, so T <= 3 keeps every value within fp32's 24 bits."""
    g = gen(seed)
    sparse = lambda *s: torch.randint(-2, 3, s, generator=g).float() * (torch.rand(*s, generator=g) < 0.03)
    half = lambda *s: torch.randint(-2, 3, s, generator=g).float() / 2
    dOut = torch.randint(-4, 5, (B, T, 256), generator=g).float()
    ACT = torch.full((B, T, 768), 0.5)
    for d in range(2):
        ACT[:, :, 384 * d + 256:384 * d + 384] = torch.randint(-1, 2, (B, T, H), generator=g).float() / 2
    W = [sparse(H, 256), sparse(H, H), sparse(H, 256), sparse(H, H)]
    return _bwd_exact(env, dict(dOut=dOut, out=half(B, T, 256), ACT=ACT, W=W, h0f=half(B, H), h0b=half(B, H)))


def _bwd_exact(env, I):
    rx, rh = ref_bwd(I["dOut"], I["out"], I["ACT"], I["W"], I["h0f"], I["h0b"], "cpu")
    assert torch.equal(rx.float().double(), rx) and torch.equal(rh.float().double(), rh), "the exact class left fp32"
    assert rx.abs().max() < 2 ** 24 and rh.abs().max() < 2 ** 24
    dxp, dh0 = run_bwd(env, I["dOut"], I["out"], I["ACT"], I["W"], I["h0f"], I["h0b"])
    assert same_bits(dxp.cpu(), rx.float()), "exact class: dxp differs from float64"
    assert same_bits(dh0.cpu(), rh.float()), "exact class: dh0 differs from float64"
    return rx.abs().max().item()


def bwd_call(env, dxp, dOut, out, ACT, W, h0f, h0b, dh0, B, T):
    return env.lib.taco_bigru_bwd_h0(_vp(dxp), _vp(dOut), _vp(out), _vp(ACT), *[_vp(w) for w in W], _vp(h0f), _vp(h0b),
                                     _vp(dh0), B, T, env.stream)


def bwd_abi(env, refusals=True):
    """2d guards: T = 0 writes a non-NULL dh0 as zeros and leaves dxp untouched, also with NULL operands of the empty
    sequence; B = 0 touches nothing; with `refusals` (as in fwd_abi), NULL operands of a non-empty launch and negative
    sizes are refused"""
    dev = env.device
    B, T = 3, 4
    ops = [nan_guarded(torch.randn(s), dev) for s in ((B, T, 256), (B, T, 256), (B, T, 768), (H, 256), (H, H), (H, 256), (H, H))]
    dOut, out, ACT, W = ops[0], ops[1], ops[2], ops[3:]
    h0 = nan_guarded(torch.randn(B, H), dev)
    xbuf, dxp = guarded((B, T, 768), dev, sentinel=True)
    hbuf, dh0 = guarded((B, 2, H), dev, sentinel=True)
    assert bwd_call(env, dxp, dOut, out, ACT, W, h0, h0, dh0, B, 0) == 0, env.lib.taco_last_error()
    env.sync()
    assert untouched(xbuf), "T = 0 wrote to dxp"
    assert bands_intact(hbuf, dh0.numel()) and bool((dh0.view(torch.int32) == 0).all()), "T = 0: dh0 is not +0"
    hbuf.view(torch.int32).fill_(SENT)
    assert bwd_call(env, None, None, None, None, W, None, None, dh0, B, 0) == 0, env.lib.taco_last_error()
    env.sync()
    assert bands_intact(hbuf, dh0.numel()) and bool((dh0.view(torch.int32) == 0).all()), "T = 0: dh0 is not +0"
    hbuf.view(torch.int32).fill_(SENT)
    for b, t in ((0, 5), (0, 0), (2, 0)):
        assert bwd_call(env, dxp, dOut, out, ACT, W, h0, h0, None, b, t) == 0
    assert bwd_call(env, dxp, dOut, out, ACT, W, h0, h0, dh0, 0, 5) == 0
    env.sync()
    assert untouched(xbuf) and untouched(hbuf), "an empty launch wrote"
    if not refusals:
        return
    for i in range(8):
        args = [dxp, dOut, out, ACT, *W]
        args[i] = None
        assert bwd_call(env, *args[:4], args[4:], h0, h0, dh0, B, T) != 0, f"NULL operand {i} accepted"
    for b, t in ((-1, 4), (3, -1)):
        assert bwd_call(env, dxp, dOut, out, ACT, W, h0, h0, dh0, b, t) != 0, f"negative size ({b}, {t}) accepted"
    env.sync()
    assert untouched(xbuf) and untouched(hbuf), "a refused call wrote"
