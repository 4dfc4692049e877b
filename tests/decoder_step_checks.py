"""Local (step-by-step) check of the persistent decoder forward, csrc/decoder.cu: every value the kernel stores at step t
is compared with float64 formed from the kernel's OWN stored values, so the bar does not grow with T and an error shows
at the first step and stage it enters.  Written once; run on the H100 by tests/test_gpu_decoder_steps.py and on any float
decoder run (tests/test_decoder_steps_host.py).

What the kernel stores is everything a step depends on: y [B,T,80r], align [B,T,Tx], the three GRU state sequences
h_save [3,T,B,256] and, with an attention window, the peaks [B,T].  models/grad.py::decoder_recompute rebuilds every
activation of every step from exactly those tensors; run over tests/mirror_kernels.py in float64 it is the local reference:

  h1(t)      GRU 1 from z(t) (rebuilt from the kernel's y(t-1), align(t-1) -> ctx, and x(t)) and the kernel's h1(t-1)
  h2(t), h3  GRU i from the kernel's h_{i-1}(t) and h_i(t-1)
  y(t)       (z(t) + the kernel's h3(t)) . W_out + b_out
  align(t)   q = the kernel's y(t) . W_q, e_j = sum_d v_d tanh(k_jd + q_d), j >= text_length (and, windowed, j outside the
             window around the kernel's p(t-1)) masked, softmax
  peak(t)    the lowest j of the highest windowed float64 score; compared where the top two scores are further apart
             than their bars
Free-running decoding is scheduled sampling with every row sampled, a zero go frame and no dropout (keep masks of ones,
keep scale 1); the previous state at step 0 is h0 / att0 or zero.

Bars, per element (u = 2^-24, the fp32 unit roundoff):

* Products.  The kernel's dense stages are 3xTF32 mma.sync products, each operand split into a TF32 head and a remainder
  whose own low 13 bits the tensor core drops: the product error is about 2^-21 |a||b| per term, and the fp32
  accumulation (three accumulators, 16 warp partials, the bias) adds a few u per term.  Those errors are independent from
  term to term, so a K-term sum's error grows as sqrt(K), not K (probabilistic rounding-error analysis, Higham and Mary,
  SIAM J. Sci. Comput. 41 (2019)): the bar is C * 2^-20 * S with S built from rss(X, W) = sqrt(X^2 . W^2), the size of
  X . W for independent errors of size X.  S follows the matrices the kernel actually multiplies (decoder.cu fused_tail:
  the first GRU takes z through the pack-time products of W_in, W_a and W_out with Wg1_x / Wc1_x; OQP forms q and the
  next p1 from s through W_out W_q and W_out[:, last 80] W1), and adds each operand's own deviation from the reference's:
      the kernel's y(t-1) vs s(t-1) . W_out + b_out:  dy = rss(|s(t-1)|, W_out) + |b_out|   (the reference reads y)
      the context vs align . values:                  rss(align, values)
      p1 (free-running rows) = rss(|s(t-1)|, W_out,80 W1) + |b_p1| + rss(dy_80, W1);  teacher rows rss(|x|, W1) + |b1|
      p2 = rss(S_p1, W2) + rss(p1, W2) + |b2|  (both times keep * scale)
      first GRU, for Wx = Wg1_x or Wc1_x:  rss(|ctx|, W_a,ctx W_in,a Wx) + rss(ctx dev, same) + rss(|p2|, W_in,p Wx)
          + rss(S_p2, same) + rss(|s(t-1)|, W_out W_a,y W_in,a Wx) + rss(dy, W_a,y W_in,a Wx) + |b_inF Wx| + h(t-1) terms
      layers 2, 3:  rss(h_{i-1}(t), Wg_x) + rss(h_i(t-1), Wg_h) + |bg|, and the same with r h for the candidate
      y:  rss(|s|, W_out) + |b_out| + rss(S_z, W_out)   (s = z + h3 with the kernel's z, which carries z's bar S_z)
      q:  rss(|s|, W_out W_q) + |b_out W_q| + rss(dy(t), W_q)
  The fold's own rounding (each folded product formed in float64 from fp32 operands and rounded once, the intermediate
  ones again in the next fold) is not bounded but computed: the folds are rebuilt here exactly as packed and in exact
  float64, and 2^-24 F = |operand . (packed - exact)| enters each bar as it is.
* Functions and element-wise steps, carried through their derivatives:
      sigmoidf_acc 2.5e-7, tanhf_acc 5e-7 absolute (common.cuh)
      gates     dr, du = s(1 - s) * C 2^-20 S_g + 2.5e-7
      candidate dc = (1 - c^2) * (C 2^-20 S_c + rss(dr h(t-1), Wc_h)) + 5e-7
      state     dh = |h(t-1) - c| du + (1 - u) dc + 2u (|(1 - u) c| + |u h(t-1)| + |h|)
  The attention forms tanh(k + q) = 1 - 2 R, R = 1/(e^{2k} e^{2q} + 1), with exp2f (2 ulp, its argument rounded: a
  relative error 2u * |k| in e^{2k}), one fma, rcp.approx (1 ulp), then e_j = sum_d v_d - 2 sum_d v_d R_d.  With
  2 R P / (P + 1) = (1 - t^2) / 2 and 2 R = 1 - t:
      de_j = ||v_d (1 - t_jd^2) (dq_d + u (|k_jd| + |q_d| + 2))||_d + 7 u ||v_d (1 - t_jd)||_d + u (4 ||v||_d + |e_j|)
  (||.||_d the root-sum-square over the 256 depths, as above; dq = q's bar; the 256-term sums are 13 roundings deep, 8 per
  lane then a 5-level butterfly: 4 ~ sqrt(13), and 7 = 3 for the fma and rcp + 4).  The softmax
  (__expf, relative 2 ulp plus u |x| from its rounded argument; the quarter statistics and the normalisation):
      dalpha_j = alpha_j (de_j + sum_k alpha_k de_k + u (3 |e_j - M| + 3 sum_k alpha_k |e_k - M| + 24)) + 2^-126
  (2^-126: __expf flushes results below the normal range to zero).  A step whose keys or query reach exp2x's clamp
  (|x| > 20.79) is scored as sum_d v_d tanhf_acc(k_jd + q_d) instead; its de_j also carries 5e-7 sum_d |v_d|.
* Calibration: C is one constant for the whole envelope, C_PROD below.  Each `Report` carries the worst measured ratio
  |kernel - reference| / bar per quantity; the figures measured on the H100 are in DESIGN.md section 3.4.

The first failing element in (t, stage, b, unit) order is where the fault sits: everything after it is checked against
the faulty state.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from types import SimpleNamespace

import torch

from tacotron_b200.models import grad
from tests import mirror_kernels as MK

U24 = 2.0 ** -24
EPS = 2.0 ** -20
C_PROD = 2.0                    # C of the product bars (calibrated on the H100, DESIGN.md section 3.4)
SIG_ERR, TANH_ERR = 2.5e-7, 5e-7
FLUSH = 2.0 ** -126
CLAMP = 20.7                    # |k|, |q| past which decoder.cu's exp2x may clamp (60 / 2.885390082 = 20.79)
STAGES = ("h1", "h2", "h3", "y", "align", "peak")
MF, UNITS = 80, 256


@dataclass
class Failure:
    t: int
    stage: str
    b: int
    unit: int
    value: float
    ref: float
    bar: float
    S: float

    def __str__(self):
        return (f"first failure at t={self.t} {self.stage} b={self.b} unit={self.unit}: kernel {self.value!r}, "
                f"float64 {self.ref!r}, bar {self.bar:.3e}, S {self.S:.3e}")


@dataclass
class Report:
    worst: dict                         # stage -> worst |kernel - reference| / bar
    first: Failure | None
    bar: dict = field(repr=False)       # stage -> [T,B,N] bars (time-major)
    ref: dict = field(repr=False)       # stage -> [T,B,N] float64 references
    ratio: dict = field(repr=False)     # stage -> [T,B,N]

    def __str__(self):
        w = ", ".join(f"{k} {v:.3f}" for k, v in self.worst.items())
        return f"worst ratio to the bar: {w}" + ("" if self.first is None else f"; {self.first}")


def rss(X, W):
    """sqrt(X^2 . W^2): the probabilistic size of X . W for independent per-term errors of size X (Higham and Mary,
    SIAM J. Sci. Comput. 41 (2019): a sum of n rounding errors grows as sqrt(n) u, not n u, with high probability)"""
    return torch.sqrt((X * X) @ (W * W))


def gru_bar(RU, cc, hp, S_g, S_c, Wc_h, c=C_PROD):
    """GRU state update h = u h(t-1) + (1 - u) c and its bar.  RU [.., 2N] = [r | u], cc [.., N] candidate, hp [.., N]
    h(t-1), S_g [.., 2N] / S_c [.., N] the sizes of the gate / candidate pre-activations' errors in units of C 2^-20,
    Wc_h [N,N] the candidate's recurrent weights"""
    N = cc.shape[-1]
    d_g = RU * (1 - RU) * (c * EPS * S_g) + SIG_ERR
    d_r, d_u = d_g[..., :N], d_g[..., N:]
    uu = RU[..., N:]
    d_c = (1 - cc * cc) * (c * EPS * S_c + rss(d_r * hp, Wc_h)) + TANH_ERR
    h = uu * hp + (1 - uu) * cc
    return h, (hp - cc).abs() * d_u + (1 - uu) * d_c + 2 * U24 * (((1 - uu) * cc).abs() + (uu * hp).abs() + h.abs())


def score_bar(th, e, v_abs, dq, k_abs, q_abs):
    """bar of the kernel's score e_j = sum_d v_d - 2 sum_d v_d R_jd (R = 1/(e^{2k} e^{2q} + 1)).  th [.., Tx, D] =
    tanh(k + q), e [.., Tx], v_abs [D], dq / k_abs / q_abs broadcasting to th: q's bar and the absolute operands"""
    t1 = v_abs * (1 - th * th) * (dq + U24 * (k_abs + q_abs + 2))
    t2 = v_abs * (1 - th)
    return (torch.sqrt((t1 * t1).sum(-1)) + 7 * U24 * torch.sqrt((t2 * t2).sum(-1))
            + U24 * (4 * torch.sqrt((v_abs * v_abs).sum()) + e.abs()))


def softmax_bar(alpha, dE, dist):
    """bar of alpha = softmax(e) over the last axis: dE the score bars, dist = |e - max e| (both 0 where masked)"""
    return (alpha * (dE + (alpha * dE).sum(-1, keepdim=True) + U24 * (3 * dist + 3 * (alpha * dist).sum(-1, keepdim=True) + 24))
            + FLUSH)


def _tm(x):
    """[B,T,...] -> time-major [T,B,...]"""
    return x.transpose(0, 1).contiguous()


def _prev(X, first):
    """X [T,B,N] -> X(t-1), `first` [B,N] (or zeros) at t = 0"""
    out = torch.empty_like(X)
    out[0] = 0 if first is None else first
    out[1:] = X[:-1]
    return out


def check(y, align, H, P, keys, values, text_length, r, mode, *, mel=None, sample_mask=None, keep=None, keep_scale=1.0,
          h0=None, att0=None, window=None, peak=None, c=C_PROD, chunk=8):
    """One decoder run, checked step by step.  y [B,T,80r], align [B,T,Tx], H [3,T,B,256] (h_save), peak [B,T] (windowed
    runs): the kernel's outputs.  P: the weights ('dec/...' names), keys / values [B,Tx,256] and text_length [B]: the
    kernel's inputs.  mode 'infer' | 'teacher' | 'sched'; mel [B,T,80r] and sample_mask [T,B] as the kernel took them,
    keep = (keep1 [T,B,256], keep2 [T,B,128]) or None, h0 [3,B,256] / att0 [B,256] or None, window (back, ahead) or
    None.  Everything is evaluated in float64 on y's device.  Returns a Report."""
    dev = y.device
    f = lambda x: None if x is None else x.to(dev, torch.float64)
    B, T, OUT = y.shape
    Tx = align.shape[2]
    Pd = {k: f(v) for k, v in P.items() if k.startswith("dec/") and torch.is_tensor(v)}
    y64, al64, H64, K64, V64 = f(y), f(align), f(H), f(keys), f(values)
    h064, att064 = f(h0), f(att0)
    tl = text_length.to(dev, torch.int64)
    if mode == "infer":                 # scheduled sampling with every row sampled, zero go frame, no dropout
        mel64 = torch.zeros(B, T, OUT, dtype=torch.float64, device=dev)
        sm = torch.ones(T, B, dtype=torch.uint8, device=dev)
    else:
        mel64 = f(mel)
        sm = None if mode == "teacher" else sample_mask.to(dev, torch.uint8)
    if keep is None:
        keep = (torch.ones(T, B, 256, dtype=torch.uint8, device=dev), torch.ones(T, B, 128, dtype=torch.uint8, device=dev))
        keep_scale = 1.0
    k1, k2 = (k.to(dev, torch.uint8) for k in keep)
    cfg = SimpleNamespace(mel_features=MF, r=r, audio_dropout_prob=1.0 - 1.0 / keep_scale)
    S = {"dec/y": y64, "dec/align": al64, "dec/H": H64, "dec/values": V64, "mel": mel64, "dec/keep1": k1, "dec/keep2": k2,
         "dec/h0": h064, "dec/att0": att064}
    if sm is not None:
        S["dec/sample_mask"] = sm
    R = grad.decoder_recompute(MK, Pd, S, cfg)
    ks = R["ks"]
    A = {k: v.abs() for k, v in Pd.items()}
    W_in, W_a, W_out = A["dec/in_proj/W"], A["dec/attn/W_a"], A["dec/out_proj/W"]
    lo = OUT - MF
    # ---- the folded products the kernel multiplies (decoder.cu fused_tail): exact, and as packed (each fold formed in
    #      float64 from fp32 operands and rounded once); E_* = |packed - exact|, the fold's own rounding ----
    f32 = lambda x: x.float().double()
    W_a_, W_in_, W_out_ = Pd["dec/attn/W_a"], Pd["dec/in_proj/W"], Pd["dec/out_proj/W"]
    b_in_, b_out_, W_q_, W1_ = Pd["dec/in_proj/b"], Pd["dec/out_proj/b"], Pd["dec/attn/W_q"], Pd["dec/prenet/W1"]
    Mc = W_a_[OUT:] @ W_in_[128:]                                                # ctx -> z
    M1 = W_a_[:OUT] @ W_in_[128:]                                                # y -> z
    M1f = f32(M1)
    Ms, Msf = W_out_ @ M1, f32(W_out_ @ M1f)                                     # s -> z
    bz, bzf = b_in_ + b_out_ @ M1, f32(b_in_ + b_out_ @ M1f)                     # z's bias, t > 0
    fold = {"Mc": (Mc, f32(Mc)), "Ms": (Ms, Msf), "bz": (bz, bzf), "bz0": (b_in_, b_in_)}
    Mq, Mp1 = W_out_ @ W_q_, W_out_[:, lo:] @ W1_
    bp1 = b_out_[lo:] @ W1_ + Pd["dec/prenet/b1"]
    Eq, Ebq = f32(Mq) - Mq, f32(b_out_ @ W_q_) - b_out_ @ W_q_                 # signed fold errors
    Ep1, Ebp1 = f32(Mp1) - Mp1, f32(bp1) - bp1
    Z = R["Z"].view(T, B, UNITS)
    Hs = [H64[i] for i in range(3)]
    s_abs = (Z + Hs[2]).abs()
    s_prev = _prev(s_abs, None)
    later = torch.ones(T, 1, 1, dtype=torch.float64, device=dev)
    later[0] = 0                                                                 # t > 0: there is an s(t-1)
    s_sig = _prev(Z + Hs[2], None)                                               # s(t-1), signed
    dy_prev = rss(s_prev, W_out) + A["dec/out_proj/b"] * later                   # the kernel's y(t-1) vs s(t-1) . W_out + b
    ctx_sig = _prev(R["CTX"].view(T, B, -1), None)                              # ctx(t-1) from the kernel's align(t-1)
    ctx_prev = ctx_sig.abs()
    ctx_dev = _prev(_tm(torch.sqrt(torch.bmm(al64 * al64, V64 * V64))), None)  # the kernel's context vs align . values
    sel = R["sel"].to(torch.bool)[..., None]
    Xin = R["Xin"]
    kk1, kk2 = k1.to(torch.float64) * ks, k2.to(torch.float64) * ks
    # pre-net: p1 of free-running rows from s(t-1) through the fold with W1 (the reference: the kernel's y(t-1)), of teacher
    # rows from the frame; S_* in units of C 2^-20, F_* the fold roundings in units of 2^-24
    S_p1 = torch.where(sel, rss(s_prev, Mp1) + bp1.abs() + rss(dy_prev[..., lo:], W1_),
                       rss(Xin.abs(), W1_) + A["dec/prenet/b1"]) * kk1
    F_p1 = torch.where(sel, (s_sig @ Ep1 + Ebp1).abs(), torch.zeros_like(S_p1)) * kk1
    P1, P2 = R["PN1"].view(T, B, -1), R["PN2"].view(T, B, -1)
    W2_ = Pd["dec/prenet/W2"]
    S_p2 = (rss(S_p1, W2_) + rss(P1, W2_) + A["dec/prenet/b2"]) * kk2
    F_p2 = rss(F_p1, W2_) * kk2

    def first_layer(Wx):
        """(S, F) of [ctx | p2] . W_cpF Wx + s(t-1) . W_sF Wx + b_inF Wx, as the kernel multiplies it (Wx = None: z)"""
        def fm(name):
            ex, pk = fold[name]
            if Wx is None:
                return ex, pk - ex
            e2 = ex @ Wx
            return e2, f32(pk @ Wx) - e2
        (Mc2, Ec2), (Ms2, Es2), (bz2, Ebz2), (bz02, Ebz02) = fm("Mc"), fm("Ms"), fm("bz"), fm("bz0")
        Mp2 = W_in_[:128] if Wx is None else W_in_[:128] @ Wx
        My2 = M1 if Wx is None else M1 @ Wx
        Ep2 = torch.zeros_like(Mp2) if Wx is None else f32(Mp2) - Mp2
        S = (rss(ctx_prev, Mc2) + rss(ctx_dev, Mc2) + rss(P2, Mp2) + rss(S_p2, Mp2) + rss(s_prev, Ms2)
             + rss(dy_prev, My2))
        Fs = ctx_sig @ Ec2 + P2 @ Ep2 + s_sig @ Es2
        S[1:] += bz2.abs()
        S[0] += bz02.abs()
        Fs[1:] += Ebz2
        Fs[0] += Ebz02
        F = Fs.abs() + rss(F_p2, Mp2)
        if att064 is not None:                  # step 0: att0 . W_in[128:] (. Wx) formed by the library's GEMM
            iz = att064 @ W_in_[128:]
            S[0] += rss(att064.abs(), W_in_[128:]) if Wx is None else rss(iz.abs(), Wx) + rss(rss(att064.abs(), W_in_[128:]), Wx)
        return S, F

    r_cF = U24 / (c * EPS)                      # a fold rounding (2^-24 F) in units of the product bar (C 2^-20)
    ref, bar, Sx = {}, {}, {}
    # ---- the three GRU layers ----
    for i in range(3):
        Wg, Wc = A[f"dec/gru{i+1}/Wg"], A[f"dec/gru{i+1}/Wc"]
        hp = _prev(Hs[i], None if h064 is None else h064[i])
        RU = R["RU"][i].view(T, B, 2 * UNITS)
        rr = RU[..., :UNITS]
        cc = R["C"][i].view(T, B, UNITS)
        if i == 0:
            Sg, Fg = first_layer(Pd["dec/gru1/Wg"][:UNITS])
            Sc, Fc = first_layer(Pd["dec/gru1/Wc"][:UNITS])
            S_g = Sg + r_cF * Fg + rss(hp, Wg[UNITS:]) + A["dec/gru1/bg"]
            S_c = Sc + r_cF * Fc + rss(rr * hp, Wc[UNITS:]) + A["dec/gru1/bc"]
        else:
            xa = Hs[i - 1]
            S_g = rss(xa, Wg[:UNITS]) + rss(hp, Wg[UNITS:]) + A[f"dec/gru{i+1}/bg"]
            S_c = rss(xa, Wc[:UNITS]) + rss(rr * hp, Wc[UNITS:]) + A[f"dec/gru{i+1}/bc"]
        ref[f"h{i+1}"], bar[f"h{i+1}"] = gru_bar(RU, cc, hp, S_g, S_c, Wc[UNITS:], c)
        Sx[f"h{i+1}"] = S_c
    # ---- output projection: s = z + h3 with the kernel's z, which carries z's bar ----
    S_z, F_z = first_layer(None)
    ref["y"] = (Z + Hs[2]) @ W_out_ + b_out_
    Sx["y"] = rss(s_abs, W_out) + A["dec/out_proj/b"] + rss(S_z + r_cF * F_z, W_out)
    bar["y"] = c * EPS * Sx["y"]
    # ---- attention: q = s . W_out W_q + b_out W_q in the kernel, the kernel's y(t) . W_q in the reference ----
    q = R["PQ"].view(T, B, UNITS)
    dq = c * EPS * (rss(s_abs, Mq) + (b_out_ @ W_q_).abs() + rss(rss(s_abs, W_out) + A["dec/out_proj/b"], W_q_)) \
        + U24 * ((Z + Hs[2]) @ Eq + Ebq).abs()
    v, va = Pd["dec/attn/v"], A["dec/attn/v"]
    j = torch.arange(Tx, device=dev)
    valid = j[None, :] < tl[:, None]                                             # [B,Tx]
    kabs = K64.abs()
    E = torch.empty(T, B, Tx, dtype=torch.float64, device=dev)
    dE = torch.empty_like(E)
    for t0 in range(0, T, chunk):
        t1 = min(T, t0 + chunk)
        qc = q[t0:t1][:, :, None, :]                                             # [tc,B,1,256]
        th = torch.tanh(K64[None] + qc)                                          # [tc,B,Tx,256]
        E[t0:t1] = (th * v).sum(-1)
        dE[t0:t1] = score_bar(th, E[t0:t1], va, dq[t0:t1][:, :, None, :], kabs[None], qc.abs())
        del th
    # a step whose keys or query reach exp2x's clamp (|x| > 20.79) is scored with tanhf_acc(k + q) instead (decoder.cu
    # scores_direct): its bar also carries tanhf_acc's bound on each of the 256 terms (rows flagged here: a superset)
    direct = (kabs.amax((1, 2)) > CLAMP)[None, :] | (q.abs().amax(-1) > CLAMP)                    # [T,B]
    dE += direct[..., None] * (TANH_ERR * va.sum())
    allowed = valid[None].expand(T, B, Tx).clone()
    if window is not None:
        back, ahead = window
        pk = peak.to(dev, torch.int64)
        pprev = torch.zeros(T, B, dtype=torch.int64, device=dev)
        pprev[1:] = pk[:, :-1].t()
        allowed &= (j >= (pprev - back).clamp_min(0)[..., None]) & (j <= (pprev + ahead)[..., None])
    Em = torch.where(allowed, E, torch.full_like(E, -math.inf))
    M = Em.max(-1, keepdim=True).values
    alpha = torch.where(allowed, torch.exp(Em - M.clamp_min(-1e300)), torch.zeros_like(E))
    alpha = alpha / alpha.sum(-1, keepdim=True).clamp_min(1e-300)
    dist = torch.where(allowed, (E - M).abs(), torch.zeros_like(E))
    dEa = torch.where(allowed, dE, torch.zeros_like(dE))
    ref["align"] = alpha
    bar["align"] = softmax_bar(alpha, dEa, dist)
    Sx["align"] = dEa
    got = {"h1": Hs[0], "h2": Hs[1], "h3": Hs[2], "y": _tm(y64), "align": _tm(al64)}
    ratio = {}
    for k in ("h1", "h2", "h3", "y", "align"):
        d = (got[k] - ref[k]).abs()
        ratio[k] = torch.where(d == 0, torch.zeros_like(d), d / bar[k]).nan_to_num(nan=math.inf)    # NaN: a failure
    if window is not None:            # peak(t): the reference's lowest maximiser, unless the kernel's is within the bars
        pk_t = peak.to(dev, torch.int64).t()                                     # [T,B]
        p_ref = torch.argmax(Em, -1)                                             # first maximal index
        e_ref = Em.gather(-1, p_ref[..., None])[..., 0]
        e_k = Em.gather(-1, pk_t.clamp(0, Tx - 1)[..., None])[..., 0]
        b2 = dE.gather(-1, p_ref[..., None])[..., 0] + dE.gather(-1, pk_t.clamp(0, Tx - 1)[..., None])[..., 0]
        rp = torch.where(pk_t == p_ref, torch.zeros_like(e_ref), (e_ref - e_k) / b2)
        rp = torch.where((pk_t < 0) | (pk_t >= Tx), torch.full_like(rp, math.inf), rp)
        ratio["peak"], ref["peak"], bar["peak"] = rp[..., None], p_ref[..., None].to(torch.float64), b2[..., None]
        got["peak"], Sx["peak"] = pk_t[..., None].to(torch.float64), b2[..., None]
    worst = {k: float(v.max()) for k, v in ratio.items()}
    first = None
    bad = {k: ~(v <= 1) for k, v in ratio.items()}
    if any(bool(b.any()) for b in bad.values()):
        tf = {k: (int(b.any(-1).any(-1).nonzero()[0, 0]) if b.any() else T) for k, b in bad.items()}
        t = min(tf.values())
        k = next(s for s in STAGES if s in tf and tf[s] == t)
        b, n = (int(x) for x in bad[k][t].nonzero()[0])
        first = Failure(t, k, b, n, float(got[k][t, b, n]), float(ref[k][t, b, n]), float(bar[k][t, b, n]), float(Sx[k][t, b, n]))
    return Report(worst, first, bar, ref, ratio)
