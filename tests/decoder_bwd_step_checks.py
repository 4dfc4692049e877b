"""Local (step-by-step) check of the persistent decoder backward, csrc/decoder_bwd.cu: every value the kernel stores at
step t is compared with float64 formed from the kernel's OWN stored outputs and the call's inputs, so the bar does not
grow with T and an error shows at the step and stage it enters.  Written once; run on the H100 by
tests/test_gpu_decoder_bwd_steps.py and on the host emulation and the float64 mirror by tests/test_decoder_bwd_steps_host.py.

What is checked at step t (descending), in the kernel's stage order (the header of decoder_bwd.cu):

  A     dscore  DSCORE(t) = a (dal - sum a dal) + dscore_add,  dal_j = DCTX(t) . values_j
        dpq     DPQ(t)_d = v_d sum_j DSCORE(t)_j (1 - tanh(k_jd + PQ(t)_d)^2)
  4'    E       E(t) = dy_ext(t) . W_out^T, the fold as the call's workspace holds it, against float64
        du3 dc3 GRU 3's head: dh = dres + carry, dres = E(t) + [DATT(t) | DPQ(t) | sel(t+1) DPN1(t+1)] . M124^T
  5/6   dr<i>   dr_pre of layer i from the stored DC_i(t)
        du<i-1> dc<i-1>  the head of layer i-1: dh = DC_i(t) . Wc_i,x^T + DG_i(t) . Wg_i,x^T + carry
        carry<i> the carry into step t-1 (at t = 0: DH0) = dh u + drh r + DG_i(t) . Wg_i,h^T
        dz      DZ(t) = dres + the layer-1 input gradient
  7'    dpn2    DPN2(t) from the stored DZ(t);  datt, dctx: DATT(t-1), DCTX(t-1) (M7 = [W_in | W_a[OUT:] W_in[128:]])
        dpn1    DPN1(t) from the stored DPN2(t) (formed in stage A of step t-1)
  after dy, dx  DY(t) = dy_ext + DATT W_a[:OUT]^T + DPQ W_q^T (+ sel(t+1) DX(t+1)),  DX(t) = DPN1(t) W1^T  (taco_gemm)
The weight folds M124 and M7 are checked on their own against float64 and reported at step T-1, stage 4' / 7'.

The carries dhc_i are not outputs, and DG / DC cannot give them back when u -> 1.  They are read back through DH0: the
kernel run on the suffix s .. T-1 alone, with H0 = H(s-1), leaves in DH0 exactly the full run's carry into step s-1
(composition is an exact law, checked bit for bit by `read_carries`).

Bars, per element (u = 2^-24).  gemm_block: each warp runs n = K/8 chained fmaf, then 8 partials and one epilogue add.
A chain's rounding errors are each u times a partial sum; summed in quadrature (Higham and Mary, SIAM J. Sci. Comput. 41
(2019)) they come to about sqrt(n/2) u rss(X, W), rss(X, W) = sqrt(X^2 . W^2), plus u per later add of the result:
      prod(X, W, K) = sqrt(K/16) rss(|X|, |W|)
  dscore  a_j (e_dal_j + sum_k a_k e_dal_k) + u (sqrt(Tx/2) rss(a, dal) + |a_j (dal_j - tot)| + |ds|),
          e_dal = u (sqrt(13/2) rss_d(dctx, values_j) + 5 |dal|)   (8 fmaf per lane then a 5-level butterfly)
  dpq     |v_d| (u sqrt(Tx/2) rss_j(ds, 1 - e^2) + 2 TANH_ERR rss_j(ds, e)) + 2 u |dpq|   (tanhf_acc, common.cuh, carried
          through d(1 - e^2) = -2 e de)
  dres    u (prod(xc, M124, 768) + 2 |dres|) about the reference formed with the folds as the workspace holds them: the
          folds' own rounding, xc . (M124 - M124_exact) + (E - E_exact), is computed exactly and enters the reference
          as it is, not bounded (the folds themselves are checked against float64 on their own); likewise dctx with Mctx
  heads   e_dh = e_in + u |dh|;  du: |(h - c) u (1 - u)| e_dh + 4 u |du|;  dc: |(1 - u)(1 - c^2)| e_dh + u (4 |dc| +
          2 |dh (1 - u)| c^2)  (1 - c*c cancels as |c| -> 1)
  dr      |h r (1 - r)| e_drh + 4 u |dr|, e_drh = u (prod(DC, Wc_h, 256) + |drh|)
  dIN     u (prod(DC, Wc_x, 256) + prod(DG, Wg_x, 512) + 2 |dIN|)   (the operand of the head below and of dz)
  carry   |u| e_dh + |r| e_drh + u (prod(DG, Wg_h, 512) + 3 |carry|)
  dz      e_dres + e_dIN + u |dz|;  dpn2, dpn1: ks u (prod + 2 |out|);  datt, dctx: u (prod + |out|)
  folds and the tail products (taco_gemm): tol sum |a||b| + u |out| per added product, tol = 2^-19 for the FFMA route
          and 2^-16 for 3xTF32 (the bars of tests/test_gpu_train_envelope.py)
Every bar but the folds' is C times that, C = C_PROD for the whole envelope, calibrated on the H100 (DESIGN.md 3.5):
these are root-mean-square estimates, and the largest of some 10^7 elements sits several of them out.  Every bar also
carries 2^-126 for results in the subnormal range (saturated gates make u (1 - u) tiny).

The first failing element in (t descending, stage, b, unit) order is where the fault sits: every later check reads the
faulty stored values.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import torch

U24 = 2.0 ** -24
C_PROD = 8.0                    # C of the bars (calibrated on the H100, DESIGN.md section 3.5)
FLUSH = 2.0 ** -126             # subnormal results: their spacing, and zero where the hardware flushes them
TANH_ERR = 5e-7                 # tanhf_acc, absolute (common.cuh)
ROUTE_TOL = {0: 2.0 ** -19, 1: 2.0 ** -16}     # taco_gemm: FFMA, 3xTF32 (tests/test_gpu_train_envelope.py)
UNITS, MF, RB = 256, 80, 32
# workspace layout of decoder_bwd.cu (floats)
WS_ZERO_END = RB * 768 + 3 * RB * UNITS + 6 * RB * UNITS + 32
WS_M124 = WS_ZERO_END
WS_M7 = WS_M124 + UNITS * 768
WS_E = WS_M7 + 640 * UNITS
WS_MAXT = 1024
WS_TOTAL = WS_E + WS_MAXT * RB * UNITS
STAGES = ("dscore", "dpq", "M124", "E", "du3", "dc3", "dr3", "du2", "dc2", "carry3", "dr2", "du1", "dc1", "carry2",
          "dr1", "dz", "carry1", "M7", "dpn2", "datt", "dctx", "dpn1", "dy", "dx")
FOLDS = ("M124", "M7")
OUTS = ("DATT", "DY", "DPQ", "DSCORE", "DCTX", "DZ", "DPN2", "DPN1", "DX")
TIME_MAJOR = ("dy_ext", "PQ", "PN1", "PN2", "sel")


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
    worst: dict                         # quantity -> worst |kernel - reference| / bar
    first: Failure | None
    ratio: dict = field(repr=False)     # quantity -> [T,B,N] (folds: the fold's shape)

    def __str__(self):
        w = ", ".join(f"{k} {v:.3f}" for k, v in self.worst.items())
        return f"worst ratio to the bar: {w}" + ("" if self.first is None else f"; {self.first}")


def rss(X, W):
    """sqrt(X^2 . W^2) over the last axis of X and the first of W"""
    return torch.sqrt((X * X) @ (W * W))


def prod(X, W, K):
    """the FFMA rounding of gemm_block's X . W (K terms, K/8 per warp chain), in units of u"""
    return math.sqrt(K / 16.0) * rss(X.abs(), W.abs())


def ws_folds(a):
    """(M124 [256,768], M7 [640,256], E [T,B,256]) as the call's workspace a['_ws'] holds them"""
    ws = a["_ws"]
    T, B = a["dy_ext"].shape[:2]
    return (ws[WS_M124:WS_M7].view(UNITS, 768), ws[WS_M7:WS_E].view(640, UNITS),
            ws[WS_E:WS_E + T * B * UNITS].view(T, B, UNITS))


def _slice_args(a, s):
    """the arguments of the kernel run on steps s .. T-1 alone, with H0 = H(s-1) and fresh outputs"""
    T, B, OUT = a["dy_ext"].shape
    Tx = a["align"].shape[2]
    n = T - s
    d = {k: v for k, v in a.items() if not k.startswith("_") and k not in OUTS and k not in ("DG", "DC", "DH0")}
    for k in TIME_MAJOR:
        d[k] = a[k][s:].contiguous()
    for k in ("RU", "C", "H"):
        d[k] = [x[s:].contiguous() for x in a[k]]
    d["align"] = a["align"][:, s:].contiguous()
    if a.get("dscore_add") is not None:
        d["dscore_add"] = a["dscore_add"][:, s:].contiguous()
    d["H0"] = [x[s - 1].contiguous() for x in a["H"]]
    e = lambda *shape: torch.full(shape, float("nan"), dtype=a["dy_ext"].dtype, device=a["dy_ext"].device)
    for k, w in (("DATT", UNITS), ("DY", OUT), ("DPQ", UNITS), ("DCTX", UNITS), ("DZ", UNITS), ("DPN2", 128),
                 ("DPN1", UNITS), ("DX", MF)):
        d[k] = e(n, B, w)
    d["DSCORE"] = e(B, n, Tx)
    d["DG"] = [e(n, B, 2 * UNITS) for _ in range(3)]
    d["DC"] = [e(n, B, UNITS) for _ in range(3)]
    d["DH0"] = e(3, B, UNITS)
    return d


def _bits(x):
    return x.contiguous().view(torch.int32) if x.dtype == torch.float32 else x.contiguous().view(torch.int64)


def suffix_mismatch(a, d, s):
    """outputs of the suffix run `d` (steps s ..) that differ in any bit from the full run's: a list of names"""
    bad = [k for k in OUTS if k != "DSCORE" and not torch.equal(_bits(a[k][s:]), _bits(d[k]))]
    if not torch.equal(_bits(a["DSCORE"][:, s:]), _bits(d["DSCORE"])):
        bad.append("DSCORE")
    for k in ("DG", "DC"):
        bad += [f"{k}{i}" for i in range(3) if not torch.equal(_bits(a[k][i][s:]), _bits(d[k][i]))]
    if "_ws" in a and "_ws" in d:
        if not torch.equal(_bits(ws_folds(a)[2][s:]), _bits(ws_folds(d)[2])):
            bad.append("E")
    return bad


def read_carries(run, a, steps, compose=True):
    """the carries into the steps `steps` (and into t - 1 for each): {t: [3,B,256]} for t in -1 .. T-1.  carry[T-1] = 0,
    carry[-1] = the full run's DH0 (when it asked for one), carry[s-1] = DH0 of `run` on the suffix s .. T-1.
    compose: every suffix output must equal the full run's bit for bit (a list of mismatches is returned)."""
    T, B = a["dy_ext"].shape[:2]
    z = torch.zeros(3, B, UNITS, dtype=a["dy_ext"].dtype, device=a["dy_ext"].device)
    carry = {T - 1: z}
    if a.get("DH0") is not None:
        carry[-1] = a["DH0"]
    need = sorted({x for t in steps for x in (t, t - 1) if 0 <= x < T - 1})
    mism = []
    for c in need:
        d = _slice_args(a, c + 1)
        run(d)
        carry[c] = d["DH0"].clone()
        if compose:
            bad = suffix_mismatch(a, d, c + 1)
            if bad:
                mism.append((c + 1, bad))
    return carry, mism


def check(a, carry, *, route=0, steps=None, c=C_PROD, exact_folds=False):
    """One decoder-backward run, checked step by step.  `a`: the call's arguments after the run (time-major, as
    kernels.decoder_bwd takes them, with the workspace in a['_ws'] unless exact_folds); carry: read_carries' dict; route:
    taco_gemm's implementation during the call (0 FFMA, 1 3xTF32); steps: the steps to check (default all; the stages
    that need a carry are checked where it is known).  Evaluated in float64 on a's device.  Returns a Report."""
    f = lambda x: None if x is None else x.double()
    dt = a["dy_ext"]
    dev = dt.device
    T, B, OUT = dt.shape
    Tx = a["align"].shape[2]
    lo = OUT - MF
    u = U24
    tol = ROUTE_TOL[route]
    steps = list(range(T)) if steps is None else sorted(set(steps))
    chk = torch.zeros(T, dtype=torch.bool, device=dev)
    chk[steps] = True
    W_a, W_q, W_out, W_in, W1, W2, v = (f(a[k]) for k in ("W_a", "W_q", "W_out", "W_in", "W1", "W2", "v"))
    Wg, Wc = [f(x) for x in a["Wg"]], [f(x) for x in a["Wc"]]
    ks = float(a["keep_scale"])
    dy_ext, PQ, PN1, PN2 = (f(a[k]) for k in ("dy_ext", "PQ", "PN1", "PN2"))
    sel = a["sel"].to(torch.float64)
    RU, Cc, H = [f(x) for x in a["RU"]], [f(x) for x in a["C"]], [f(x) for x in a["H"]]
    al = f(a["align"]).transpose(0, 1)                                           # [T,B,Tx]
    V, Kk = f(a["values"]), f(a["keys"])
    dsa = None if a.get("dscore_add") is None else f(a["dscore_add"]).transpose(0, 1)
    DATT, DPQ, DCTX, DZ, DPN2, DPN1, DY, DX = (f(a[k]) for k in ("DATT", "DPQ", "DCTX", "DZ", "DPN2", "DPN1", "DY", "DX"))
    DS = f(a["DSCORE"]).transpose(0, 1)
    DG, DC = [f(x) for x in a["DG"]], [f(x) for x in a["DC"]]
    H0 = a.get("H0")
    hprev = [torch.cat([(torch.zeros(1, B, UNITS, dtype=torch.float64, device=dev) if H0 is None else f(H0[i])[None]),
                        H[i][:-1]]) for i in range(3)]
    # ---- folds: exact, and as the kernel used them ----
    M124x = torch.cat([W_out @ W_a[:OUT], W_out @ W_q, W_out[:, lo:] @ W1], 1)  # [256,768]
    Mctx = W_a[OUT:] @ W_in[128:]
    Ex = dy_ext @ W_out.t()
    if exact_folds:
        M124p, Mctxp, Ep = M124x, Mctx, Ex
        M7p = torch.cat([W_in, Mctx])
    else:
        M124p, M7p, Ep = (x.double() for x in ws_folds(a))
        Mctxp = M7p[384:]
    A = lambda x: x.abs()
    ratio, ref, bar, got, size = {}, {}, {}, {}, {}

    def put(name, g, r, b):
        d = (g - r).abs()
        b = b + FLUSH
        ratio[name] = torch.where(d == 0, torch.zeros_like(d), d / b).nan_to_num(nan=math.inf)
        got[name], ref[name], bar[name], size[name] = g, r, b, b / (c * u)       # size: the bar in units of C u

    # folds on their own (route bars), and E per step
    M124b = tol * torch.cat([A(W_out) @ A(W_a[:OUT]), A(W_out) @ A(W_q), A(W_out[:, lo:]) @ A(W1)], 1) + u * A(M124x)
    put("M124", M124p, M124x, M124b)
    M7x = torch.cat([W_in, Mctx])
    M7b = torch.cat([torch.zeros_like(W_in), tol * (A(W_a[OUT:]) @ A(W_in[128:]))]) + u * A(M7x)
    put("M7", M7p, M7x, M7b)
    Eb = tol * (A(dy_ext) @ A(W_out).t()) + u * A(Ex)
    put("E", Ep, Ex, Eb)
    # ---- stage A: the attention of step t ----
    dal = torch.einsum("tbd,bjd->tbj", DCTX, V)
    e_dal = u * (math.sqrt(13 / 2) * torch.sqrt(torch.einsum("tbd,bjd->tbj", DCTX * DCTX, V * V)) + 5 * A(dal))
    tot = (al * dal).sum(-1, keepdim=True)
    dsr = al * (dal - tot)
    e_ds = (al * (e_dal + (al * e_dal).sum(-1, keepdim=True))
            + u * (math.sqrt(Tx / 2) * torch.sqrt((al * al * dal * dal).sum(-1, keepdim=True)) + A(dsr) + 2 * A(dsr)))
    if dsa is not None:
        dsr = dsr + dsa
        e_ds = e_ds + u * A(dsr)
    put("dscore", DS, dsr, c * e_ds)
    dpq = torch.empty(T, B, UNITS, dtype=torch.float64, device=dev)
    e_dpq = torch.empty_like(dpq)
    for t0 in range(0, T, 8):
        t1 = min(T, t0 + 8)
        th = torch.tanh(Kk[None] + PQ[t0:t1][:, :, None, :])                    # [tc,B,Tx,256]
        w = 1 - th * th
        ds = DS[t0:t1][..., None]
        dpq[t0:t1] = v * (ds * w).sum(2)
        e_dpq[t0:t1] = A(v) * (u * math.sqrt(Tx / 2) * torch.sqrt((ds * ds * w * w).sum(2))
                               + 2 * TANH_ERR * torch.sqrt((ds * ds * th * th).sum(2)))
        del th, w
    e_dpq = e_dpq + 2 * u * A(dpq)
    put("dpq", DPQ, dpq, c * e_dpq)
    # ---- stage 4': dres and GRU 3's head ----
    nxt = torch.zeros(T, B, UNITS, dtype=torch.float64, device=dev)
    nxt[:-1] = sel[1:, :, None] * DPN1[1:]
    xc = torch.cat([DATT, DPQ, nxt], -1)                                          # [T,B,768]
    dres = Ep + xc @ M124p.t()                                                    # with the folds as the kernel used them
    e_dres = c * u * (prod(xc, M124x.t(), 768) + 2 * A(dres))
    have = torch.zeros(T, dtype=torch.bool, device=dev)
    CR = torch.full((T, 3, B, UNITS), math.nan, dtype=torch.float64, device=dev)
    for t, x in carry.items():
        if t >= 0:
            CR[t], have[t] = x.double(), True
    CRo = torch.full_like(CR, math.nan)                                           # the carry out of step t (into t-1)
    have_o = torch.zeros(T, dtype=torch.bool, device=dev)
    for t in range(T):
        if (t - 1) in carry:
            CRo[t], have_o[t] = carry[t - 1].double(), True

    def head(i, din, e_in):
        """GRU layer i's head from the gradient `din` arriving at h_i(t) (error e_in) and the carry: (dh, e_dh)"""
        dh = din + CR[:, i]
        e_dh = e_in + c * u * A(dh)
        r_, uu, cc = RU[i][..., :UNITS], RU[i][..., UNITS:], Cc[i]
        gu = (hprev[i] - cc) * uu * (1 - uu)
        gc = (1 - uu) * (1 - cc * cc)
        du, dc = dh * gu, dh * gc
        put(f"du{i+1}", DG[i][..., UNITS:], du, A(gu) * e_dh + c * u * 4 * A(du))
        put(f"dc{i+1}", DC[i], dc, A(gc) * e_dh + c * u * (4 * A(dc) + 2 * A(dh * (1 - uu)) * cc * cc))
        return dh, e_dh

    dh, e_dh = head(2, dres, e_dres)
    for i in (2, 1, 0):
        Wc_x, Wc_h = Wc[i][:UNITS], Wc[i][UNITS:]
        Wg_x, Wg_h = Wg[i][:UNITS], Wg[i][UNITS:]
        r_, uu = RU[i][..., :UNITS], RU[i][..., UNITS:]
        drh = DC[i] @ Wc_h.t()
        e_drh = c * u * (prod(DC[i], Wc_h.t(), 256) + A(drh))
        g = hprev[i] * r_ * (1 - r_)
        dr = drh * g
        put(f"dr{i+1}", DG[i][..., :UNITS], dr, A(g) * e_drh + c * u * 4 * A(dr))
        din = DC[i] @ Wc_x.t() + DG[i] @ Wg_x.t()
        e_din = c * u * (prod(DC[i], Wc_x.t(), 256) + prod(DG[i], Wg_x.t(), 512) + 2 * A(din))
        co = dh * uu + drh * r_ + DG[i] @ Wg_h.t()
        e_co = A(uu) * e_dh + A(r_) * e_drh + c * u * (prod(DG[i], Wg_h.t(), 512) + 3 * A(co))
        put(f"carry{i+1}", CRo[:, i], co, e_co)
        if i > 0:
            dh, e_dh = head(i - 1, din, e_din)
        else:
            dz = dres + din
            e_dz = e_dres + e_din + c * u * A(dz)
            put("dz", DZ, dz, e_dz)
    # ---- stage 7' ----
    m2 = (PN2 > 0).double()
    dpn2 = m2 * ks * (DZ @ W_in[:128].t())
    e_dpn2 = c * u * m2 * ks * (prod(DZ, W_in[:128].t(), 256) + 2 * A(DZ @ W_in[:128].t()))
    put("dpn2", DPN2, dpn2, e_dpn2)
    nanrow = torch.full((1, B, UNITS), math.nan, dtype=torch.float64, device=dev)
    datt = DZ @ W_in[128:].t()
    e_datt = c * u * (prod(DZ, W_in[128:].t(), 256) + A(datt))
    put("datt", torch.cat([nanrow, DATT[:-1]]), datt, e_datt)
    dctx = DZ @ Mctxp.t()
    e_dctx = c * u * (prod(DZ, Mctx.t(), 256) + A(dctx))
    put("dctx", torch.cat([nanrow, DCTX[:-1]]), dctx, e_dctx)
    for k in ("datt", "dctx"):
        ratio[k][0] = 0                                                          # step 0 forms no DATT(-1), DCTX(-1)
    m1 = (PN1 > 0).double()
    p1 = DPN2 @ W2.t()
    e_dpn1 = c * u * m1 * ks * (prod(DPN2, W2.t(), 128) + 2 * A(p1))
    put("dpn1", DPN1, m1 * ks * p1, e_dpn1)
    # ---- after the kernel: taco_gemm products ----
    dxr = DPN1 @ W1.t()
    e_dx = c * (tol * (A(DPN1) @ A(W1).t()) + u * A(dxr))
    put("dx", DX, dxr, e_dx)
    dyr = dy_ext + DATT @ W_a[:OUT].t() + DPQ @ W_q.t()
    e_dy = tol * (A(DATT) @ A(W_a[:OUT]).t() + A(DPQ) @ A(W_q).t()) + u * (A(dy_ext) + 2 * A(dyr))
    tail = torch.zeros_like(dyr)
    tail[:-1, :, lo:] = sel[1:, :, None] * DX[1:]
    dyr = dyr + tail
    e_dy = c * (e_dy + u * A(dyr) * (tail != 0))
    put("dy", DY, dyr, e_dy)
    # ---- the steps checked, and where a carry was known ----
    need_in = {"du3", "dc3", "dr3", "du2", "dc2", "dr2", "du1", "dc1", "dr1", "dz", "carry3", "carry2", "carry1"}
    for k, r in ratio.items():
        if k in FOLDS:
            continue
        m = chk.clone()
        if k in need_in:
            m &= have
        if k.startswith("carry"):
            m &= have_o
        r[~m] = 0
    worst = {k: float(r.max()) if r.numel() else 0.0 for k, r in ratio.items()}
    first = None
    bad = {k: ~(r <= 1) for k, r in ratio.items()}
    if any(bool(b.any()) for b in bad.values()):
        last = {}
        for k, b in bad.items():
            if not b.any():
                continue
            if k in FOLDS:
                last[k] = T - 1
            else:
                last[k] = int(b.flatten(1).any(1).nonzero().max())
        t = max(last.values())
        k = next(s for s in STAGES if last.get(s) == t)
        if k in FOLDS:
            n = int(bad[k].flatten().nonzero()[0, 0])
            idx = divmod(n, bad[k].shape[1])
            first = Failure(t, k, -1, n, float(got[k][idx]), float(ref[k][idx]), float(bar[k][idx]), float(size[k][idx]))
        else:
            b, n = (int(x) for x in bad[k][t].nonzero()[0])
            first = Failure(t, k, b, n, float(got[k][t, b, n]), float(ref[k][t, b, n]), float(bar[k][t, b, n]),
                            float(size[k][t, b, n]))
    return Report(worst, first, ratio)


def make_args(r, B, Tx, T, *, seed=0, sched=True, lengths=None, speakers=0, ga=False, keep_scale=2.0, gate_scale=1.0,
              key_scale=1.0, device="cpu", dtype=torch.float32, P=None):
    """the arguments of one taco_decoder_bwd call (time-major, as kernels.decoder_bwd takes them) with outputs filled
    with NaN.  The saved activations are drawn in their ranges rather than from a forward run -- the check is local, so
    it needs the kernel's inputs, not a consistent history: r, u = sigmoid, c, h = tanh (of N(0, gate_scale^2): gate_scale
    large saturates them), alignments a softmax over the text, pre-net activations relu with about half of them zero.
    sched: sel from a random half of the rows (sel(0) = 0); speakers: H0 rows of a table that size; ga: dscore_add from
    the guided attention loss (tests/mirror_kernels_guided.py) at g = 0.2, lam = 10; key_scale scales keys and PQ."""
    from oracle import tacotron_oracle as O
    from tests import mirror_kernels_guided as MKG
    from tests.util import ocfg
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    if P is None:
        P = O.init_params(ocfg(r=r, T=T, vocab=20), seed=1, trained_like=True)
    OUT = 80 * r
    tl = (torch.randint(max(1, Tx // 2), Tx + 1, (B,), generator=g) if lengths is None else lengths).to(torch.int64)
    tl[0] = Tx
    live = torch.arange(Tx)[None, :] < tl[:, None]                                       # [B,Tx]
    values = rn(B, Tx, UNITS) * 0.5 * live[..., None]
    keys = values @ P["dec/attn/W_mem"].double() * key_scale * 8
    sc = torch.where(live[:, None, :], rn(B, T, Tx) * 2, torch.full((B, T, Tx), -math.inf, dtype=torch.float64))
    align = torch.softmax(sc, -1)
    RU = [torch.sigmoid(rn(T, B, 2 * UNITS) * 2 * gate_scale) for _ in range(3)]
    Cs = [torch.tanh(rn(T, B, UNITS) * gate_scale) for _ in range(3)]
    H = [torch.tanh(rn(T, B, UNITS) * gate_scale) for _ in range(3)]
    sel = (torch.rand(T, B, generator=g) < 0.5).to(torch.uint8) if sched else torch.zeros(T, B, dtype=torch.uint8)
    sel[0] = 0
    a = {"W_a": P["dec/attn/W_a"], "W_q": P["dec/attn/W_q"], "W_out": P["dec/out_proj/W"], "W_in": P["dec/in_proj/W"],
         "W1": P["dec/prenet/W1"], "W2": P["dec/prenet/W2"], "v": P["dec/attn/v"],
         "Wg": [P[f"dec/gru{i+1}/Wg"] for i in range(3)], "Wc": [P[f"dec/gru{i+1}/Wc"] for i in range(3)],
         "dy_ext": rn(T, B, OUT) * 0.01, "RU": RU, "C": Cs, "H": H, "align": align, "values": values, "keys": keys,
         "PQ": rn(T, B, UNITS) * key_scale, "PN1": torch.relu(rn(T, B, UNITS)), "PN2": torch.relu(rn(T, B, 128)),
         "sel": sel, "keep_scale": keep_scale, "text_length": tl.to(torch.int32)}
    if speakers:
        table = torch.tanh(rn(speakers, 3, UNITS))
        ids = torch.randint(0, speakers, (B,), generator=g)
        a["H0"] = [table[ids, i].contiguous() for i in range(3)]
        a["DH0"] = torch.empty(3, B, UNITS)
    if ga:
        steps = torch.randint(max(1, T // 2), T + 1, (B,), generator=g).to(torch.int32)
        dsa = torch.empty(B, T, Tx, dtype=torch.float64)
        MKG.guided_attention(dsa, torch.empty(1, dtype=torch.float64), align, tl.to(torch.int32), steps, 0.2, 10.0)
        a["dscore_add"] = dsa
    for k, w in (("DATT", UNITS), ("DY", OUT), ("DPQ", UNITS), ("DCTX", UNITS), ("DZ", UNITS), ("DPN2", 128),
                 ("DPN1", UNITS), ("DX", MF)):
        a[k] = torch.empty(T, B, w)
    a["DSCORE"] = torch.empty(B, T, Tx)
    a["DG"] = [torch.empty(T, B, 2 * UNITS) for _ in range(3)]
    a["DC"] = [torch.empty(T, B, UNITS) for _ in range(3)]
    if "DH0" not in a:
        a["DH0"] = torch.empty(3, B, UNITS)

    def cv(x):
        if isinstance(x, list):
            return [cv(y) for y in x]
        if not torch.is_tensor(x):
            return x
        if x.dtype.is_floating_point:
            x = x.to(torch.float32).to(dtype)             # the kernel's fp32 values, exactly, in `dtype`
        return x.to(device).contiguous()
    a = {k: cv(v) for k, v in a.items()}
    for k in OUTS:
        a[k].fill_(math.nan)
    for k in ("DG", "DC"):
        for x in a[k]:
            x.fill_(math.nan)
    a["DH0"].fill_(math.nan)
    return a
