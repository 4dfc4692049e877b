"""TEST INFRASTRUCTURE ONLY -- a torch-CPU restatement of the *training* kernel namespace
(tacotron_b200/kernels.py, i.e. the taco_*_bwd / taco_gemm / taco_adam entry points of include/taco_b200.h).

Two uses:
  * `-m "not gpu"`: tacotron_b200/models/grad.py (the hand-written backward orchestration) is run with this
    namespace on CPU tensors and compared with torch.autograd over the oracle -- that pins the HOST logic
    (what is multiplied with what, which rows are shifted, where gradients accumulate);
  * `-m gpu`: every CUDA training kernel is compared with the function of the same name here.
The product never imports this module (the only in-package implementation of the namespace is the CUDA
one, which raises if libtaco_b200.so is missing).

Semantics are stated in the docstrings; they ARE the specification of the CUDA kernels.
"""
from __future__ import annotations

import math

import torch

ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_TANH = 0, 1, 2, 3


def empty(shape, like, dtype=None):
    return torch.empty(shape, dtype=dtype or like.dtype, device=like.device)


def padded_rows(rows, cols, like):
    return torch.empty((rows, cols), dtype=like.dtype)


def zeros(shape, like, dtype=None):
    return torch.zeros(shape, dtype=dtype or like.dtype, device=like.device)


def _shift_rows(A, sh, period):
    """rows i -> A[i+sh] if i and i+sh lie in the same block of `period` rows (and inside A), else 0."""
    R = A.shape[0]
    period = period or R
    out = torch.zeros_like(A)
    idx = torch.arange(R, device=A.device)
    src = idx + sh
    ok = (src >= 0) & (src < R) & (torch.div(idx, period, rounding_mode="floor") == torch.div(src.clamp(0, R - 1), period, rounding_mode="floor"))
    out[idx[ok]] = A[src[ok]]
    return out


def gemm(C, A, B, *, ta=False, tb=False, beta=0.0, shift=0, period=0, taps=1, dshift=0, kper=0, b_tap_stride=0,
         batch=1, a_bstride=0, b_bstride=0, c_bstride=0, bshift=0):
    """C_z[M,N] = beta*C_z + sum_k opA_z[m,k] * opB_z[k,n]   for z in range(batch)   (fp32, exact products)

    C is the [M,N] view of batch 0; batch z lives c_bstride ELEMENTS further (same for A/B with a_/b_bstride).
    ta=False: A stored [M,K];  opA[m,k] = A[m + sh(k), k]   sh(k) = shift + z*bshift + (k // kper)*dshift (kper>0)
    ta=True : A stored [K,M];  opA[m,k] = A[k + sh, m]      sh = shift + z*bshift
              a shifted row outside its block of `period` stored rows (period=0: all rows one block) reads as 0.
    tb=False: B stored [K,N];  tb=True: B stored [N,K'] per K-segment: opB[(j,kk), n] = B[j*b_tap_stride + n*ldb + kk]
              (taps segments of kper columns; taps=1: plain [N,K]).
    """
    assert C.dim() == 2 and A.dim() == 2 and B.dim() == 2
    M, N = C.shape
    for z in range(batch):
        Cz = _offset_view(C, z * c_bstride)
        Az = _offset_view(A, z * a_bstride)
        Bz = _offset_view(B, z * b_bstride)
        sh0 = shift + z * bshift
        acc = torch.zeros(M, N, dtype=C.dtype, device=C.device)
        if ta:
            assert taps == 1
            Ash = _shift_rows(Az, sh0, period)                 # [K, M]
            Bm = Bz.t() if tb else Bz
            acc = Ash.t() @ Bm
        else:
            if taps == 1:
                Ash = _shift_rows(Az, sh0, period)
                Bm = Bz.t() if tb else Bz
                acc = Ash @ Bm
            else:
                assert tb and kper > 0 and Az.shape[1] == kper
                for j in range(taps):
                    Ash = _shift_rows(Az, sh0 + j * dshift, period)     # [M, kper]
                    Bj = _offset_view(Bz, j * b_tap_stride)              # [N, kper]
                    acc = acc + Ash @ Bj.t()
        if beta == 0.0:
            Cz.copy_(acc)
        else:
            Cz.mul_(beta).add_(acc)


def _offset_view(t, off):
    if off == 0:
        return t
    return torch.as_strided(t, t.shape, t.stride(), t.storage_offset() + off)


def conv_dx(dX, dZ, W, T, beta=0.0):
    """data gradient of tf.layers.conv1d('same') / dense (taps = 1):
    dX[b,s,c] = beta*dX + sum_j sum_n dZ[b, s - tap0 - j, n] * W[j,c,n],  tap0 = -((taps-1)//2), zero outside [0,T).
    dX [B*T,Cin], dZ [B*T,Cout] (2-D views, possibly strided), W [taps,Cin,Cout]."""
    taps, Cin, Cout = W.shape
    tap0 = -((taps - 1) // 2)
    gemm(dX, dZ, W.reshape(taps * Cin, Cout)[:Cin], tb=True, beta=beta, shift=-tap0, dshift=-1, kper=Cout, taps=taps,
         b_tap_stride=Cin * Cout, period=T)


def colsum(out, A, Bm=None, R=None, beta=1.0):
    """out[n] = beta*out[n] + sum_m A[m,n] * (Bm is None ? 1 : Bm[m,n] - (R is None ? 0 : R[m,n]))"""
    if Bm is None:
        s = A.sum(0)
    elif R is None:
        s = (A * Bm).sum(0)
    else:
        s = (A * (Bm - R)).sum(0)
    out.mul_(beta).add_(s)


def bias_act_(Cm, bias, act):
    """in place: C[m,n] = act(C[m,n] + bias[n])   (bias may be None)"""
    v = Cm if bias is None else Cm + bias
    if act == ACT_RELU:
        v = torch.relu(v)
    elif act == ACT_SIGMOID:
        v = torch.sigmoid(v)
    elif act == ACT_TANH:
        v = torch.tanh(v)
    Cm.copy_(v)


def mul_shift(out, X, Hm, shift, period):
    """out[m,n] = X[m,n] * H[m+shift, n]  (0 when the shifted row leaves its block of `period` rows)"""
    out.copy_(X * _shift_rows(Hm, shift, period))


def epi_bwd(dZ, dY, Y, relu, scale=None, shift=None, gain=1.0, R=None):
    """Backward of the taco_linear_fwd epilogue  y = (act(z) * scale + shift) * keep*gain (+ R):
         dZ = dY * gain * scale[n] * mask,  mask = 1 (no relu) or
              relu, no scale:  Y > 0              (Y = relu(z)*keep*gain: zero when dropped or dead)
              relu, scale   :  (Y - R - shift[n]) * scale[n] > 0
    dZ may alias dY."""
    g = dY * gain
    if scale is not None:
        g = g * scale
    if relu:
        if scale is None:
            mask = Y > 0
        else:
            base = Y if R is None else Y - R
            mask = (base - shift) * scale > 0
        g = g * mask.to(g.dtype)
    dZ.copy_(g)


def bn_param_grad(dgamma, dbeta, S1, S2, gamma, beta):
    """y = gamma*(a-mean)*rstd + beta  =>  dbeta += S1 = sum dY ;  dgamma += (S2 - beta*S1)/gamma,  S2 = sum dY*y"""
    dbeta.add_(S1)
    dgamma.add_((S2 - beta * S1) / gamma)


def maxpool_bwd(dX, dP, X):
    """X,dP,dX [B,T,C]; forward P[t] = max(X[t], X[t+1]) (t<T-1), P[T-1] = X[T-1]; ties go to X[t] (first)."""
    B, T, C = X.shape
    dX.zero_()
    if T == 1:
        dX.copy_(dP)
        return
    first = (X[:, :-1] >= X[:, 1:]).to(dP.dtype)
    dX[:, :-1] += dP[:, :-1] * first
    dX[:, 1:] += dP[:, :-1] * (1 - first)
    dX[:, -1] += dP[:, -1]


def highway_fwd(Y, Pm, X):
    """P [M,2U] = [h_pre | t_pre] (biases included);  Y = relu(h)*sigmoid(t) + X*(1-sigmoid(t))"""
    U = X.shape[1]
    Hh = torch.relu(Pm[:, :U])
    Tt = torch.sigmoid(Pm[:, U:])
    Y.copy_(Hh * Tt + X * (1 - Tt))


def highway_bwd(dP, dXd, dY, Pm, X):
    """dP [M,2U] = [dY*T*(h>0) | dY*(H-X)*T*(1-T)] ;  dXd = dY*(1-T)   (direct path only)"""
    U = X.shape[1]
    h = Pm[:, :U]
    Hh = torch.relu(h)
    Tt = torch.sigmoid(Pm[:, U:])
    dP[:, :U] = dY * Tt * (h > 0).to(dY.dtype)
    dP[:, U:] = dY * (Hh - X) * Tt * (1 - Tt)
    dXd.copy_(dY * (1 - Tt))


def l1_bwd(dA, A, Bt, beta=0.0):
    """dA = beta*dA + sign(A - B)   (d/dA sum|A-B|; 0 at equality)"""
    s = torch.sign(A - Bt)
    if beta == 0.0:
        dA.copy_(s)
    else:
        dA.mul_(beta).add_(s)


def scatter_add_rows(dTable, ids, dRows):
    """dTable[ids[m], :] += dRows[m, :]   (ids clamped to [0, V) like taco_gather_rows)"""
    V = dTable.shape[0]
    idx = ids.reshape(-1).to(torch.int64).clamp(0, V - 1)
    dTable.index_add_(0, idx, dRows.reshape(idx.numel(), -1))


def bigru_bwd(dxp, dOut, out, ACT, Wg_h_fw, Wc_h_fw, Wg_h_bw, Wc_h_bw):
    """Serial part of the bidirectional-GRU backward (hidden 128).
    out [B,T,256] forward output (fw|bw); ACT [B,T,768] activated gates in the xp layout
    (dir*384 + [r 0:128 | u 128:256 | c 256:384]); dOut [B,T,256]; dxp [B,T,768] <- pre-activation gradients."""
    B, T, _ = out.shape
    Hn = 128
    for d, (Wg, Wc) in enumerate(((Wg_h_fw, Wc_h_fw), (Wg_h_bw, Wc_h_bw))):
        carry = torch.zeros(B, Hn, dtype=out.dtype)
        order = range(T - 1, -1, -1) if d == 0 else range(T)
        for t in order:
            tp = t - 1 if d == 0 else t + 1
            hprev = out[:, tp, d * Hn:(d + 1) * Hn] if 0 <= tp < T else torch.zeros(B, Hn, dtype=out.dtype)
            a = ACT[:, t, d * 384:(d + 1) * 384]
            r, u, c = a[:, :Hn], a[:, Hn:2 * Hn], a[:, 2 * Hn:]
            dh = dOut[:, t, d * Hn:(d + 1) * Hn] + carry
            du_pre = dh * (hprev - c) * u * (1 - u)
            dc_pre = dh * (1 - u) * (1 - c * c)
            drh = dc_pre @ Wc.t()
            dr_pre = drh * hprev * r * (1 - r)
            carry = dh * u + drh * r + torch.cat([dr_pre, du_pre], -1) @ Wg.t()
            dxp[:, t, d * 384:(d + 1) * 384] = torch.cat([dr_pre, du_pre, dc_pre], -1)


def dec_inputs(Xin, sel, mel, y, sample_mask, r, sched):
    """Decoder step inputs (last of the r frames), time-major.  Xin [T,B,80], sel [T,B] uint8.
    x_0 = mel[:,0]; x_t = sched and sample_mask[t-1,b] ? y[:,t-1] : mel[:,t]; sel marks the sampled rows."""
    T, B, mf = Xin.shape
    lo = (r - 1) * mf
    for t in range(T):
        x = mel[:, t, lo:lo + mf].clone()
        s = torch.zeros(B, dtype=torch.bool, device=mel.device)
        if t > 0 and sched:
            s = sample_mask[t - 1].to(torch.bool)
            x = torch.where(s[:, None], y[:, t - 1, lo:lo + mf], x)
        Xin[t] = x
        sel[t] = s.to(torch.uint8)


def decoder_bwd(a):
    """Serial part of the attention-decoder backward.  `a` is a namespace/dict (see grad.decoder_bwd) with
    time-major saved activations and outputs; every output is the PRE-ACTIVATION gradient of its linear stage so
    that all weight gradients become batched GEMMs afterwards."""
    T, B, OUT = a["dy_ext"].shape
    U = 256
    mf = a["DX"].shape[2]
    lo = OUT - mf
    dt = a["dy_ext"].dtype
    z = lambda n: torch.zeros(B, n, dtype=dt)
    dattn = z(256)
    dh = [z(U), z(U), z(U)]
    dx_next = z(mf)
    W_a, W_q, W_out, W_in, W1, W2 = a["W_a"], a["W_q"], a["W_out"], a["W_in"], a["W1"], a["W2"]
    ks = a["keep_scale"]
    for t in range(T - 1, -1, -1):
        a["DATT"][t] = dattn
        t1 = dattn @ W_a.t()                                    # [B, OUT+256]
        dctx = t1[:, OUT:]
        a["DCTX"][t] = dctx
        al = a["align"][:, t]                                   # [B,Tx]
        dal = torch.einsum("bd,bjd->bj", dctx, a["values"])
        dscore = al * (dal - (al * dal).sum(-1, keepdim=True))
        a["DSCORE"][:, t] = dscore
        e = torch.tanh(a["keys"] + a["PQ"][t][:, None, :])
        dpq = (dscore[:, :, None] * a["v"] * (1 - e * e)).sum(1)
        a["DPQ"][t] = dpq
        dy = a["dy_ext"][t] + t1[:, :OUT] + dpq @ W_q.t()
        if t + 1 < T:
            s = a["sel"][t + 1].to(dt)[:, None]
            dy = dy.clone()
            dy[:, lo:] += s * dx_next
        a["DY"][t] = dy
        dres = dy @ W_out.t()
        dIN = dres                                               # gradient w.r.t. h3 from the residual/out-proj
        for i in (2, 1, 0):
            Hi = a["H"][i]
            hprev = Hi[t - 1] if t > 0 else z(U)
            r_, u_, c_ = a["RU"][i][t][:, :U], a["RU"][i][t][:, U:], a["C"][i][t]
            dhi = dIN + dh[i]
            du_pre = dhi * (hprev - c_) * u_ * (1 - u_)
            dc_pre = dhi * (1 - u_) * (1 - c_ * c_)
            a["DC"][i][t] = dc_pre
            t2 = dc_pre @ a["Wc"][i].t()                         # [B, 2U]: [dIN_c | drh]
            drh = t2[:, U:]
            dr_pre = drh * hprev * r_ * (1 - r_)
            dg = torch.cat([dr_pre, du_pre], -1)
            a["DG"][i][t] = dg
            t3 = dg @ a["Wg"][i].t()                             # [B, 2U]: [dIN_g | dh_g]
            dh[i] = dhi * u_ + drh * r_ + t3[:, U:]
            dIN = t2[:, :U] + t3[:, :U]
        dz = dres + dIN
        a["DZ"][t] = dz
        t4 = dz @ W_in.t()                                       # [B, 384]: [dpn2 | dattn(t-1)]
        dattn = t4[:, 128:]
        dpn2 = t4[:, :128] * ks * (a["PN2"][t] > 0).to(dt)
        a["DPN2"][t] = dpn2
        dpn1 = (dpn2 @ W2.t()) * ks * (a["PN1"][t] > 0).to(dt)
        a["DPN1"][t] = dpn1
        dx_next = dpn1 @ W1.t()
        a["DX"][t] = dx_next


def attn_bwd_post(dkeys, dv, DSCORE, keys, PQ, v):
    """dkeys[b,j,d] = sum_t DSCORE[b,t,j] * v[d] * (1 - e^2),  dv[d] += sum_{b,t,j} DSCORE[b,t,j] * e,
    e = tanh(keys[b,j,d] + PQ[t,b,d]).   PQ is time-major [T,B,256]."""
    B, T, Tx = DSCORE.shape
    dkeys.zero_()
    for t in range(T):
        e = torch.tanh(keys + PQ[t][:, None, :])
        ds = DSCORE[:, t][:, :, None]
        dkeys += ds * v * (1 - e * e)
        dv += (ds * e).sum((0, 1))


def sumsq(out, x):
    """out[0] = sum x^2 (accumulated in double)"""
    out[0] = (x.double() ** 2).sum().to(out.dtype)


def adam_step(p, g, m, v, lr_t, b1, b2, eps, clip, sumsq_t):
    """g *= clip / max(sqrt(sumsq), clip) (clip <= 0: no clipping, tacotron.py:179);  m,v,p <- TF Adam (oracle/tf12.py adam_tf) with lr_t precomputed."""
    gn = torch.sqrt(sumsq_t[0])
    scale = clip / torch.maximum(gn, torch.tensor(float(clip), dtype=gn.dtype)) if clip > 0 else torch.ones_like(gn)   # cap_grads <= 0: unclipped
    gc = g * scale
    m.mul_(b1).add_(gc * (1 - b1))
    v.mul_(b2).add_(gc * gc * (1 - b2))
    p.sub_(lr_t * m / (torch.sqrt(v) + eps))


def epi_fwd_keep_(X, keep, gain):
    """in place: X = keep ? X*gain : 0   (tf.layers.dropout with an explicit keep mask, SURVEY A.11)"""
    X.mul_(keep.to(X.dtype) * gain)


def mask_rows(dst, src, length):
    """dst[b,t,:] = t < length[b] ? src[b,t,:] : 0   (taco_mask_rows)"""
    B, T, _ = src.shape
    m = (torch.arange(T)[None, :] < length[:, None].to(torch.int64)).to(src.dtype)
    dst.copy_(src * m[:, :, None])


# ------------------------------------------------------------------------------------------------------------
# Griffin-Lim glue kernels (SURVEY 8(f) rank 1; audio.py:67-97).  FFTs are library calls (torch.fft); these are the
# fused steps between them.  n = frames, NB = 1 + n_fft/2 bins, L = hop*(n-1) samples.
# ------------------------------------------------------------------------------------------------------------
def _hann_padded(win_length, n_fft, dtype):
    n = torch.arange(win_length, dtype=torch.float64)
    w = 0.5 - 0.5 * torch.cos(2.0 * math.pi * n / win_length)
    out = torch.zeros(n_fft, dtype=torch.float64)
    lp = (n_fft - win_length) // 2
    out[lp:lp + win_length] = w
    return out.to(dtype)


def gl_init(full, mag, spec, phase_u, r, scale=None, shift=None):
    """reshape_frames(forward=False) (audio.py:30-35) + de-normalisation + exp + initial phase:
    frame f of block b4 = f // 4r holds spec[t = 4*b4 + (f % 4r) % 4,  c*F : (c+1)*F],  c = (f % 4r) // 4;
    mag = exp(v*scale + shift); full = mag * exp(2 pi i phase_u).   spec [B,T,F*r]; mag/phase_u [B,n,F]; full complex."""
    B, n, F = mag.shape
    f = torch.arange(n)
    b4, rem = f // (4 * r), f % (4 * r)
    c, tl = rem // 4, rem % 4
    t = 4 * b4 + tl
    cols = c[:, None] * F + torch.arange(F)[None, :]                         # [n, F]
    v = spec[:, t[:, None], cols]                                             # [B, n, F]
    if scale is not None:
        v = v * scale[cols] + shift[cols]
    m = torch.exp(v)
    mag.copy_(m)
    ang = 2.0 * math.pi * phase_u
    full.copy_(torch.complex(m * torch.cos(ang), m * torch.sin(ang)))


def gl_ola(y, fr, hop, win_length):
    """librosa.istft after the inverse FFT: y[s] = sum_t w[p - t*hop] fr[t, p - t*hop] / sum_t w^2[p - t*hop],
    p = s + n_fft/2 (centre trim), division only where the window sum exceeds tiny.  fr [B,n,n_fft] real, y [B,L]."""
    B, n, n_fft = fr.shape
    w = _hann_padded(win_length, n_fft, fr.dtype)
    tot = torch.zeros(B, n_fft + hop * (n - 1), dtype=fr.dtype)
    ss = torch.zeros(n_fft + hop * (n - 1), dtype=fr.dtype)
    for t in range(n):
        tot[:, t * hop:t * hop + n_fft] += fr[:, t] * w
        ss[t * hop:t * hop + n_fft] += w * w
    nz = ss > torch.finfo(fr.dtype).tiny
    tot[:, nz] = tot[:, nz] / ss[nz]
    y.copy_(tot[:, n_fft // 2:n_fft // 2 + y.shape[1]])


def gl_frame(frw, y, hop, win_length):
    """librosa.stft before the FFT: frw[t, j] = w[j] * ypad[t*hop + j], ypad = reflect-padded y by n_fft/2."""
    B, n, n_fft = frw.shape
    w = _hann_padded(win_length, n_fft, y.dtype)
    yp = torch.nn.functional.pad(y[:, None, :], (n_fft // 2, n_fft // 2), mode="reflect")[:, 0]
    for t in range(n):
        frw[:, t] = yp[:, t * hop:t * hop + n_fft] * w


def normalize_f16(out, x, mean, std):
    """out = f32( f16( f32( f16( f32(x) - f32(mean) ) ) / std ) )   (data_input.py:61-64 then :38-39)"""
    d = (x.float() - mean.float()).half()
    out.copy_((d.float() / std).half().float())


def rfft2048(X, x):
    """X = rfft(x) over the last axis (unnormalised)"""
    X.copy_(torch.fft.rfft(x, dim=-1))


def irfft2048(x, X):
    """x = irfft(X, n=2048) over the last axis"""
    x.copy_(torch.fft.irfft(X, n=2048, dim=-1))


def gl_phase(full, mag, rebuilt):
    """full = mag * exp(i angle(rebuilt))   (audio.py:84,87; angle(0) = 0)"""
    a = rebuilt.abs()
    unit = torch.where(a > 0, rebuilt / torch.where(a > 0, a, torch.ones_like(a)), torch.ones_like(rebuilt))
    full.copy_(unit * mag)
