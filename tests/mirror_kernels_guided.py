"""TEST INFRASTRUCTURE ONLY -- tests/mirror_kernels_spkdec.py plus the torch-CPU restatements of taco_guided_attention and
of taco_decoder_bwd with dscore_add (the guided attention loss).  This module is the kernel namespace `K` that
tacotron_b200/models/grad.py runs over on CPU for a model trained with Config.guided_attention > 0, with or without the
speaker-conditioned decoder; the docstrings are the specification of the kernels."""
from __future__ import annotations

import torch

from tests.mirror_kernels_spkdec import *      # noqa: F401,F403  (the speaker-conditioned decoder namespace, unchanged)
from tests import guided_attention_oracle as GA
from tests import mirror_kernels_spkdec as _SD


def guided_attention_partial_count(B, T):
    return B * T


def guided_attention(dscore, loss, align, text_length, speech_steps, g, lam, partial=None):
    """dscore [B,T,Tx] <- lam * align * (W - s) on the mask t < speech_steps[b], j < min(text_length[b], Tx), 0 elsewhere
    (s = sum_j align W of the row); loss [1] <- lam * sum align W, summed per row and then over the rows in float64.
    W as tests/guided_attention_oracle.py states it."""
    B, T, Tx = align.shape
    W, mask = GA.band(text_length, speech_steps, T, Tx, g, align.dtype)
    s = (align * W).sum(-1)
    dscore.copy_(torch.where(mask, lam * align * (W - s[..., None]), torch.zeros_like(align)))
    loss.copy_((lam * s.double().sum()).reshape(loss.shape).to(loss.dtype))


def decoder_bwd(a):
    """tests/mirror_kernels_spkdec.py::decoder_bwd (H0 / DH0 optional), with a['dscore_add'] ([B,T,Tx], or absent / None)
    added to the softmax backward's dscore of every step before it feeds dpq and DSCORE."""
    add = a.get("dscore_add")
    if add is None:
        return _SD.decoder_bwd(a)
    H0, DH0 = a.get("H0"), a.get("DH0")
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
        t1 = dattn @ W_a.t()
        dctx = t1[:, OUT:]
        a["DCTX"][t] = dctx
        al = a["align"][:, t]
        dal = torch.einsum("bd,bjd->bj", dctx, a["values"])
        dscore = al * (dal - (al * dal).sum(-1, keepdim=True)) + add[:, t]
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
        dIN = dres
        for i in (2, 1, 0):
            Hi = a["H"][i]
            hprev = Hi[t - 1] if t > 0 else (H0[i] if H0 is not None else z(U))
            r_, u_, c_ = a["RU"][i][t][:, :U], a["RU"][i][t][:, U:], a["C"][i][t]
            dhi = dIN + dh[i]
            du_pre = dhi * (hprev - c_) * u_ * (1 - u_)
            dc_pre = dhi * (1 - u_) * (1 - c_ * c_)
            a["DC"][i][t] = dc_pre
            t2 = dc_pre @ a["Wc"][i].t()
            drh = t2[:, U:]
            dr_pre = drh * hprev * r_ * (1 - r_)
            dg = torch.cat([dr_pre, du_pre], -1)
            a["DG"][i][t] = dg
            t3 = dg @ a["Wg"][i].t()
            dh[i] = dhi * u_ + drh * r_ + t3[:, U:]
            dIN = t2[:, :U] + t3[:, :U]
        dz = dres + dIN
        a["DZ"][t] = dz
        t4 = dz @ W_in.t()
        dattn = t4[:, 128:]
        dpn2 = t4[:, :128] * ks * (a["PN2"][t] > 0).to(dt)
        a["DPN2"][t] = dpn2
        dpn1 = (dpn2 @ W2.t()) * ks * (a["PN1"][t] > 0).to(dt)
        a["DPN1"][t] = dpn1
        dx_next = dpn1 @ W1.t()
        a["DX"][t] = dx_next
    if DH0 is not None:
        for i in range(3):
            DH0[i] = dh[i]
