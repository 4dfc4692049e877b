"""TEST INFRASTRUCTURE ONLY -- tests/mirror_kernels_spk.py plus the torch-CPU restatement of taco_decoder_bwd with an
initial GRU state (H0 / DH0, the speaker-conditioned decoder).  This module is the kernel namespace `K` that
tacotron_b200/models/grad.py runs over on CPU for such a model; the docstring is the specification of the kernel."""
from __future__ import annotations

import torch

from tests.mirror_kernels_spk import *        # noqa: F401,F403  (the multi-speaker namespace, unchanged)
from tests import mirror_kernels as _MK


def decoder_bwd(a):
    """tests/mirror_kernels.py::decoder_bwd, with a['H0'] (three [B,256] initial states h_i(-1), or absent / None = zero)
    as the h(t-1) of step 0, and a['DH0'] ([3,B,256], or absent / None) <- the GRU carries left after step 0 =
    d(loss)/d(h_i(-1))."""
    H0, DH0 = a.get("H0"), a.get("DH0")
    if H0 is None and DH0 is None:
        return _MK.decoder_bwd(a)
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
