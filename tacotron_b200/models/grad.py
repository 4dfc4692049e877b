"""Hand-written backward of the Tacotron hot path (reference: the graph that ``tf.gradients`` differentiates
for ``Tacotron.add_train_op``, models/tacotron.py:167-185, i.e. the reverse of models/tacotron.py:107-165 and
models/ops.py:27-132).

There is no autograd here: every function below is the reverse of one forward block, written against the
kernel namespace ``K`` (tacotron_b200/kernels.py = the taco_gemm / taco_*_bwd entry points of
include/taco_b200.h).  Arguments:

    K  kernel namespace (all arithmetic happens there)
    P  parameters   name -> tensor   (TF layouts, tacotron_b200/params.py)
    G  gradients    name -> tensor   (same shapes; ACCUMULATED into -- zero them before a step)
    S  saved forward activations  name -> tensor  (written by the train-mode forward, models/tacotron.py)

The only torch calls in this file are allocation, views and pure data movement (copy / transpose); the same
code therefore runs unchanged over tests/mirror_kernels.py on CPU tensors, which is how the host logic is pinned
against torch.autograd over the oracle (tests/test_grad_host.py).

Design notes (H100): all weight gradients and every data gradient outside the three recurrences are large
batched GEMMs (rows = B*T); the recurrences keep only the truly serial data-gradient chain in their
persistent kernels (taco_bigru_bwd: one CTA per (utterance, direction); taco_decoder_bwd: one cooperative
kernel for all T steps) and emit PRE-ACTIVATION gradients for every step so that their weight gradients become
batched GEMMs too.  Gates are not stored by the forward: they are recomputed in batch from the saved hidden
states (h(t-1) is a one-row shift of the saved output), which costs one forward-sized GEMM but no serial work.
"""
from __future__ import annotations

ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_TANH = 0, 1, 2, 3
BN_EPS = 1e-3


def _v2(t):
    """[..., C] -> [rows, C] view"""
    return t.reshape(-1, t.shape[-1])


# ------------------------------------------------------------------------------------------------------------
# dense / conv1d('same') backward
# ------------------------------------------------------------------------------------------------------------
def dense_bwd(K, dY, X, W, gW, gb=None, dX=None, beta_dx=0.0):
    """y = x.W + b (W [in,out]).  dY,X,dX are 2-D (possibly strided) views."""
    if dX is not None:
        K.conv_dx(dX, dY, W.reshape(1, W.shape[0], W.shape[1]), dY.shape[0], beta=beta_dx)
    K.gemm(gW, X, dY, ta=True, beta=1.0)
    if gb is not None:
        K.colsum(gb, dY)


def conv_bwd(K, dZ, X, W, gW, gb, T, dX=None, beta_dx=0.0):
    """tf.layers.conv1d('same') (SURVEY A.2): z[b,t,n] = sum_j sum_c x[b,t+tap0+j,c] W[j,c,n], tap0 = -((k-1)//2).
    dZ [B*T,Cout] (may be a strided column slice), X [B*T,Cin], W/gW [k,Cin,Cout]."""
    taps, Cin, Cout = W.shape
    tap0 = -((taps - 1) // 2)
    if dX is not None:     # dx[b,s,c] = sum_j sum_n dz[b, s-tap0-j, n] W[j,c,n]
        K.conv_dx(dX, dZ, W, T, beta=beta_dx)
    # dW[j,c,n] = sum_{b,t} x[b,t+tap0+j,c] dz[b,t,n]  -- one batch entry per tap
    K.gemm(gW.reshape(taps * Cin, Cout)[:Cin], X, dZ, ta=True, beta=1.0, shift=tap0, bshift=1, batch=taps,
           c_bstride=Cin * Cout, period=T)
    K.colsum(gb, dZ)


def bn_act_bwd(K, P, G, pre, dY, Y, relu, R=None, affine=None):
    """y = BN_inference(act(z)) (+R)  (SURVEY A.4: gamma*(a-mean)/sqrt(var+eps)+beta, moving stats constant).
    Returns dZ (in place over dY) after accumulating dgamma/dbeta.  `affine` = the (scale, shift) pair the forward
    used: the relu mask is recovered as (y - shift)*scale > 0, which is exact only with bit-identical scale/shift
    (a dead unit gives y == shift exactly because the forward computes fma(0, scale, shift))."""
    gamma, beta = P[f"{pre}/bn_gamma"], P[f"{pre}/bn_beta"]
    scale, shift = affine if affine is not None else S_affine(P, pre)
    N = dY.shape[1]
    S1 = K.zeros((N,), dY)
    S2 = K.zeros((N,), dY)
    K.colsum(S1, dY)
    K.colsum(S2, dY, Y, R)
    K.bn_param_grad(G[f"{pre}/bn_gamma"], G[f"{pre}/bn_beta"], S1, S2, gamma, beta)
    K.epi_bwd(dY, dY, Y, relu, scale=scale, shift=shift, R=R)
    return dY


def S_affine(P, pre):
    """Folded inference batch-norm affine (same expression as ops.bn_affine); recomputed per call (tiny)."""
    scale = P[f"{pre}/bn_gamma"] / (P[f"{pre}/bn_var"] + BN_EPS).sqrt()
    shift = P[f"{pre}/bn_beta"] - P[f"{pre}/bn_mean"] * scale
    return scale.contiguous(), shift.contiguous()


# ------------------------------------------------------------------------------------------------------------
# highway (models/ops.py:27-46)
# ------------------------------------------------------------------------------------------------------------
def highway_bwd(K, P, G, S, pre, tag, dY, x_outer=None, spk=None):
    """dY [M,128] -> gradient w.r.t. the layer input.  S[tag+'_in'] = input of the T/H denses (after the optional
    width-changing dense), S[tag+'_P'] = [h_pre | t_pre].  x_outer = input of the optional dense (ops.py:29-30).
    spk = (s_l [B,128], ds_l [B,128], T) for a speaker-conditioned layer (ops.py:101-107): its dense sees [x_outer | s_l],
    computed forward as x_outer.Wd[:128] + u, u = s_l.Wd[128:] + bd per utterance; ds_l is accumulated into."""
    X = _v2(S[f"{tag}_in"])
    Pm = _v2(S[f"{tag}_P"])
    M, U = X.shape
    dP = K.empty((M, 2 * U), dY)
    dX = K.empty((M, U), dY)
    K.highway_bwd(dP, dX, dY, Pm, X)
    dH, dT = dP[:, :U], dP[:, U:]
    K.gemm(dX, dH, P[f"{pre}/WH"], tb=True, beta=1.0)
    K.gemm(dX, dT, P[f"{pre}/WT"], tb=True, beta=1.0)
    K.gemm(G[f"{pre}/WH"], X, dH, ta=True, beta=1.0)
    K.gemm(G[f"{pre}/WT"], X, dT, ta=True, beta=1.0)
    K.colsum(G[f"{pre}/bH"], dH)
    K.colsum(G[f"{pre}/bT"], dT)
    if spk is not None:
        s_l, ds_l, T = spk
        Wd = P[f"{pre}/Wd"]
        Xo = _v2(x_outer)
        dXo = K.empty(Xo.shape, dY)
        dense_bwd(K, dX, Xo, Wd[:128], G[f"{pre}/Wd"][:128], dX=dXo)
        du = K.zeros((Xo.shape[0] // T, U), dY)
        K.colsum_seg(du, dX, T)                                  # du[b] = sum_t d(proj)[b,t]
        K.gemm(G[f"{pre}/Wd"][128:], s_l, du, ta=True, beta=1.0)
        K.colsum(G[f"{pre}/bd"], du)
        K.gemm(ds_l, du, Wd[128:], tb=True, beta=1.0)
        return dXo
    if f"{pre}/Wd" in P:
        Xo = _v2(x_outer)
        dXo = K.empty(Xo.shape, dY)
        dense_bwd(K, dX, Xo, P[f"{pre}/Wd"], G[f"{pre}/Wd"], G[f"{pre}/bd"], dX=dXo)
        return dXo
    return dX


# ------------------------------------------------------------------------------------------------------------
# bidirectional GRU (models/ops.py:118-128, SURVEY A.5)
# ------------------------------------------------------------------------------------------------------------
def bigru_bwd(K, P, G, S, p, dOut, dh0=None):
    """dOut [B,T,256] -> dHin [B*T,128].  When the forward started from an initial state S[p+'/h0'] [B,128] (both
    directions, ops.py:111-126), dh0 [B,2,128] receives d(loss)/d(initial state) per direction."""
    out, xp, hin = S[f"{p}/gru_out"], S[f"{p}/xp"], S[f"{p}/hw_out"]
    h0 = S.get(f"{p}/h0")
    B, T, _ = out.shape
    M = B * T
    out2, hin2 = _v2(out), _v2(hin)
    ACT = K.empty((M, 768), out)
    ACT.copy_(_v2(xp))                                   # x-side products + biases (data movement only)
    RH = K.empty((M, 256), out)
    ACT3, RH3 = ACT.view(B, T, 768), RH.view(B, T, 256)
    names = (f"{p}/gru_fw", f"{p}/gru_bw")
    for d, dn in enumerate(names):
        Wg, Wc = P[f"{dn}/Wg"], P[f"{dn}/Wc"]
        sh = -1 if d == 0 else 1                         # h(t-1) in processing order: previous row (fw) / next row (bw)
        first = 0 if d == 0 else T - 1                   # first processed step: its h(t-1) is the initial state
        Hd = out2[:, d * 128:(d + 1) * 128]
        g = ACT[:, d * 384:d * 384 + 256]
        c = ACT[:, d * 384 + 256:(d + 1) * 384]
        K.gemm(g, Hd, Wg[128:], beta=1.0, shift=sh, period=T)
        if h0 is not None:
            K.gemm(ACT3[:, first, d * 384:d * 384 + 256], h0, Wg[128:], beta=1.0)
        K.bias_act_(g, None, ACT_SIGMOID)
        RHd = RH[:, d * 128:(d + 1) * 128]
        K.mul_shift(RHd, g[:, :128], Hd, sh, T)
        if h0 is not None:
            K.mul_shift(RH3[:, first, d * 128:(d + 1) * 128], ACT3[:, first, d * 384:d * 384 + 128], h0, 0, 0)
        K.gemm(c, RHd, Wc[128:], beta=1.0)
        K.bias_act_(c, None, ACT_TANH)
    dxp = K.empty((M, 768), out)
    if h0 is None:
        K.bigru_bwd(dxp.view(B, T, 768), dOut, out, ACT.view(B, T, 768), P[f"{names[0]}/Wg"][128:], P[f"{names[0]}/Wc"][128:],
                    P[f"{names[1]}/Wg"][128:], P[f"{names[1]}/Wc"][128:])
    else:
        K.bigru_bwd_h0(dxp.view(B, T, 768), dOut, out, ACT.view(B, T, 768), P[f"{names[0]}/Wg"][128:], P[f"{names[0]}/Wc"][128:],
                       P[f"{names[1]}/Wg"][128:], P[f"{names[1]}/Wc"][128:], h0, h0, dh0)
    if "_capture" in S:
        S["_capture"][f"{p}/bigru_bwd"] = {"dxp": dxp.view(B, T, 768), "dOut": dOut, "out": out, "ACT": ACT.view(B, T, 768)}
    dHin = K.empty((M, 128), out)
    for d, dn in enumerate(names):
        Wg, Wc = P[f"{dn}/Wg"], P[f"{dn}/Wc"]
        sh = -1 if d == 0 else 1
        Hd = out2[:, d * 128:(d + 1) * 128]
        RHd = RH[:, d * 128:(d + 1) * 128]
        dg = dxp[:, d * 384:d * 384 + 256]
        dc = dxp[:, d * 384 + 256:(d + 1) * 384]
        K.gemm(dHin, dg, Wg[:128], tb=True, beta=0.0 if d == 0 else 1.0)
        K.gemm(dHin, dc, Wc[:128], tb=True, beta=1.0)
        K.gemm(G[f"{dn}/Wg"][:128], hin2, dg, ta=True, beta=1.0)
        K.gemm(G[f"{dn}/Wg"][128:], Hd, dg, ta=True, beta=1.0, shift=sh, period=T)
        if h0 is not None:
            first = 0 if d == 0 else T - 1
            K.gemm(G[f"{dn}/Wg"][128:], h0, dxp.view(B, T, 768)[:, first, d * 384:d * 384 + 256], ta=True, beta=1.0)
        K.gemm(G[f"{dn}/Wc"][:128], hin2, dc, ta=True, beta=1.0)
        K.gemm(G[f"{dn}/Wc"][128:], RHd, dc, ta=True, beta=1.0)
        K.colsum(G[f"{dn}/bg"], dg)
        K.colsum(G[f"{dn}/bc"], dc)
    return dHin


# ------------------------------------------------------------------------------------------------------------
# CBHG (models/ops.py:48-132)
# ------------------------------------------------------------------------------------------------------------
def cbhg_bwd(K, P, G, S, p, dOut, Kb, c, n_hw=4):
    """dOut [B,T,256] -> d(input) [B*T,Cin]."""
    x_in = S[f"{p}/x_in"]
    B, T, Cin = x_in.shape
    X = _v2(x_in)
    M = B * T
    Sv = S.get(f"{p}/spk_s")                                                  # speaker-conditioned CBHG (ops.py:101-115)
    dh0 = K.empty((B, 2, 128), dOut) if Sv is not None else None
    dH = bigru_bwd(K, P, G, S, p, dOut, dh0=dh0)                              # [M,128]
    dSv = K.zeros(Sv.shape, dOut) if Sv is not None else None
    for l in range(n_hw - 1, -1, -1):
        if Sv is not None:
            spk = (Sv[:, 128 * l:128 * (l + 1)], dSv[:, 128 * l:128 * (l + 1)], T)
            dH = highway_bwd(K, P, G, S, f"{p}/highway{l}", f"{p}/hw{l}", dH, x_outer=S[f"{p}/hw{l}_x"], spk=spk)
        else:
            dH = highway_bwd(K, P, G, S, f"{p}/highway{l}", f"{p}/hw{l}", dH, x_outer=S[f"{p}/res"])
    if Sv is not None:
        speaker_bwd(K, P, G, S, p, dSv, dh0, n_hw)
    dRes = dH                                                                  # [M,Cin]  (res = proj2_bn + x_in)
    dIn = K.empty((M, Cin), dRes)
    dIn.copy_(dRes)                                                            # residual branch (ops.py:92)
    # proj2: BN(conv3(proj1)) -- no activation, residual added after
    bn_act_bwd(K, P, G, f"{p}/proj2", dRes, _v2(S[f"{p}/res"]), relu=False, R=X, affine=S.get(f"{p}/proj2/bn_affine"))
    P1 = _v2(S[f"{p}/proj1"])
    dP1 = K.empty(P1.shape, dRes)
    conv_bwd(K, dRes, P1, P[f"{p}/proj2/W"], G[f"{p}/proj2/W"], G[f"{p}/proj2/b"], T, dX=dP1)
    # proj1: BN(relu(conv3(bank_pool)))
    bn_act_bwd(K, P, G, f"{p}/proj1", dP1, P1, relu=True, affine=S.get(f"{p}/proj1/bn_affine"))
    pool = _v2(S[f"{p}/bank_pool"])
    dPool = K.empty(pool.shape, dRes)
    conv_bwd(K, dP1, pool, P[f"{p}/proj1/W"], G[f"{p}/proj1/W"], G[f"{p}/proj1/b"], T, dX=dPool)
    # max-pool(2,1,same) then BN(relu(bank convs))
    bank_bn = S[f"{p}/bank_bn"]
    dBank = K.empty(pool.shape, dRes)
    K.maxpool_bwd(dBank.view(B, T, -1), dPool.view(B, T, -1), bank_bn)
    bn_act_bwd(K, P, G, f"{p}/bank", dBank, _v2(bank_bn), relu=True, affine=S.get(f"{p}/bank/bn_affine"))
    co = c[0]
    for k in range(1, Kb + 1):
        conv_bwd(K, dBank[:, (k - 1) * co:k * co], X, P[f"{p}/bank/W{k}"], G[f"{p}/bank/W{k}"], G[f"{p}/bank/b{k}"], T,
                 dX=dIn, beta_dx=1.0)
    return dIn


def speaker_bwd(K, P, G, S, p, dSv, dh0, n_hw):
    """Reverse of ops._speaker_terms: S = relu(e.[Ws_0 .. Ws_{n-1} | Ws_init] + bs), e = speaker table rows of
    S['speaker'].  dSv [B,128*(n_hw+1)] holds the highway layers' ds_l; the initial-state block gets dh0_fw + dh0_bw."""
    Sv, e = S[f"{p}/spk_s"], S[f"{p}/spk_e"]
    B = Sv.shape[0]
    K.colsum_seg(dSv[:, 128 * n_hw:], dh0.view(2 * B, 128), 2)                # both directions start from the same state
    K.epi_bwd(dSv, dSv, Sv, True)                                              # relu
    de = K.empty(e.shape, e)
    names = [f"highway{l}" for l in range(n_hw)] + ["gru_init"]
    for i, nm in enumerate(names):
        blk = dSv[:, 128 * i:128 * (i + 1)]
        K.gemm(G[f"{p}/{nm}/Ws"], e, blk, ta=True, beta=1.0)
        K.colsum(G[f"{p}/{nm}/bs"], blk)
        K.gemm(de, blk, P[f"{p}/{nm}/Ws"], tb=True, beta=0.0 if i == 0 else 1.0)
    K.scatter_add_rows(G["speaker/embed"], S["speaker"], de)


# ------------------------------------------------------------------------------------------------------------
# pre-net on the embedding table (models/tacotron.py:38-44, :111-114)
# ------------------------------------------------------------------------------------------------------------
def enc_prenet_bwd(K, P, G, S, dL2, keep_scale):
    """dL2 [B*Tx,128] -> embedding / pre-net gradients.  Forward (ops.pre_net with ids): t1 = relu(table.W1+b1)
    on the V table rows, l1 = gather(t1, ids)*keep1*ks, l2 = relu(l1.W2+b2)*keep2*ks."""
    l1, l2, t1, ids = _v2(S["enc/prenet/l1"]), _v2(S["enc/prenet/l2"]), S["enc/prenet/t1"], S["text"]
    table = P["embedding"]
    K.epi_bwd(dL2, dL2, l2, True, gain=keep_scale)
    dL1 = K.empty(l1.shape, dL2)
    dense_bwd(K, dL2, l1, P["enc/prenet/W2"], G["enc/prenet/W2"], G["enc/prenet/b2"], dX=dL1)
    # through dropout+gather: d t1[v] = sum over rows with id v of dL1 * ks * [l1 > 0 or kept]; l1 > 0 <=> kept and t1 > 0
    K.epi_bwd(dL1, dL1, l1, True, gain=keep_scale)
    dT1 = K.zeros(t1.shape, dL2)
    K.scatter_add_rows(dT1, ids, dL1)
    # rows of t1 that are relu-dead got mask 0 above already (l1 = 0 there), so dT1 is the pre-activation gradient
    dense_bwd(K, dT1, table, P["enc/prenet/W1"], G["enc/prenet/W1"], G["enc/prenet/b1"], dX=G["embedding"], beta_dx=1.0)


# ------------------------------------------------------------------------------------------------------------
# attention decoder (models/tacotron.py:46-105, 136-138)
# ------------------------------------------------------------------------------------------------------------
def decoder_recompute(K, P, S, cfg):
    """Batched recomputation (time-major, rows = t*B + b) of every decoder activation the backward needs, from the
    tensors the forward kernel saved: y, alignments, the three GRU state sequences.  Returns a dict."""
    y, align, Hs = S["dec/y"], S["dec/align"], S["dec/H"]
    values = S["dec/values"]
    B, T, OUT = y.shape
    Tx = align.shape[2]
    mf, r = cfg.mel_features, cfg.r
    U = 256
    M = T * B
    ks = 1.0 / (1.0 - cfg.audio_dropout_prob)
    R = {"T": T, "B": B, "OUT": OUT, "ks": ks}
    Ytm = y.transpose(0, 1).contiguous()                                      # [T,B,OUT]  (data movement)
    R["Ytm"] = Ytm
    # step inputs and pre-net (tacotron.py:64-71, :38-44)
    Xin = K.empty((T, B, mf), y)
    sel = K.empty((T, B), y, dtype=S["dec/keep1"].dtype)
    K.dec_inputs(Xin, sel, S["mel"], y, S.get("dec/sample_mask"), r, S.get("dec/sample_mask") is not None)
    R["Xin"], R["sel"] = Xin, sel
    PN1 = K.empty((M, 256), y)
    K.gemm(PN1, _v2(Xin), P["dec/prenet/W1"])
    K.bias_act_(PN1, P["dec/prenet/b1"], ACT_RELU)
    K.epi_fwd_keep_(PN1, _v2(S["dec/keep1"]), ks)
    PN2 = K.empty((M, 128), y)
    K.gemm(PN2, PN1, P["dec/prenet/W2"])
    K.bias_act_(PN2, P["dec/prenet/b2"], ACT_RELU)
    K.epi_fwd_keep_(PN2, _v2(S["dec/keep2"]), ks)
    R["PN1"], R["PN2"] = PN1, PN2
    # context and attention vector (AttentionWrapper, A.6): ctx = align . values ; attn = [y, ctx] . W_a
    CTXbm = K.empty((B, T, 256), y)
    K.gemm(CTXbm[0], align[0], values[0], batch=B, a_bstride=T * Tx, b_bstride=Tx * 256, c_bstride=T * 256)
    CTX = CTXbm.transpose(0, 1).contiguous()                                  # [T,B,256]
    R["CTX"] = CTX
    W_a = P["dec/attn/W_a"]
    ATT = K.empty((M, 256), y)
    K.gemm(ATT, _v2(Ytm), W_a[:OUT])
    K.gemm(ATT, _v2(CTX), W_a[OUT:], beta=1.0)
    R["ATT"] = ATT
    # InputProjectionWrapper: z(t) = [pn2(t), attn(t-1)] . W_in + b_in
    W_in = P["dec/in_proj/W"]
    h0, att0 = S.get("dec/h0"), S.get("dec/att0")                              # speaker-conditioned decoder: h_i(-1), a(-1)
    R["h0"], R["att0"] = h0, att0
    Z = K.empty((M, U), y)
    K.gemm(Z, PN2, W_in[:128])
    K.gemm(Z, ATT, W_in[128:], beta=1.0, shift=-B)
    if att0 is not None:                                                       # step 0 rows: a(-1) instead of zero
        K.gemm(Z[:B], att0, W_in[128:], beta=1.0)
    K.bias_act_(Z, P["dec/in_proj/b"], ACT_NONE)
    R["Z"] = Z
    # the three GRU layers: gates from the saved state sequences
    R["RU"], R["C"], R["RH"], R["IN"], R["H"] = [], [], [], [], []
    inp = Z
    for i in range(3):
        Wg, Wc = P[f"dec/gru{i+1}/Wg"], P[f"dec/gru{i+1}/Wc"]
        Hi = _v2(Hs[i])                                                       # [M,U]
        RU = K.empty((M, 2 * U), y)
        K.gemm(RU, inp, Wg[:U])
        K.gemm(RU, Hi, Wg[U:], beta=1.0, shift=-B)
        if h0 is not None:                                                     # step 0 rows: h_i(-1) instead of zero
            K.gemm(RU[:B], h0[i], Wg[U:], beta=1.0)
        K.bias_act_(RU, P[f"dec/gru{i+1}/bg"], ACT_SIGMOID)
        RHm = K.empty((M, U), y)
        K.mul_shift(RHm, RU[:, :U], Hi, -B, 0)
        if h0 is not None:
            K.mul_shift(RHm[:B], RU[:B, :U], h0[i], 0, 0)
        Cc = K.empty((M, U), y)
        K.gemm(Cc, inp, Wc[:U])
        K.gemm(Cc, RHm, Wc[U:], beta=1.0)
        K.bias_act_(Cc, P[f"dec/gru{i+1}/bc"], ACT_TANH)
        R["RU"].append(RU); R["C"].append(Cc); R["RH"].append(RHm); R["IN"].append(inp); R["H"].append(Hi)
        inp = Hi
    PQ = K.empty((M, 256), y)
    K.gemm(PQ, _v2(Ytm), P["dec/attn/W_q"])
    R["PQ"] = PQ
    return R


def decoder_bwd(K, P, G, S, cfg, dY_ext):
    """dY_ext [B,T,80r] = gradient arriving at seq2seq_output (loss + post-net).  Returns dEncoded [B,Tx,256]."""
    R = decoder_recompute(K, P, S, cfg)
    T, B, OUT, ks = R["T"], R["B"], R["OUT"], R["ks"]
    U = 256
    M = T * B
    align, values, keys = S["dec/align"], S["dec/values"], S["dec/keys"]
    Tx = align.shape[2]
    like = dY_ext
    mf = cfg.mel_features
    tm = lambda n: K.empty((T, B, n), like)
    a = {
        "dy_ext": dY_ext.transpose(0, 1).contiguous(),
        "W_a": P["dec/attn/W_a"], "W_q": P["dec/attn/W_q"], "W_out": P["dec/out_proj/W"], "W_in": P["dec/in_proj/W"],
        "W1": P["dec/prenet/W1"], "W2": P["dec/prenet/W2"], "v": P["dec/attn/v"],
        "Wg": [P[f"dec/gru{i+1}/Wg"] for i in range(3)], "Wc": [P[f"dec/gru{i+1}/Wc"] for i in range(3)],
        "RU": [x.view(T, B, 2 * U) for x in R["RU"]], "C": [x.view(T, B, U) for x in R["C"]],
        "H": [x.view(T, B, U) for x in R["H"]],
        "align": align, "values": values, "keys": keys, "PQ": R["PQ"].view(T, B, 256),
        "PN1": R["PN1"].view(T, B, 256), "PN2": R["PN2"].view(T, B, 128), "sel": R["sel"], "keep_scale": ks,
        "text_length": S["text_length"],
        "DATT": tm(256), "DY": tm(OUT), "DPQ": tm(256), "DSCORE": K.empty((B, T, Tx), like), "DCTX": tm(256),
        "DG": [tm(2 * U) for _ in range(3)], "DC": [tm(U) for _ in range(3)], "DZ": tm(U), "DPN2": tm(128), "DPN1": tm(256),
        "DX": tm(mf), "max_ctas": getattr(cfg, "max_ctas", None),
    }
    h0, att0 = R["h0"], R["att0"]
    if h0 is not None:
        a["H0"] = [h0[i] for i in range(3)]
        a["DH0"] = K.empty((3, B, U), like)
    if S.get("dec/dscore_ga") is not None:                # guided attention loss: its d(loss)/d(score), added to the
        a["dscore_add"] = S["dec/dscore_ga"]              # softmax backward's dscore of every step
    K.decoder_bwd(a)
    if "_capture" in S:                                   # tests: expose the serial kernel's arguments and outputs
        S["_capture"]["decoder_bwd"] = a
    DATT, DY, DPQ, DZ =_v2(a["DATT"]), _v2(a["DY"]), _v2(a["DPQ"]), _v2(a["DZ"])
    Ytm2, CTX2 = _v2(R["Ytm"]), _v2(R["CTX"])
    # attention layer / query layer / output projection
    K.gemm(G["dec/attn/W_a"][:OUT], Ytm2, DATT, ta=True, beta=1.0)
    K.gemm(G["dec/attn/W_a"][OUT:], CTX2, DATT, ta=True, beta=1.0)
    K.gemm(G["dec/attn/W_q"], Ytm2, DPQ, ta=True, beta=1.0)
    K.gemm(G["dec/out_proj/W"], R["Z"], DY, ta=True, beta=1.0)                 # res = z + h3 (ResidualWrapper)
    K.gemm(G["dec/out_proj/W"], R["H"][2], DY, ta=True, beta=1.0)
    K.colsum(G["dec/out_proj/b"], DY)
    for i in range(3):
        DG, DC = _v2(a["DG"][i]), _v2(a["DC"][i])
        n = f"dec/gru{i+1}"
        K.gemm(G[f"{n}/Wg"][:U], R["IN"][i], DG, ta=True, beta=1.0)
        K.gemm(G[f"{n}/Wg"][U:], R["H"][i], DG, ta=True, beta=1.0, shift=-B)
        K.gemm(G[f"{n}/Wc"][:U], R["IN"][i], DC, ta=True, beta=1.0)
        K.gemm(G[f"{n}/Wc"][U:], R["RH"][i], DC, ta=True, beta=1.0)
        K.colsum(G[f"{n}/bg"], DG)
        K.colsum(G[f"{n}/bc"], DC)
    K.gemm(G["dec/in_proj/W"][:128], R["PN2"], DZ, ta=True, beta=1.0)
    K.gemm(G["dec/in_proj/W"][128:], R["ATT"], DZ, ta=True, beta=1.0, shift=-B)
    K.colsum(G["dec/in_proj/b"], DZ)
    if h0 is not None:                                                         # step-0 products of the initial state
        for i in range(3):
            K.gemm(G[f"dec/gru{i+1}/Wg"][U:], h0[i], _v2(a["DG"][i])[:B], ta=True, beta=1.0)
        K.gemm(G["dec/in_proj/W"][128:], att0, DZ[:B], ta=True, beta=1.0)
        decoder_speaker_bwd(K, P, G, S, DZ[:B], a["DH0"])
    DPN2, DPN1 = _v2(a["DPN2"]), _v2(a["DPN1"])
    K.gemm(G["dec/prenet/W2"], R["PN1"], DPN2, ta=True, beta=1.0)
    K.colsum(G["dec/prenet/b2"], DPN2)
    K.gemm(G["dec/prenet/W1"], _v2(R["Xin"]), DPN1, ta=True, beta=1.0)
    K.colsum(G["dec/prenet/b1"], DPN1)
    # memory: keys = values . W_mem ; values = encoded * length mask
    dkeys = K.empty((B, Tx, 256), like)
    K.attn_bwd_post(dkeys, G["dec/attn/v"], a["DSCORE"], keys, a["PQ"], P["dec/attn/v"])
    dvalues = K.empty((B, Tx, 256), like)
    # dvalues[b] = align[b]^T . DCTX[:, b]   (DCTX is time-major: row stride B*256, batch stride 256)
    K.gemm(dvalues[0], align[0], a["DCTX"][:, 0], ta=True, batch=B, a_bstride=T * Tx, b_bstride=256, c_bstride=Tx * 256)
    dk2, dv2 = _v2(dkeys), _v2(dvalues)
    K.gemm(dv2, dk2, P["dec/attn/W_mem"], tb=True, beta=1.0)
    K.gemm(G["dec/attn/W_mem"], _v2(values), dk2, ta=True, beta=1.0)
    dEnc = K.empty((B, Tx, 256), like)
    K.mask_rows(dEnc, dvalues, S["text_length"])
    return dEnc


def decoder_speaker_bwd(K, P, G, S, DZ0, DH0):
    """Reverse of ops.decoder_speaker_state: S = e.[Wa | Wh1 | Wh2 | Wh3] + b, relu on the three state blocks, e = speaker
    table rows of S['speaker'].  DZ0 [B,256] = d(loss)/d(z(0)), DH0 [3,B,256] = d(loss)/d(h_i(-1)) (taco_decoder_bwd)."""
    Sv, e = S["dec/spk_s"], S["dec/spk_e"]
    B = Sv.shape[0]
    W_in = P["dec/in_proj/W"]
    dSv = K.empty(Sv.shape, Sv)
    K.gemm(dSv[:, :256], DZ0, W_in[128:], tb=True)                             # d a(-1) = dz(0) . W_in[128:]^T
    dSv[:, 256:].view(B, 3, 256).copy_(DH0.transpose(0, 1))                     # (data movement)
    K.epi_bwd(dSv[:, 256:], dSv[:, 256:], Sv[:, 256:], True)                   # relu of the state blocks
    de = K.empty(e.shape, e)
    for i, nm in enumerate(("attn", "h1", "h2", "h3")):
        blk = dSv[:, 256 * i:256 * (i + 1)]
        K.gemm(G[f"dec/spk/{nm}/W"], e, blk, ta=True, beta=1.0)
        K.colsum(G[f"dec/spk/{nm}/b"], blk)
        K.gemm(de, blk, P[f"dec/spk/{nm}/W"], tb=True, beta=0.0 if i == 0 else 1.0)
    K.scatter_add_rows(G["speaker/embed"], S["speaker"], de)


# ------------------------------------------------------------------------------------------------------------
# whole model: reverse of Tacotron.inference + add_loss_op (models/tacotron.py:107-165)
# ------------------------------------------------------------------------------------------------------------
def model_bwd(K, P, G, S, cfg):
    """Accumulates d(loss)/d(param) into G for loss = sum|seq2seq_output - mel| + sum|output - stft|, plus the guided
    attention loss when S['dec/dscore_ga'] holds its gradient with respect to the attention scores."""
    y, out = S["dec/y"], S["post/out"]
    B, T, OUT = y.shape
    mf, r = cfg.mel_features, cfg.r
    F = cfg.fft_size
    post = _v2(S["post/cbhg/gru_out"])                                         # [B*T*r, 256]
    out2 = out.reshape(-1, F)
    dOut = K.padded_rows(out2.shape[0], F, y)           # 1025 columns in a 1028-float pitch: TMA-readable by the dX / dW kernels
    K.l1_bwd(dOut, out2, S["stft"].reshape(-1, F))
    dPost = K.empty(post.shape, y)
    dense_bwd(K, dOut, post, P["post/dense/W"], G["post/dense/W"], G["post/dense/b"], dX=dPost)
    dPostIn = cbhg_bwd(K, P, G, S, "post/cbhg", dPost.view(B, T * r, 256), cfg_post_K(cfg), cfg_post_c(cfg))   # [B*T*r, 80]
    dY = dPostIn.view(B, T, OUT)
    K.l1_bwd(_v2(dY), _v2(y), _v2(S["mel"]), beta=1.0)
    dEnc = decoder_bwd(K, P, G, S, cfg, dY)
    dPre = cbhg_bwd(K, P, G, S, "enc/cbhg", dEnc, cfg_enc_K(cfg), cfg_enc_c(cfg))
    enc_prenet_bwd(K, P, G, S, dPre, 1.0 / (1.0 - cfg.char_dropout_prob))


def cfg_enc_K(cfg): return getattr(cfg, "enc_K", 16)
def cfg_enc_c(cfg): return getattr(cfg, "enc_c", (128, 128, 128))
def cfg_post_K(cfg): return getattr(cfg, "post_K", 8)
def cfg_post_c(cfg): return getattr(cfg, "post_c", (128, 256, 80))
