"""Host-side mirror of the reference's ``models/ops.py`` over the sm_90a C-ABI.

Same surface as the reference -- ``highway``, ``CBHG``, ``InferenceHelper`` (models/ops.py:5-132)
-- plus the north-star spellings ``pre_net``, ``conv1d_banks``, ``highwaynet``,
``attention_decoder``.  Tensors are fp32 CUDA ``torch.Tensor`` s in TF's NWC layout; every
arithmetic op is a call into ``libtaco_b200.so`` (tacotron_b200/_lib.py).  No CPU fallback.

TF-1 builds a graph inside ``tf.variable_scope`` s; here the equivalent is a ``Scope`` (a
ParamStore + name prefix) taken from the innermost ``variable_scope(...)`` context, so call
sites read like the reference:

    with variable_scope(store, 'enc'):
        encoded = CBHG(pre_out, None, K=16, c=[128,128,128], gru_units=128)
"""
from __future__ import annotations

import contextlib
import ctypes as C
import numbers

import torch

from .. import _lib as L
from ..params import BN_EPS

# ----------------------------------------------------------------------------------------------
# scopes + derived (kernel-layout) buffers
# ----------------------------------------------------------------------------------------------
_scope_stack = []


class Scope:
    def __init__(self, store, prefix=""):
        self.store = store
        self.prefix = prefix.strip("/")

    def name(self, n):
        return f"{self.prefix}/{n}" if self.prefix else n

    def p(self, n):
        return self.store[self.name(n)]

    def has(self, n):
        return self.name(n) in self.store

    def sub(self, n):
        return Scope(self.store, self.name(n))


@contextlib.contextmanager
def variable_scope(store_or_name, prefix=None):
    """``with variable_scope(store, 'enc'):`` or nested ``with variable_scope('cbhg'):``."""
    if prefix is None and isinstance(store_or_name, str):
        parent = current_scope()
        sc = parent.sub(store_or_name)
    else:
        sc = Scope(store_or_name, prefix or "")
    _scope_stack.append(sc)
    try:
        yield sc
    finally:
        _scope_stack.pop()


def current_scope():
    if not _scope_stack:
        raise RuntimeError("no variable_scope active: wrap the call in `with variable_scope(store, prefix):`")
    return _scope_stack[-1]


# ----------------------------------------------------------------------------------------------
# train-mode activation saving: inside `with saving(S):` every op records the tensors the hand-written
# backward (models/grad.py) needs, under the names grad.py reads, and uses the un-fused variants whose
# intermediates must exist in memory (bank max-pool input, highway pre-activations).
# ----------------------------------------------------------------------------------------------
_save = None


@contextlib.contextmanager
def saving(S):
    global _save
    prev, _save = _save, S
    try:
        yield S
    finally:
        _save = prev


class Runtime:
    """Per-store kernel-side state: precision mode, derived operand buffers, scratch buffers."""

    def __init__(self, store, precision="tf32"):
        assert precision in ("tf32", "fp32", "fp32x3")
        self.store = store
        self.precision = precision
        # 'fp32x3': wgmma tensor cores with the error-compensated 3xTF32 split (fp32-grade products, ~1e-6);
        # 'tf32': single-pass TF32 products; 'fp32': exact-product FFMA kernel (cross-check path)
        self.impl = {"tf32": L.IMPL_TC, "fp32": L.IMPL_SIMT, "fp32x3": L.IMPL_TC3}[precision]
        self.derived = {}
        self.derived_version = {}
        self.scratch = {}

    def buf(self, tag, shape, dtype=torch.float32):
        key = (tag, tuple(shape), dtype)
        t = self.scratch.get(key)
        if t is None:
            t = torch.empty(shape, dtype=dtype, device=self.store.device)
            self.scratch[key] = t
        return t

    def get(self, key, builder):
        """Derived buffer cache keyed on the store version (rebuilt in place after an update)."""
        if self.derived_version.get(key) != self.store.version:
            self.derived[key] = builder(self.derived.get(key))
            self.derived_version[key] = self.store.version
        return self.derived[key]


def runtime(store, precision=None):
    rt = getattr(store, "_runtime", None)
    if rt is None or (precision is not None and rt.precision != precision):
        rt = Runtime(store, precision or "tf32")
        store._runtime = rt
    return rt


def _cpad(c):
    return (c + 31) // 32 * 32


def _pack(rt, key, W, taps, Cin, N, ld=None, row0=0, dst=None, n_total=None):
    """TF [taps][C][N] -> K-major TF32 operand rows [row0, row0+N) of dst (tensor-core path).  For the 3xTF32 path
    dst has 2*n_total rows: the hi heads in rows [0, n_total), the lo remainders in rows [n_total, 2 n_total)."""
    ld = ld or taps * _cpad(Cin)
    n_total = n_total or N
    x3 = rt.impl == L.IMPL_TC3
    if dst is None:
        dst = torch.zeros(((2 if x3 else 1) * n_total, ld), dtype=torch.float32, device=W.device)
    if x3:
        L.check(L.lib().taco_pack_weight_x3(L.ptr(W), taps, Cin, N, C.c_void_p(dst.data_ptr() + row0 * ld * 4),
                                            C.c_void_p(dst.data_ptr() + (n_total + row0) * ld * 4), ld, L.current_stream()),
                "taco_pack_weight_x3")
    else:
        L.check(L.lib().taco_pack_weight(L.ptr(W), taps, Cin, N, C.c_void_p(dst.data_ptr() + row0 * ld * 4), ld,
                                         L.current_stream()), "taco_pack_weight")
    return dst


def packed_weight(rt, name, W, taps, Cin, N):
    if rt.impl == L.IMPL_SIMT:
        return None
    return rt.get(("pack", name), lambda old: _pack(rt, name, W.contiguous(), taps, Cin, N, dst=old))


def bn_affine(rt, sc):
    """Inference-mode batch_normalization folded to y = x*scale + shift (SURVEY A.4)."""
    def build(old):
        scale = sc.p("bn_gamma") / torch.sqrt(sc.p("bn_var") + BN_EPS)
        shift = sc.p("bn_beta") - sc.p("bn_mean") * scale
        if old is not None:
            old[0].copy_(scale); old[1].copy_(shift)
            return old
        return (scale.contiguous(), shift.contiguous())
    return rt.get(("bn", sc.prefix), build)


# ----------------------------------------------------------------------------------------------
# the one contraction primitive
# ----------------------------------------------------------------------------------------------
def linear(rt, x, W, Wp, N, *, taps=1, bank_K=0, bank_cout=0, bias=None, act=L.ACT_NONE, scale=None, shift=None,
           keep=None, keep_scale=1.0, residual=None, highway_x=None, pool=False, out=None, tag="lin", bias_utt=None):
    """x [B,T,C] (contiguous) -> [B,T,N'] through taco_linear_fwd.  See include/taco_b200.h."""
    assert x.dim() == 3 and x.is_cuda and x.dtype == torch.float32 and x.stride(2) == 1
    B, T, Cin = x.shape
    assert x.stride(0) == T * x.stride(1)
    n_out = N // 2 if highway_x is not None else N
    if out is None:
        out = rt.buf(tag, (B, T, n_out))
    d = L.LinearDesc()
    d.X = x.data_ptr(); d.ldx = x.stride(1); d.B = B; d.T = T; d.C = Cin
    d.taps = taps; d.tap0 = -((taps - 1) // 2); d.N = N
    d.bank_K = bank_K; d.bank_cout = bank_cout
    d.W = W.data_ptr() if W is not None else None
    if Wp is not None:
        d.Wp = Wp.data_ptr(); d.ldwp = Wp.stride(0)
    d.Y = out.data_ptr(); d.ldy = out.stride(1)
    d.bias = bias.data_ptr() if bias is not None else None
    d.act = act
    d.scale = scale.data_ptr() if scale is not None else None
    d.shift = shift.data_ptr() if shift is not None else None
    if keep is not None:
        assert keep.dtype == torch.uint8 and keep.is_contiguous() and keep.numel() == B * T * n_out
        d.keep = keep.data_ptr()
    d.keep_scale = float(keep_scale)
    if residual is not None:
        assert residual.stride(-1) == 1
        d.residual = residual.data_ptr(); d.ldr = residual.stride(-2)
    if highway_x is not None:
        d.epilogue = L.EPI_HIGHWAY
        d.hx = highway_x.data_ptr(); d.ldhx = highway_x.stride(-2)
    d.pool = 1 if pool else 0
    if bias_utt is not None:                                    # [B, >= N] per-utterance bias, unit inner stride
        assert bias_utt.dim() == 2 and bias_utt.shape[0] == B and bias_utt.stride(1) == 1
        d.bias_utt = bias_utt.data_ptr(); d.ldbu = bias_utt.stride(0)
    d.impl = rt.impl
    L.check(L.lib().taco_linear_fwd(C.byref(d), L.current_stream()), f"taco_linear_fwd[{tag}]")
    return out


def _dropout_mask(shape, rate, device):
    return (torch.rand(shape, device=device) >= rate).to(torch.uint8)


# ----------------------------------------------------------------------------------------------
# Tacotron.pre_net (models/tacotron.py:38-44) -- lives on the model in the reference; the
# north-star surface lists it under ops, so it is defined here and bound as a method there.
# ----------------------------------------------------------------------------------------------
def pre_net(inputs, units=(256, 128), dropout=0.5, train=True, masks=None, scope=None, ids=None):
    """dense(256,relu) -> dropout -> dense(128,relu) -> dropout.  `inputs` [B,T,Cin].
    With `ids` (int32 [B,T]) `inputs` is the embedding TABLE [V,Cin]: layer 1 is then applied to
    the V table rows once and gathered (identical arithmetic per row, V << B*T)."""
    sc = scope or current_scope().sub("prenet")
    rt = runtime(sc.store)
    W1, b1, W2, b2 = sc.p("W1"), sc.p("b1"), sc.p("W2"), sc.p("b2")
    ks = 1.0 / (1.0 - dropout)
    if ids is not None:
        V, Cin = inputs.shape
        B, T = ids.shape
        t1 = linear(rt, inputs.view(1, V, Cin), W1, packed_weight(rt, sc.name("W1"), W1, 1, Cin, units[0]), units[0],
                    bias=b1, act=L.ACT_RELU, tag=sc.name("t1"))
        m1 = m2 = None
        if train:
            m1, m2 = masks if masks is not None else (_dropout_mask((B, T, units[0]), dropout, ids.device),
                                                      _dropout_mask((B, T, units[1]), dropout, ids.device))
        l1 = rt.buf(sc.name("l1"), (B, T, units[0]))
        L.check(L.lib().taco_gather_rows(L.ptr(t1), L.ptr(ids), B * T, units[0], V, L.ptr(m1), ks, L.ptr(l1),
                                         L.current_stream()), "taco_gather_rows")
    else:
        B, T, Cin = inputs.shape
        m1 = m2 = None
        if train:
            m1, m2 = masks if masks is not None else (_dropout_mask((B, T, units[0]), dropout, inputs.device),
                                                      _dropout_mask((B, T, units[1]), dropout, inputs.device))
        l1 = linear(rt, inputs, W1, packed_weight(rt, sc.name("W1"), W1, 1, Cin, units[0]), units[0], bias=b1,
                    act=L.ACT_RELU, keep=m1, keep_scale=ks, tag=sc.name("l1"))
    l2 = linear(rt, l1, W2, packed_weight(rt, sc.name("W2"), W2, 1, units[0], units[1]), units[1], bias=b2,
                act=L.ACT_RELU, keep=m2, keep_scale=ks, tag=sc.name("l2"))
    if _save is not None and ids is not None:
        _save[sc.name("t1")] = t1.view(V, units[0]); _save[sc.name("l1")] = l1; _save[sc.name("l2")] = l2
    return l2


# ----------------------------------------------------------------------------------------------
# conv bank (models/ops.py:54-71): K conv1d 'same' + relu, concat, batch-norm, max-pool(2,1,same)
# ----------------------------------------------------------------------------------------------
def conv1d_banks(inputs, K=16, cout=128, scope=None):
    sc = scope or current_scope().sub("bank")
    rt = runtime(sc.store)
    B, T, Cin = inputs.shape
    Wall = sc.store.span(sc.name("W1"), sc.name(f"W{K}"))
    ball = sc.store.span(sc.name("b1"), sc.name(f"b{K}"))
    scale, shift = bn_affine(rt, sc)
    Wp = None
    if rt.impl != L.IMPL_SIMT:
        def build(old):
            ld = K * _cpad(Cin)
            rows = K * cout * (2 if rt.impl == L.IMPL_TC3 else 1)
            dst = old if old is not None else torch.zeros((rows, ld), dtype=torch.float32, device=inputs.device)
            for k in range(1, K + 1):
                _pack(rt, None, sc.p(f"W{k}"), k, Cin, cout, ld=ld, row0=(k - 1) * cout, dst=dst, n_total=K * cout)
            return dst
        Wp = rt.get(("pack", sc.name("bank")), build)
        if _save is None:
            return linear(rt, inputs, Wall, Wp, K * cout, bank_K=K, bank_cout=cout, bias=ball, act=L.ACT_RELU, scale=scale,
                          shift=shift, pool=True, tag=sc.name("pool"))
    bank = linear(rt, inputs, Wall, Wp, K * cout, bank_K=K, bank_cout=cout, bias=ball, act=L.ACT_RELU, scale=scale,
                  shift=shift, tag=sc.name("bn"))
    pooled = rt.buf(sc.name("pool"), (B, T, K * cout))
    L.check(L.lib().taco_maxpool_fwd(L.ptr(bank), L.ptr(pooled), B, T, K * cout, L.current_stream()), "taco_maxpool_fwd")
    if _save is not None:
        _save[sc.name("bn")] = bank; _save[sc.name("pool")] = pooled; _save[sc.name("bn_affine")] = (scale, shift)
    return pooled


# ----------------------------------------------------------------------------------------------
# highway (models/ops.py:27-46)
# ----------------------------------------------------------------------------------------------
def _highway_weights(rt, sc, units):
    """[WH | WT] [units, 2 units], [bH | bT] and the packed operand of one highway layer"""
    def build_w(old):
        w = torch.cat([sc.p("WH"), sc.p("WT")], dim=1)
        if old is not None:
            old.copy_(w); return old
        return w.contiguous()

    def build_b(old):
        b = torch.cat([sc.p("bH"), sc.p("bT")])
        if old is not None:
            old.copy_(b); return old
        return b.contiguous()
    Whw = rt.get(("hw_w", sc.prefix), build_w)
    bhw = rt.get(("hw_b", sc.prefix), build_b)
    return Whw, bhw, packed_weight(rt, sc.name("hw"), Whw, 1, units, 2 * units)


def highway(inputs, units=128, scope=None):
    sc = scope or current_scope()
    rt = runtime(sc.store)
    B, T, Cin = inputs.shape
    if Cin != units:                                            # ops.py:29-30
        Wd, bd = sc.p("Wd"), sc.p("bd")
        inputs = linear(rt, inputs, Wd, packed_weight(rt, sc.name("Wd"), Wd, 1, Cin, units), units, bias=bd,
                        tag=sc.name("d"))
    Whw, bhw, Wp = _highway_weights(rt, sc, units)
    if _save is not None:                                       # train: keep [h_pre | t_pre] for the backward
        from .. import kernels as K
        Pm = linear(rt, inputs, Whw, Wp, 2 * units, bias=bhw, tag=sc.name("P"))
        out = rt.buf(sc.name("out"), (B, T, units))
        K.highway_fwd(out.view(-1, units), Pm.view(-1, 2 * units), inputs.view(-1, units))
        _save[sc.name("in")] = inputs; _save[sc.name("P")] = Pm
        return out
    return linear(rt, inputs, Whw, Wp, 2 * units, bias=bhw, highway_x=inputs, tag=sc.name("out"))


highwaynet = highway


def highway_stack(inputs, num_layers=4, scope=None):
    """Inference: the width-fixing dense (inputs not 128 wide, ops.py:29-30), `num_layers` highway layers (scopes
    highway0, highway1, ...) and the bi-GRU input products of the same scope as ONE kernel (taco_highway_stack_fwd,
    fp32x3 only): the activations between the layers never leave the SM.  Returns xp [B,T,768], bit-identical to
    highway() x num_layers followed by the products bidirectional_gru() computes itself."""
    sc = scope or current_scope()
    rt = runtime(sc.store)
    assert rt.impl == L.IMPL_TC3, "the fused highway stack is implemented for precision 'fp32x3'"
    assert 1 <= num_layers <= L.HIGHWAY_STACK_MAX
    assert inputs.dim() == 3 and inputs.stride(2) == 1
    B, T, Cin = inputs.shape
    assert inputs.stride(0) == T * inputs.stride(1)
    d = L.HighwayStackDesc()
    d.X = inputs.data_ptr(); d.ldx = inputs.stride(1); d.M = B * T; d.C = Cin
    if Cin != 128:
        dsc = sc.sub("highway0")
        Wd = dsc.p("Wd")
        Wdp = packed_weight(rt, dsc.name("Wd"), Wd, 1, Cin, 128)
        d.Wd_p = Wdp.data_ptr(); d.ldwd = Wdp.stride(0); d.bd = dsc.p("bd").data_ptr()
    d.L = num_layers
    for l in range(num_layers):
        _, bhw, Wp = _highway_weights(rt, sc.sub(f"highway{l}"), 128)
        d.hw_p[l] = Wp.data_ptr(); d.hw_b[l] = bhw.data_ptr(); d.ldhw = Wp.stride(0)
    _, bx, Wxp = _gru_input_weights(rt, sc)
    d.xp_p = Wxp.data_ptr(); d.ldxp = Wxp.stride(0); d.xp_b = bx.data_ptr()
    xp = rt.buf(sc.name("xp"), (B, T, 768))
    d.Y = xp.data_ptr(); d.ldy = xp.stride(1)
    d.impl = rt.impl
    L.check(L.lib().taco_highway_stack_fwd(C.byref(d), L.current_stream()), "taco_highway_stack_fwd")
    return xp


# ----------------------------------------------------------------------------------------------
# bidirectional GRU (models/ops.py:118-128)
# ----------------------------------------------------------------------------------------------
def _gru_input_weights(rt, sc, Cin=128):
    """Input-side operand of both GRU directions, [Wg_fw | Wc_fw | Wg_bw | Wc_bw][:Cin] [Cin, 768], its bias and its
    packed form (the products xp that taco_bigru_fwd reads)"""
    fw, bw = sc.sub("gru_fw"), sc.sub("gru_bw")

    def build_w(old):
        w = torch.cat([fw.p("Wg")[:Cin], fw.p("Wc")[:Cin], bw.p("Wg")[:Cin], bw.p("Wc")[:Cin]], dim=1)
        if old is not None:
            old.copy_(w); return old
        return w.contiguous()

    def build_b(old):
        b = torch.cat([fw.p("bg"), fw.p("bc"), bw.p("bg"), bw.p("bc")])
        if old is not None:
            old.copy_(b); return old
        return b.contiguous()
    Wx = rt.get(("gru_wx", sc.prefix), build_w)                  # [128, 768]
    bx = rt.get(("gru_bx", sc.prefix), build_b)
    return Wx, bx, packed_weight(rt, sc.name("gru_wx"), Wx, 1, Cin, 768)


def bidirectional_gru(inputs, gru_units=128, scope=None, h0=None, xp=None):
    """h0: None (zero state) or the [B,128] initial state of both directions (initial_state_fw = initial_state_bw,
    models/ops.py:111-126).  xp: the input products [B,T,768] when the caller has computed them (CBHG's fused highway
    stack); `inputs` is then not read."""
    sc = scope or current_scope()
    rt = runtime(sc.store)
    assert gru_units == 128, "the persistent GRU kernel is specialised for 128 units"
    fw, bw = sc.sub("gru_fw"), sc.sub("gru_bw")
    if xp is None:
        assert inputs.shape[-1] == 128, "the persistent GRU kernel is specialised for 128 units"
        B, T, Cin = inputs.shape
        Wx, bx, Wxp = _gru_input_weights(rt, sc, Cin)
        xp = linear(rt, inputs, Wx, Wxp, 768, bias=bx, tag=sc.name("xp"))
    else:
        assert xp.dim() == 3 and xp.shape[-1] == 768 and xp.is_contiguous()
        B, T, Cin = xp.shape[0], xp.shape[1], 128
    out = rt.buf(sc.name("gru_out"), (B, T, 2 * gru_units))
    if h0 is None:
        L.check(L.lib().taco_bigru_fwd(L.ptr(xp), L.ptr(fw.p("Wg")[Cin:]), L.ptr(fw.p("Wc")[Cin:]), L.ptr(bw.p("Wg")[Cin:]),
                                       L.ptr(bw.p("Wc")[Cin:]), L.ptr(out), B, T, L.current_stream()), "taco_bigru_fwd")
    else:
        assert h0.shape == (B, gru_units) and h0.is_contiguous()
        L.check(L.lib().taco_bigru_fwd_h0(L.ptr(xp), L.ptr(fw.p("Wg")[Cin:]), L.ptr(fw.p("Wc")[Cin:]), L.ptr(bw.p("Wg")[Cin:]),
                                          L.ptr(bw.p("Wc")[Cin:]), L.ptr(h0), L.ptr(h0), L.ptr(out), B, T, L.current_stream()),
                "taco_bigru_fwd_h0")
    if _save is not None:
        _save[sc.name("hw_out")] = inputs; _save[sc.name("xp")] = xp; _save[sc.name("gru_out")] = out
    return out


# ----------------------------------------------------------------------------------------------
# CBHG (models/ops.py:48-132)
# ----------------------------------------------------------------------------------------------
def _speaker_terms(sc, e, n_hw):
    """Speaker conditioning of a CBHG (models/ops.py:101-115) from e [B,16]: the n_hw highway speaker denses and the
    bi-GRU initial-state dense as ONE contraction over the concatenated [16, 128*(n_hw+1)] weight (S = relu(e.Ws + bs)),
    then per highway layer the per-utterance part of its width-fixing dense, u_l = s_l.Wd_l[128:] + bd_l.
    Returns (S [B,128*(n_hw+1)], [u_l [B,128]], h0 [B,128] contiguous)."""
    rt = runtime(sc.store)
    B, E = e.shape
    names = [f"highway{l}" for l in range(n_hw)] + ["gru_init"]

    def build_w(old):
        w = torch.cat([sc.p(f"{n}/Ws") for n in names], dim=1)
        if old is not None:
            old.copy_(w); return old
        return w.contiguous()

    def build_b(old):
        b = torch.cat([sc.p(f"{n}/bs") for n in names])
        if old is not None:
            old.copy_(b); return old
        return b.contiguous()
    Ws = rt.get(("spk_w", sc.prefix), build_w)
    bs = rt.get(("spk_b", sc.prefix), build_b)
    NS = 128 * len(names)
    Sv = linear(rt, e.view(1, B, E), Ws, packed_weight(rt, sc.name("spk_w"), Ws, 1, E, NS), NS, bias=bs, act=L.ACT_RELU,
                tag=sc.name("spk_s")).view(B, NS)
    us = []
    for l in range(n_hw):
        Wu = sc.p(f"highway{l}/Wd")[128:]
        u = linear(rt, Sv.view(1, B, NS)[:, :, 128 * l:128 * (l + 1)], Wu, packed_weight(rt, sc.name(f"highway{l}/Wd_s"), Wu, 1, 128, 128),
                   128, bias=sc.p(f"highway{l}/bd"), tag=sc.name(f"highway{l}/u"))
        us.append(u.view(B, 128))
    h0 = rt.buf(sc.name("gru_h0"), (B, 128))
    h0.copy_(Sv[:, 128 * n_hw:])                                  # the kernel reads [B][128] rows (data movement only)
    return Sv, us, h0


def CBHG(inputs, speaker_embed=None, K=16, c=[128, 128, 128], gru_units=128, num_highway_layers=4, num_conv_proj=2,
         trace=None):
    """speaker_embed: None, or e [B,16] (multi-speaker encoder, models/ops.py:101-115): layer l's highway input is
    [h | tile(s_l)], computed as h.Wd_l[:128] plus the per-utterance bias u_l; the bi-GRU starts from relu(e.Wg + bg)."""
    assert num_conv_proj == len(c) - 1                           # ops.py:75
    with variable_scope("cbhg") as sc:
        rt = runtime(sc.store)
        B, T, Cin = inputs.shape
        conv_bank = conv1d_banks(inputs, K=K, cout=c[0], scope=sc.sub("bank"))
        conv_proj = conv_bank
        cin = K * c[0]
        for layer in range(num_conv_proj):
            psc = sc.sub(f"proj{layer + 1}")
            last = layer == num_conv_proj - 1
            W, b = psc.p("W"), psc.p("b")
            scale, shift = bn_affine(rt, psc)
            conv_proj = linear(rt, conv_proj, W, packed_weight(rt, psc.name("W"), W, 3, cin, c[layer + 1]), c[layer + 1],
                               taps=3, bias=b, act=L.ACT_NONE if last else L.ACT_RELU, scale=scale, shift=shift,
                               residual=inputs if last else None, tag=psc.name("out"))   # +inputs: ops.py:92
            cin = c[layer + 1]
            if _save is not None:
                _save[psc.name("bn_affine")] = (scale, shift)
                _save[sc.name("res" if last else f"proj{layer + 1}")] = conv_proj
        h = conv_proj
        if trace is not None:
            trace[sc.name("bank_pool")] = conv_bank
            trace[sc.name("res")] = conv_proj
        if _save is not None:
            _save[sc.name("x_in")] = inputs
            _save[sc.name("bank_bn")] = _save[sc.name("bank/bn")]
            _save[sc.name("bank_pool")] = conv_bank
        h0 = None
        if speaker_embed is not None:
            assert speaker_embed.shape == (B, 16) and speaker_embed.is_contiguous()
            Sv, us, h0 = _speaker_terms(sc, speaker_embed, num_highway_layers)
            if _save is not None:
                _save[sc.name("spk_e")] = speaker_embed; _save[sc.name("spk_s")] = Sv; _save[sc.name("h0")] = h0
        if (_save is None and trace is None and speaker_embed is None and rt.impl == L.IMPL_TC3 and gru_units == 128
                and 1 <= num_highway_layers <= L.HIGHWAY_STACK_MAX):
            # inference: highway layers + bi-GRU input products in one kernel, same bits as the layer-by-layer route below
            return bidirectional_gru(None, gru_units, scope=sc, xp=highway_stack(h, num_highway_layers, scope=sc))
        for layer in range(num_highway_layers):
            hsc = sc.sub(f"highway{layer}")
            if speaker_embed is not None:                         # width-fixing dense of [h | tile(s_l)] (ops.py:29-30)
                Wx = hsc.p("Wd")[:128]
                x_outer = h
                h = linear(rt, h, Wx, packed_weight(rt, hsc.name("Wd_x"), Wx, 1, 128, 128), 128, bias_utt=us[layer],
                           tag=hsc.name("d"))
                if _save is not None:
                    _save[sc.name(f"hw{layer}_x")] = x_outer
            h = highway(h, scope=hsc)
            if _save is not None:
                _save[sc.name(f"hw{layer}_in")] = _save[sc.name(f"highway{layer}/in")]
                _save[sc.name(f"hw{layer}_P")] = _save[sc.name(f"highway{layer}/P")]
        if trace is not None:
            trace[sc.name("highway_out")] = h
        out = bidirectional_gru(h, gru_units, scope=sc, h0=h0)
        if trace is not None:
            trace[sc.name("out")] = out
        return out


# ----------------------------------------------------------------------------------------------
# InferenceHelper (models/ops.py:5-25): first input zeros, next input = previous output, never
# finished.  The persistent decoder kernel implements exactly this policy as TACO_DEC_INFER; the
# class carries the policy choice and reproduces the helper protocol for host-side use.
# ----------------------------------------------------------------------------------------------
class InferenceHelper:
    decoder_mode = L.DEC_INFER

    def __init__(self, batch_size, out_size):
        self._batch_size = batch_size
        self._out_size = out_size

    @property
    def batch_size(self):
        return self._batch_size

    def initialize(self, device="cuda"):
        finished = torch.zeros(self._batch_size, dtype=torch.bool, device=device)
        next_inputs = torch.zeros(self._batch_size, self._out_size, dtype=torch.float32, device=device)
        return finished, next_inputs

    def sample(self, time, outputs, state):
        return torch.zeros(32, dtype=torch.int32, device=outputs.device)   # ops.py:15 (hard-coded 32)

    def next_inputs(self, time, outputs, state, sample_ids=None):
        finished = torch.zeros(self._batch_size, dtype=torch.bool, device=outputs.device)
        return finished, outputs, state


# ----------------------------------------------------------------------------------------------
# attention decoder (models/tacotron.py:46-105,136-138): one persistent kernel for all T steps
# ----------------------------------------------------------------------------------------------
def decoder_speaker_state(sc, e):
    """Speaker conditioning of the decoder (Config.speaker_decoder) from e [B,16]: the initial attention vector
    a(-1) = e.Wa + ba (the reference's commented-out line, models/tacotron.py:96-97) and the initial GRU states
    h_i(-1) = relu(e.Wh_i + bh_i), as ONE contraction S = e.[Wa | Wh1 | Wh2 | Wh3] + b with the relu on the three state
    blocks.  Returns (S [B,1024], h0 [3,B,256], att0 [B,256]); h0 / att0 contiguous, the decoder kernel's layouts."""
    rt = runtime(sc.store)
    B, E = e.shape
    names = ("attn", "h1", "h2", "h3")

    def build_w(old):
        w = torch.cat([sc.p(f"spk/{n}/W") for n in names], dim=1)
        if old is not None:
            old.copy_(w); return old
        return w.contiguous()

    def build_b(old):
        b = torch.cat([sc.p(f"spk/{n}/b") for n in names])
        if old is not None:
            old.copy_(b); return old
        return b.contiguous()
    Ws = rt.get(("spk_w", sc.prefix), build_w)
    bs = rt.get(("spk_b", sc.prefix), build_b)
    NS = 256 * len(names)
    Sv = linear(rt, e.view(1, B, E), Ws, packed_weight(rt, sc.name("spk_w"), Ws, 1, E, NS), NS, bias=bs,
                tag=sc.name("spk_s")).view(B, NS)
    L.check(L.lib().taco_bias_act(C.c_void_p(Sv.data_ptr() + 256 * 4), NS, B, NS - 256, None, L.ACT_RELU, L.current_stream()),
            "taco_bias_act")
    h0 = rt.buf(sc.name("spk_h0"), (3, B, 256))
    h0.copy_(Sv[:, 256:].view(B, 3, 256).transpose(0, 1))           # the kernel reads [3][B][256] (data movement only)
    att0 = rt.buf(sc.name("spk_att0"), (B, 256))
    att0.copy_(Sv[:, :256])
    if _save is not None:
        _save[sc.name("spk_e")] = e; _save[sc.name("spk_s")] = Sv; _save[sc.name("h0")] = h0; _save[sc.name("att0")] = att0
    return Sv, h0, att0


def _decoder_weights(sc):
    w = L.DecoderWeights()
    w.pre_W1 = sc.p("prenet/W1").data_ptr(); w.pre_b1 = sc.p("prenet/b1").data_ptr()
    w.pre_W2 = sc.p("prenet/W2").data_ptr(); w.pre_b2 = sc.p("prenet/b2").data_ptr()
    w.in_W = sc.p("in_proj/W").data_ptr(); w.in_b = sc.p("in_proj/b").data_ptr()
    for i in range(3):
        w.gru_Wg[i] = sc.p(f"gru{i+1}/Wg").data_ptr(); w.gru_bg[i] = sc.p(f"gru{i+1}/bg").data_ptr()
        w.gru_Wc[i] = sc.p(f"gru{i+1}/Wc").data_ptr(); w.gru_bc[i] = sc.p(f"gru{i+1}/bc").data_ptr()
    w.out_W = sc.p("out_proj/W").data_ptr(); w.out_b = sc.p("out_proj/b").data_ptr()
    w.att_Wq = sc.p("attn/W_q").data_ptr(); w.att_v = sc.p("attn/v").data_ptr(); w.att_Wa = sc.p("attn/W_a").data_ptr()
    return w


# launch geometry of the forward decoder kernel (csrc/decoder.cu): a row group of 8 utterances runs on 32 co-resident CTAs
# (one per SM), a launch runs as many independent row groups as the CTA budget allows, up to 4 (32 utterances, the size of
# its workspace), also when it has fewer utterances: a grid sized to the utterances was measured slower (see DESIGN.md)
DEC_GROUP_ROWS = 8
DEC_GROUP_CTAS = 32
DEC_MAX_GROUPS = 4


def decoder_budget(capacity, max_ctas=None):
    """CTAs the decoder kernels may use: the device's co-resident `capacity`, capped by `max_ctas` (None or 0 = no cap).
    Raises TacoError, before anything is launched, for a cap below one row group or a device that cannot hold one."""
    if max_ctas is not None and max_ctas != 0 and max_ctas < DEC_GROUP_CTAS:
        raise L.TacoError(f"max_ctas={max_ctas}: the decoder kernels need at least {DEC_GROUP_CTAS} CTAs (None = the device's capacity)")
    if capacity < DEC_GROUP_CTAS:
        raise L.TacoError(f"only {capacity} decoder CTAs can be co-resident on this device; the decoder needs {DEC_GROUP_CTAS}")
    return capacity if not max_ctas else min(int(max_ctas), capacity)


def decoder_plan(B, capacity, max_ctas=None):
    """The forward decoder launches for B utterances: [(b0, nb, ctas)], utterances b0..b0+nb-1 on `ctas` CTAs.  Each launch
    runs the row groups the budget allows (min(4, budget // 32) groups of 32 CTAs) and takes up to 8 utterances per group."""
    groups = min(DEC_MAX_GROUPS, decoder_budget(capacity, max_ctas) // DEC_GROUP_CTAS)
    rows = DEC_GROUP_ROWS * groups
    return [(b0, min(rows, B - b0), DEC_GROUP_CTAS * groups) for b0 in range(0, B, rows)]


INT32_MAX = 2 ** 31 - 1


def attention_window(window):
    """None (no window) or (back, ahead) -> None or a tuple of two ints with back >= 0 and ahead >= 1: the positions
    step t of free-running decoding may attend are max(0, p(t-1) - back) .. p(t-1) + ahead, p(t-1) = the previous
    step's attention peak (p(-1) = 0).  Both must fit taco_decoder_args' int32 fields.  Raises TacoError, before
    anything is launched, for anything else."""
    if window is None:
        return None
    try:
        back, ahead = window
    except (TypeError, ValueError):
        raise L.TacoError(f"attention window {window!r}: expected None or (back, ahead)") from None
    for name, v, lo in (("back", back, 0), ("ahead", ahead, 1)):
        if isinstance(v, bool) or not isinstance(v, numbers.Integral):
            raise L.TacoError(f"attention window {window!r}: {name} must be an integer, got {type(v).__name__}")
        if v < lo:
            raise L.TacoError(f"attention window {window!r}: {name} must be >= {lo}, got {v}")
        if v > INT32_MAX:                     # the C ABI's int32 fields (any bound >= Tx already allows every position)
            raise L.TacoError(f"attention window {window!r}: {name} must be <= {INT32_MAX}, got {v}")
    return int(back), int(ahead)


def stop_rule_hold(hold):
    """None (no stop rule) or hold -> None or an int >= 1: the decoder steps in a row whose attention peaks must all lie
    at or past the last real character before a row ends (the end-of-text stop rule of free-running decoding).  It must
    fit taco_decoder_args' int32 field.  Raises TacoError, before anything is launched, for anything else."""
    if hold is None:
        return None
    if isinstance(hold, bool) or not isinstance(hold, numbers.Integral):
        raise L.TacoError(f"stop rule hold {hold!r}: expected None or an integer >= 1, got {type(hold).__name__}")
    if not 1 <= hold <= INT32_MAX:
        raise L.TacoError(f"stop rule hold {hold!r}: must be in [1, {INT32_MAX}]")
    return int(hold)


def stop_positions(text, text_length):
    """stop_at int32 [B] on text's device, without a host synchronisation: the position of each row's last real
    character, max(min(n_b, N_b, Tx) - 1, 0), with n_b = the non-zero ids of text row b (id 0 is <pad>) and N_b =
    text_length[b].  N_b alone is not it: load_prompts counts the raw line, newline included, in text_length while
    dropping out-of-vocabulary characters from the ids, so position N_b - 1 is usually padding."""
    B, Tx = text.shape
    n = (text != 0).sum(dim=1)
    last = torch.minimum(torch.minimum(n, text_length.to(n.dtype)), torch.full_like(n, Tx)) - 1
    return last.clamp_(min=0).to(torch.int32)


def stop_rule_end_steps(peaks, stop_at, hold):
    """The stop rule on a host array of peaks [B, T] (each step's attention peak p(t)): end_step [B] int64 = t + 1 for
    the first t with p(t - hold + 1), ..., p(t) all >= stop_at[b], or T.  The kernel applies the same rule to its own
    peaks as it decodes."""
    import numpy as np
    p = np.asarray(peaks)
    B, T = p.shape
    at = np.asarray(stop_at).reshape(B, 1)
    end = np.full(B, T, dtype=np.int64)
    run = np.zeros(B, dtype=np.int64)
    for t in range(T):
        run = np.where(p[:, t] >= at[:, 0], run + 1, 0)
        hit = (run >= hold) & (end == T)
        end[hit] = t + 1
    return end


def stopped_steps(end_step, T):
    """decoder steps Tacotron.inference keeps from a stopped decode of T steps: T' = min(T, 4 ceil(max_b end_step / 4)),
    whole blocks of 4 steps as reshape_frames needs.  Reads end_step to the host (one synchronisation)."""
    e = int(end_step.max()) if torch.is_tensor(end_step) else int(max(end_step))
    return min(int(T), 4 * ((e + 3) // 4))


def decoder_fwd_launches(lib, plan, w, t, mode, T, r, keep_scale, max_ctas, stream, window=None, hold=None):
    """One taco_decoder_fwd per entry of `plan` over the full-batch tensors `t` (dict: packed, keys, values, text_length,
    y, align, workspace, and mel, sample_mask, keep1, keep2, h_save, step_ns, h0, att0, peak or None).  [B]-major tensors
    (peak [B][T] among them) are passed from row b0; the [T][B]-major ones (sample_mask, keep1, keep2, h_save) and the
    initial states h0 [3][B][256], att0 [B][256] whole, with row0 = b0 and row_stride = B.  window: None or (back, ahead)
    (attention_window), passed as given: taco_decoder_fwd checks it against the mode.  hold: None or the stop rule's hold
    (stop_rule_hold), with t['stop_at'] and t['end_step'] int32 [B], passed from row b0 like peak."""
    B = t["keys"].shape[0]
    Tx = t["keys"].shape[1]
    ptr = lambda x, b0=0: None if x is None else x[b0:].data_ptr()
    for b0, nb, _ in plan:
        a = L.DecoderArgs()
        a.weights = C.pointer(w)
        a.packed = t["packed"].data_ptr(); a.keys = ptr(t["keys"], b0); a.values = ptr(t["values"], b0)
        a.text_length = ptr(t["text_length"], b0)
        a.mode = mode
        a.mel = ptr(t.get("mel"), b0)
        a.sample_mask = ptr(t.get("sample_mask")); a.keep1 = ptr(t.get("keep1")); a.keep2 = ptr(t.get("keep2"))
        a.h_save = ptr(t.get("h_save"))
        a.row0 = b0; a.row_stride = B
        a.keep_scale = keep_scale
        a.B = nb; a.Tx = Tx; a.T = T; a.r = r
        a.y = ptr(t["y"], b0); a.align = ptr(t["align"], b0); a.workspace = t["workspace"].data_ptr()
        a.step_ns = ptr(t.get("step_ns"))
        a.h0 = ptr(t.get("h0")); a.att0 = ptr(t.get("att0"))
        a.max_ctas = int(max_ctas or 0)
        if window is not None:
            a.win_back, a.win_ahead = window
        a.peak = ptr(t.get("peak"), b0)
        a.stop_at = ptr(t.get("stop_at"), b0); a.end_step = ptr(t.get("end_step"), b0)
        if hold is not None:
            a.stop_hold = hold
        L.check(lib.taco_decoder_fwd(C.byref(a), stream), "taco_decoder_fwd")


def attention_decoder(encoded, text_length, r, T, mode=L.DEC_INFER, mel=None, sample_mask=None, drop_masks=None,
                      dropout=0.5, scope=None, step_ns=None, max_ctas=None, h0=None, att0=None, window=None,
                      stop_hold=None, stop_at=None):
    """encoded [B,Tx,256], text_length int32 [B] -> (seq2seq_output [B,T,80r], alignments [B,T,Tx]).
    h0 [3,B,256] / att0 [B,256]: initial GRU states / attention vector (speaker-conditioned decoder), None = zero.
    window: None, or (back, ahead) in free-running mode (attention_window): each step attends only near the previous
    step's peak, and the result is (seq2seq_output, alignments, peaks int32 [B,T]) with each step's peak position.
    stop_hold, stop_at: None, or the end-of-text stop rule in free-running mode, both set: hold (stop_rule_hold) >= 1 and
    stop_at int32 [B] (stop_positions).  Row b ends after step t when p(t - hold + 1), ..., p(t) >= stop_at[b];
    end_step[b] = t + 1, or T.  Each row group of 8 stops decoding within _lib.DECODER_STOP_LAG steps of its last row's
    end; the steps it did not decode hold 0 in y and alignments and -1 in the peaks.  The result is then
    (seq2seq_output, alignments, peaks, end_step int32 [B]), on the device (nothing is read to the host).
    max_ctas caps the CTAs (SMs) the decoder kernel may occupy (None = all the device holds); the batch is decoded in as
    many launches of up to 8 x (max_ctas // 32) utterances as it needs (decoder_plan)."""
    from .. import kernels as K
    B, Tx, D = encoded.shape
    assert D == 256
    window = attention_window(window)
    if window is not None and mode != L.DEC_INFER:
        raise L.TacoError(f"attention window {window}: only free-running decoding (mode DEC_INFER) takes a window, mode is {mode}")
    hold = stop_rule_hold(stop_hold)
    if (hold is None) != (stop_at is None):
        raise L.TacoError(f"stop rule: stop_hold={stop_hold!r} and stop_at {'set' if stop_at is not None else 'None'}: "
                          f"give both or neither")
    if hold is not None:
        if mode != L.DEC_INFER:
            raise L.TacoError(f"stop rule: only free-running decoding (mode DEC_INFER) stops at the end of the text, mode is {mode}")
        if not (stop_at.dtype == torch.int32 and stop_at.is_contiguous() and tuple(stop_at.shape) == (B,)
                and stop_at.device == encoded.device):
            raise L.TacoError(f"stop rule: stop_at must be a contiguous int32 tensor of shape [{B}] on {encoded.device}, got "
                              f"{stop_at.dtype} {stop_at.device} {tuple(stop_at.shape)}")
    sc = scope or current_scope()
    rt = runtime(sc.store)
    lib = L.lib()
    plan = decoder_plan(B, K.decoder_capacity()[0], max_ctas)     # (raises before any launch for a budget below 32)
    out_w = 80 * r
    y = rt.buf(sc.name("y"), (B, T, out_w))
    align = rt.buf(sc.name("align"), (B, T, Tx))
    # BahdanauAttention memory: values = length-masked encoder states, keys = values . W_mem (tacotron.py:48-52)
    values = rt.buf(sc.name("values"), (B, Tx, D))
    L.check(lib.taco_mask_rows(L.ptr(encoded), L.ptr(text_length), L.ptr(values), B, Tx, D, L.current_stream()), "taco_mask_rows")
    Wm = sc.p("attn/W_mem")
    keys = linear(rt, values, Wm, packed_weight(rt, sc.name("attn/W_mem"), Wm, 1, D, 256), 256, tag=sc.name("keys"))

    w = _decoder_weights(sc)

    def build_pack(old):
        dst = old if old is not None else torch.empty(lib.taco_decoder_packed_bytes(r) // 4, dtype=torch.float32,
                                                      device=encoded.device)
        L.check(lib.taco_decoder_pack(C.byref(w), r, L.ptr(dst), L.current_stream()), "taco_decoder_pack")
        return dst
    packed = rt.get(("dec_pack", sc.prefix, r), build_pack)
    ws = rt.buf(sc.name("dec_ws"), (lib.taco_decoder_workspace_bytes(32, Tx, T, r) // 4,))
    rt.dec_ws = ws                                               # (per-slot time stamps live in its tail; see decoder.cu)
    ks = 1.0 / (1.0 - dropout)
    hs = None
    if _save is not None:                                        # train: the three GRU state sequences feed the backward
        assert B <= 32, "training decodes at most 32 utterances per rank (the backward kernel's limit)"
        hs = rt.buf(sc.name("H"), (3, T, B, 256))
        _save[sc.name("H")] = hs; _save[sc.name("values")] = values; _save[sc.name("keys")] = keys
        _save[sc.name("y")] = y; _save[sc.name("align")] = align
        if drop_masks is not None:
            _save[sc.name("keep1")], _save[sc.name("keep2")] = drop_masks
        if mode == L.DEC_SCHED:
            _save[sc.name("sample_mask")] = sample_mask
    t = {"packed": packed, "keys": keys, "values": values, "text_length": text_length, "y": y, "align": align,
         "workspace": ws, "step_ns": step_ns, "h_save": hs, "h0": h0, "att0": att0}
    if h0 is not None:
        assert h0.shape == (3, B, 256) and h0.is_contiguous()
    if att0 is not None:
        assert att0.shape == (B, 256) and att0.is_contiguous()
    if mode != L.DEC_INFER:
        assert mel is not None and mel.is_contiguous() and mel.shape == (B, T, out_w)
        t["mel"] = mel
    if mode == L.DEC_SCHED:
        assert sample_mask is not None and sample_mask.dtype == torch.uint8 and sample_mask.shape == (T, B)
        assert sample_mask.is_contiguous()
        t["sample_mask"] = sample_mask
    if drop_masks is not None:
        k1, k2 = drop_masks
        assert k1.dtype == torch.uint8 and k1.shape == (T, B, 256) and k2.shape == (T, B, 128)
        assert k1.is_contiguous() and k2.is_contiguous()
        t["keep1"], t["keep2"] = k1, k2
    if window is not None or hold is not None:
        t["peak"] = rt.buf(sc.name("peak"), (B, T), torch.int32)
    if hold is not None:
        t["stop_at"] = stop_at
        t["end_step"] = rt.buf(sc.name("end_step"), (B,), torch.int32)
    decoder_fwd_launches(lib, plan, w, t, mode, T, r, ks, max_ctas, L.current_stream(), window, hold)
    if hold is not None:
        return y, align, t["peak"], t["end_step"]
    return (y, align) if window is None else (y, align, t["peak"])
