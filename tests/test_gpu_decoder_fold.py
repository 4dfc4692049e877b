"""-m gpu: the decoder's first GRU stage with the input projection folded in.  z(t) = [ctx(t-1) | p2(t)] . W_cpF +
s(t-1) . W_sF + b_inF is never formed on the step's dependent chain: the G1 stage multiplies [ctx | p2] and s(t-1) by
pack-time products with Wg1_x and Wc1_x (csrc/decoder.cu fused_tail).

  * the folded blocks of the packed buffer against float64 products of the raw parameters;
  * the free-running decoder at the benchmark's C2 shape (B = 32, Tx = 128, r = 5) against the float64 oracle, step 0
    (no s, no context: the t = 0 biases and initial-state terms) and the later steps apart, with and without a
    speaker-conditioned initial state.  Bar: 1e-4 of the tensor's max magnitude, the decoder bar for T <= 20.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import tacotron_oracle as O
from tests import speaker_decoder_oracle as SD
from tests.test_gpu_decoder_envelope import _run_forward
from tests.test_gpu_speaker_decoder import _dec_case, _run
from tests.util import assert_close, ocfg

pytestmark = pytest.mark.gpu

U, NS = 256, 32
# segments of csrc/decoder.cu build_seg_table, in order: (K, FL, warps, k-tile slots per warp)
SEGS = ([(384, 4, 16, 3)] * 2 + [(256, 4, 16, 2)] * 2          # G1_CP, Z1_CP, G1_S, Z1_S
        + [(256, 4, 16, 2)] * 5 + [(256, 2, 16, 2)] * 5         # G_H0..2, G_X1..2; C_X1..2, C_RH0..2
        + [(256, 4, 16, 2)] * 2 + [(80, 2, 16, 2), (256, 2, 8, 4)])   # Y, QP, PM, P2


def _seg_offsets():
    offs, o = [], 0
    for K, FL, nw, kpw in SEGS:
        offs.append(o)
        o += NS * nw * kpw * 32 * FL
    return offs, (o + 63) // 64 * 64


def _unpack_split(packed, seg):
    """a 16-column (FL = 4) segment whose slice cs holds columns 8cs..8cs+7 and 256+8cs..256+8cs+7 -> [K][512]"""
    K, FL, nw, kpw = SEGS[seg]
    assert FL == 4
    off = _seg_offsets()[0][seg]
    blk = packed[off: off + NS * nw * kpw * 32 * FL].reshape(NS, nw, kpw, 32, FL)
    cs, w, i, lane, e = np.meshgrid(np.arange(NS), np.arange(nw), np.arange(kpw), np.arange(32), np.arange(FL), indexing="ij")
    kt = w + nw * i
    m = (lane >> 2) + 8 * (e & 1)
    k = kt * 8 + (lane & 3) + 4 * (e >> 1)
    col = np.where(m < 8, 8 * cs + m, U + 8 * cs + m - 8)
    live = kt < K // 8
    out = np.full((K, 2 * U), np.nan)
    out[k[live], col[live]] = blk[live]
    return out


def _check(got, ref, what, rel=1e-6):
    ref = ref.numpy()
    assert not np.isnan(got).any(), f"{what}: entries the pack never wrote"
    err = np.abs(got - ref).max() / np.abs(ref).max()
    assert err <= rel, f"{what}: max error {err:.3e} of the max magnitude (bar {rel:.0e})"


@pytest.mark.parametrize("r", [2, 5])
def test_folded_blocks_match_float64_products(r):
    from tacotron_b200 import Config, _lib as L
    from tacotron_b200.models import ops
    from tacotron_b200.params import ParamStore, model_shapes
    p = O.init_params(ocfg(r=r, T=8, vocab=20), seed=1, trained_like=True)
    st = ParamStore(model_shapes(Config(r=r, vocab_size=20)), "cuda")
    st.load(p)
    ops.runtime(st, "fp32")
    w = ops._decoder_weights(ops.Scope(st, "dec"))
    lib = L.lib()
    dst = torch.full((lib.taco_decoder_packed_bytes(r) // 4,), float("nan"), device="cuda")
    L.check(lib.taco_decoder_pack(C.byref(w), r, L.ptr(dst), L.current_stream()), "taco_decoder_pack")
    packed = dst.cpu().double().numpy()

    d = {k[4:]: v.double() for k, v in p.items() if k.startswith("dec/")}
    out = 80 * r
    Wa, Win, bin_ = d["attn/W_a"], d["in_proj/W"], d["in_proj/b"]
    Wg1x, Wc1x, bg1 = d["gru1/Wg"][:U], d["gru1/Wc"][:U], d["gru1/bg"]
    W_cpF = torch.cat([Wa[out:] @ Win[128:], Win[:128]])
    M1 = Wa[:out] @ Win[128:]
    W_sF = d["out_proj/W"] @ M1
    b_inF = bin_ + d["out_proj/b"] @ M1
    _check(_unpack_split(packed, 0), W_cpF @ Wg1x, f"r={r} G1 gates [ctx | p2]")
    _check(_unpack_split(packed, 1), torch.cat([W_cpF @ Wc1x, W_cpF], 1), f"r={r} G1 [candidate x | z] [ctx | p2]")
    _check(_unpack_split(packed, 2), W_sF @ Wg1x, f"r={r} G1 gates s(t-1)")
    _check(_unpack_split(packed, 3), torch.cat([W_sF @ Wc1x, W_sF], 1), f"r={r} G1 [candidate x | z] s(t-1)")

    # biases at the start of the packed tail: b_g1F, b_g1F0, b_z1F, b_z1F0 (t > 0, then t = 0)
    t0 = _seg_offsets()[1]
    tail = packed[t0: t0 + 4 * 2 * U].reshape(4, 2 * U)
    _check(tail[0], b_inF @ Wg1x + bg1, f"r={r} gate bias t > 0")
    _check(tail[1], bin_ @ Wg1x + bg1, f"r={r} gate bias t = 0")
    _check(tail[2], torch.cat([b_inF @ Wc1x, b_inF]), f"r={r} [candidate x | z] bias t > 0")
    _check(tail[3], torch.cat([bin_ @ Wc1x, bin_]), f"r={r} [candidate x | z] bias t = 0")


def _check_steps(y, a, y_ref, a_ref, what):
    assert not torch.isnan(y).any() and not torch.isnan(a).any(), f"{what}: NaN in the output"
    for sl, name in ((slice(0, 1), "t = 0"), (slice(1, None), "t > 0")):
        assert_close(y[:, sl], y_ref[:, sl], 1e-4, f"{what} y {name}")
        assert_close(a[:, sl], a_ref[:, sl], 1e-4, f"{what} align {name}")


def test_c2_free_running_matches_oracle():
    y, a, y_ref, a_ref, _ = _run_forward(5, 32, 128, 12, "infer")
    _check_steps(y, a, y_ref, a_ref, "C2 decoder")


def test_c2_free_running_with_initial_state_matches_oracle():
    r, B, Tx, T = 5, 32, 128, 12
    cfg, p, encoded, inp, dec_m, sm, h0, att0, st = _dec_case(r, B, Tx, T)
    y_ref, a_ref = SD.decoder(encoded, inp["text_length"], p, cfg, "infer", T, h0, att0, mel=inp["mel"])
    y, a = _run(st, r, T, "infer", encoded, inp, dec_m, sm, h0, att0)
    _check_steps(y, a, y_ref, a_ref, "C2 speaker decoder")
