"""-m gpu: the persistent decoder forward (taco_decoder_fwd) checked step by step against float64 formed from its own
stored state (tests/decoder_step_checks.py), over the range its ABI accepts.

Every run writes into NaN-poisoned y, align, h_save and peak, each inside a guard band of sentinel words: after the run
every cell must be written and no guard word may change (the multi-launch row0 / row_stride addressing above all).

Cases: the C2 step (B = 32, Tx = 128 ragged, T = 200, r = 5) in every mode, with dropout and with a 109-speaker initial
state; r = 1..6; one Tx in each weight-residency set of test_gpu_decoder_envelope.py with whole attention quarters masked;
single- and multi-launch batches and one row group per launch; T = 1 and T = 1000; the attention window; saturated gates
and keys / queries past exp2x's clamp; three exact laws bit for bit; and the check's sensitivity to each weight.

Each check prints its worst |kernel - float64| / bar per quantity (h1, h2, h3, y, align, peak).
"""
import ctypes as C
import math

import pytest
import torch

from oracle import tacotron_oracle as O
from tacotron_b200 import _lib as L
from tacotron_b200.models import ops
from tests import decoder_step_checks as DC
from tests import speaker_decoder_oracle as SD
from tests.test_gpu_attention_window import WINDOWS
from tests.test_gpu_decoder_envelope import short_lengths
from tests.util import ocfg

pytestmark = pytest.mark.gpu
PAD = 1024                      # guard band, words, on each side of every output
SENT = 0x7FA5A5A5               # signalling-NaN bit patterns no arithmetic produces: the guard words,
POISON = 0x7FBADBAD             # and every output cell before the run (peaks: an impossible position)
POISON_PEAK = -(2 ** 31)
KEEP_SCALE = 2.0                # 1 / (1 - audio dropout 0.5)
MODES = {"infer": L.DEC_INFER, "teacher": L.DEC_TEACHER, "sched": L.DEC_SCHED}
DEC = ["prenet/W1", "prenet/b1", "prenet/W2", "prenet/b2", "in_proj/W", "in_proj/b", "out_proj/W", "out_proj/b",
       "attn/W_q", "attn/v", "attn/W_a"] + [f"gru{i}/{n}" for i in (1, 2, 3) for n in ("Wg", "bg", "Wc", "bc")]


class _Scope:
    def __init__(self, t):
        self.t = t

    def p(self, name):
        return self.t["dec/" + name]


def _guarded(shape, dtype):
    n = math.prod(shape)
    buf = torch.empty(n + 2 * PAD, dtype=dtype, device="cuda")
    buf.view(torch.int32).fill_(SENT)
    body = buf[PAD:PAD + n].view(shape)
    body.view(torch.int32).fill_(POISON if dtype.is_floating_point else POISON_PEAK)
    return buf, body


def _guard_intact(buf, n):
    w = buf.view(torch.int32)
    return bool((w[:PAD] == SENT).all()) and bool((w[PAD + n:] == SENT).all())


def case(r, B, Tx, T, lengths=None, seed=0, speakers=0):
    """weights (trained-like), encoder output, lengths, mel, keep masks, sample mask; with `speakers`, the
    speaker-conditioned decoder's initial state (h0, att0) of random speakers of a table that size"""
    if speakers:
        cfg = SD.SpkDecOracleConfig(r=r, max_decode_iter=T, vocab_size=20, num_speakers=speakers)
        p = SD.init_params(cfg, seed=1, trained_like=True)
    else:
        cfg = ocfg(r=r, T=T, vocab=20)
        p = O.init_params(cfg, seed=1, trained_like=True)
    g = torch.Generator().manual_seed(seed)
    encoded = torch.randn(B, Tx, 256, generator=g) * 0.5
    inp = O.synthetic_inputs(cfg, B, Tx, T, seed=seed, ragged=True)
    tl = inp["text_length"] if lengths is None else lengths
    _, dm = O.dropout_masks(cfg, B, Tx, T, seed=2)
    sm = O.sched_mask(cfg, B, T, seed=3)
    c = dict(r=r, p=p, encoded=encoded, tl=tl, mel=inp["mel"], keep=dm, sm=sm, T=T, h0=None, att0=None)
    if speakers:
        e = p["speaker/embed"][torch.randint(0, speakers, (B,), generator=g)]
        c["h0"], c["att0"] = SD.initial_state(p, e)
    return c


def memory(encoded, tl, W_mem):
    """values = length-masked encoder output, keys = values . W_mem, formed in float64 and given to both sides in fp32"""
    Tx = encoded.shape[1]
    values = encoded.double() * (torch.arange(Tx)[None, :] < tl[:, None].to(torch.int64))[..., None]
    return values.float(), (values @ W_mem.double()).float()


def run(c, mode, window=None, max_ctas=None, keys=None, p=None, encoded=None):
    """one taco_decoder_fwd per launch of ops.decoder_plan into guarded, NaN-poisoned outputs -> dict of outputs and
    the memory it read.  p / encoded / keys override the case's."""
    p = c["p"] if p is None else p
    encoded = c["encoded"] if encoded is None else encoded
    r, T, tl = c["r"], c["T"], c["tl"]
    B, Tx, _ = encoded.shape
    values, k = memory(encoded, tl, p["dec/attn/W_mem"])
    keys = k if keys is None else keys
    lib = L.lib()
    t = {k_: p[k_].float().cuda().contiguous() for k_ in ("dec/" + n for n in DEC)}
    w = ops._decoder_weights(_Scope(t))
    packed = torch.empty(lib.taco_decoder_packed_bytes(r) // 4, dtype=torch.float32, device="cuda")
    L.check(lib.taco_decoder_pack(C.byref(w), r, L.ptr(packed), L.current_stream()), "taco_decoder_pack")
    shapes = {"y": ((B, T, 80 * r), torch.float32), "align": ((B, T, Tx), torch.float32),
              "h_save": ((3, T, B, 256), torch.float32)}
    if window is not None:
        shapes["peak"] = ((B, T), torch.int32)
    bufs, outs = {}, {}
    for name, (shape, dt) in shapes.items():
        bufs[name], outs[name] = _guarded(shape, dt)
    a = {"packed": packed, "keys": keys.cuda().contiguous(), "values": values.cuda(), "text_length": tl.cuda(),
         "workspace": torch.zeros(lib.taco_decoder_workspace_bytes(32, Tx, T, r) // 4, device="cuda"), **outs}
    if mode != "infer":
        a["mel"] = c["mel"].float().cuda().contiguous()
        a["keep1"], a["keep2"] = (m.cuda().contiguous() for m in c["keep"])
    if mode == "sched":
        a["sample_mask"] = c["sm"].cuda().contiguous()
    if c["h0"] is not None:
        a["h0"] = c["h0"].float().cuda().contiguous()
        a["att0"] = c["att0"].float().cuda().contiguous()
    plan = ops.decoder_plan(B, _capacity(), max_ctas)
    ops.decoder_fwd_launches(lib, plan, w, a, MODES[mode], T, r, KEEP_SCALE, max_ctas, L.current_stream(), window)
    torch.cuda.synchronize()
    for name, (shape, dt) in shapes.items():
        assert _guard_intact(bufs[name], math.prod(shape)), f"{name}: a guard word changed"
        unwritten = outs[name].view(torch.int32) == (POISON if dt.is_floating_point else POISON_PEAK)
        assert not unwritten.any(), f"{name}: {int(unwritten.sum())} cells left unwritten"
    return {"y": outs["y"].clone(), "align": outs["align"].clone(), "H": outs["h_save"].clone(),
            "peak": outs["peak"].clone() if window is not None else None, "keys": keys, "values": values}


def _capacity():
    from tacotron_b200 import kernels as K
    return K.decoder_capacity()[0]


def check(c, mode, out, window=None, p=None):
    """decoder_step_checks.check on one run (the reference keeps the case's weights unless `p` is given)"""
    return DC.check(out["y"], out["align"], out["H"], c["p"] if p is None else p, out["keys"], out["values"], c["tl"],
                    c["r"], mode, mel=c["mel"], sample_mask=c["sm"], keep=None if mode == "infer" else c["keep"],
                    keep_scale=KEEP_SCALE, h0=c["h0"], att0=c["att0"], window=window, peak=out["peak"])


def assert_local(c, mode, what, window=None, **kw):
    out = run(c, mode, window=window, **kw)
    rep = check(c, mode, out, window=window, p=kw.get("p"))
    print(f"{what}: {rep}")
    assert rep.first is None, f"{what}: {rep.first}"
    return out, rep


# ---------------------------------------------------------------------------------------------------------------------
# the C2 step
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["infer", "teacher", "sched"])
def test_c2(mode):
    assert_local(case(5, 32, 128, 200), mode, f"C2 {mode}")


@pytest.mark.parametrize("mode", ["infer", "sched"])
def test_c2_speaker_state(mode):
    """step 0 is where the init_* terms of h0 / att0 enter"""
    assert_local(case(5, 32, 128, 200, speakers=109), mode, f"C2 109-speaker state {mode}")


# ---------------------------------------------------------------------------------------------------------------------
# r, Tx, B, T
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["infer", "sched"])
@pytest.mark.parametrize("r", [1, 2, 3, 4, 5, 6])
def test_r(r, mode):
    """r = 1 and r = 3 leave whole output slices of OQP without columns"""
    assert_local(case(r, 9, 37, 60), mode, f"r={r} {mode}")


@pytest.mark.parametrize("Tx", [1, 7, 128, 140, 150, 170, 185, 200, 215, 230, 256])
def test_tx_residency(Tx):
    """one Tx in every weight-residency set, lengths that mask whole attention quarters"""
    c = case(5, 32, Tx, 40, lengths=short_lengths(Tx, 32))
    assert_local(c, "infer", f"Tx={Tx} infer")
    assert_local(c, "teacher", f"Tx={Tx} teacher")


@pytest.mark.parametrize("B", [1, 8, 9, 31, 32, 33, 64])
def test_batch(B):
    """B > 32: several launches, h_save at the row stride"""
    assert_local(case(5, B, 64, 50), "sched", f"B={B} sched")


def test_one_row_group_per_launch():
    assert_local(case(5, 32, 64, 50), "sched", "B=32 max_ctas=32", max_ctas=32)


@pytest.mark.parametrize("B,T", [(9, 1), (1, 1000), (32, 1000)])
def test_length(B, T):
    assert_local(case(5, B, 128, T), "infer", f"B={B} T={T}")


# ---------------------------------------------------------------------------------------------------------------------
# attention window: alignments and peaks, locally
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("window", WINDOWS)
@pytest.mark.parametrize("Tx,T", [(128, 200), (256, 100)])
def test_window(Tx, T, window):
    c = case(5, 32, Tx, T, lengths=None if Tx == 128 else short_lengths(Tx, 32))
    assert_local(c, "infer", f"Tx={Tx} window={window}", window=window)


# ---------------------------------------------------------------------------------------------------------------------
# magnitudes
# ---------------------------------------------------------------------------------------------------------------------
def _recurrent_x3(p):
    q = dict(p)
    for i in (1, 2, 3):
        for n in ("Wg", "Wc"):
            W = p[f"dec/gru{i}/{n}"].clone()
            W[256:] *= 3
            q[f"dec/gru{i}/{n}"] = W
    return q


@pytest.mark.parametrize("mode", ["infer", "sched"])
def test_saturated_gates(mode):
    c = case(5, 32, 128, 200)
    c["p"] = _recurrent_x3(c["p"])
    assert_local(c, mode, f"recurrent weights x3 {mode}")


@pytest.mark.parametrize("scale", [30.0, 60.0])
def test_keys_and_queries_past_the_exp2x_clamp(scale):
    """keys and q(t) beyond +-20.8, where exp2x clamps e^{2k} and e^{2q}: many (k, q) pairs of opposite sign have a
    moderate sum, where tanh(k + q) is far from +-1 and the clamped product gives it wrong (before the direct form,
    alpha 0.016396 where float64 gives 0.016430 at scale 30, bar 1.3e-5)"""
    c = case(2, 9, 64, 30)
    g = torch.Generator().manual_seed(7)
    keys = torch.randn(9, 64, 256, generator=g) * scale
    q = dict(c["p"])
    q["dec/attn/W_q"] = c["p"]["dec/attn/W_q"] * scale
    c["p"] = q
    assert (keys.abs() > 20.8).float().mean() > 0.3
    assert_local(c, "infer", f"|keys| ~ {scale}", keys=keys)


# ---------------------------------------------------------------------------------------------------------------------
# exact laws, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
def _rows(c, idx):
    d = dict(c)
    d["encoded"], d["tl"], d["mel"] = c["encoded"][idx], c["tl"][idx], c["mel"][idx]
    d["keep"] = tuple(m[:, idx] for m in c["keep"])
    d["sm"] = c["sm"][:, idx]
    if c["h0"] is not None:
        d["h0"], d["att0"] = c["h0"][:, idx], c["att0"][idx]
    return d


@pytest.mark.parametrize("mode", ["infer", "sched"])
def test_row_independence(mode):
    """an utterance decoded in row slot b of a batch equals the same utterance decoded alone"""
    c = case(5, 32, 128, 120, speakers=109)
    full = run(c, mode)
    for b in (0, 13, 31):
        one = run(_rows(c, [b]), mode)
        assert torch.equal(full["y"][b:b + 1], one["y"]) and torch.equal(full["align"][b:b + 1], one["align"]), b
        assert torch.equal(full["H"][:, :, b:b + 1], one["H"]), b


def test_nan_in_one_utterance_leaves_the_others_bit_identical():
    c = case(5, 32, 128, 120)
    base = run(c, "infer")
    enc = c["encoded"].clone()
    enc[11, 0, 5] = float("nan")
    bad = run(c, "infer", encoded=enc)
    others = [b for b in range(32) if b != 11]
    assert torch.equal(base["y"][others], bad["y"][others]) and torch.equal(base["align"][others], bad["align"][others])
    assert torch.equal(base["H"][:, :, others], bad["H"][:, :, others])
    assert torch.isnan(bad["y"][11]).any()


def test_two_runs_give_the_same_bits():
    c = case(5, 32, 128, 200)
    a, b = run(c, "sched"), run(c, "sched")
    for k in ("y", "align", "H"):
        assert torch.equal(a[k], b[k]), k


# ---------------------------------------------------------------------------------------------------------------------
# sensitivity: one weight matrix perturbed before taco_decoder_pack, the float64 reference keeps the original
# ---------------------------------------------------------------------------------------------------------------------
# weight, the (t, stage) where it first enters, and the largest relative perturbation 2^k the check must still flag
# (measured smallest flagged on an H100 80GB HBM3 at 700 W: 2^-18, -15, -18, -16, -18, -18; at those the free-running
# C2 comparison sees at most 1.4e-5 of max|y|, under its 2e-4 bar).  Each weight is scaled by 1 + 2^k, k = -4, -5, ...
# until the check passes.  No flagged run may fail before the weight enters; near the smallest flagged perturbation the
# first failure can sit later than the entry (at h3(1) for Wc3, whose r h half is zero at t = 0; at y(1) for W_a, where
# y's bar is relatively tighter than the gates').
SENSITIVITY = [
    ("dec/gru3/Wc", 0, "h3", -16),
    ("dec/gru1/Wg", 0, "h1", -14),
    ("dec/out_proj/W", 0, "y", -17),
    ("dec/attn/W_q", 0, "align", -14),
    ("dec/attn/W_a", 1, "h1", -16),
    ("dec/attn/v", 0, "align", -16),
]


@pytest.mark.parametrize("name,t,stage,k_max", SENSITIVITY)
def test_sensitivity(name, t, stage, k_max):
    from tests.util import relerr
    c = case(5, 32, 128, 200)
    smallest = None
    for k in range(-4, -31, -1):
        q = dict(c["p"])
        q[name] = c["p"][name] * (1 + 2.0 ** k)
        out = run(c, "infer", p=q)
        f = check(c, "infer", out).first
        if f is None:
            break
        assert (f.t, DC.STAGES.index(f.stage)) >= (t, DC.STAGES.index(stage)), f"{name} x (1 + 2^{k}): {f}"
        if k >= k_max + 8:                          # a perturbation far above the bars: flagged where it enters
            assert (f.t, f.stage) == (t, stage), f"{name} x (1 + 2^{k}): {f}"
        smallest, flagged = k, out
    assert smallest is not None and smallest <= k_max, f"{name}: smallest flagged perturbation 2^{smallest} > 2^{k_max}"
    # what the free-running C2 comparison (test_gpu_model.py: max and mean |diff| <= 2e-4 of the float64 oracle's) sees
    pd = {k_: v.double() for k_, v in c["p"].items()}
    y_ref, a_ref = O.decoder(c["encoded"].double(), c["tl"], pd, ocfg(r=5, T=200, vocab=20), "infer", 200)
    print(f"{name}: smallest flagged 2^{smallest}; free running there: y {relerr(flagged['y'], y_ref)}, "
          f"align {relerr(flagged['align'], a_ref)}")
