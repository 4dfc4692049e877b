"""-m gpu: the persistent decoder backward (taco_decoder_bwd) checked step by step against float64 formed from its own
stored outputs (tests/decoder_bwd_step_checks.py), over the range its ABI accepts.

Every run writes into NaN-poisoned outputs, each inside a guard band of sentinel words: after the run every cell must be
written and no guard word may change.  The carries are read back through DH0 of suffix runs, and every suffix run must
reproduce the full run's outputs at its steps bit for bit (composition).

Cases: the C2 step (B = 32, Tx = 128 ragged, T = 200, r = 5) with teacher forcing, scheduled sampling, the guided
attention's dscore_add and a 109-speaker initial state, on both taco_gemm routes of the folds; r = 1..6; Tx = 1, 7, 67, 129,
256 with lengths that end inside attention quarters; B = 1, 31, 32; T = 1, 2 and 1024; one row group of 32 CTAs (no
weight cache); saturated gates; keys and queries where 1 - e^2 underflows.  Exact laws bit for bit: rows alone and
permuted, NaN isolation, determinism, exact zeros.  The check's sensitivity to one input element.  The limits.

Each check prints its worst |kernel - float64| / bar per quantity.
"""
import math
import time

import pytest
import torch

from tacotron_b200 import _lib as L
from tests import decoder_bwd_step_checks as DB
from tests.test_gpu_decoder_envelope import short_lengths

pytestmark = pytest.mark.gpu
PAD = 1024                      # guard band, words, on each side of every output
SENT = 0x7FA5A5A5               # signalling-NaN bit patterns no arithmetic produces: the guard words,
POISON = 0x7FBADBAD             # and every output cell before the run


def _guarded(shape):
    n = math.prod(shape)
    buf = torch.empty(n + 2 * PAD, dtype=torch.float32, device="cuda")
    buf.view(torch.int32).fill_(SENT)
    body = buf[PAD:PAD + n].view(shape)
    body.view(torch.int32).fill_(POISON)
    return buf, body


def _outputs(a):
    for k in DB.OUTS:
        yield k, None, a[k]
    for k in ("DG", "DC"):
        for i in range(3):
            yield k, i, a[k][i]
    yield "DH0", None, a["DH0"]


def run(a):
    """kernels.decoder_bwd into guarded, poisoned outputs (replacing a's), then the guards and the coverage"""
    from tacotron_b200 import kernels as K
    bufs = []
    for k, i, x in list(_outputs(a)):
        buf, body = _guarded(tuple(x.shape))
        bufs.append((k, i, buf, x.numel()))
        if i is None:
            a[k] = body
        else:
            a[k][i] = body
    K.decoder_bwd(a)
    torch.cuda.synchronize()
    for k, i, buf, n in bufs:
        w = buf.view(torch.int32)
        assert bool((w[:PAD] == SENT).all()) and bool((w[PAD + n:] == SENT).all()), f"{k}{i}: a guard word changed"
        assert not bool((w[PAD:PAD + n] == POISON).any()), f"{k}{i}: cells left unwritten"


def args(r, B, Tx, T, **kw):
    a = DB.make_args(r, B, Tx, T, device="cuda", **kw)
    if kw.get("ga"):                               # dscore_add from the library's own guided-attention kernel
        from tacotron_b200 import kernels as K
        g = torch.Generator().manual_seed(11)
        steps = torch.randint(max(1, T // 2), T + 1, (B,), generator=g).to(torch.int32).cuda()
        dsa = torch.empty(B, T, Tx, device="cuda")
        K.guided_attention(dsa, torch.empty(1, device="cuda"), a["align"], a["text_length"].cuda(), steps, 0.2, 10.0)
        a["dscore_add"] = dsa
    return a


def exact_zeros(a, what):
    T, B = a["dy_ext"].shape[:2]
    Tx = a["align"].shape[2]
    if a.get("dscore_add") is None:
        past = torch.arange(Tx, device="cuda")[None, None, :] >= a["text_length"].cuda()[:, None, None].long()
        assert bool((a["DSCORE"][past.expand(B, T, Tx)] == 0).all()), f"{what}: DSCORE past text_length"
    assert bool((a["DPN1"][a["PN1"] <= 0] == 0).all()), f"{what}: DPN1 where PN1 <= 0"
    assert bool((a["DPN2"][a["PN2"] <= 0] == 0).all()), f"{what}: DPN2 where PN2 <= 0"
    assert bool((a["DATT"][T - 1] == 0).all()) and bool((a["DCTX"][T - 1] == 0).all()), f"{what}: DATT / DCTX (T-1)"


def assert_local(a, what, steps=None, route=0):
    from tacotron_b200 import kernels as K
    prev = K.set_gemm_impl(route)
    try:
        t0 = time.perf_counter()
        run(a)
        exact_zeros(a, what)
        T = a["dy_ext"].shape[0]
        carry, mism = DB.read_carries(run, a, range(T) if steps is None else steps)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
    finally:
        K.set_gemm_impl(prev)
    assert not mism, f"{what}: suffix runs differ from the full run: {mism[:4]}"
    rep = DB.check(a, carry, route=route, steps=steps)
    print(f"{what}: {rep} (kernel + {len(carry) - 1} suffix runs {t1 - t0:.1f} s, check {time.perf_counter() - t1:.1f} s)")
    assert rep.first is None, f"{what}: {rep.first}"
    return rep


# ---------------------------------------------------------------------------------------------------------------------
# the C2 step, both routes of the folds and the tail
# ---------------------------------------------------------------------------------------------------------------------
C2 = dict(teacher=dict(sched=False), sched=dict(), ga=dict(ga=True), speakers=dict(speakers=109))


@pytest.mark.parametrize("route", [0, 1])
@pytest.mark.parametrize("name", list(C2))
def test_c2(name, route):
    assert_local(args(5, 32, 128, 200, **C2[name]), f"C2 {name} route {route}", route=route)


def test_c2_from_a_forward_run():
    """the arguments grad.decoder_bwd builds from an fp32 decoder forward (scheduled sampling, dropout)"""
    from tacotron_b200.models import grad
    from tests import grad_util, mirror_kernels as MK
    from tests.test_gpu_decoder_envelope import _setup
    cfg, p, encoded, mel, tl, dec_m, sm = _setup(5, 32, 128, 200)
    S = {"mel": mel, "text_length": tl, "dec/keep1": dec_m[0], "dec/keep2": dec_m[1], "_capture": {}, "dec/sample_mask": sm}
    grad_util.decoder_saving(encoded, tl, p, cfg, 200, mel, dec_m, sm, S)
    grad.decoder_bwd(MK, p, {k: torch.zeros_like(v) for k, v in p.items()}, S, cfg,
                     torch.randn(32, 200, 400, generator=torch.Generator().manual_seed(5)))
    cap = {k: v for k, v in S["_capture"]["decoder_bwd"].items() if not k.startswith("_")}
    a = {k: ([t.cuda().contiguous() for t in v] if isinstance(v, list) else v.cuda().contiguous() if torch.is_tensor(v) else v)
         for k, v in cap.items()}
    a["DH0"] = torch.empty(3, 32, 256, device="cuda")
    assert_local(a, "C2 from a forward run")


# ---------------------------------------------------------------------------------------------------------------------
# r, Tx, B, T, the grid
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("r", [1, 2, 3, 4, 5, 6])
def test_r(r):
    assert_local(args(r, 9, 37, 40), f"r={r}")


@pytest.mark.parametrize("Tx", [1, 7, 67, 129, 256])
def test_tx(Tx):
    """the Tx % 8 and Tx % 32 tails of stage A, lengths inside attention quarters"""
    assert_local(args(5, 32, Tx, 40, lengths=short_lengths(Tx, 32)), f"Tx={Tx}")


@pytest.mark.parametrize("B", [1, 31, 32])
def test_batch(B):
    assert_local(args(5, B, 64, 50), f"B={B}")


@pytest.mark.parametrize("T", [1, 2])
def test_short(T):
    assert_local(args(5, 32, 64, T, speakers=109), f"T={T}")


def test_longest():
    """T = 1024, the workspace's last E row: every step"""
    assert_local(args(5, 32, 128, 1024), "T=1024")


def test_one_row_group_without_weight_cache():
    a = args(5, 32, 128, 200)
    a["max_ctas"] = 32
    assert_local(a, "C2 max_ctas=32")


# ---------------------------------------------------------------------------------------------------------------------
# magnitudes
# ---------------------------------------------------------------------------------------------------------------------
def test_saturated_gates():
    """u, r -> 0 or 1 and |c| -> 1: the carries cannot be recovered from DG / DC there"""
    a = args(5, 32, 128, 200, gate_scale=8.0)
    sat = (a["RU"][0] < 1e-3) | (a["RU"][0] > 1 - 1e-3)
    assert sat.float().mean() > 0.5
    assert_local(a, "saturated gates")


def test_one_minus_e2_underflows():
    """keys and queries large enough that tanh(k + q) rounds to +-1: 1 - e^2 is exactly 0 in fp32"""
    a = args(5, 32, 128, 100, key_scale=40.0)
    assert (a["keys"].abs() > 10).float().mean() > 0.3
    assert_local(a, "|keys| ~ 40")


# ---------------------------------------------------------------------------------------------------------------------
# exact laws, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
BATCHED = ("align", "values", "keys", "dscore_add", "DSCORE", "text_length")


def _rows(a, idx):
    idx_t = torch.as_tensor(idx, device="cuda")
    d = {}
    for k, v in a.items():
        if k.startswith("_") or not (torch.is_tensor(v) or isinstance(v, list)):
            d[k] = v
        elif k in ("Wg", "Wc") or k in ("W_a", "W_q", "W_out", "W_in", "W1", "W2", "v"):
            d[k] = v
        elif k == "H0":
            d[k] = [x[idx_t].contiguous() for x in v]
        elif isinstance(v, list):
            d[k] = [x[:, idx_t].contiguous() for x in v]
        elif k in BATCHED:
            d[k] = v[idx_t.to(v.device)].contiguous()
        elif k == "DH0":
            d[k] = v[:, idx_t].contiguous()
        else:
            d[k] = v[:, idx_t].contiguous()
    return d


def _same(a, b, idx):
    idx_t = torch.as_tensor(idx, device="cuda")
    sub = _rows(a, idx)
    for k, i, x in _outputs(b):
        y = sub[k] if i is None else sub[k][i]
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), (k, i, idx)


def test_rows_alone_and_permuted():
    a = args(5, 32, 128, 120, speakers=109, ga=True)
    run(a)
    for idx in ([0], [13], [31], [3, 7, 30]):
        d = _rows(a, idx)
        run(d)
        _same(a, d, idx)
    perm = torch.randperm(32, generator=torch.Generator().manual_seed(3)).tolist()
    d = _rows(a, perm)
    run(d)
    _same(a, d, perm)


def test_nan_in_one_row_stays_there():
    a = args(5, 32, 128, 120)
    run(a)
    d = _rows(a, list(range(32)))
    d["dy_ext"][60, 11, 5] = float("nan")
    run(d)
    others = [b for b in range(32) if b != 11]
    _same(_rows(a, others), _rows(d, others), list(range(31)))
    assert torch.isnan(d["DZ"][:, 11]).any()


def test_two_runs_give_the_same_bits():
    a = args(5, 32, 128, 200, ga=True)
    run(a)
    d = _rows(a, list(range(32)))
    run(d)
    _same(a, d, list(range(32)))


def test_limits():
    from tacotron_b200 import kernels as K
    a = args(1, 2, 8, 1025)
    with pytest.raises(L.TacoError, match="T=1025 exceeds 1024 steps per launch"):
        K.decoder_bwd(a)
    a = args(1, 33, 8, 4)
    with pytest.raises(L.TacoError, match=r"B=33 must be in \[1,32\] per launch"):
        K.decoder_bwd(a)


# ---------------------------------------------------------------------------------------------------------------------
# sensitivity: one element of one input perturbed for the kernel only, the float64 reference keeps the original
# ---------------------------------------------------------------------------------------------------------------------
# input, its element (list index or None, t, b, n), and the (t, stage) where it first enters.  Each element is scaled by
# 1 + 2^k, k = -4, -5, ... until the check passes; no flagged run may fail before the entry, and far above the smallest
# flagged perturbation the first failure is the entry itself.  Measured smallest flagged on an H100 80GB HBM3 at 700 W:
# RU 2^-16, C 2^-18, H 2^-17, PQ 2^-12 (PQ enters through the sum over Tx of 1 - e^2, which a relative change moves least).
SENSITIVITY = [
    ("RU", (2, 150, 7, 256 + 40), (150, "du3"), -12),
    ("C", (1, 150, 7, 40), (150, "du2"), -12),
    ("H", (0, 149, 7, 40), (150, "du1"), -12),
    ("PQ", (None, 150, 7, 40), (150, "dpq"), -12),
]


@pytest.mark.parametrize("name,el,entry,k_max", SENSITIVITY)
def test_sensitivity(name, el, entry, k_max):
    base = args(5, 32, 128, 200)
    i, t, b, n = el
    steps = sorted({entry[0] - 1, entry[0], entry[0] + 1})
    smallest = None
    for k in range(-4, -31, -1):
        a = _rows(base, list(range(32)))
        x = a[name] if i is None else a[name][i]
        orig = x.clone()
        x[t, b, n] = x[t, b, n] * (1 + 2.0 ** k)
        run(a)
        carry, _ = DB.read_carries(run, a, steps, compose=False)
        if i is None:
            a[name] = orig
        else:
            a[name][i] = orig
        f = DB.check(a, carry, steps=steps).first
        if f is None:
            break
        assert (-f.t, DB.STAGES.index(f.stage)) >= (-entry[0], DB.STAGES.index(entry[1])), f"{name} x (1 + 2^{k}): {f}"
        if k >= k_max + 8:
            assert (f.t, f.stage) == entry, f"{name} x (1 + 2^{k}): {f}"
        smallest = k
    print(f"{name}{el}: smallest flagged 2^{smallest}")
    assert smallest is not None and smallest <= k_max, f"{name}: smallest flagged perturbation 2^{smallest} > 2^{k_max}"


def test_a_relu_mask_flip_is_flagged_where_it_enters():
    base = args(5, 32, 128, 200)
    a = _rows(base, list(range(32)))
    t, b = 120, 4
    n = int((a["PN1"][t, b] > 0).nonzero()[0, 0])
    a["PN1"][t, b, n] = 0.0
    run(a)
    carry, _ = DB.read_carries(run, a, [t - 1, t, t + 1], compose=False)
    a["PN1"] = base["PN1"]
    f = DB.check(a, carry, steps=[t - 1, t, t + 1]).first
    assert f is not None and (f.t, f.stage, f.b, f.unit) == (t, "dpn1", b, n), str(f)
