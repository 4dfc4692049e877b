"""CPU: the step-by-step check of the decoder backward (tests/decoder_bwd_step_checks.py) on the float64 mirror and on the
kernel itself under the host emulation (tests/cuda_emu, the one-CTA build tests/test_cuda_emu.py also drives): the
mirror shows float64-level ratios, the emulated kernel passes, suffix runs compose bit for bit, one corrupted stored
element is reported at exactly its (t, stage, b, unit), a fold rounded to TF32 is flagged where it is first used, and
the bars of one small case match a hand restatement."""
import math

import pytest
import torch

from tests import decoder_bwd_step_checks as DB
from tests import mirror_kernels_guided as MKG
from tests.emulator import KernelsOver, emu  # noqa: F401  (the emulated library, built once per process)


def _mirror(a):
    MKG.decoder_bwd(a)


def _emu_run(lib):
    """kernels.decoder_bwd over the emulated library, on CPU tensors (the workspace is kept in a['_ws'])"""
    return KernelsOver(lib).decoder_bwd


def test_workspace_layout(emu):  # noqa: F811
    assert emu.taco_decoder_bwd_workspace_bytes() == DB.WS_TOTAL * 4


@pytest.mark.parametrize("kw", [dict(), dict(sched=False), dict(speakers=109, ga=True), dict(gate_scale=6.0)],
                         ids=["sched", "teacher", "speakers+ga", "saturated"])
def test_float64_mirror_passes_at_float64_level(kw):
    a = DB.make_args(3, 4, 11, 7, dtype=torch.float64, **kw)
    _mirror(a)
    carry, _ = DB.read_carries(_mirror, a, range(7), compose=False)
    rep = DB.check(a, carry, exact_folds=True)
    assert rep.first is None, str(rep)
    assert max(rep.worst.values()) < 1e-4, str(rep)            # fp32 kernels sit near 1


@pytest.mark.parametrize("r,B,Tx,T,kw", [(2, 3, 9, 5, dict()), (1, 2, 7, 4, dict(speakers=109, ga=True)),
                                         (6, 2, 12, 3, dict(sched=False)), (3, 1, 1, 2, dict())])
def test_emulated_kernel_passes_and_suffixes_compose(emu, r, B, Tx, T, kw):  # noqa: F811
    run = _emu_run(emu)
    a = DB.make_args(r, B, Tx, T, **kw)
    run(a)
    carry, mism = DB.read_carries(run, a, range(T))
    assert not mism, f"suffix runs differ from the full run: {mism}"
    rep = DB.check(a, carry)
    print(rep)
    assert rep.first is None, str(rep)


@pytest.fixture(scope="module")
def small_run(emu):  # noqa: F811
    run = _emu_run(emu)
    a = DB.make_args(2, 3, 9, 5)
    run(a)
    carry, _ = DB.read_carries(run, a, range(5))
    return a, carry


@pytest.mark.parametrize("where", [
    ("DSCORE", 3, 1, 4, "dscore"), ("DPQ", 2, 0, 17, "dpq"), ("DC", 2, 4, 2, 200, "dc3"), ("DG", 1, 3, 1, 300, "du2"),
    ("DG", 0, 1, 0, 5, "dr1"), ("DZ", 0, 2, 100, "dz"), ("DPN2", 4, 2, 64, "dpn2"), ("DATT", 2, 1, 7, "datt"),
    ("DCTX", 0, 0, 255, "dctx"), ("DPN1", 3, 1, 9, "dpn1"), ("DX", 1, 2, 79, "dx"), ("DY", 4, 0, 3, "dy")],
    ids=lambda w: f"{w[0]}{'' if len(w) == 5 else w[1]}")
def test_one_corrupted_element_is_reported_where_it_sits(small_run, where):
    a0, carry = small_run
    a = {k: ([x.clone() for x in v] if isinstance(v, list) else v.clone() if torch.is_tensor(v) else v) for k, v in a0.items()}
    if len(where) == 6:
        name, i, t, b, n, stage = where
        x = a[name][i]
    else:
        name, t, b, n, stage = where
        x = a[name]
    idx = (b, t, n) if name == "DSCORE" else (t, b, n)
    x[idx] = x[idx] * (1 + 2.0 ** -12) + 1e-9
    rep = DB.check(a, carry)
    t_rep = t + 1 if name in ("DATT", "DCTX") else t            # DATT(t), DCTX(t) are formed in stage 7' of step t + 1
    f = rep.first
    unit = n - 256 if stage.startswith("du") else n             # du_pre is the second half of DG
    assert f is not None and (f.t, f.stage, f.b, f.unit) == (t_rep, stage, b, unit), str(rep)


def test_corrupted_carry_is_reported_at_its_step(small_run):
    a, carry0 = small_run
    carry = dict(carry0)
    carry[1] = carry0[1].clone()
    carry[1][1, 2, 33] *= 1 + 2.0 ** -8
    f = DB.check(a, carry).first
    assert f is not None and (f.t, f.stage, f.b, f.unit) == (2, "carry2", 2, 33), str(f)


@pytest.mark.parametrize("fold,stage", [("M124", "M124"), ("M7", "M7")])
def test_fold_rounded_to_tf32_is_flagged_where_first_used(small_run, fold, stage):
    a0, carry = small_run
    a = dict(a0)
    ws = a0["_ws"].clone()
    lo, hi = (DB.WS_M124, DB.WS_M7) if fold == "M124" else (DB.WS_M7 + 384 * DB.UNITS, DB.WS_E)
    ws[lo:hi] = (ws[lo:hi].view(torch.int32) & ~0x1FFF).view(torch.float32)        # TF32: 10 mantissa bits
    a["_ws"] = ws
    f = DB.check(a, carry).first
    T = a["dy_ext"].shape[0]
    assert f is not None and f.t == T - 1 and f.stage == stage, str(f)


def test_bars_match_a_hand_restatement(small_run):
    """dpn1 and dr3 of one element, restated from the formulas of the module docstring"""
    a, carry = small_run
    rep = DB.check(a, carry)
    t, b, n = 2, 1, 7
    u, c, ks = 2.0 ** -24, DB.C_PROD, float(a["keep_scale"])
    d2 = a["DPN2"][t, b].double()
    W2 = a["W2"].double()
    p1 = float(d2 @ W2[n])
    rss = math.sqrt(float((d2 * d2) @ (W2[n] * W2[n])))
    bar = c * u * ks * (math.sqrt(128 / 16) * rss + 2 * abs(p1)) if a["PN1"][t, b, n] > 0 else 0.0
    got = float(a["DPN1"][t, b, n])
    want = ks * p1 if a["PN1"][t, b, n] > 0 else 0.0
    r = 0.0 if got == want else abs(got - want) / (bar + DB.FLUSH)
    assert math.isclose(float(rep.ratio["dpn1"][t, b, n]), r, rel_tol=1e-6, abs_tol=1e-12)   # (the difference cancels: float64 order)
    # dr3 = drh h(t-1) r (1 - r),  drh = DC3(t) . Wc3_h^T
    dc = a["DC"][2][t, b].double()
    Wh = a["Wc"][2].double()[256 + n]
    drh = float(dc @ Wh)
    e_drh = c * u * (math.sqrt(256 / 16) * math.sqrt(float((dc * dc) @ (Wh * Wh))) + abs(drh))
    rr = float(a["RU"][2][t, b, n])
    hp = float(a["H"][2][t - 1, b, n])
    g = hp * rr * (1 - rr)
    bar = abs(g) * e_drh + c * u * 4 * abs(drh * g) + DB.FLUSH
    got = float(a["DG"][2][t, b, n])
    r = 0.0 if got == drh * g else abs(got - drh * g) / bar
    assert math.isclose(float(rep.ratio["dr3"][t, b, n]), r, rel_tol=1e-6, abs_tol=1e-12)   # (the difference cancels: float64 order)
