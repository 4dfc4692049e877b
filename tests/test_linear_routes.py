"""Which kernel instantiation and epilogue taco_linear_fwd launches, as the library itself reports it
(taco_linear_route: host only, no GPU).  Pins the dispatch conditions at their boundaries, the argument checks, and
that the GPU envelope (tests/test_gpu_linear_envelope.py) runs every instantiation x epilogue x epilogue-field
combination the dispatcher allows."""
import pytest

from tacotron_b200 import _lib as L
from tests.linear_envelope_cases import CASES, FEATURES, TC_IMPLS, Case, check_route, instantiation, route


def _route(impl="fp32x3", **kw):
    kw.setdefault("name", "probe")
    return route(Case(**kw), impl)


# ------------------------------------------------------------------------------------------------------------------
# pinned routes
# ------------------------------------------------------------------------------------------------------------------
def test_bn32_at_the_33_tile_boundary():
    # fp32x3 takes 32-column n-tiles when (m-tiles x 128-column n-tiles) <= 132 / 4 = 33 and N >= 64
    assert _route(B=33, T=128, C=256, N=128)[:2] == (32, 6)
    assert _route(B=34, T=128, C=256, N=128)[:2] == (128, 2)
    assert _route(B=11, T=384, C=256, N=128)[:2] == (32, 6)           # 3 m-tiles per utterance
    assert _route(B=11, T=385, C=256, N=128)[:2] == (128, 2)          # 4
    assert _route(B=16, T=128, C=256, N=256)[:2] == (32, 6)           # 2 n-tiles: 32 tiles
    assert _route(B=17, T=128, C=256, N=256)[:2] == (128, 2)          # 34
    assert _route(B=1, T=300, C=256, N=1025)[:2] == (32, 6)           # the post dense of one utterance: 27 tiles
    assert _route(B=32, T=128, C=2048, N=128, taps=3)[:2] == (32, 6)  # the encoder-side long-K conv projection


def test_bn32_needs_n64_and_fp32x3_plain():
    assert _route(B=1, T=128, C=32, N=64)[:2] == (32, 6)
    assert _route(B=1, T=128, C=32, N=63)[:2] == (128, 2)
    assert _route(B=1, T=128, C=32, N=64, pool=True)[:2] == (128, 2)
    assert _route(B=1, T=128, C=32, N=256, bank_K=2)[:2] == (128, 2)
    assert _route(B=1, T=128, C=128, N=256, highway=True)[:3] == (256, 2, 1)
    assert _route("tf32", B=1, T=128, C=32, N=64)[:2] == (128, 2)


def test_tf32_ring_depth_at_8_and_9_k_iterations():
    assert _route("tf32", B=64, T=1000, C=256, N=128)[:2] == (128, 2)           # 8 k-chunks
    assert _route("tf32", B=64, T=1000, C=257, N=128)[:2] == (128, 3)           # 9
    assert _route("tf32", B=64, T=1000, C=64, N=128, taps=4)[:2] == (128, 2)    # 4 taps x 2 chunks
    assert _route("tf32", B=64, T=1000, C=96, N=128, taps=3)[:2] == (128, 3)    # 3 taps x 3 chunks
    assert _route("tf32", B=2, T=100, C=32, N=128, bank_K=1)[:2] == (128, 3)    # banks always take the 3-stage ring
    assert _route("tf32", B=2, T=100, C=128, N=256, highway=True)[:3] == (256, 2, 1)
    assert _route("fp32x3", B=64, T=1000, C=257, N=128)[:2] == (128, 2)


@pytest.mark.parametrize("direct,transposing", [
    (dict(), dict(transposing="ldy")),                                       # ldy % 4 != 0
    (dict(), dict(transposing="y_align")),                                   # Y not 16-byte aligned
    (dict(), dict(N=126)),                                                   # N % 4 != 0
    (dict(residual=True), dict(residual=True, transposing="ldr")),           # ldr % 4 != 0
    (dict(keep=True, N=112), dict(keep=True, N=120)),                        # keep needs N % 16 == 0
    (dict(N=256, highway=True), dict(N=256, highway=True, transposing="ldhx")),
    (dict(N=256, highway=True), dict(N=256, highway=True, transposing="ldy")),   # highway: ldy against U = 128
    (dict(pool=True), dict(pool=True, transposing="y_align")),
    (dict(N=256, bank_K=2, pool=True), dict(N=256, bank_K=2, pool=True, transposing="ldy")),
])
def test_direct_or_transposing_epilogue(direct, transposing):
    base = dict(B=4, T=300, C=128, N=128)
    for impl in TC_IMPLS:
        assert _route(impl, **{**base, **direct})[3] == 1
        assert _route(impl, **{**base, **transposing})[3] == 0


def test_direct_epilogue_alignment_conditions():
    """Alignment of each operand the register-direct epilogue touches with 16-byte vectors."""
    from tests.linear_envelope_cases import Layout, desc, stand_in_addresses
    for field, kw in (("Y", {}), ("residual", dict(residual=True)), ("hx", dict(highway=True, N=256)),
                      ("keep", dict(keep=True))):
        c = Case(name="align", **{**dict(B=2, T=50, C=128, N=128), **kw})
        lay = Layout(c)
        a = stand_in_addresses(c, lay)
        assert L.linear_route(desc(c, "tf32", a, lay))[3] == 1
        a[field] += 4 if field != "keep" else 8
        assert L.linear_route(desc(c, "tf32", a, lay))[3] == 0, field


def test_pool_tile_stride_and_simt_route():
    assert _route("tf32", B=3, T=381, C=80, N=128, taps=3, pool=True)[4] == 127
    assert _route("fp32x3", B=3, T=381, C=80, N=1024, bank_K=8, pool=True)[4] == 127
    assert _route("tf32", B=3, T=381, C=80, N=128, taps=3)[4] == 128
    assert _route("fp32", B=3, T=381, C=80, N=128, taps=3) == (64, 1, 0, 0, 64)
    assert _route("fp32", B=3, T=381, C=128, N=256, highway=True) == (64, 1, 1, 0, 64)


# ------------------------------------------------------------------------------------------------------------------
# argument checks: a stride too small for its row would make the kernel overwrite / read the next row
# ------------------------------------------------------------------------------------------------------------------
def _rejected(impl, field, value, msg, **kw):
    """field may be one name or several ("residual+ldr") set to the same value"""
    from tests.linear_envelope_cases import Layout, desc, stand_in_addresses
    kw.setdefault("B", 2); kw.setdefault("T", 10); kw.setdefault("C", 32); kw.setdefault("N", 128)
    c = Case(name="bad", **kw)
    lay = Layout(c)
    d = desc(c, impl, stand_in_addresses(c, lay), lay)
    L.linear_route(d)                                            # the descriptor itself is accepted
    for f in field.split("+"):
        setattr(d, f, value)
    with pytest.raises(L.TacoError, match=msg):
        L.linear_route(d)


@pytest.mark.parametrize("impl", ["fp32", "tf32", "fp32x3"])
def test_stride_checks(impl):
    _rejected(impl, "ldy", 127, r"ldy 127 < 128")
    _rejected(impl, "ldy", 127, r"ldy 127 < 128", N=256, C=128, highway=True)
    _rejected(impl, "ldr", 100, r"ldr 100 < N 128", residual=True)
    _rejected(impl, "ldhx", 124, r"ldhx 124 < U 128", N=256, C=128, highway=True)
    _rejected(impl, "ldbu", 127, r"ldbu >= N", bias_utt=True)
    _rejected(impl, "ldx", 31, r"ldx < C")


def test_field_checks():
    _rejected("fp32", "pool", 1, r"SIMT\): fused max-pool")
    for impl in ("fp32", "tf32", "fp32x3"):
        for field in ("keep", "residual+ldr", "scale"):
            _rejected(impl, field, 1 << 40, r"highway epilogue takes only bias and hx", N=256, C=128, highway=True)
        _rejected(impl, "act", L.ACT_RELU, r"highway epilogue takes only bias and hx", N=256, C=128, highway=True)
    for impl in TC_IMPLS:
        _rejected(impl, "keep", 1 << 40, r"pool cannot be combined", pool=True)
        _rejected(impl, "ldwp", 32, r"ldwp too small", taps=3)
        _rejected(impl, "ldx", 33, r"multiples of 4 floats", C=32)


# ------------------------------------------------------------------------------------------------------------------
# the GPU envelope's case list
# ------------------------------------------------------------------------------------------------------------------
def test_envelope_cases_take_their_intended_routes():
    names = [c.name for c in CASES]
    assert len(names) == len(set(names))
    for c in CASES:
        for impl in c.impls:
            check_route(c, impl, route(c, impl))


def _combos(case_list):
    got = set()
    for c in case_list:
        for impl in c.impls:
            if impl == "fp32":
                continue
            try:
                r = route(c, impl)
            except L.TacoError:
                continue
            for f in c.features():
                got.add(instantiation(impl, r) + (r[3], f))
    return got


def test_envelope_covers_every_route_the_dispatcher_allows():
    """Probe the dispatcher with every epilogue field on both layouts over shapes that reach each condition, and
    require the envelope to run each (instantiation, direct/transposing, field) the library accepts."""
    probes = [dict(B=1, T=1, C=32, N=64), dict(B=1, T=1, C=32, N=48), dict(B=64, T=1000, C=256, N=128),
              dict(B=64, T=1000, C=257, N=128), dict(B=3, T=129, C=33, N=80, taps=7), dict(B=32, T=128, C=2048, N=128, taps=3),
              dict(B=33, T=128, C=256, N=128), dict(B=34, T=128, C=256, N=128), dict(B=2, T=300, C=80, N=512, bank_K=4),
              dict(B=1, T=40000, C=128, N=256, highway=True)]
    feats = {"plain": {}, "keep": dict(keep=True), "residual": dict(residual=True), "pool": dict(pool=True),
             "bias_utt": dict(bias_utt=True)}
    assert set(feats) == set(FEATURES)
    probe_cases = [Case(name="probe", **p, **fk, transposing=tr, impls=TC_IMPLS)
                   for p in probes for fk in feats.values() for tr in ("", "ldy")]
    allowed = _combos(probe_cases)
    covered = _combos(CASES)
    # six instantiations: fp32x3 {32/6, 128/2, highway 256/2}, tf32 {128/2, 128/3, highway 256/2}
    assert {k[:4] for k in allowed} == {("fp32x3", 32, 6, 0), ("fp32x3", 128, 2, 0), ("fp32x3", 256, 2, 1),
                                        ("tf32", 256, 2, 1), ("tf32", 128, 2, 0), ("tf32", 128, 3, 0)}
    missing = sorted(allowed - covered)
    assert not missing, f"routes the envelope never runs: {missing}"


def test_envelope_grid_reaches_the_listed_edges():
    cs = CASES
    assert {1, 8, 31, 32, 33, 80, 128, 256, 1024, 2048} <= {c.C for c in cs}
    assert {8, 48, 80, 128, 256, 768, 1025} <= {c.N for c in cs}
    assert {1, 2, 127, 128, 129, 255, 256, 257, 1000} <= {c.T for c in cs}
    assert {1, 3, 32} <= {c.B for c in cs}
    assert {1, 2, 3, 4, 5, 7} <= {c.taps for c in cs}
    assert any(c.taps > c.T and c.B > 1 for c in cs)
    assert {"tf", "zero", "left"} <= {c.tap0 for c in cs if c.taps > 1}
    assert {L.ACT_NONE, L.ACT_RELU, L.ACT_SIGMOID, L.ACT_TANH} <= {c.act for c in cs}
    assert {N % 32 for c in cs if c.keep and not c.transposing for N in [c.N]} >= {0, 16}
    assert any(c.keep and c.N % 16 for c in cs)
    assert {1, 2, 4, 8, 16} <= {c.bank_K for c in cs if c.pool}
    assert {1, 2, 126, 127, 128, 129, 253, 254, 255, 256, 381} <= {c.T for c in cs if c.pool and not c.bank_K}
    assert {1, 2, 126, 127, 128, 129, 253, 254, 255, 256, 381} <= {c.T for c in cs if c.pool}
    assert {1, 127, 128, 129, 40000} <= {c.B * c.T for c in cs if c.highway}
    assert all("fp32" not in c.impls for c in cs if c.pool)
