"""-m gpu: the fused CBHG highway stack (taco_highway_stack_fwd: width-fixing dense + 4 highway layers + the bi-GRU input
products in one kernel) against the unfused sequence (ops.linear dense + ops.highway x 4 + the xp ops.linear), bit for
bit, on random weights; and CBHG's inference route through it against its layer-by-layer route."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _store(cin, seed, K=4):
    """a CBHG's variables (params.cbhg_shapes, scope 'cbhg'), filled with random weights and non-zero biases"""
    from tacotron_b200.params import ParamStore, cbhg_shapes
    shapes = cbhg_shapes("cbhg", cin, K, [128, 128, cin])
    st = ParamStore(shapes, "cuda")
    g = torch.Generator().manual_seed(seed)
    for n, (s, kind) in st.shapes.items():
        if kind in ("dense", "conv"):
            fan_in = s[0] if kind == "dense" else s[0] * s[1]
            t = torch.randn(s, generator=g) / fan_in ** 0.5
        elif kind == "var":
            t = torch.rand(s, generator=g) + 0.5
        else:
            t = 0.5 * torch.randn(s, generator=g)
        st.views[n].copy_(t)
    st.version += 1
    return st


def _unfused(ops, rt, sc, x, n_hw):
    h = x
    for l in range(n_hw):
        h = ops.highway(h, scope=sc.sub(f"highway{l}"))
    Wx, bx, Wxp = ops._gru_input_weights(rt, sc)
    return ops.linear(rt, h, Wx, Wxp, 768, bias=bx, tag="ref_xp").clone()


@pytest.mark.parametrize("B,T,C", [
    (32, 1000, 80),      # post-net at the C2 shape (32 x 200 frames x r = 5)
    (32, 128, 128),      # encoder at the C2 shape
    (3, 997, 80), (3, 997, 128),   # rows not a multiple of the 128-row tile
    (1, 1, 80), (1, 1, 128),       # a single row
    (1, 500, 80), (1, 140, 128),   # B = 1 at the C5 shape (T r = 500, Tx = 140)
])
def test_fused_matches_unfused_bitwise(B, T, C):
    from tacotron_b200.models import ops
    st = _store(C, seed=B * 7919 + T + C)
    rt = ops.runtime(st, "fp32x3")
    x = torch.randn(B, T, C, generator=torch.Generator().manual_seed(T), device="cpu").cuda()
    sc = ops.Scope(st, "cbhg")
    ref = _unfused(ops, rt, sc, x, 4)
    got = ops.highway_stack(x, 4, scope=sc).clone()
    torch.cuda.synchronize()
    assert got.shape == (B, T, 768)
    assert torch.isfinite(ref).all()
    diff = (got.view(torch.int32) != ref.view(torch.int32)).sum().item()
    assert diff == 0, f"{diff} of {ref.numel()} elements differ; max |d| = {(got - ref).abs().max().item():.3e}"


def test_fused_leaves_nothing_but_xp():
    """rows past M are neither read nor written: the elements around the output stay as they were"""
    from tacotron_b200.models import ops
    st = _store(128, seed=5)
    rt = ops.runtime(st, "fp32x3")
    sc = ops.Scope(st, "cbhg")
    x = torch.randn(2, 70, 128, device="cuda")
    ref = _unfused(ops, rt, sc, x, 4)
    big = torch.full((3 * 70 * 768,), 7.0, device="cuda")
    out = big[:2 * 70 * 768].view(2, 70, 768)
    rt.scratch[(sc.name("xp"), (2, 70, 768), torch.float32)] = out     # make highway_stack write into a known buffer
    got = ops.highway_stack(x, 4, scope=sc)
    torch.cuda.synchronize()
    assert got.data_ptr() == out.data_ptr()
    assert torch.equal(got, ref)
    assert (big[2 * 70 * 768:] == 7.0).all()


@pytest.mark.parametrize("B,T,C", [(4, 300, 80), (4, 96, 128)])
def test_cbhg_inference_route_matches_layer_by_layer(B, T, C):
    """CBHG takes the fused route at inference (fp32x3, no trace); a traced call keeps the layer-by-layer route: the
    outputs of both are the same bits"""
    from tacotron_b200 import _lib as L
    from tacotron_b200.models import ops
    st = _store(C, seed=C + T)
    ops.runtime(st, "fp32x3")
    x = torch.randn(B, T, C, device="cuda")
    with ops.variable_scope(st, ""):
        ops.CBHG(x, K=4, c=[128, 128, C])                       # packs the weights once (not counted below)
        n0 = L.lib().taco_launch_count()
        fused = ops.CBHG(x, K=4, c=[128, 128, C]).clone()
        n_fused = L.lib().taco_launch_count() - n0
        n0 = L.lib().taco_launch_count()
        trace = {}
        layered = ops.CBHG(x, K=4, c=[128, 128, C], trace=trace).clone()
        n_layered = L.lib().taco_launch_count() - n0
    torch.cuda.synchronize()
    assert torch.equal(fused, layered)
    # the layered route: (dense) + 4 highway + xp = 5 or 6 launches; the fused route: 1
    assert n_layered - n_fused == (5 if C == 128 else 6) - 1
