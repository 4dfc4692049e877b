"""-m gpu: the configuration bench.py times, end to end: Tacotron.inference with precision 'fp32x3', CUDA graphs and the
default features (no attention window, no stop rule), at the C2 shape (B = 32, Tx = 128 ragged, T = 200, r = 5) and the
C5 shape (B = 1, Tx = 140, T = 500), with trained-like oracle weights.
  * graph replay == eager untraced call == traced call, bit for bit.  The untraced calls take the fused highway stack
    (one taco_highway_stack_fwd per CBHG), the traced call the layer-by-layer route: 9 launches more (the encoder's
    4 highway layers + xp against 1, the post-net's dense + 4 highway layers + xp against 1);
  * seq2seq_output, alignments and output are within 2e-4 (max and mean, tests/util.assert_close) of the float64 oracle
    run on the same float32 parameter values, for the batch that captured the graphs and for a second batch replayed
    through them;
  * after load_params with a second parameter set the replay equals a fresh model with those parameters, bit for bit."""
from types import SimpleNamespace

import pytest
import torch

from oracle import tacotron_oracle as O
from tacotron_b200 import Config, Tacotron
from tacotron_b200 import _lib as L
from tacotron_b200 import kernels as K
from tests.bwd_tc_envelope_checks import recording
from tests.util import assert_close, to_cuda

pytestmark = pytest.mark.gpu
TOL = 2e-4
SHAPES = {"C2": (32, 128, 200, True), "C5": (1, 140, 500, False)}
LAYERED_EXTRA = (4 + 1 - 1) + (1 + 4 + 1 - 1)     # encoder CBHG (C = 128) + post-net CBHG (C = 80)


def _model(T, params):
    m = Tacotron(Config(r=5, vocab_size=64, max_decode_iter=T, precision="fp32x3", cuda_graph=True), None, train=False)
    m.load_params(params)
    return m


def _oracle(p, inp, cfg):
    return O.inference({k: v.double() for k, v in p.items()}, inp, cfg, train=False)


@pytest.fixture(scope="module", params=list(SHAPES))
def shape(request):
    """the model, its inputs and the float64 oracle results, computed once per shape"""
    B, Tx, T, ragged = SHAPES[request.param]
    cfg = O.OracleConfig(r=5, max_decode_iter=T, vocab_size=64)
    p = O.init_params(cfg, seed=1, trained_like=True)
    inp = [O.synthetic_inputs(cfg, B, Tx, T, seed=s, ragged=ragged, with_targets=False) for s in (0, 5)]
    return SimpleNamespace(name=request.param, T=T, cfg=cfg, p=p, inp=inp, ref=[_oracle(p, x, cfg) for x in inp],
                           model=_model(T, p))


def _call(m, inp, **kw):
    """(seq2seq_output, alignments, output) cloned, the taco_highway_stack_fwd calls and the launches of one call"""
    n0 = L.lib().taco_launch_count()
    with recording(K) as rec:
        y, out = m.inference(to_cuda(inp), train=False, **kw)
        res = (y.clone(), m.alignments.clone(), out.clone())
    torch.cuda.synchronize()
    return res, rec.calls.count("taco_highway_stack_fwd"), L.lib().taco_launch_count() - n0


def _same_bits(a, b, what):
    for x, y, n in zip(a, b, ("seq2seq_output", "alignments", "output")):
        assert x.shape == y.shape, f"{what} {n}: {tuple(x.shape)} vs {tuple(y.shape)}"
        diff = int((x.contiguous().view(torch.int32) != y.contiguous().view(torch.int32)).sum())
        assert diff == 0, f"{what} {n}: {diff} elements differ, max |d| {(x - y).abs().max().item():.3e}"


def _against_oracle(got, ref, what):
    y, a, out = got
    y_ref, out_ref, a_ref = ref
    assert_close(y, y_ref, TOL, f"{what} seq2seq_output")
    assert_close(a, a_ref, TOL, f"{what} alignments")
    assert_close(out, out_ref, TOL, f"{what} output")


def test_graph_eager_traced_and_oracle(shape):
    m = shape.model
    graphed, n_hs, _ = _call(m, shape.inp[0])                 # 2 eager warm-up calls + the capture, 2 CBHGs each
    assert n_hs == 6, f"{shape.name}: {n_hs} taco_highway_stack_fwd calls while capturing"
    replay, n_hs, n_replay = _call(m, shape.inp[0])
    assert n_hs == 0 and n_replay == 0, "the second call must replay the graphs"
    _same_bits(replay, graphed, f"{shape.name} replay vs capture")
    m.config.cuda_graph = False
    try:
        eager, n_hs, n_eager = _call(m, shape.inp[0])
        assert n_hs == 2, f"{shape.name}: the untraced eager call made {n_hs} fused calls"
        traced, n_hs, n_traced = _call(m, shape.inp[0], trace={})
        assert n_hs == 0, f"{shape.name}: the traced call took the fused route"
    finally:
        m.config.cuda_graph = True
    assert n_traced - n_eager == LAYERED_EXTRA, f"{shape.name}: {n_traced} traced vs {n_eager} untraced launches"
    _same_bits(graphed, eager, f"{shape.name} graph vs eager")
    _same_bits(eager, traced, f"{shape.name} eager vs traced")
    _against_oracle(graphed, shape.ref[0], shape.name)


def test_second_batch_through_the_graphs(shape):
    m = shape.model
    _call(m, shape.inp[0])
    got, n_hs, _ = _call(m, shape.inp[1])
    assert n_hs == 0
    _against_oracle(got, shape.ref[1], f"{shape.name} second batch")


def test_load_params_refreshes_the_replay(shape):
    m = shape.model
    _call(m, shape.inp[0])
    p2 = O.init_params(shape.cfg, seed=7, trained_like=True)
    m.load_params(p2)
    try:
        got, _, _ = _call(m, shape.inp[1])
        again, _, n = _call(m, shape.inp[1])
        assert n == 0
        fresh, _, _ = _call(_model(shape.T, p2), shape.inp[1])
        _same_bits(got, fresh, f"{shape.name} after load_params vs a fresh model")
        _same_bits(again, fresh, f"{shape.name} replay after load_params vs a fresh model")
    finally:
        m.load_params(shape.p)
