"""GPU tests of the summaries (csrc/summary.cu, kernels.histogram, train.train(summary_dir=...), test.test(summary_dir=...)):
taco_histogram against its torch-CPU mirror with NaN-poisoned workspace and outputs, up to the 32.8 M floats of the
benchmark's training `output`, run to run bit-identical; the training driver's event file on the toy corpus of
test_gpu_z_data.py (tags, steps, scalars, the step-4 output histogram against the oracle, no effect on the other outputs);
the synthesis driver's audio and image summaries."""
import math
import os

import numpy as np
import pytest
import torch

from tacotron_b200 import summary as S
from tests import mirror_kernels_summary as MKS
from tests.test_gpu_z_data import _dataset
from tests.test_summary import NLIM, _events, check_result, edge_values

pytestmark = pytest.mark.gpu


def _kernel(x):
    from tacotron_b200 import kernels as K
    lim = torch.from_numpy(S.histogram_limits()).cuda()
    K._hist_ws.pop(x.device, None)
    K._hist_ws[x.device] = torch.full((K.L.lib().taco_histogram_workspace_bytes() // 8,), float("nan"), dtype=torch.float64,
                                      device=x.device).view(torch.uint8)          # NaN-poisoned workspace
    res = torch.full((NLIM + 5,), float("nan"), dtype=torch.float64, device=x.device).view(torch.int64)
    K.histogram(res, x, lim)
    return res


@pytest.mark.parametrize("n", [1, 3, 4097, 32 * 1000 * 1025, "edge"])
def test_histogram_kernel_against_mirror(n):
    if n == "edge":
        x = torch.from_numpy(edge_values())
    else:
        g = torch.Generator().manual_seed(n)
        x = torch.randn(n, generator=g) * torch.exp(torch.randn(n, generator=g) * (8 if n < 10000 else 1.5))
    got = _kernel(x.cuda())
    got2 = _kernel(x.cuda())
    torch.cuda.synchronize()
    assert torch.equal(got, got2)                                    # bit-identical from run to run
    want = torch.empty(NLIM + 5, dtype=torch.int64)
    MKS.histogram(want, x, torch.from_numpy(S.histogram_limits()))
    got = got.cpu()
    assert torch.equal(got[:NLIM + 3], want[:NLIM + 3])             # counts, non-finite count, min, max exact
    xf = x.double()
    xf = xf[torch.isfinite(xf)]
    s, sq = got[NLIM + 3:].view(torch.float64).tolist()
    ws, wsq = want[NLIM + 3:].view(torch.float64).tolist()
    assert abs(s - ws) <= 1e-12 * float(xf.abs().sum()) and abs(sq - wsq) <= 1e-12 * float((xf * xf).sum())
    if n == "edge":
        check_result(got, x.numpy(), sums_exact=False)


def _train(root, monkeypatch, summaries):
    from tacotron_b200 import train as trainer
    from tacotron_b200.models.tacotron import Config, Tacotron
    os.makedirs(root, exist_ok=True)
    _dataset(root)
    monkeypatch.chdir(root)
    torch.manual_seed(0)
    cfg = Config()
    cfg.data_path, cfg.save_path, cfg.restore = "data/toy/", "toy/tacotron", False
    logs = []
    m = trainer.train(Tacotron, cfg, num_steps=4, log=logs.append, save_every=2,
                      summary_dir="log/toy/tacotron/train" if summaries else None)
    torch.cuda.synchronize()
    return m, logs


def _files(root):
    out = {}
    for d, _, fs in os.walk(root):
        for f in fs:
            p = os.path.join(d, f)
            out[os.path.relpath(p, root)] = open(p, "rb").read()
    return out


def test_train_driver_summaries(tmp_path, monkeypatch):
    from tests import summary_oracle as SO
    m, _ = _train(str(tmp_path / "a"), monkeypatch, True)
    ev = _events(str(tmp_path / "a" / "log/toy/tacotron/train"))
    assert ev[0][2] == "brain.Event:2"
    tags = {}
    for step, _, _, vals in ev[1:]:
        tags.setdefault(step, []).extend(t for t, _ in vals)
    merged = list(S.HISTOGRAM_TAGS) + list(S.SCALAR_TAGS)
    assert sorted(tags) == [1, 2, 3, 4]
    for step in (1, 3):
        assert tags[step] == merged
    for step in (2, 4):
        assert sorted(tags[step]) == sorted(merged + [f"ideal_{step}/audio/0", f"sample_{step}/audio/0", f"attention_{step}/image/0"])
    last = {t: v for step, _, _, vals in ev[1:] if step == 4 for t, v in vals}
    assert last["loss"].simple_value == float(m.loss)
    assert last["seq2seq_loss"].simple_value == float(m.seq2seq_loss)
    assert last["output_loss"].simple_value == float(m.output_loss)
    assert last["cap_grads/global_gradient_norm"].simple_value == float(m.grad_sumsq.sqrt())
    # the step-4 output histogram against the oracle
    out = m.output.detach().cpu().numpy().reshape(-1)
    h = SO.Histogram()
    for v in out.tolist():
        h.add(v)
    hp = last["post-process/output"].histo
    bl, bc = h.encode()
    assert list(hp.bucket_limit) == bl and list(hp.bucket) == bc
    assert (hp.min, hp.max, hp.num) == (h.min, h.max, h.num)
    od = out.astype(np.float64)
    assert abs(hp.sum - math.fsum(od)) <= 1e-12 * float(np.abs(od).sum())
    assert abs(hp.sum_squares - math.fsum(od * od)) <= 1e-12 * float((od * od).sum())
    # the audio summaries are the waveforms the driver writes next to the checkpoint, unnormalised
    au = last["sample_4/audio/0"].audio
    assert au.sample_rate == 16000.0 and au.content_type == "audio/wav" and au.length_frames > 0
    # without summary_dir: no event file and the same outputs.  The training step is not bit-reproducible (the split-K
    # weight gradients add with float atomics), so the two runs agree to that rounding carried through four steps:
    # parameters within the 2 lr per step that two Adam updates can differ by, the alignments within 0.05.
    _train(str(tmp_path / "b"), monkeypatch, False)
    fa, fb = _files(str(tmp_path / "a")), _files(str(tmp_path / "b"))
    assert not os.path.exists(str(tmp_path / "b" / "log"))
    fa = {k: v for k, v in fa.items() if not k.startswith("log" + os.sep)}
    assert sorted(fa) == sorted(fb)
    for k in fa:
        pa, pb = os.path.join(str(tmp_path / "a"), k), os.path.join(str(tmp_path / "b"), k)
        if k.endswith(".npz"):
            za, zb = np.load(pa), np.load(pb)
            assert sorted(za.files) == sorted(zb.files), k
            for f in za.files:
                if za[f].dtype.kind == "f":
                    assert np.abs(za[f].astype(np.float64) - zb[f]).max() <= 8 * m.config.init_lr * 1.5, (k, f)
                else:
                    assert np.array_equal(za[f], zb[f]), (k, f)
        elif k.endswith("_attention.npy"):
            assert np.abs(np.load(pa) - np.load(pb)).max() <= 0.05, k
        elif k.endswith(".wav"):
            assert fa[k][:44] == fb[k][:44], k                       # same format and length
        elif k.startswith("data" + os.sep):
            assert fa[k] == fb[k], k


def test_synthesis_driver_summaries(tmp_path, monkeypatch):
    from tacotron_b200 import test as synth
    from tacotron_b200.models.tacotron import Config, Tacotron
    _train(str(tmp_path), monkeypatch, False)
    cfg = Config()
    cfg.data_path, cfg.save_path = "data/toy/", "toy/tacotron"
    waves = synth.test(Tacotron, cfg, ["abc de\n", "hello, you\n", "abc de\n"], log=lambda *a: None,
                       summary_dir="log/toy/tacotron/test")
    ev = _events("log/toy/tacotron/test")
    assert len(ev) == 4 and all(step == 0 for step, _, _, _ in ev)
    texts = [S.clean_tag(open(f"log/toy/tacotron/test/{n}.txt").read()) for n in range(3)]
    assert texts[0] == texts[2] != texts[1]
    want = [[f"{texts[0]}/audio/0", f"{texts[0]}_1/image/0"], [f"{texts[1]}/audio/0", f"{texts[1]}_1/image/0"],
            [f"{texts[0]}_2/audio/0", f"{texts[0]}_3/image/0"]]
    for n, (_, _, _, vals) in enumerate(ev[1:]):
        assert [t for t, _ in vals] == want[n]
        au, im = vals[0][1].audio, vals[1][1].image
        assert au.encoded_audio_string == S.wav_bytes(waves[n].cpu().numpy(), 16000)
        assert au.length_frames == waves[n].numel() and im.colorspace == 4
        al = np.load(f"log/toy/tacotron/test/{n}_attention.npy")
        assert (im.height, im.width) == S.attention_rgba(al).shape[:2]
