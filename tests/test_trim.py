"""The synthesis tail trim on the CPU: the torch mirror of taco_speech_frames against the float64 oracle, the
validation of invert_speech, and the packed Griffin-Lim orchestration over the mirror kernels against the padded one."""
import numpy as np
import pytest
import torch

from tacotron_b200 import audio
from tests import mirror_kernels as MK
from tests import mirror_kernels_trim as MKT
from tests import trim_oracle as TO


def _affine(r, seed):
    g = np.random.RandomState(seed)
    return (g.rand(1025 * r) * 2 + 1).astype(np.float32), (g.randn(1025 * r) * 2 - 5).astype(np.float32)


def trim_cases(r):
    """(name, spec float32 [B, T, 1025 r], scale, shift, expected frames): every finite frame is at least
    0.5 dB from its threshold (asserted), so float32 cannot flip it"""
    T = {1: 24, 2: 16, 5: 8}[r]
    blk, n = 4 * r, 4 * r * (T // 4)
    cases = []
    for aff in (False, True):
        scale, shift = _affine(r, 3) if aff else (None, None)
        sfx = "_affine" if aff else ""
        ends = [n // 2 - 1, n, n - 1, 1]                       # quiet tail, all voiced, tail < one block, k_min floor
        spec = TO.speech_like(len(ends), T, r, ends, seed=r, scale=scale, shift=shift)
        want = [blk * -(-e // blk) for e in ends]
        want[3] = blk * -(-5 // blk)
        cases.append(("speech" + sfx, spec, scale, shift, want))
        last = TO.speech_like(1, T, r, [n], seed=7 + r, scale=scale, shift=shift)      # only the last frame voiced
        q = TO.speech_like(1, T, r, [0], seed=7 + r, scale=scale, shift=shift)
        lastonly = q.copy()
        tq, tl, c = 4 * ((n - 1) // blk), (n - 1) % 4, ((n - 1) % blk) // 4
        lastonly[0, tq + tl, c * 1025:(c + 1) * 1025] = last[0, tq + tl, c * 1025:(c + 1) * 1025]
        cases.append(("last_frame" + sfx, lastonly, scale, shift, [n]))
    base = TO.speech_like(4, T, r, [n // 2] * 4, seed=11)
    base[0, 1, 5] = np.nan
    base[1, T - 1, 7] = np.inf
    base[2, 0, :1025] = -np.inf                                 # a whole frame of -inf: e = -inf
    base[3, 2, 9] = -np.inf                                     # one -inf bin: e stays finite
    cases.append(("nonfinite", base, None, None, [n, n, n, blk * -(-(n // 2) // blk)]))
    return cases


@pytest.mark.parametrize("r", [1, 2, 5])
def test_speech_frames_mirror_matches_oracle(r):
    for name, spec, scale, shift, want in trim_cases(r):
        assert TO.margin_db(spec, r, scale, shift) >= 0.5, name
        ref = TO.speech_frames(spec, r, scale, shift)
        got = torch.empty(spec.shape[0], dtype=torch.int32)
        sc = None if scale is None else torch.from_numpy(scale)
        sh = None if shift is None else torch.from_numpy(shift)
        MKT.speech_frames(got, torch.from_numpy(spec), r, sc, sh)
        assert got.tolist() == ref.tolist() == want, (name, got.tolist(), ref.tolist(), want)


def test_speech_frames_threshold():
    """top_db moves the end: a tail 40 dB below the speech is speech at 60 dB and silence at 20 dB"""
    r, T = 2, 16
    spec = TO.speech_like(1, T, r, [16], seed=1)
    quiet = TO.speech_like(1, T, r, [32], seed=1)
    tail = TO.frame_space(quiet[0], r).copy()
    lo = TO.frame_space(spec[0], r)
    lo[16:] = tail[16:] - 40 * TO.LN10_OVER_10 / 2                  # 40 dB of power
    nb = T // 4
    spec[0] = lo.reshape(nb, r, 4, 1025).transpose(0, 2, 1, 3).reshape(nb * 4, r * 1025)
    assert min(TO.margin_db(spec, r, top_db=db) for db in (60.0, 20.0)) >= 0.5
    assert TO.speech_frames(spec, r, top_db=60.0).tolist() == [32]
    assert TO.speech_frames(spec, r, top_db=20.0).tolist() == [16]
    for db in (60.0, 20.0):
        got = torch.empty(1, dtype=torch.int32)
        MKT.speech_frames(got, torch.from_numpy(spec), r, top_db=db)
        assert got.tolist() == TO.speech_frames(spec, r, top_db=db).tolist()


@pytest.mark.parametrize("bad", [[8, 7], [8, 4], [8, 40], [8], [8, 8, 8]])
def test_invert_speech_rejects_bad_frames(bad):
    r, T = 2, 16                                                # n = 32, blocks of 8
    spec = torch.zeros(2, T, 1025 * r, dtype=torch.float64)
    with pytest.raises(ValueError):
        audio.invert_speech(spec, r, torch.tensor(bad, dtype=torch.int32), n_iter=0, K=MKT)


def test_invert_speech_rejects_a_short_utterance_at_r1():
    spec = torch.zeros(1, 8, 1025, dtype=torch.float64)
    with pytest.raises(ValueError):
        audio.invert_speech(spec, 1, torch.tensor([4], dtype=torch.int32), n_iter=0, K=MKT)


@pytest.mark.parametrize("r,T,frames,n_iter", [(1, 12, [8, 12, 8], 2), (2, 8, [16, 8], 3), (5, 8, [20, 40], 1)])
def test_packed_orchestration_equals_padded_on_truncated_spectrogram(r, T, frames, n_iter):
    g = torch.Generator().manual_seed(5)
    B = len(frames)
    spec = torch.randn(B, T, 1025 * r, generator=g, dtype=torch.float64) * 0.5
    mean = torch.randn(1025 * r, generator=g, dtype=torch.float64) * 0.1
    std = torch.rand(1025 * r, generator=g, dtype=torch.float64) + 0.5
    N = sum(frames)
    pu = torch.rand(N, 1025, generator=g, dtype=torch.float64)
    ys = audio.invert_speech(spec, r, torch.tensor(frames, dtype=torch.int32), n_iter=n_iter, stft_mean=mean, stft_std=std,
                             phase_u=pu, K=MKT)
    off = np.concatenate([[0], np.cumsum(frames)])
    for b in range(B):
        assert ys[b].shape == (300 * (frames[b] - 1),)
        ref = audio.invert_spectrogram(spec[b:b + 1, :frames[b] // r], r, n_iter=n_iter, stft_mean=mean, stft_std=std,
                                       phase_u=pu[off[b]:off[b + 1]][None], K=MK)[0]
        assert torch.equal(ys[b], ref), b
