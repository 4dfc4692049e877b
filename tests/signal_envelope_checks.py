"""The signal kernels that make integer decisions from float reductions or carry a long recurrence or tap sum, over their
envelope, against float64: taco_trim_bounds (trim_kernel, csrc/features.cu), taco_speech_frames / taco_speech_bounds
(frame_power_kernel + speech_end_kernel / speech_bounds_kernel), taco_join_segments and taco_de_emphasis (csrc/audio.cu)
and taco_resample (csrc/resample.cu).  Written once, run on the H100 by tests/test_gpu_z_signal_envelope.py and under
the host emulation (tests/cuda_emu) by tests/test_signal_envelope_host.py.

Every check takes a tests.stft_envelope_checks.Env (kernel namespace K, library, device, stream) and reuses its guarded
buffers: outputs are prefilled with a sentinel bit pattern inside PAD words of it that must survive, operands sit inside
NaN bands.  Every reference is float64 from the kernel's own float32 operands, through the existing oracles
(feature_oracle.trim, trim_oracle.log_power / speech_frames, longform_oracle.speech_bounds / join_segments,
griffin_lim_oracle.de_emphasis, resample_oracle.resample_loop).

u = 2^-24, u64 = 2^-53, SAFETY = 2 on every bar that is not rigorous as stated.

Integer decisions.  A frame is DECIDED when its float64 quantity is further from the threshold than the sum of the two
quantities' bars.  The kernel's answer must equal the float64 answer when every frame that can change it is decided;
otherwise it must be one of the answers reachable by flipping only undecided frames (first in {first decided} + the
undecided frames before it, last likewise).
* trim: the quantity is q_f = db_f - db_max + top_db (non-silent when q_f > 0), db = 10 log10(max(1e-10, e)).  The
  kernel sums each hop-block of squares with fp64 fmas (hop roundings), adds `per` blocks and divides (per + 1); the
  oracle's mean is a pairwise sum (log2(frame_length) + 1): e is within R u64 relative in both, R = hop + per + 2 +
  log2(frame_length) + 1, so db within 10/ln10 2 R u64 + 4 u64 |db| between them (log10 and the product by 10 rounded
  once each).  SAFETY times that, for the frame and for the maximum: about 1e-12 dB, so every planted margin (0.01 dB)
  and every random one here is decided and the bounds must match bit for bit.
* speech: e = m + log sum_k exp(2v'_k - m), v' = fmaf(v, scale, shift).  Term k has a relative error of
  4u (expf, 2 ulp) + u |2v'_k - m| (the subtraction) + 2u |v'_k| (the fmaf, with the affine only); the lane sums and
  the 5-level butterfly add (ceil(F/32) + 5) u of the (positive) sum; logf 2u |log s|; the final add u |e|.  The
  per-term errors are weighted by the terms (sum_k t_k d_k / sum_k t_k in float64).  The threshold
  thr = E - top_db * 0.2302585f adds u |top_db c| twice (the product, the constant's rounding) and u |thr|; the maximum
  E is one of the e_f, within the largest bar of the utterance.  margin_f = e_f - (E - top_db ln10/10) decided when
  |margin_f| > SAFETY (bar_f + bar_max) + bar_thr.

Values.
* join: out = float32(float64(src w)) with w = sin^2(pi (j + 0.5) / (2 fade)) in double (exact to ~1e-15).  The
  float64 reference (longform_oracle.join_segments) spells c as 0.5 - 0.5 cos(.), whose cancellation costs 4 u64 / w
  relative; so the kernel must give float32(ref) bit for bit, and a float32 neighbour only where ref lies within
  tol = 1e-15 + 4 u64 / w relative of a rounding boundary.  Worst figure: |out - ref| / (half an ulp of ref + tol |ref|).
* de_emphasis: y_i = x_i + c y_{i-1}.  A term c^(i-j) x_j reaches output i through at most i - j roundings of products
  of powers of c (runs' a *= c and p *= c, the butterfly's a *= oa, the warp totals wa: a product tree of i - j leaves
  has i - j - 1 internal nodes) and through the additions on its path: <= 16 in the run's fmaf chain, 5 butterfly
  levels, <= 15 warp totals in the serial pass, the yin fmaf and the output fmaf inside its tile (38), 17 more for the
  carry into the next tile, and 22 per further tile crossed, at least 8192 samples each (< 0.003 per sample of
  distance).  Each addition's rounding is u of a partial sum bounded by A_i, A the float64 recurrence over |x|:
      |y - y64|_i <= SAFETY u (1.003 B_i + 55 A_i),   B_i = sum_{j<=i} c^(i-j) A_j
  i.e. K u B_i with K = 1.003 + 55 A_i / B_i <= 56.  Local: behind a loud burst the bar decays with the signal.  c = 0
  must return the input bit for bit.
* resample: bit for bit against the sequential loop (resample_oracle.resample_loop's arithmetic, evaluated at chosen
  outputs by loop_at, which is checked against resample_loop itself), and against the float64 sum of the same taps
  within taps u sum |w x| (taps float32 roundings of partial sums bounded by sum |w x|; rigorous to first order).
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from tests import feature_oracle as FO
from tests import griffin_lim_oracle as GO
from tests import longform_oracle as LO
from tests import resample_oracle as RO
from tests import trim_oracle as TO
from tests.stft_envelope_checks import NAN, SENT, Env, Out, _frac, _p, operand, same_bits  # noqa: F401

U = 2.0 ** -24
U64 = 2.0 ** -53
SAFETY = 2.0
LN10_10 = math.log(10.0) / 10.0
C_LN10_10 = float(np.float32(0.230258509299404568))       # the kernels' float32 constant
SMS = 132
DE_L = 55                                                 # additions on a de_emphasis path (module docstring)
RS_GRID = 65535 * 256                                      # outputs one resample_kernel launch covers without a stride


def rng(seed):
    return np.random.RandomState(seed)


def _sent_bits(t):
    return t.contiguous().view(torch.int32) == SENT


# ------------------------------------------------------------------------------------------------------------------
# the decision rule
# ------------------------------------------------------------------------------------------------------------------
def reachable(margin, bar):
    """(firsts, lasts): the first / last positive frame over every flip of the undecided frames (|margin| <= bar);
    None stands for "no positive frame".  Singletons when every frame that can change them is decided."""
    pos = np.flatnonzero(margin > bar)
    und = np.flatnonzero(~(np.abs(margin) > bar))
    if pos.size:
        return ({int(pos[0])} | {int(u) for u in und if u < pos[0]}, {int(pos[-1])} | {int(u) for u in und if u > pos[-1]})
    return {None} | {int(u) for u in und}, {None} | {int(u) for u in und}


# ------------------------------------------------------------------------------------------------------------------
# 1. taco_trim_bounds
# ------------------------------------------------------------------------------------------------------------------
def trim_db(x, frame_length, hop):
    """(db_f, bar_f) of feature_oracle.trim's frames: db = 10 log10(max(1e-10, mean square)), float64, and its bar"""
    x64 = np.asarray(x, np.float32).astype(np.float64)
    yp = np.pad(x64, frame_length // 2, mode="reflect")
    nf = 1 + len(x64) // hop
    w = np.lib.stride_tricks.sliding_window_view(yp, frame_length)[::hop][:nf]
    e = np.einsum("ij,ij->i", w, w) / frame_length
    db = 10.0 * np.log10(np.maximum(1e-10, e))
    R = hop + frame_length // hop + 2 + frame_length.bit_length()
    return db, SAFETY * (10.0 / math.log(10.0) * 2 * R * U64 + 4 * U64 * np.abs(db))


def run_trim(env, waves, frame_length, hop, top_db, base=0):
    """bounds int32 [B, 2] of the kernel on `waves` packed end to end from sample `base` of y (NaN before it)"""
    lens = [len(w) for w in waves]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64) + base
    y = np.full(base + sum(lens), np.nan, np.float32)
    for w, a in zip(waves, off[:-1]):
        y[a:a + len(w)] = w
    o = Out((len(waves), 2), env.device, torch.int32)
    env.K.trim_bounds(o.t, operand(torch.from_numpy(y), env.device), operand(torch.from_numpy(off), env.device),
                      frame_length, hop, top_db)
    env.sync()
    assert o.bands_intact(), "trim_bounds wrote outside bounds"
    assert len(waves) == 0 or o.written(), "trim_bounds left bounds unwritten"
    return o.t.cpu().numpy()


def trim_check(env, waves, frame_length, hop, top_db=60.0, base=0, ref_hop=None, oracle=True):
    """the kernel's bounds of every utterance within the decision rule (reference at ref_hop, default the kernel's);
    where every frame is decided, also feature_oracle.trim's own answer.  Returns (bounds, undecided utterances)."""
    ref_hop = ref_hop or hop
    got = run_trim(env, waves, frame_length, hop, top_db, base)
    t32 = float(np.float32(top_db))
    undecided = 0
    for b, w in enumerate(waves):
        db, bar = trim_db(w, frame_length, ref_hop)
        imax = int(np.argmax(db))
        firsts, lasts = reachable(db - db[imax] + t32, bar + bar[imax])
        want = {(0, 0) if f is None else (f * ref_hop, min(len(w), (l + 1) * ref_hop))
                for f in firsts for l in lasts if (f is None) == (l is None)}
        g = tuple(int(v) for v in got[b])
        assert g in want, f"trim_bounds utterance {b} (len {len(w)}, {frame_length}/{hop}): {g}, float64 allows {sorted(want)}"
        if len(want) > 1:
            undecided += 1
        elif oracle:
            assert g == tuple(int(v) for v in FO.trim(w, t32, frame_length, ref_hop)[1]), f"feature_oracle.trim, {b}"
    return got, undecided


def envelope_wave(n, seed, lo_db=-90.0):
    """noise under a random piecewise-constant envelope between lo_db and 0 dB (speech-like bursts and pauses)"""
    g = rng(seed)
    edges = np.sort(g.randint(0, n, size=max(2, n // 3000)))
    lvl = np.repeat(g.uniform(lo_db, 0.0, size=len(edges) + 1), np.diff(np.concatenate([[0], edges, [n]])))
    return (g.randn(n) * 10 ** (lvl / 20)).astype(np.float32)


def impulse_waves(nf, frame_length, hop, frames, seed):
    """one utterance of nf frames per f in `frames`: a unit impulse at sample f*hop (clipped to the last sample) over
    noise 80 dB below a frame holding it, so the loud frames are those holding the impulse and first / last sweep
    every tile edge"""
    n = (nf - 1) * hop + 1
    g = rng(seed)
    out = []
    for f in frames:
        x = (g.randn(n) * 1e-4 / math.sqrt(frame_length)).astype(np.float32)
        x[min(f * hop, n - 1)] = 1.0
        out.append(x)
    return out


def planted_waves(frame_length, hop, delta_db, seed):
    """runs of constant amplitude: quiet (-100 dB), a planted run at -60 + delta_db, loud (0 dB), a second planted run,
    quiet.  Every frame inside a run has exactly its amplitude's power; frames straddling a run edge are >= 1.2 dB
    away from -60."""
    g = rng(seed)
    a = float(np.float32(10 ** ((-60.0 + delta_db) / 20)))
    runs = [(3 * frame_length + 7, 1e-5), (2 * frame_length, a), (2 * frame_length, 1.0), (2 * frame_length, a),
            (3 * frame_length + hop // 2 + 3, 1e-5)]
    x = np.concatenate([np.full(n, v) * np.where(g.rand(n) < 0.5, -1.0, 1.0) for n, v in runs]).astype(np.float32)
    return x


def trim_lengths(frame_length, hop):
    """frame_length/2 + 1, multiples of hop +- 1, and nf = 255, 256, 257, 512, 513 frames (both ends of each)"""
    ls = {frame_length // 2 + 1, frame_length // 2 + 2}
    for k in (2, 3, 17, 64):
        ls |= {k * hop - 1, k * hop, k * hop + 1}
    for nf in (255, 256, 257, 512, 513):
        ls |= {(nf - 1) * hop, nf * hop - 1}
    return sorted(v for v in ls if v > frame_length // 2)


# ------------------------------------------------------------------------------------------------------------------
# 2. taco_speech_frames / taco_speech_bounds
# ------------------------------------------------------------------------------------------------------------------
def to_spec(v, T, r):
    """v [B, n, F] in gl_init's frame space -> spec float32 [B, T, F r]; rows past 4 (T/4) NaN (never read)"""
    B, n, F = v.shape
    nb = T // 4
    spec = torch.full((B, T, F * r), NAN)
    spec[:, :4 * nb] = torch.as_tensor(v, dtype=torch.float32).reshape(B, nb, r, 4, F).permute(0, 1, 3, 2, 4) \
        .reshape(B, 4 * nb, r * F)
    return spec


def speech_e_bars(spec, r, scale=None, shift=None, device="cpu"):
    """(e64 [B, n], bar [B, n]) float64 numpy: each frame's log power and the bar of the kernel's float32 value"""
    B, T, W = spec.shape
    F, nb = W // r, T // 4
    v = spec[:, :4 * nb].to(device).double().reshape(B, nb, 4, r, F).permute(0, 1, 3, 2, 4).reshape(B, 4 * nb * r, F)
    c = torch.arange(4 * nb * r, device=device) % (4 * r) // 4
    if scale is not None:
        v = v * scale.to(device).double().view(r, F)[c] + shift.to(device).double().view(r, F)[c]
    x = 2 * v
    m = x.max(-1, keepdim=True).values
    t = torch.exp(x - m)
    s = t.sum(-1)
    d = 4 * U + U * (x - m).abs() + (2 * U * v.abs() if scale is not None else 0.0)
    rel = (t * d).sum(-1) / s
    e = m[..., 0] + s.log()
    bar = rel + (math.ceil(F / 32) + 5) * U + 2 * U * s.log().abs() + U * e.abs()
    return e.cpu().numpy(), bar.cpu().numpy()


def run_speech(env, spec, r, scale=None, shift=None, top_db=60.0):
    """(frames [B], bounds [B, 3]) of both entry points; frames bit-identical to bounds[:, 2]"""
    B = spec.shape[0]
    dev = env.device
    of, ob = Out((B,), dev, torch.int32), Out((B, 3), dev, torch.int32)
    sp, sc, sh = operand(spec, dev), operand(scale, dev), operand(shift, dev)
    env.K.speech_frames(of.t, sp, r, sc, sh, top_db)
    env.K.speech_bounds(ob.t, sp, r, sc, sh, top_db)
    env.sync()
    assert of.bands_intact() and ob.bands_intact(), "speech_frames / speech_bounds wrote outside their outputs"
    assert of.written() and ob.written(), "speech_frames / speech_bounds left outputs unwritten"
    fr, bd = of.t.cpu().numpy(), ob.t.cpu().numpy()
    assert np.array_equal(fr, bd[:, 2]), "speech_bounds' frame count differs from speech_frames'"
    return fr, bd


def speech_check(env, spec, r, scale=None, shift=None, top_db=60.0, ref_top_db=None):
    """both entry points within the decision rule at ref_top_db (default top_db); exactly longform_oracle.speech_bounds
    and trim_oracle.speech_frames wherever decided.  Returns (bounds, undecided utterances)."""
    ref_top_db = top_db if ref_top_db is None else ref_top_db
    B, T, W = spec.shape
    n, blk = 4 * r * (T // 4), 4 * r
    kmin = -(-5 // blk)
    fr, bd = run_speech(env, spec, r, scale, shift, top_db)
    e, bar = speech_e_bars(spec, r, scale, shift, env.device)
    t32 = float(np.float32(top_db))
    sc_np = None if scale is None else scale.numpy()
    sh_np = None if shift is None else shift.numpy()
    ref = LO.speech_bounds(spec.numpy(), r, sc_np, sh_np, ref_top_db)
    ref_fr = TO.speech_frames(spec.numpy(), r, sc_np, sh_np, ref_top_db)
    assert np.array_equal(ref[:, 2], ref_fr)
    undecided = 0
    for b in range(B):
        g = tuple(int(v) for v in bd[b])
        if not np.all(np.isfinite(e[b])):
            assert g == (0, n, n), f"speech_bounds utterance {b}: not finite, got {g}"
            continue
        E = e[b].max()
        thr_bar = 2 * U * t32 * C_LN10_10 + U * (abs(E) + t32 * C_LN10_10)
        tot = SAFETY * (bar[b] + bar[b].max()) + thr_bar
        margin = e[b] - (E - ref_top_db * LN10_10)
        firsts, lasts = reachable(margin, tot)
        want = {(f, l + 1, blk * min(max(-(-(l + 1) // blk), kmin), T // 4)) for f in firsts for l in lasts}
        assert g in want, f"speech_bounds utterance {b} (T={T}, r={r}): {g}, float64 allows {sorted(want)}"
        if len(want) > 1:
            undecided += 1
        else:
            assert g == tuple(int(v) for v in ref[b]), f"speech_bounds utterance {b}: {g}, oracle {tuple(ref[b])}"
    return bd, undecided


def speech_map(env, T, r, F, seed=0):
    """index-coded: utterance b has one loud frame, f = b (every f < n); rows past 4 (T/4) NaN.  Exact {f, f + 1,
    4r clamp(ceil((f + 1) / 4r), ceil(5 / 4r), T/4)}"""
    n, blk = 4 * r * (T // 4), 4 * r
    g = torch.Generator().manual_seed(seed)
    v = -40.0 + torch.rand(n, n, F, generator=g)
    v[torch.arange(n), torch.arange(n)] = torch.rand(n, F, generator=g)
    _, bd = run_speech(env, to_spec(v, T, r), r)
    f = np.arange(n)
    k = np.minimum(np.maximum((f + blk) // blk, -(-5 // blk)), T // 4)
    want = np.stack([f, f + 1, blk * k], 1)
    bad = np.flatnonzero((bd != want).any(1))
    assert bad.size == 0, f"speech map T={T} r={r}: frame {bad[0]} gives {tuple(bd[bad[0]])}, want {tuple(want[bad[0]])}"


def planted_spec(T, r, F, delta_db, top_db=60.0):
    """two utterances: loud frames (v = 0) in the middle, frames planted at top_db - delta_db / top_db + delta_db
    below them near both ends, the rest 200 nats down"""
    n = 4 * r * (T // 4)
    v = torch.full((2, n, F), -100.0)
    v[:, n // 3:n // 2] = 0.0
    for b, s in enumerate((-1.0, 1.0)):
        vp = -(top_db + s * delta_db) * LN10_10 / 2
        v[b, [1, n - 2]] = vp
    return to_spec(v, T, r)


def speech_at_threshold(env, r, top_db=60.0):
    """F = 1 makes e = 2v exactly (expf(0) = 1, logf(1) = 0): with the loudest frame at e = 0 the threshold is
    -fl32(top_db * 0.2302585f) whichever way the kernel contracts it.  A frame exactly at it is voiced (>=), one a
    float32 step below is not."""
    T = 16
    n = 4 * r * (T // 4)
    thr = -float(np.float32(np.float32(top_db) * np.float32(C_LN10_10)))
    below = float(np.nextafter(np.float32(thr), np.float32(-np.inf)))
    v = torch.full((4, n, 1), -100.0)
    v[:, n // 2] = 0.0
    v[0, 0], v[0, n - 2] = thr / 2, thr / 2                          # at the threshold: first = 0, last = n - 2
    v[1, 0], v[1, n - 2] = below / 2, below / 2                      # a step below: only the loud frame
    v[2, n - 1] = thr / 2                                            # at the threshold, the last frame
    v[3, 1], v[3, n - 1] = thr / 2, below / 2
    _, bd = run_speech(env, to_spec(v, T, r), r, top_db=top_db)
    blk = 4 * r
    fr = lambda l: blk * min(max(-(-(l + 1) // blk), -(-5 // blk)), T // 4)  # noqa: E731
    want = [(0, n - 1, fr(n - 2)), (n // 2, n // 2 + 1, fr(n // 2)), (n // 2, n, fr(n - 1)), (1, n // 2 + 1, fr(n // 2))]
    assert [tuple(int(x) for x in row) for row in bd] == want, f"threshold rule (r={r}): {bd.tolist()} != {want}"


def ramp_spec(B, T, r, F, seed, nan_rows=True):
    """log magnitudes whose loudness falls along each utterance at a random rate (the threshold crossed at a random
    frame), bins spread by N(0, 1.5)"""
    n = 4 * r * (T // 4)
    g = torch.Generator().manual_seed(seed)
    rate = torch.rand(B, 1, 1, generator=g) * 40 + 5
    f = torch.arange(n, dtype=torch.float32)[None, :, None] / n
    v = -rate * f + torch.randn(B, n, F, generator=g) * 1.5 + torch.randn(B, n, 1, generator=g) * 0.5
    return to_spec(v, T, r)


def speech_nonfinite(env, B, T, r, F, seed):
    """NaN, +Inf and an all -Inf frame, each in its own utterance: that one gives {0, n, n}, the others their bits"""
    spec = ramp_spec(B, T, r, F, seed)
    _, base = run_speech(env, spec, r)
    n = 4 * r * (T // 4)
    for b, (t, col, val) in zip((1, 2, 3), ((0, 3, NAN), (T // 4 * 4 - 1, F * r - 1, float("inf")), (5, None, -math.inf))):
        s = spec.clone()
        if col is None:
            s[b, t, :F] = val
        else:
            s[b, t, col] = val
        _, bd = run_speech(env, s, r)
        assert tuple(bd[b]) == (0, n, n), f"speech_bounds: {val} in utterance {b} gives {tuple(bd[b])}"
        keep = np.arange(B) != b
        assert np.array_equal(bd[keep], base[keep]), f"speech_bounds: a {val} frame changed another utterance"


# ------------------------------------------------------------------------------------------------------------------
# 3. taco_join_segments
# ------------------------------------------------------------------------------------------------------------------
def make_segments(lens, src_len, seed, gap=5):
    """rows {src_start, dst_start, len} placed left to right in out with random gaps (0 .. gap; at least 1 after an
    empty row, which check_segments would otherwise see inside its neighbour once shuffled), random src starts, then
    shuffled; -> (seg int64 [S, 3], out_len)"""
    g = rng(seed)
    seg = np.zeros((len(lens), 3), np.int64)
    d = int(g.randint(0, gap + 1))
    for s, n in enumerate(lens):
        seg[s] = (g.randint(0, src_len - n + 1), d, n)
        d += n + int(g.randint(0, gap + 1)) + (n == 0)
    return seg[g.permutation(len(lens))], d + 3


def join_check(env, src, seg, out_len, fade, ref_fade=None):
    """the kernel's out against longform_oracle.join_segments at ref_fade (default fade): float32(ref) bit for bit,
    a neighbour only within tol of a rounding boundary, every other sample untouched.  Returns (worst fraction,
    neighbours taken)."""
    ref_fade = ref_fade or fade
    o = Out((out_len,), env.device)
    env.K.join_segments(o.t, operand(torch.from_numpy(src), env.device), seg, fade)
    env.sync()
    assert o.bands_intact(), "join_segments wrote outside out"
    got = o.t.cpu()
    ref = LO.join_segments(np.full(out_len, np.nan), src, seg, ref_fade)
    w = LO.join_segments(np.full(out_len, np.nan), np.ones(len(src)), seg, ref_fade)
    cov = ~np.isnan(ref)
    assert bool(_sent_bits(got)[torch.from_numpy(~cov)].all()), "join_segments wrote outside its segments"
    g = got.numpy()[cov].astype(np.float64)
    r, tol = ref[cov], 1e-15 + 4 * U64 / w[cov]
    lo, hi = r - tol * np.abs(r), r + tol * np.abs(r)
    ok = (g >= lo.astype(np.float32)) & (g <= hi.astype(np.float32))
    if not ok.all():
        i = int(np.flatnonzero(~ok)[0])
        raise AssertionError(f"join_segments (fade {fade}, reference {ref_fade}): {int((~ok).sum())} samples off; "
                             f"first: {g[i]!r}, float64 {r[i]!r}")
    nb = int((g != r.astype(np.float32)).sum())
    half = np.spacing(np.abs(r).astype(np.float32)).astype(np.float64) / 2
    return float(np.max(np.abs(g - r) / (half + tol * np.abs(r) + 1e-300), initial=0.0)), nb


def join_abi_skips(env):
    """through the C ABI: rows outside [0, out_len) (negative start, destination or length, or past the end) write
    nothing; the valid rows around them are written as through K.join_segments"""
    src = torch.from_numpy(rng(1).randn(500).astype(np.float32))
    out_len = 300
    good = np.array([[0, 0, 40], [100, 60, 50], [7, 250, 50]], np.int64)
    bad = np.array([[-1, 120, 10], [0, -1, 10], [0, 140, -3], [0, 260, 41], [0, 301, 0], [0, 2 ** 40, 5]], np.int64)
    seg = np.concatenate([bad[:3], good, bad[3:]])
    o = Out((out_len,), env.device)
    sd = operand(torch.from_numpy(seg), env.device)
    rc = env.lib.taco_join_segments(_p(o.t), out_len, _p(operand(src, env.device)), _p(sd), len(seg),
                                    int(max(seg[:, 2].max(), 0)), 16, env.stream)
    assert rc == 0, env.lib.taco_last_error().decode()
    env.sync()
    o2 = Out((out_len,), env.device)
    env.K.join_segments(o2.t, operand(src, env.device), good, 16)
    env.sync()
    assert o.bands_intact() and same_bits(o.t, o2.t), "join_segments: a segment outside out wrote"


# ------------------------------------------------------------------------------------------------------------------
# 4. taco_de_emphasis
# ------------------------------------------------------------------------------------------------------------------
def de_signal(kind, n, seed):
    g = rng(seed)
    if kind == "noise":
        return g.randn(n).astype(np.float32)
    if kind == "burst":                                  # 2000 loud samples, then 1e-6 noise for the rest
        x = (g.randn(n) * 1e-6).astype(np.float32)
        x[:min(n, 2000)] = g.randn(min(n, 2000)) * 1e3
        return x
    if kind == "dc":
        return np.full(n, 0.75, np.float32)
    if kind == "alt":
        return np.where(np.arange(n) % 2 == 0, 1.0, -1.0).astype(np.float32)
    raise ValueError(kind)


def run_de(env, x, start, c):
    """the kernel in place on a buffer holding x over [start[0], start[S]) and the sentinel elsewhere; checks that
    every sample outside (and the PAD bands) is untouched.  Returns the buffer."""
    N = len(x)
    o = Out((N,), env.device)
    a, b = int(start[0]), int(start[-1])
    o.t[a:b] = torch.from_numpy(x[a:b]).to(env.device)
    env.K.de_emphasis(o.t, np.asarray(start, np.int64), c)
    env.sync()
    assert o.bands_intact(), "de_emphasis wrote outside y"
    sb = _sent_bits(o.t.cpu())
    assert bool(sb[:a].all()) and bool(sb[b:].all()), "de_emphasis wrote outside [start[0], start[S])"
    return o.t.cpu().numpy()


def de_check(env, x, start, c, ref_c=None):
    """worst |y - y64| / bar over every segment (reference at ref_c, default the kernel's c)"""
    c = float(np.float32(c))
    ref_c = c if ref_c is None else float(np.float32(ref_c))
    y = run_de(env, x, start, c)
    a, b = int(start[0]), int(start[-1])
    if c == 0.0:
        assert same_bits(torch.from_numpy(y[a:b]), torch.from_numpy(x[a:b])), "de_emphasis at c = 0 is not the input"
    x64 = np.asarray(x, np.float64)
    y64 = GO.de_emphasis(x64, start, ref_c)[a:b]
    A = GO.de_emphasis(np.abs(x64), start, ref_c)
    Bs = GO.de_emphasis(A, start, ref_c)[a:b]
    bar = SAFETY * U * (1.003 * Bs + DE_L * A[a:b])
    return _frac(torch.from_numpy(np.abs(y[a:b].astype(np.float64) - y64)), torch.from_numpy(bar + 1e-300),
                 f"de_emphasis (c={c}, reference {ref_c})")


DE_LENGTHS = [0, 1, 15, 16, 17, 8191, 8192, 8193, 16383, 16385, 3 * 8192 + 5]


def de_segments(lens, first=3, tail=5):
    start = np.concatenate([[first], first + np.cumsum(lens)]).astype(np.int64)
    return start, int(start[-1]) + tail


def de_laws(env, x, start, c, picks):
    """bit for bit: a NaN in one segment leaves the others; a segment alone gives its bits in the batch"""
    y = run_de(env, x, start, c)
    S = len(start) - 1
    nz = [s for s in range(S) if start[s + 1] > start[s]]
    s = nz[len(nz) // 2]
    xn = x.copy()
    xn[(start[s] + start[s + 1]) // 2] = np.nan
    yn = run_de(env, xn, start, c)
    keep = np.ones(len(x), bool)
    keep[start[s]:start[s + 1]] = False
    assert same_bits(torch.from_numpy(yn[keep]), torch.from_numpy(y[keep])), "de_emphasis: a NaN crossed segments"
    for s in picks:
        ya = run_de(env, x, start[s:s + 2], c)
        sl = slice(int(start[s]), int(start[s + 1]))
        assert same_bits(torch.from_numpy(ya[sl]), torch.from_numpy(y[sl])), f"de_emphasis segment {s} differs alone"


def de_sensitivity(env, x, start, c, ks):
    """largest k (smallest perturbation) whose kernel run at c (1 + 2^-k) the check flags against the reference at c"""
    flagged = []
    for k in ks:
        ck = float(np.float32(c * (1 + 2.0 ** -k)))
        if ck == float(np.float32(c)):
            continue
        try:
            de_check(env, x, start, ck, ref_c=c)
        except AssertionError:
            flagged.append(k)
    return max(flagged) if flagged else None


# ------------------------------------------------------------------------------------------------------------------
# 5. taco_resample
# ------------------------------------------------------------------------------------------------------------------
def loop_at(x, ratio, wd, step, treg, ts):
    """resample_oracle.resample_loop's outputs at indices ts (from its register treg), vectorised over ts in the loop's
    order of operations; with the float64 sums of the same taps, sum |w x| and the tap counts"""
    xd = np.asarray(x, np.float32).astype(np.float64)
    win, delta = wd[:, 0], wd[:, 1]
    nwin, n_in = len(win), len(xd)
    scale = min(1.0, ratio)
    tr = treg[ts]
    n = tr.astype(np.int64)
    frac = scale * (tr - n)
    y = np.zeros(len(ts), np.float32)
    s64, sabs, taps = np.zeros(len(ts)), np.zeros(len(ts)), np.zeros(len(ts), np.int64)
    for side in (0, 1):
        if side:
            frac = scale - frac
        idx = frac * RO.NUM_TABLE
        off = idx.astype(np.int64)
        eta = idx - off
        cnt = np.minimum(n + 1, (nwin - off) // step) if side == 0 else np.minimum(n_in - n - 1, (nwin - off) // step)
        for i in range(int(cnt.max(initial=0))):
            m = i < cnt
            o = np.where(m, off + i * step, 0)
            w = win[o] + eta * delta[o]
            xv = xd[np.where(m, n - i if side == 0 else n + 1 + i, 0)]
            y = np.where(m, (y.astype(np.float64) + w * xv).astype(np.float32), y)
            s64 += np.where(m, w * xv, 0.0)
            sabs += np.where(m, np.abs(w * xv), 0.0)
        taps += np.maximum(cnt, 0)
    return y, s64, sabs, taps


def rs_setup(lens, sr_orig, sr_new):
    from tacotron_b200 import audio
    ratio = float(sr_new) / sr_orig
    sizes = [RO.lengths(n, sr_orig, sr_new) for n in lens]
    wd, step = audio.resample_filter(sr_orig, sr_new)
    treg = audio.resample_register(ratio, max(s[0] for s in sizes))
    return ratio, sizes, np.array(wd), step, treg


def run_resample(env, waves, sr_orig, sr_new, treg=None):
    lens = [len(w) for w in waves]
    ratio, sizes, wd, step, treg0 = rs_setup(lens, sr_orig, sr_new)
    treg = treg0 if treg is None else treg
    in_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    out_off = np.concatenate([[0], np.cumsum([s[1] for s in sizes])]).astype(np.int64)
    dev = env.device
    o = Out((int(out_off[-1]),), dev)
    env.K.resample(o.t, operand(torch.from_numpy(np.concatenate(waves)), dev), operand(torch.from_numpy(in_off), dev),
                   operand(torch.from_numpy(out_off), dev), operand(torch.from_numpy(wd), dev), step, ratio,
                   operand(torch.from_numpy(treg), dev))
    env.sync()
    assert o.bands_intact() and o.written(), "resample: guards"
    return o.t.cpu().numpy(), out_off, sizes, ratio, wd, step, treg0


def resample_check(env, waves, sr_orig, sr_new, sample=None, treg=None, loop=False):
    """every utterance: zero tail exact, outputs (all, or `sample(b, n_out)` of them) bit for bit the loop's and within
    taps u sum |w x| of the float64 sum.  loop=True also runs resample_oracle.resample_loop whole (small inputs) and
    requires loop_at to match it.  Returns the worst fraction."""
    y, out_off, sizes, ratio, wd, step, treg0 = run_resample(env, waves, sr_orig, sr_new, treg)
    worst = 0.0
    for b, w in enumerate(waves):
        yb = y[out_off[b]:out_off[b + 1]]
        n_out, n_fix = sizes[b]
        assert np.all(yb[n_out:] == 0) and not np.signbit(yb[n_out:]).any(), f"resample {b}: zero tail"
        ts = np.arange(n_out) if sample is None else np.unique(sample(b, n_out))
        want, s64, sabs, taps = loop_at(w, ratio, wd, step, treg0, ts)
        if loop:
            full = RO.resample_loop(w, sr_orig, sr_new)
            assert same_bits(torch.from_numpy(want), torch.from_numpy(full[ts])), "loop_at differs from resample_loop"
        bad = np.flatnonzero(yb[ts].view(np.int32) != want.view(np.int32))
        if bad.size:
            t = int(ts[bad[0]])
            raise AssertionError(f"resample {sr_orig}->{sr_new} utterance {b} (n_in {len(w)}): {bad.size} outputs "
                                 f"differ from the loop; first t = {t}: {yb[t]!r} != {want[bad[0]]!r}")
        bar = taps * U * sabs * (1 + 2.0 ** -20) + 1e-300
        worst = max(worst, _frac(torch.from_numpy(np.abs(yb[ts].astype(np.float64) - s64)), torch.from_numpy(bar),
                                 f"resample {sr_orig}->{sr_new} against the float64 sum"))
    return worst


def resample_lengths(sr_orig, sr_new):
    """the fewest samples giving an output, shorter than a wing, both wings clamped at once, one side clamped, long"""
    ratio = float(sr_new) / sr_orig
    one = 1
    while int(one * ratio) < 1:
        one += 1
    wing = int(64 / min(1.0, ratio))
    return [one, one + 1, 7, wing // 2 + 1, wing - 1, wing + 1, 2 * wing - 1, 2 * wing + 3, 3 * wing + 11]


def resample_abi_nan(env, sr_orig=48000, sr_new=16000, n_in=601):
    """through the C ABI with a register shorter than the output: t >= treg_len is NaN, t >= n_out the zero tail,
    the rest the loop's bits"""
    x = rng(3).randn(n_in).astype(np.float32)
    ratio, sizes, wd, step, treg = rs_setup([n_in], sr_orig, sr_new)
    n_out, n_fix = sizes[0]
    tl = n_out - 17
    dev = env.device
    o = Out((n_fix,), dev)
    args = [operand(torch.from_numpy(v), dev) for v in (x, np.array([0, n_in], np.int64), np.array([0, n_fix], np.int64),
                                                         wd, treg[:tl])]
    rc = env.lib.taco_resample(_p(o.t), _p(args[0]), _p(args[1]), _p(args[2]), 1, _p(args[3]), wd.shape[0], step,
                               C.c_double(ratio), _p(args[4]), tl, env.stream)
    assert rc == 0, env.lib.taco_last_error().decode()
    env.sync()
    y = o.t.cpu().numpy()
    assert o.bands_intact()
    assert np.isnan(y[tl:n_out]).all() and np.all(y[n_out:] == 0), "resample: t >= treg_len not NaN / tail not 0"
    want = loop_at(x, ratio, wd, step, treg, np.arange(tl))[0]
    assert same_bits(torch.from_numpy(y[:tl]), torch.from_numpy(want)), "resample with a short register"


def resample_sensitivity(env, x, sr_orig, sr_new, sample):
    """the kernel on the register of ratio one ulp up: (outputs the bit check flags, float64-bar fraction)"""
    from tacotron_b200 import audio
    ratio, sizes, wd, step, treg = rs_setup([len(x)], sr_orig, sr_new)
    treg_up = audio.resample_register(float(np.nextafter(ratio, np.inf)), len(treg))
    y = run_resample(env, [x], sr_orig, sr_new, treg=treg_up)[0]
    ts = np.unique(sample)
    want = loop_at(x, ratio, wd, step, treg, ts)[0]
    return int((y[ts].view(np.int32) != want.view(np.int32)).sum())
