"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY.  The resampling inside the reference's ``librosa.load(fname, mono=True, sr=sr)``
(audio.py:39) when a file is not at `sr`: librosa 0.6 ``resample(y, orig_sr, target_sr, res_type='kaiser_best',
fix=True)`` over resampy 0.2.2's ``resample`` / ``resample_f``, restated from the published algorithm.  Neither librosa
nor resampy is installed here, so parity with a resampy build stays unpinned; what is pinned is this arithmetic:

  filter  resampy's kaiser_best table: num_zeros = 64, precision = 9 (512 entries per zero crossing), Kaiser beta
          14.769656459379492, rolloff 0.9475937167399596; win = kaiser(2n+1, beta)[n:] * rolloff *
          sinc(rolloff * linspace(0, 64, n+1)), n = 512 * 64 (32769 float64 values).  When ratio = sr_new / sr_orig < 1
          the table is scaled by ratio; delta[:-1] = diff(win), delta[-1] = 0.
  lengths n_out = int(n_in * ratio) (resampy; n_out < 1 is an error), then zero-padded to ceil(n_in * ratio) (librosa's
          fix_length).
  loop    scale = min(1, ratio), step = int(scale * 512), time register treg[t] = treg[t-1] + 1/ratio summed in float64
          one output at a time.  For output t: n = int(treg[t]), frac = scale*(treg[t] - n), idx = frac*512,
          off = int(idx), eta = idx - off; left wing i < min(n+1, (nwin-off)//step): y += (win[o] + eta*delta[o]) * x[n-i]
          with o = off + i*step; then frac = scale - frac gives off and eta of the right wing,
          k < min(n_in-n-1, (nwin-off)//step): y += (...) * x[n+k+1].  The weight and the product are float64; y is
          float32 and rounded after every add (numba's `y[t] += weight * x[..]` on a float32 array), no fused
          multiply-add, left wing before right wing.

`resample` vectorises the loop over t and keeps each output's tap order; `resample_loop` is the loop itself, for small
inputs.
"""
from __future__ import annotations

import numpy as np

NUM_ZEROS, NUM_TABLE = 64, 512
BETA, ROLLOFF = 14.769656459379492, 0.9475937167399596


def kaiser_best():
    """resampy's kaiser_best half window (float64 [32769]) before any ratio scaling"""
    from scipy.signal.windows import kaiser
    n = NUM_TABLE * NUM_ZEROS
    return kaiser(2 * n + 1, BETA)[n:] * (ROLLOFF * np.sinc(ROLLOFF * np.linspace(0, NUM_ZEROS, n + 1)))


def filter_table(ratio):
    """(win, delta) float64 as resampy.resample hands them to resample_f"""
    win = kaiser_best()
    if ratio < 1:
        win *= ratio
    delta = np.zeros_like(win)
    delta[:-1] = np.diff(win)
    return win, delta


def lengths(n_in, sr_orig, sr_new):
    ratio = float(sr_new) / sr_orig
    return int(n_in * ratio), int(np.ceil(n_in * ratio))


def time_register(ratio, n):
    """treg[0 .. n): the float64 register resample_f advances by 1/ratio after every output"""
    inc = 1.0 / ratio
    treg = np.zeros(n)
    acc = 0.0
    for t in range(1, n):
        acc = acc + inc
        treg[t] = acc
    return treg


def _positions(treg, scale):
    n = treg.astype(np.int64)
    frac = scale * (treg - n)
    idx = frac * NUM_TABLE
    off = idx.astype(np.int64)
    return n, frac, off, idx - off


def resample(x, sr_orig, sr_new, treg=None):
    """librosa.resample(x, sr_orig, sr_new, res_type='kaiser_best') for a float32 mono signal -> float32 [ceil(n*ratio)].
    treg: other positions in place of the time register (to show what the register's rounding does)."""
    x = np.asarray(x, dtype=np.float32)
    ratio = float(sr_new) / sr_orig
    n_in = len(x)
    n_out, n_fix = lengths(n_in, sr_orig, sr_new)
    if n_out < 1:
        raise ValueError(f"{n_in} samples at {sr_orig} Hz are too few to resample to {sr_new} Hz")
    win, delta = filter_table(ratio)
    nwin = len(win)
    scale = min(1.0, ratio)
    step = int(scale * NUM_TABLE)
    xd = x.astype(np.float64)
    y = np.zeros(n_out, dtype=np.float32)
    n, frac, off, eta = _positions(time_register(ratio, n_out) if treg is None else treg[:n_out], scale)

    def wing(count, off, eta, src):
        nonlocal y
        for i in range(int(count.max(initial=0))):
            m = i < count
            o = np.where(m, off + i * step, 0)
            w = win[o] + eta * delta[o]
            s = (y.astype(np.float64) + w * xd[np.where(m, src(i), 0)]).astype(np.float32)
            y = np.where(m, s, y)

    wing(np.minimum(n + 1, (nwin - off) // step), off, eta, lambda i: n - i)
    frac = scale - frac
    idx = frac * NUM_TABLE
    off = idx.astype(np.int64)
    wing(np.minimum(n_in - n - 1, (nwin - off) // step), off, idx - off, lambda i: n + i + 1)
    return np.concatenate([y, np.zeros(n_fix - n_out, np.float32)])


def resample_loop(x, sr_orig, sr_new):
    """resampy 0.2.2's resample_f written out sample by sample (slow: small inputs only), zero-padded as librosa does"""
    x = np.asarray(x, dtype=np.float32)
    ratio = float(sr_new) / sr_orig
    n_out, n_fix = lengths(len(x), sr_orig, sr_new)
    win, delta = filter_table(ratio)
    nwin, n_orig = len(win), len(x)
    scale = min(1.0, ratio)
    time_increment = 1.0 / ratio
    index_step = int(scale * NUM_TABLE)
    time_register = 0.0
    y = np.zeros(n_fix, dtype=np.float32)
    for t in range(n_out):
        n = int(time_register)
        frac = scale * (time_register - n)
        index_frac = frac * NUM_TABLE
        offset = int(index_frac)
        eta = index_frac - offset
        for i in range(min(n + 1, (nwin - offset) // index_step)):
            weight = win[offset + i * index_step] + eta * delta[offset + i * index_step]
            y[t] = np.float32(float(y[t]) + weight * float(x[n - i]))
        frac = scale - frac
        index_frac = frac * NUM_TABLE
        offset = int(index_frac)
        eta = index_frac - offset
        for k in range(min(n_orig - n - 1, (nwin - offset) // index_step)):
            weight = win[offset + k * index_step] + eta * delta[offset + k * index_step]
            y[t] = np.float32(float(y[t]) + weight * float(x[n + k + 1]))
        time_register += time_increment
    return y
