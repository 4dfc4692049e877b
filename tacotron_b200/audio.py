"""Spectrogram inversion on the GPU -- host-side mirror of the reference's ``audio.py`` inversion surface
(``reshape_frames`` :23-35, ``invert_spectrogram`` :67-75, ``griffinlim`` :77-97), SURVEY.md section 8(f) rank 1:
it sits inside BASELINE config 5's end-to-end latency (test.py:64) and would dominate it on the CPU.

Design: a batch of utterances stays on the device for all iterations.  The two transforms per iteration are the library's
own shared-memory FFT kernels (csrc/audio.cu ``taco_rfft2048`` / ``taco_irfft2048``: radix-4 Stockham, one CTA per frame --
round 1 called cuFFT through ``torch.fft`` here); everything between them is four fused kernels of libtaco_b200.so:

    gl_init   reshape_frames(forward=False) + de-normalisation + exp + initial phase  ->  magnitude, first spectrum
    gl_ola    window, overlap-add, window-sum-square normalisation, centre trim        (the tail of librosa.istft)
    gl_frame  reflect padding, framing, window                                         (the head of librosa.stft)
    gl_phase  mag * rebuilt/|rebuilt|                                                  (audio.py:84,87)

so one iteration is irfft2048 -> gl_ola -> gl_frame -> rfft2048 -> gl_phase: 5 launches of this library, ~20 MB of HBM traffic per utterance of
500 frames.  All arithmetic goes through the kernel namespace K (tacotron_b200/kernels.py); tests run the same
orchestration over tests/mirror_kernels.py on CPU tensors against the numpy oracle (oracle/audio_oracle.py).
``speech_frames`` / ``invert_speech`` are the opt-in tail trim of synthesis: where each utterance's speech ends
(taco_speech_frames), then the same loop over only the kept frames of the batch, packed end to end.
``momentum`` (every inversion entry point) is fast Griffin-Lim: gl_phase_momentum in place of gl_phase, with two rebuilt
buffers written in turn.  ``de_emphasis`` undoes preprocessing's pre-emphasis on synthesised waveforms (taco_de_emphasis).

Feature extraction (the reference's ``process_audio``, audio.py:38-65, used by tacotron_b200/preprocess.py) is the
analysis half of the same transform: trim_bounds -> feature_frames -> rfft2048 -> feature_spec, four launches per chunk of
utterances (csrc/features.cu).  ``load_wav`` reads a WAV file the way ``librosa.load(f, mono=True, sr=sr)`` does when no
resampling is needed and rejects a file at another rate.  ``read_wav`` returns the file's rate instead, and
``resample_batch`` / ``process_audio_batch(rates=...)`` do librosa.load's resampling on the device (csrc/resample.cu:
librosa 0.6's kaiser_best over resampy 0.2.2's loop, one launch per source rate in a chunk).
"""
from __future__ import annotations

import functools

import numpy as np
import torch

n_fft = 2048            # audio.py:10
win_length = 1200       # audio.py:11
hop_length = 300        # audio.py:12
maximum_audio_length = 108000   # audio.py:13
F_BINS = 1 + n_fft // 2
PRE_EMPHASIS = 0.97     # audio.py:53
N_MELS = 80             # audio.py:57
MEL_SR = 22050          # librosa's default sr: melspectrogram(S=stft) builds its basis at this rate, not the file's
TRIM_TOP_DB, TRIM_FRAME, TRIM_HOP = 60.0, 2048, 512     # librosa.effects.trim defaults (audio.py:42)
STFT_FRAMES = 1 + maximum_audio_length // hop_length     # 361
MIN_SAMPLES = n_fft // 2 + 1                             # shorter signals cannot be reflect-padded by n_fft/2
RS_ZEROS, RS_TABLE = 64, 512                             # resampy's kaiser_best: 64 zero crossings, 2^9 entries each
RS_BETA, RS_ROLLOFF = 14.769656459379492, 0.9475937167399596


def feature_frames_per_utterance(r):
    """rows of the stored arrays: 4*(361 // 4r) frames survive reshape_frames; the reference allocates
    maximum_audio_length // (hop*r) rows (preprocess.py:178).  The two agree for r in {1, 2, 3, 5, 6}.  At r = 4 they
    do not (88 vs 90), and the reference fails on the assignment (preprocess.py:194); its guard (audio.py:46) never
    fires because `% 4*r` is `(x % 4) * r`."""
    if r < 1:
        raise ValueError(f"r = {r} is not supported for preprocessing (use r in 1, 2, 3, 5, 6)")
    rows, stored = 4 * (STFT_FRAMES // (4 * r)), maximum_audio_length // (hop_length * r)
    if rows != stored:
        raise ValueError(f"r = {r} is not supported for preprocessing: reshape_frames keeps {rows} rows of "
                         f"{maximum_audio_length} samples, but the stored arrays have {stored} (use r in 1, 2, 3, 5, 6)")
    return rows


def load_wav(path, sr):
    """librosa.load(path, mono=True, sr=sr) (audio.py:39) for a WAV file already at `sr` (see read_wav); a file at another
    rate is an error (read_wav + resample_batch convert it)."""
    x, rate = read_wav(path)
    if rate != sr:
        raise ValueError(f"{path}: sample rate {rate} Hz, expected {sr} Hz (load_wav does not resample; preprocess with "
                         f"--resample to convert it)")
    return x


def read_wav(path):
    """a WAV file as librosa.load(path, mono=True, sr=None) reads it -> (float32 samples, rate): int16 / 32768, int32 and
    24-bit / 2^31, (uint8 - 128) / 128, float as stored, channels averaged in float32."""
    from scipy.io import wavfile
    rate, x = wavfile.read(path)
    if x.dtype == np.int16:
        x = x.astype(np.float32) / np.float32(32768.0)
    elif x.dtype == np.int32:
        x = (x.astype(np.float64) / 2147483648.0).astype(np.float32)
    elif x.dtype == np.uint8:
        x = (x.astype(np.float32) - np.float32(128.0)) / np.float32(128.0)
    elif x.dtype.kind == "f":
        x = x.astype(np.float32)
    else:
        raise ValueError(f"{path}: unsupported WAV sample format {x.dtype}")
    if x.ndim == 2:
        x = np.mean(x, axis=1, dtype=np.float32)
    return np.ascontiguousarray(x), int(rate)


def resample_lengths(n_in, sr_orig, sr_new, what="signal"):
    """(n_out, n_fix) of librosa.resample: resampy computes int(n_in * ratio) samples (fewer than one is an error naming
    `what`), librosa zero-pads them to ceil(n_in * ratio)"""
    ratio = float(sr_new) / sr_orig
    n_out, n_fix = int(n_in * ratio), int(np.ceil(n_in * ratio))
    if n_out < 1:
        raise ValueError(f"{what}: {n_in} samples at {sr_orig} Hz are too few to resample to {sr_new} Hz")
    return n_out, n_fix


@functools.lru_cache(maxsize=None)
def _kaiser_best():
    from scipy.signal.windows import kaiser
    n = RS_TABLE * RS_ZEROS
    return kaiser(2 * n + 1, RS_BETA)[n:] * (RS_ROLLOFF * np.sinc(RS_ROLLOFF * np.linspace(0, RS_ZEROS, n + 1)))


def resample_filter(sr_orig, sr_new):
    """resampy 0.2.2's kaiser_best table as resample_f receives it for ratio = sr_new / sr_orig -> (win_delta float64
    [32769, 2] = {win, delta}, step).  win = kaiser(2n+1, beta)[n:] * rolloff * sinc(rolloff * linspace(0, 64, n+1)),
    n = 512*64, scaled by ratio when ratio < 1; delta[:-1] = diff(win), delta[-1] = 0; step = int(min(1, ratio) * 512).
    Restated from the published algorithm: parity with a resampy build is not pinned."""
    return _resample_filter(float(sr_new) / sr_orig)


@functools.lru_cache(maxsize=None)
def _resample_filter(ratio):
    win = _kaiser_best().copy()
    if ratio < 1:
        win *= ratio
    wd = np.zeros((len(win), 2))
    wd[:, 0] = win
    wd[:-1, 1] = np.diff(win)
    wd.flags.writeable = False
    return wd, int(min(1.0, ratio) * RS_TABLE)


def resample_register(ratio, n):
    """resample_f's time register for the first n outputs: treg[0] = 0, treg[t] = treg[t-1] + 1/ratio in float64, summed
    in order (np.cumsum is that recurrence).  Not t/ratio: the kernels reproduce the truncations of the running sum."""
    treg = np.zeros(n)
    np.cumsum(np.full(n - 1, 1.0 / ratio), out=treg[1:])
    return treg


_rs_dev = {}


def _resample_on(ratio, n, device):
    """the table and a time register of at least n entries on `device`, cached per ratio; the register grows (its
    prefix does not change) when a longer utterance arrives"""
    key = (str(device), ratio)
    wd, treg = _rs_dev.get(key, (None, None))
    if wd is None:
        wd = torch.from_numpy(_resample_filter(ratio)[0].copy()).to(device)
    if treg is None or treg.numel() < n:
        treg = torch.from_numpy(resample_register(ratio, n)).to(device)
    _rs_dev[key] = (wd, treg)
    return wd, treg


def _upload(waves, device):
    cuda = torch.device(device).type == "cuda"
    y = torch.from_numpy(np.concatenate(waves).astype(np.float32, copy=False) if len(waves) else np.zeros(0, np.float32))
    return (y.pin_memory() if cuda else y).to(device, non_blocking=True)


def _resample_device(waves, rates, sr, K, device):
    """the chunk on `device`, packed end to end in order with every utterance at `sr` -> (y, lengths int64).  One
    resample launch per source rate; an utterance already at `sr` is copied unchanged."""
    lens = np.array([len(w) for w in waves], dtype=np.int64)
    groups = {}
    for b, q in enumerate(rates):
        if int(q) != sr:
            groups.setdefault(int(q), []).append(b)
    sizes = {b: resample_lengths(int(lens[b]), q, sr, f"utterance {b}") for q, idx in groups.items() for b in idx}
    same = [b for b in range(len(waves)) if b not in sizes]
    parts = [None] * len(waves)
    if same:
        y = _upload([waves[b] for b in same], device)
        off = np.concatenate([[0], np.cumsum(lens[same])])
        for j, b in enumerate(same):
            parts[b] = y[off[j]:off[j + 1]]
    for q, idx in groups.items():
        ratio = float(sr) / q
        n_out = max(sizes[b][0] for b in idx)
        in_off = np.concatenate([[0], np.cumsum(lens[idx])]).astype(np.int64)
        out_off = np.concatenate([[0], np.cumsum([sizes[b][1] for b in idx])]).astype(np.int64)
        out = torch.empty(int(out_off[-1]), dtype=torch.float32, device=device)
        wd, treg = _resample_on(ratio, n_out, device)
        K.resample(out, _upload([waves[b] for b in idx], device), torch.from_numpy(in_off).to(device),
                   torch.from_numpy(out_off).to(device), wd, _resample_filter(ratio)[1], ratio, treg[:n_out])
        for j, b in enumerate(idx):
            parts[b] = out[out_off[j]:out_off[j + 1]]
            lens[b] = sizes[b][1]
    return torch.cat(parts) if parts else torch.zeros(0, dtype=torch.float32, device=device), lens


def resample_batch(waves, rates, sr, K=None, device="cuda"):
    """librosa.resample(w, rates[b], sr, res_type='kaiser_best') (librosa 0.6 over resampy 0.2.2, as librosa.load(f,
    sr=sr) applies it; audio.py:39) for each mono float32 waveform -> list of float32 numpy arrays of ceil(n*sr/rate)
    samples.  A waveform already at `sr` is returned unchanged.  The arithmetic is resampy's loop, bit for bit, as restated
    in resample_filter / resample_register (tests/resample_oracle.py); parity with resampy itself is not pinned."""
    y, lens = _resample_device(waves, rates, sr, K or _K(), device)
    y = y.cpu().numpy()
    off = np.concatenate([[0], np.cumsum(lens)])
    return [y[off[b]:off[b + 1]].copy() for b in range(len(waves))]


def mel_basis(sr=MEL_SR, n_mels=N_MELS):
    """librosa.filters.mel(sr, n_fft=2048, n_mels, dtype=float32) (librosa 0.6-0.9: Slaney mel scale, fmin 0, fmax sr/2,
    norm=1) -> basis float32 [n_mels, 1025] and the range [lo, hi) of bins each filter covers (int32 [n_mels] each).
    Each row is rounded to float32, then scaled by the area normalisation in float64 and rounded again, as librosa's
    in-place `weights *= enorm` does."""
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0

    def hz_to_mel(f):
        return min_log_mel + np.log(f / min_log_hz) / logstep if f >= min_log_hz else f / f_sp

    mels = np.linspace(hz_to_mel(0.0), hz_to_mel(sr / 2.0), n_mels + 2)
    mel_f = np.where(mels >= min_log_mel, min_log_hz * np.exp(logstep * (mels - min_log_mel)), f_sp * mels)
    fftfreqs = np.linspace(0, sr / 2.0, F_BINS, endpoint=True)
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    weights = np.zeros((n_mels, F_BINS), dtype=np.float32)
    for i in range(n_mels):
        weights[i] = np.maximum(0, np.minimum(-ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]))
    weights *= (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]
    lo = np.zeros(n_mels, dtype=np.int32)
    hi = np.zeros(n_mels, dtype=np.int32)
    for i in range(n_mels):
        nz = np.flatnonzero(weights[i])
        if nz.size:
            lo[i], hi[i] = nz[0], nz[-1] + 1
    return weights, lo, hi


_mel_dev = {}


def _mel_on(device):
    key = str(device)
    if key not in _mel_dev:
        _mel_dev[key] = tuple(torch.from_numpy(a).to(device) for a in mel_basis())
    return _mel_dev[key]


def process_audio_batch(waves, r, K=None, device="cuda", out_dtype=torch.float16, rates=None, sr=None):
    """The reference's process_audio (audio.py:38-65) for a chunk of mono float32 waveforms (numpy, each at least
    1025 samples): trim silence, drop an utterance longer than maximum_audio_length after trimming, zero-pad, pre-emphasise,
    STFT, mel, log, reshape_frames(forward=True).  Returns (mel [n, T, 80 r], stft [n, T, 1025 r], keep [N] bool) with
    the n = keep.sum() kept utterances in order, T = feature_frames_per_utterance(r); the arrays are on `device`.
    rates: the waveforms' sample rates; each one not at `sr` is first resampled to `sr` on the device as librosa.load does
    (resample_batch), and the 1025-sample minimum applies to the result."""
    K = K or _K()
    T = feature_frames_per_utterance(r)
    y = None
    if rates is not None and any(int(q) != sr for q in rates):
        if sr is None:
            raise ValueError("process_audio_batch: rates given without the target rate sr")
        y, lens = _resample_device(waves, rates, sr, K, device)
    else:
        lens = np.array([len(w) for w in waves], dtype=np.int64)
    short = np.flatnonzero(lens < MIN_SAMPLES)
    if short.size:
        raise ValueError(f"utterance {int(short[0])} has {int(lens[short[0]])} samples; at least {MIN_SAMPLES} are needed")
    N = len(waves)
    offsets = np.zeros(N + 1, dtype=np.int64)
    np.cumsum(lens, out=offsets[1:])
    if y is None:
        y = _upload(waves, device)
    bounds = torch.empty((N, 2), dtype=torch.int32, device=device)
    K.trim_bounds(bounds, y, torch.from_numpy(offsets).to(device), TRIM_FRAME, TRIM_HOP, TRIM_TOP_DB)
    b = bounds.cpu().numpy().astype(np.int64)
    kept_len = b[:, 1] - b[:, 0]
    keep = kept_len <= maximum_audio_length
    idx = np.flatnonzero(keep)
    n = len(idx)
    mel = torch.empty((n, T, N_MELS * r), dtype=out_dtype, device=device)
    stft = torch.empty((n, T, F_BINS * r), dtype=out_dtype, device=device)
    if n:
        start = torch.from_numpy(offsets[idx] + b[idx, 0]).to(device)
        length = torch.from_numpy(kept_len[idx].astype(np.int32)).to(device)
        frw = torch.empty((n, STFT_FRAMES, n_fft), dtype=torch.float32, device=device)
        K.feature_frames(frw, y, start, length, maximum_audio_length, hop_length, win_length, PRE_EMPHASIS)
        X = torch.empty((n, STFT_FRAMES, F_BINS), dtype=torch.complex64, device=device)
        K.rfft2048(X, frw)
        del frw
        basis, lo, hi = _mel_on(device)
        K.feature_spec(stft, mel, X, basis, lo, hi, r)
    return mel, stft, keep


def process_audio(fname, sr=16000, r=2, K=None, device="cuda"):
    """audio.process_audio(fname, sr=sr) (audio.py:38-65) with r explicit: (mel [T, 80 r], stft [T, 1025 r]) float16 numpy
    arrays, or (None, None) when the trimmed utterance is longer than maximum_audio_length."""
    mel, stft, keep = process_audio_batch([load_wav(fname, sr)], r, K=K, device=device)
    if not keep[0]:
        return None, None
    return mel[0].cpu().numpy(), stft[0].cpu().numpy()


def _K():
    from . import kernels
    return kernels


def reshape_frames(signal, r, forward=False):
    """audio.reshape_frames (audio.py:23-35) as a pure index permutation on a torch tensor (any device).
    forward=False: [T, F*r] -> [4r*(T//4), F]; forward=True: [F, n] -> [4*(n//4r), F*r]."""
    if forward:
        Fd, n = signal.shape
        nb = n // (4 * r)
        s = signal[:, :nb * 4 * r].reshape(Fd, nb, r, 4)                     # frame = 4r*b + 4c + tl
        return s.permute(1, 3, 2, 0).reshape(nb * 4, r * Fd)                 # row = 4b + tl, col = c*F + k
    T, W = signal.shape
    Fd = W // r
    nb = T // 4
    s = signal[:nb * 4].reshape(nb, 4, r, Fd)                                # [b, tl, c, k]
    return s.permute(0, 2, 1, 3).reshape(nb * 4 * r, Fd)                     # frame = 4r*b + 4c + tl


def griffinlim_batch(spec, r, n_iter=50, scale=None, shift=None, phase_u=None, K=None, generator=None, momentum=0.0):
    """spec [B, T, 1025*r] (log magnitudes in the decoder's r-frames-per-step layout, optionally normalised:
    magnitude = exp(spec*scale + shift), the driver's ``out*stft_std + stft_mean`` of test.py:64) -> waveforms [B, L],
    L = hop*(4r*(T//4) - 1).  phase_u: uniform [0,1) initial phases [B, n, 1025] (audio.py:81), drawn if None.
    momentum in [0, 1]: fast Griffin-Lim (_gl_iterations); 0 is the reference's plain loop."""
    K = K or _K()
    gl_check(n_iter, momentum)
    B, T, W = spec.shape
    assert W == F_BINS * r, (W, r)
    n = 4 * r * (T // 4)
    assert n >= 2, "need at least one block of 4 decoder steps"
    L = hop_length * (n - 1)
    assert L > n_fft // 2, f"{n} frames are fewer than the reflect padding of the STFT needs (>= 5)"
    rdt = spec.dtype
    cdt = torch.complex64 if rdt == torch.float32 else torch.complex128
    if phase_u is None:
        phase_u = torch.rand((B, n, F_BINS), dtype=rdt, device=spec.device, generator=generator)
    mag = torch.empty((B, n, F_BINS), dtype=rdt, device=spec.device)
    full = torch.empty((B, n, F_BINS), dtype=cdt, device=spec.device)
    y = torch.empty((B, L), dtype=rdt, device=spec.device)
    frw = torch.empty((B, n, n_fft), dtype=rdt, device=spec.device)
    _gl_iterations(K, full, mag, spec, phase_u, r, scale, shift, y, frw, n_iter, momentum=momentum)
    return y


def gl_check(n_iter, momentum):
    """n_iter an integer >= 0 and momentum a number in [0, 1], else ValueError naming the value; -> beta =
    momentum / (1 + momentum), the weight of the previous iterate in fast Griffin-Lim's update"""
    if isinstance(n_iter, bool) or not isinstance(n_iter, (int, np.integer)) or n_iter < 0:
        raise ValueError(f"Griffin-Lim: n_iter = {n_iter!r} must be an integer >= 0")
    try:
        m = float(momentum)
    except (TypeError, ValueError):
        m = float("nan")
    if isinstance(momentum, bool) or not 0.0 <= m <= 1.0:
        raise ValueError(f"Griffin-Lim: momentum = {momentum!r} must be a number in [0, 1]")
    return m / (1.0 + m)


def _gl_iterations(K, full, mag, spec, phase_u, r, scale, shift, y, frw, n_iter, rebuilt=None, packed=None, momentum=0.0):
    """frw [B, n, 2048] doubles as the istft frame buffer: irfft writes it, gl_ola consumes it, gl_frame refills it.
    packed: (off, max_frames) of invert_speech's packed layout (rows off[b]:off[b+1] per utterance), None for [B, n, .].
    momentum > 0: fast Griffin-Lim (Perraudin, Balazs & Sondergaard 2013; librosa >= 0.7), angles = d/|d| with
    d = rebuilt - beta*rebuilt_prev, beta = momentum/(1 + momentum).  rebuilt: one buffer like full, or the two the FFT
    writes in turn when momentum > 0 (the other holds the previous iterate, so nothing is copied).  momentum = 0 is the
    plain loop, launch for launch."""
    beta = gl_check(n_iter, momentum)
    if rebuilt is None:
        rebuilt = torch.empty_like(full) if beta == 0 else (torch.empty_like(full), torch.empty_like(full))
    elif beta > 0 and not isinstance(rebuilt, tuple):
        raise ValueError("Griffin-Lim with momentum needs two rebuilt buffers")
    if packed is None:
        K.gl_init(full, mag, spec, phase_u, r, scale, shift)
        ola = functools.partial(K.gl_ola, y, frw, hop_length, win_length)
        frame = functools.partial(K.gl_frame, frw, y, hop_length, win_length)
    else:
        off, nmax = packed
        K.gl_init_packed(full, mag, spec, phase_u, off, r, nmax, scale, shift)
        ola = functools.partial(K.gl_ola_packed, y, frw, off, nmax, hop_length, win_length)
        frame = functools.partial(K.gl_frame_packed, frw, y, off, nmax, hop_length, win_length)
    for it in range(n_iter + 1):
        K.irfft2048(frw, full)                                               # inverse real FFT of every frame
        ola()
        if it == n_iter:
            break
        frame()
        if beta == 0:
            K.rfft2048(rebuilt, frw)                                         # real FFT of every re-framed, windowed frame
            K.gl_phase(full, mag, rebuilt)
            continue
        cur, prev = rebuilt[it % 2], rebuilt[(it + 1) % 2]
        K.rfft2048(cur, frw)
        if it == 0:                                                          # rebuilt_prev = 0
            K.gl_phase(full, mag, cur)
        else:
            K.gl_phase_momentum(full, mag, cur, prev, beta)


def speech_frames(spec, r, stft_mean=None, stft_std=None, top_db=TRIM_TOP_DB, K=None):
    """STFT frames to keep of each utterance of spec [B, T, 1025*r] (the post-net output, de-normalised with stft_std /
    stft_mean like invert_spectrogram) -> int32 [B] on spec's device, without a host synchronisation.  A frame is speech
    when its power is within top_db of the utterance's loudest frame; frames[b] is the end of the last one, rounded up to
    whole blocks of 4r frames (decoder steps [0, frames[b]/r)), at least 5 frames, and all 4r*(T//4) frames when the
    spectrogram is not finite.  The training targets end in log(1e-8) padding frames, so a trained model is taught to go
    quiet after its speech; the rule is reasoned from that, not observed on a trained model's output."""
    K = K or _K()
    scale, shift = (stft_std, stft_mean) if stft_std is not None else (None, None)
    frames = torch.empty(spec.shape[0], dtype=torch.int32, device=spec.device)
    K.speech_frames(frames, spec.contiguous(), r, scale, shift, top_db)
    return frames


def stop_frames(end_step, r, T, frames=None):
    """STFT frames to invert of each utterance of a decode the end-of-text stop rule ended (Tacotron.end_steps, T = the
    steps the call returned) -> int32 [B] on end_step's device, without a host synchronisation: min(4r ceil(end_step[b] /
    4), 4r (T // 4)), at least the 5 frames invert_speech needs, and at most frames[b] when frames (e.g. speech_frames
    with --trim-tail) is given."""
    n = 4 * r * (T // 4)
    lo = -(-5 // (4 * r)) * 4 * r
    f = ((end_step.to(torch.int64) + 3) // 4 * (4 * r)).clamp(min=min(lo, n), max=n)
    if frames is not None:
        f = torch.minimum(f, frames.to(torch.int64))
    return f.to(torch.int32)


def invert_speech(spec, r, frames, n_iter=50, stft_mean=None, stft_std=None, phase_u=None, K=None, generator=None,
                  momentum=0.0):
    """invert_spectrogram on the first frames[b] STFT frames of each utterance only (frames: speech_frames or the
    caller's, a multiple of 4r in [5, 4r*(T//4)] each) -> list of B 1-D waveforms of hop*(frames[b]-1) samples.  The kept
    frames are packed end to end, so one iteration is still 5 launches; utterance b equals invert_spectrogram on
    spec[b:b+1, :frames[b]//r] with the same initial phases.  phase_u: packed uniform [0,1) phases [sum(frames), 1025],
    drawn on the device if None.  Reads frames to the host once."""
    y, start = invert_speech_packed(spec, r, frames, n_iter, stft_mean, stft_std, phase_u, K, generator, momentum)
    return [y[start[b]:start[b + 1]] for b in range(len(start) - 1)]


def invert_speech_packed(spec, r, frames, n_iter=50, stft_mean=None, stft_std=None, phase_u=None, K=None, generator=None,
                         momentum=0.0):
    """invert_speech's waveforms as the one flat buffer Griffin-Lim writes: (y, start) with utterance b in
    y[start[b]:start[b+1]] (start int64 numpy [B+1])"""
    K = K or _K()
    gl_check(n_iter, momentum)
    B, T, W = spec.shape
    assert W == F_BINS * r, (W, r)
    n = 4 * r * (T // 4)
    fr = np.asarray(frames.cpu() if torch.is_tensor(frames) else frames).astype(np.int64).reshape(-1)
    if fr.shape != (B,):
        raise ValueError(f"invert_speech: {fr.size} frame counts for {B} utterances")
    bad = np.flatnonzero((fr % (4 * r) != 0) | (fr < 5) | (fr > n))
    if bad.size:
        b = int(bad[0])
        raise ValueError(f"invert_speech: frames[{b}] = {int(fr[b])} must be a multiple of 4r = {4 * r} in [5, {n}]")
    off = np.zeros(B + 1, dtype=np.int64)
    np.cumsum(fr, out=off[1:])
    N, nmax = int(off[-1]), int(fr.max())
    rdt, dev = spec.dtype, spec.device
    cdt = torch.complex64 if rdt == torch.float32 else torch.complex128
    if phase_u is None:
        phase_u = torch.rand((N, F_BINS), dtype=rdt, device=dev, generator=generator)
    elif phase_u.shape != (N, F_BINS):
        raise ValueError(f"invert_speech: phase_u must be the packed [{N}, {F_BINS}], got {tuple(phase_u.shape)}")
    scale, shift = (stft_std, stft_mean) if stft_std is not None else (None, None)
    mag = torch.empty((N, F_BINS), dtype=rdt, device=dev)
    full = torch.empty((N, F_BINS), dtype=cdt, device=dev)
    y = torch.empty(hop_length * (N - B), dtype=rdt, device=dev)
    frw = torch.empty((N, n_fft), dtype=rdt, device=dev)
    _gl_iterations(K, full, mag, spec.contiguous(), phase_u.contiguous(), r, scale, shift, y, frw, n_iter,
                   packed=(torch.from_numpy(off).to(dev), nmax), momentum=momentum)
    return y, hop_length * (off - np.arange(B + 1))


def speech_bounds(spec, r, stft_mean=None, stft_std=None, top_db=TRIM_TOP_DB, K=None):
    """Where each utterance's speech starts and ends in spec [B, T, 1025*r] (de-normalised like speech_frames) -> int32
    [B, 3] on spec's device, without a host synchronisation: {f0, f1, frames} = the first voiced STFT frame, the last
    voiced frame + 1, and exactly speech_frames' frame count; {0, n, n} when the spectrogram is not finite."""
    K = K or _K()
    scale, shift = (stft_std, stft_mean) if stft_std is not None else (None, None)
    bounds = torch.empty((spec.shape[0], 3), dtype=torch.int32, device=spec.device)
    K.speech_bounds(bounds, spec.contiguous(), r, scale, shift, top_db)
    return bounds


JOIN_FADE_S = 0.01      # raised-cosine fade at every cut of a joined waveform


def kept_samples(f0, f1, frames):
    """samples [a, b) of an utterance's invert_speech output (hop*(frames-1) samples) that long-form synthesis keeps for
    speech bounds (f0, f1): from one hop before the first voiced frame to the last voiced frame's hop"""
    L = hop_length * (frames - 1)
    return max(hop_length * (f0 - 1), 0), min(hop_length * f1, L)


def join_speech(out, src, seg, sr, K=None):
    """out[d:d+n] = src[a:a+n] with a raised-cosine fade of 10 ms (JOIN_FADE_S at sr) at both ends, for every row
    {a, d, n} of seg int64 [S, 3] (host); one launch.  The segments must lie inside src and out and not overlap in out;
    samples of out outside them are left as they are."""
    K = K or _K()
    K.join_segments(out, src, seg, max(1, int(round(sr * JOIN_FADE_S))))


class GriffinLimGraph:
    """The same 5-launches-per-iteration loop captured ONCE into a CUDA graph for a fixed (B, T, r, n_iter) and replayed:
    251 launches (and their Python / ctypes overhead, ~0.1 ms per iteration of host time) collapse into one
    graph launch.  Inputs are copied into static device buffers; the result is the static `y` (valid until the next call).
    Opt-in: `invert_spectrogram(...)` stays eager.  momentum > 0: fast Griffin-Lim, with the second rebuilt buffer among
    the static ones."""

    def __init__(self, B, T, r, n_iter=50, device="cuda", with_affine=True, momentum=0.0):
        K = _K()
        beta = gl_check(n_iter, momentum)
        self.B, self.T, self.r, self.n_iter, self.momentum = B, T, r, n_iter, momentum
        n = 4 * r * (T // 4)
        L = hop_length * (n - 1)
        assert L > n_fft // 2
        dev = torch.device(device)
        f32 = dict(dtype=torch.float32, device=dev)
        self.spec = torch.zeros((B, T, F_BINS * r), **f32)
        self.phase_u = torch.zeros((B, n, F_BINS), **f32)
        self.scale = torch.ones((F_BINS * r,), **f32) if with_affine else None
        self.shift = torch.zeros((F_BINS * r,), **f32) if with_affine else None
        self.mag = torch.empty((B, n, F_BINS), **f32)
        self.full = torch.empty((B, n, F_BINS), dtype=torch.complex64, device=dev)
        self.y = torch.empty((B, L), **f32)
        self.frw = torch.empty((B, n, n_fft), **f32)
        self.rebuilt = torch.empty_like(self.full) if beta == 0 else (torch.empty_like(self.full), torch.empty_like(self.full))
        args = (K, self.full, self.mag, self.spec, self.phase_u, r, self.scale, self.shift, self.y, self.frw, n_iter, self.rebuilt)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):                     # warm-up outside capture: lazy module loads
            _gl_iterations(*args, momentum=momentum)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            _gl_iterations(*args, momentum=momentum)

    def __call__(self, spec, stft_mean=None, stft_std=None, phase_u=None, generator=None):
        self.spec.copy_(spec.reshape(self.spec.shape), non_blocking=True)
        if self.scale is not None:
            if stft_std is not None:
                self.scale.copy_(stft_std, non_blocking=True); self.shift.copy_(stft_mean, non_blocking=True)
            else:
                self.scale.fill_(1.0); self.shift.zero_()
        if phase_u is None:
            self.phase_u.uniform_(0.0, 1.0, generator=generator)             # audio.py:81 (in place, on the device)
        else:
            self.phase_u.copy_(phase_u.reshape(self.phase_u.shape), non_blocking=True)
        self.graph.replay()
        return self.y


def griffinlim(spectrogram, n_iter=50, phase_u=None, K=None, momentum=0.0):
    """audio.griffinlim for ONE magnitude spectrogram [1025, frames] (audio.py:77) -> waveform [hop*(frames-1)]."""
    Fd, n = spectrogram.shape
    assert Fd == F_BINS
    spec = torch.log(spectrogram.t().contiguous().clamp_min(1e-30))[None]    # reuse the batch path with r = 1 layout
    # r=1: reshape_frames(forward=False) is the identity on whole blocks of 4 frames
    assert n % 4 == 0, "frame count must be a multiple of 4 (the reference always produces 4r-frame blocks)"
    pu = None if phase_u is None else phase_u[None]
    return griffinlim_batch(spec, 1, n_iter=n_iter, phase_u=pu, K=K, momentum=momentum)[0]


def invert_spectrogram(spec, r, n_iter=50, stft_mean=None, stft_std=None, phase_u=None, K=None, momentum=0.0):
    """audio.invert_spectrogram (audio.py:67-75) with the driver's de-normalisation folded in.
    spec [T, 1025*r] or [B, T, 1025*r] on the device -> waveform(s).  momentum: fast Griffin-Lim (griffinlim_batch)."""
    single = spec.dim() == 2
    s = spec[None] if single else spec
    scale, shift = (stft_std, stft_mean) if stft_std is not None else (None, None)
    if phase_u is not None and single:
        phase_u = phase_u[None]
    y = griffinlim_batch(s.contiguous(), r, n_iter=n_iter, scale=scale, shift=shift, phase_u=phase_u, K=K, momentum=momentum)
    return y[0] if single else y


def de_emphasis(y, start=None, K=None):
    """Undo preprocessing's pre-emphasis (PRE_EMPHASIS, audio.py:53) on synthesised waveforms, in place: y[i] = x[i] +
    PRE_EMPHASIS*y[i-1] over each segment [start[s], start[s+1]) of y, zero state before start[s] (scipy.signal.lfilter
    ([1], [1, -PRE_EMPHASIS], .) per segment).  y: contiguous fp32 on the device.  start (host int64 [S+1]): None for the
    rows of a [B, L] y, else e.g. invert_speech_packed's start or the spans of long-form lines.  One launch; no host
    synchronisation.  Returns y."""
    K = K or _K()
    if start is None:
        if y.dim() != 2:
            raise ValueError(f"de_emphasis: without start, y must be [B, L], got {tuple(y.shape)}")
        start = np.arange(y.shape[0] + 1, dtype=np.int64) * y.shape[1]
    elif torch.is_tensor(start):
        start = start.cpu().numpy()
    K.de_emphasis(y, start, PRE_EMPHASIS)
    return y
