"""Preprocessing: WAV corpora -> the training arrays ``data/<set>/{texts,text_lens,mels,stfts,speech_lens[,speakers]}.npy``
and ``meta.pkl`` that ``tacotron_b200.data_input.load_from_npy`` reads.  Host mirror of the reference's ``preprocess.py``
(same names: ``prepare_arctic / prepare_nancy / prepare_vctk``, ``process_char``, ``pad_to_dense``, ``save_to_npy``,
``save_vocab``, ``preprocess``) with the feature extraction on the GPU (``audio.process_audio_batch``).

    python -m tacotron_b200.preprocess {arctic,nancy,vctk} [--data-dir data/] [-r 2] [--resample]

Kept from the reference: the file layouts of the three corpora (preprocess.py:41-117); characters enter the vocabulary in
first-seen order with <pad> = 0, including the characters of utterances that are later dropped (:186-189); texts are
int64, zero-padded to the longest kept prompt; text_lens int64; speech_lens is the padded frame count of every utterance;
meta.pkl = {'vocab', 'r', 'sr'} in pickle protocol 2; the spectrograms are float16 (:179-180).

Deliberate deviations:
  * speakers.npy holds the speakers of the KEPT utterances.  The reference saves all of them (:204-205), which misaligns
    speakers and utterances whenever one is dropped.
  * meta['sr'] is the rate actually used.  The reference always writes 16000 (save_vocab is called without sr, :208).
  * r = 4 (and any r outside 1-6) is rejected: the reference crashes on it (see audio.feature_frames_per_utterance).
  * a file whose rate differs from the corpus rate is an error naming the file unless --resample is given; with it, such
    a file is resampled on the GPU as the reference's librosa.load(f, sr=sr) does (audio.resample_batch: librosa 0.6's
    kaiser_best over resampy 0.2.2's loop, restated; parity with resampy itself is not pinned).  A file too short to
    give one resampled sample is an error naming it, and so is a file shorter than 1025 samples at the corpus rate (too
    short for the STFT's reflect padding).

Work is done in chunks.  A reader thread decodes the WAVs of the next chunk while the GPU works on the current one; the
float16 results are copied to pinned host buffers asynchronously and written to ``np.lib.format.open_memmap`` files while
the next chunk is on the GPU, so a Nancy-sized stfts.npy (~9 GB at r = 2) never has to fit in memory.  The files are
allocated for every listed utterance; after the last chunk the row count in their headers is set to the number of kept
utterances and the files are truncated.
"""
from __future__ import annotations

import argparse
import ast
import glob
import os
import pickle as pkl
import queue
import threading

import numpy as np
import torch

from . import audio

SR = {"arctic": 16000, "nancy": 16000, "vctk": 24000}     # preprocess.py:217
CHUNK = 64


def prepare_arctic(data_dir):
    """preprocess.py:41-60: <data_dir>/arctic/etc/arctic.data lines `( id "text" )`, wavs in arctic/wav/<id>.wav"""
    prompts, audio_files = [], []
    with open(os.path.join(data_dir, "arctic", "etc", "arctic.data")) as tff:
        for line in tff:
            spl = line.split()
            prompts.append(" ".join(spl[2:-1])[1:-1])
            audio_files.append(os.path.join(data_dir, "arctic", "wav", f"{spl[1]}.wav"))
    return {"prompts": prompts, "audio_files": audio_files}


def prepare_nancy(data_dir):
    """preprocess.py:62-79: <data_dir>/nancy/prompts.data lines `( id "text." )` (the character before the closing quote is
    dropped, as in the reference), wavs in nancy/wavn/<id>.wav"""
    prompts, audio_files = [], []
    with open(os.path.join(data_dir, "nancy", "prompts.data")) as ttf:
        for line in ttf:
            prompts.append(line[line.find('"') + 1:line.rfind('"') - 1])
            audio_files.append(os.path.join(data_dir, "nancy", "wavn", line.split()[1] + ".wav"))
    return {"prompts": prompts, "audio_files": audio_files}


def prepare_vctk(data_dir):
    """preprocess.py:81-117: speakers from the ID column of vctk/speaker-info.txt (ids in file order), prompts from
    vctk/txt/p<ID>/*.txt, wavs in vctk/wav48/p<ID>/: the original 48 kHz files with --resample (preprocess(...,
    resample=True)), otherwise files already converted to 24 kHz."""
    root = os.path.join(data_dir, "vctk")
    with open(os.path.join(root, "speaker-info.txt")) as f:
        header = f.readline().split()
        col = header.index("ID")
        ids = [line.split()[col] for line in f if line.strip()]
    speaker_ids = {uid: i for i, uid in enumerate(ids)}
    prompts, audio_files, speakers = [], [], []
    for uid in ids:
        for txt in sorted(glob.glob(os.path.join(root, "txt", f"p{uid}", "*.txt"))):
            f = os.path.basename(txt)[:-4]
            with open(txt) as tff:
                prompts.append(tff.read().strip())
            audio_files.append(os.path.join(root, "wav48", f[:4], f + ".wav"))
            speakers.append(speaker_ids[f[1:4]])
    return {"prompts": prompts, "audio_files": audio_files, "speakers": speakers}


prepare_functions = {"arctic": prepare_arctic, "nancy": prepare_nancy, "vctk": prepare_vctk}


def process_char(char, vocab, ivocab):
    """preprocess.py:130-135 with the vocabulary passed in instead of module globals"""
    if char not in vocab:
        vocab[char] = len(vocab)
        ivocab[vocab[char]] = char
    return vocab[char]


def pad_to_dense(inputs):
    """preprocess.py:137-146 for 1-D id sequences: int64 [N, longest], zero-padded"""
    max_len = max(len(t) for t in inputs)
    out = np.zeros((len(inputs), max_len), dtype=np.int64)
    for i, t in enumerate(inputs):
        out[i, :len(t)] = t
    return out


def save_to_npy(texts, text_lens, speech_lens, out_dir):
    """preprocess.py:148-159 for the small arrays (mels / stfts are streamed by `preprocess`)"""
    for name, arr in (("texts", pad_to_dense(texts)), ("text_lens", np.asarray(text_lens, dtype=np.int64)),
                      ("speech_lens", np.asarray(speech_lens, dtype=np.int64))):
        np.save(os.path.join(out_dir, name + ".npy"), arr, allow_pickle=False)


def save_vocab(out_dir, ivocab, r, sr):
    """preprocess.py:161-166, with the rate actually used"""
    with open(os.path.join(out_dir, "meta.pkl"), "wb") as vf:
        pkl.dump({"vocab": ivocab, "r": r, "sr": sr}, vf, protocol=2)


def _shrink_npy(path, rows):
    """set the leading dimension in the header of a version 1.0 .npy file to `rows` (padding the header to its old
    length) and truncate the data to match"""
    with open(path, "r+b") as f:
        head = f.read(10)
        assert head[:6] == b"\x93NUMPY" and head[6] == 1, "expected a version 1.0 .npy header"
        hlen = int.from_bytes(head[8:10], "little")
        d = ast.literal_eval(f.read(hlen).decode("latin1"))        # the header is a Python dict literal (numpy format)
        shape = (rows,) + tuple(d["shape"][1:])
        text = "{'descr': %r, 'fortran_order': %r, 'shape': %r, }" % (d["descr"], d["fortran_order"], shape)
        assert len(text) + 1 <= hlen
        f.seek(10)
        f.write((text + " " * (hlen - len(text) - 1) + "\n").encode("latin1"))
        f.truncate(10 + hlen + rows * int(np.prod(shape[1:])) * np.dtype(d["descr"]).itemsize)


def _reader(files, sr, chunk, q, resample=False):
    """queues (i, chunk of samples), or with `resample` (i, chunk of (samples, rate))"""
    try:
        for i in range(0, len(files), chunk):
            if not resample:
                q.put((i, [audio.load_wav(f, sr) for f in files[i:i + chunk]]))
                continue
            items = [audio.read_wav(f) for f in files[i:i + chunk]]
            for f, (x, rate) in zip(files[i:i + chunk], items):
                if rate != sr:
                    audio.resample_lengths(len(x), rate, sr, f)          # raises, naming the file, if nothing is left
            q.put((i, items))
        q.put(None)
    except BaseException as e:                                    # re-raised in the consumer
        q.put(e)


def preprocess(data, out_dir, r=2, sr=16000, chunk=CHUNK, K=None, device="cuda", log=print, resample=False):
    """preprocess.py:168-208: features of every listed utterance into <out_dir>; returns the number kept.  resample: a
    file at another rate is resampled to `sr` on the device (librosa.load's kaiser_best, audio.resample_batch) instead
    of being an error; meta['sr'] is `sr` either way."""
    os.makedirs(out_dir, exist_ok=True)
    T = audio.feature_frames_per_utterance(r)
    vocab, ivocab = {"<pad>": 0}, {0: "<pad>"}
    all_texts = [[process_char(c, vocab, ivocab) for c in text] for text in data["prompts"]]
    N = len(all_texts)
    files = data["audio_files"]
    assert len(files) == N
    mels = np.lib.format.open_memmap(os.path.join(out_dir, "mels.npy"), mode="w+", dtype=np.float16, shape=(N, T, audio.N_MELS * r))
    stfts = np.lib.format.open_memmap(os.path.join(out_dir, "stfts.npy"), mode="w+", dtype=np.float16, shape=(N, T, audio.F_BINS * r))
    cuda = torch.device(device).type == "cuda"
    q = queue.Queue(maxsize=2)
    th = threading.Thread(target=_reader, args=(files, sr, chunk, q, resample), daemon=True)
    th.start()
    kept = []
    count = 0
    pending = None

    def flush(p):
        nonlocal count
        mel_h, stft_h, ev = p
        if ev is not None:
            ev.synchronize()
        n = mel_h.shape[0]
        mels[count:count + n] = mel_h.numpy()
        stfts[count:count + n] = stft_h.numpy()
        count += n

    while True:
        item = q.get()
        if isinstance(item, BaseException):
            raise item
        if item is None:
            break
        i, waves = item
        rates = None
        if resample:
            waves, rates = [x for x, _ in waves], [rate for _, rate in waves]
        try:
            mel, stft, keep = audio.process_audio_batch(waves, r, K=K, device=device, rates=rates, sr=sr)
        except ValueError as e:
            raise ValueError(f"chunk starting at {files[i]}: {e}") from None
        kept.extend(i + np.flatnonzero(keep))
        if cuda:
            mel_h = torch.empty(mel.shape, dtype=mel.dtype, pin_memory=True)
            stft_h = torch.empty(stft.shape, dtype=stft.dtype, pin_memory=True)
            mel_h.copy_(mel, non_blocking=True)
            stft_h.copy_(stft, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
        else:
            mel_h, stft_h, ev = mel, stft, None
        if pending is not None:
            flush(pending)                        # disk writes of the previous chunk overlap this chunk's GPU work
        pending = (mel_h, stft_h, ev)
        log(f"{min(i + len(waves), N)}/{N} utterances, {len(kept)} kept")
    if pending is not None:
        flush(pending)
    th.join()
    if not kept:
        raise ValueError("no utterance is at most %d samples long after trimming" % audio.maximum_audio_length)
    mels.flush(); stfts.flush()
    del mels, stfts
    for name in ("mels", "stfts"):
        _shrink_npy(os.path.join(out_dir, name + ".npy"), len(kept))
    save_to_npy([all_texts[k] for k in kept], [len(all_texts[k]) for k in kept], [T] * len(kept), out_dir)
    if "speakers" in data:
        np.save(os.path.join(out_dir, "speakers.npy"), np.asarray(data["speakers"], dtype=np.int64)[kept], allow_pickle=False)
    save_vocab(out_dir, ivocab, r, sr)
    return len(kept)


def main(argv=None):
    parser = argparse.ArgumentParser(description="WAV corpus -> training arrays (feature extraction on the GPU)")
    parser.add_argument("dataset", choices=sorted(prepare_functions))
    parser.add_argument("--data-dir", default="data/")
    parser.add_argument("-r", type=int, default=2, help="decoder frames per step the arrays are laid out for")
    parser.add_argument("--resample", action="store_true",
                        help="resample files at other rates to the corpus rate on the GPU (librosa.load's kaiser_best), "
                             "e.g. VCTK's 48 kHz originals, instead of rejecting them")
    args = parser.parse_args(argv)
    audio.feature_frames_per_utterance(args.r)
    data = prepare_functions[args.dataset](args.data_dir)
    sr = SR[args.dataset]
    n = preprocess(data, os.path.join(args.data_dir, args.dataset), r=args.r, sr=sr, resample=args.resample)
    print(f"{n} of {len(data['prompts'])} utterances written to {os.path.join(args.data_dir, args.dataset)}")


if __name__ == "__main__":
    main()
