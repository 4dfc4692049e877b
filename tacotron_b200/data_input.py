"""Input side of the path -- host mirror of the reference's ``data_input.py`` (SURVEY.md section 8(f) rank 3).

Same surface: ``load_meta``, ``load_from_npy``, ``build_dataset``, ``load_prompts``, ``pad`` (data_input.py:20-113), with
the TF input pipeline replaced by what feeds a H100 well:

  * the float16 spectrogram arrays (preprocess.py:179-180) are NOT normalised / widened on the host.  They stay float16
    (memory-mapped or in RAM); a batch is gathered into PINNED float16 staging buffers by a background thread, copied
    H2D on a side stream (half the PCIe bytes of a float32 feed: 2 x 70 MB instead of 2 x 141 MB per C2 batch) and
    normalised + cast on the device by ``taco_normalize_f16`` -- bit-identical to the reference's in-place float16
    statements (data_input.py:61-64) followed by ``tf.cast(.., tf.float32)`` (:38-39);
  * ``dataset.repeat().shuffle(10000).batch(32)`` (data_input.py:27-30) is an index stream with TF's shuffle-buffer
    semantics (fill a buffer with the next 10000 indices, emit a uniformly random slot, refill it) -- the order is a
    valid TF order, not TF's exact RNG stream;
  * one batch is always in flight (double-buffered), so H2D of step i+1 overlaps the compute of step i.

The only arithmetic here is the sample mean / std (numpy on 100 utterances, as in the reference); everything per batch
is data movement plus the one device kernel.
"""
from __future__ import annotations

import os
import pickle as pkl
import threading

import numpy as np
import torch

BATCH_SIZE = 32                 # data_input.py:14
SHUFFLE_BUFFER_SIZE = 10000     # data_input.py:15
MAX_TEXT_LEN = 140              # data_input.py:17


def load_meta(data_path):
    """data_input.py:110-113 -- {'r': .., 'vocab': {id: char}} written by preprocess.py:148-166"""
    with open(os.path.join(data_path, "meta.pkl"), "rb") as vf:
        return pkl.load(vf)


def load_from_npy(dirname, mmap=True, rng=None):
    """data_input.py:42-85.  Returns (arrays, names, num_speakers, stft_mean, stft_std) like the reference, plus the
    mel statistics in arrays['_stats'].  The spectrogram arrays are returned AS STORED (float16, un-normalised): the
    normalisation happens per batch on the device (see module docstring); `stft_mean` (float16) and `stft_std`
    (float32) are the de-normalisation constants the drivers keep (train.py:31-33, test.py:27-28)."""
    j = lambda n: os.path.join(dirname, n)
    mode = "r" if mmap else None
    text = np.asarray(np.load(j("texts.npy")), dtype=np.int32)                            # :43, :66
    text_length = np.asarray(np.load(j("text_lens.npy")), dtype=np.int32)                 # :44, :67
    stft = np.load(j("stfts.npy"), mmap_mode=mode)                                        # :46
    mel = np.load(j("mels.npy"), mmap_mode=mode)                                          # :48
    rng = rng or np.random
    index = rng.randint(len(stft), size=100)                                              # :54 (a sample, to bound memory)
    stft_s, mel_s = np.asarray(stft[index]), np.asarray(mel[index])                       # same element order as the reference
    stft_mean = np.mean(stft_s, axis=(0, 1))                                              # :56  (float16 like the input)
    mel_mean = np.mean(mel_s, axis=(0, 1))                                                # :57
    stft_std = np.std(stft_s, axis=(0, 1), dtype=np.float32)                              # :58
    mel_std = np.std(mel_s, axis=(0, 1), dtype=np.float32)                                # :59
    # NOTE (reference): reconstruct zero frames as the paper suggests -> every speech_length = padded length   :71-72
    speech_length = np.ones(text.shape[0], dtype=np.int32) * mel.shape[1]
    arrays = {"text": text, "text_length": text_length, "stft": stft, "mel": mel, "speech_length": speech_length,
              "_stats": {"stft_mean": stft_mean, "stft_std": stft_std, "mel_mean": mel_mean, "mel_std": mel_std}}
    names = ["text", "text_length", "stft", "mel", "speech_length"]
    num_speakers = 1
    if os.path.exists(j("speakers.npy")):                                                 # :79-83
        arrays["speaker"] = np.load(j("speakers.npy"))
        names.append("speaker")
        num_speakers = int(np.max(arrays["speaker"])) + 1
    return arrays, names, num_speakers, stft_mean, stft_std


def shuffled_indices(n, buffer_size=SHUFFLE_BUFFER_SIZE, seed=0):
    """Infinite index stream of ``Dataset.from_tensor_slices(..).repeat().shuffle(buffer_size)`` (data_input.py:27-29)."""
    assert n > 0 and buffer_size > 0
    rng = np.random.RandomState(seed)
    buf = [i % n for i in range(buffer_size)]             # repeat() comes first, so the buffer always fills completely
    src = buffer_size
    while True:
        k = rng.randint(len(buf))
        yield buf[k]
        buf[k] = src % n
        src += 1


class DeviceBatches:
    """``build_dataset`` (data_input.py:20-40) for a CUDA consumer: iterator of input dicts of DEVICE tensors
    {'text' i32 [B,Tx], 'text_length' i32 [B], 'stft' f32 [B,T,1025r], 'mel' f32 [B,T,80r], 'speech_length' i32 [B]}, plus 'speaker' i32 [B] when the arrays have speaker ids.
    shard=(rank, world): data parallel ranks draw disjoint batches from the same shuffled stream."""

    def __init__(self, arrays, batch_size=BATCH_SIZE, buffer_size=SHUFFLE_BUFFER_SIZE, seed=0, device="cuda", shard=(0, 1), K=None):
        self.a = arrays
        self.B = batch_size
        self.device = torch.device(device)
        self.cuda = self.device.type == "cuda"
        self.rank, self.world = shard
        self.idx = shuffled_indices(len(arrays["text"]), buffer_size, seed)
        if K is None:
            from . import kernels as K
        self.K = K
        st = arrays["_stats"]
        self.stats = {k: torch.from_numpy(np.ascontiguousarray(v)).to(self.device) for k, v in st.items()}
        self.dev_index = torch.cuda.current_device() if self.cuda else None
        self.stream = torch.cuda.Stream() if self.cuda else None
        self.slots = [self._alloc(), self._alloc()]
        self.pending = None
        self.cur = 0
        self._launch(0)

    def _alloc(self):
        a, B = self.a, self.B
        pin = self.cuda

        def host(shape, dtype):
            t = torch.empty(shape, dtype=dtype)
            return t.pin_memory() if pin else t
        h = {"text": host((B,) + a["text"].shape[1:], torch.int32), "text_length": host((B,), torch.int32),
             "speech_length": host((B,), torch.int32), "stft": host((B,) + a["stft"].shape[1:], torch.float16),
             "mel": host((B,) + a["mel"].shape[1:], torch.float16)}
        if "speaker" in a:                            # multi-speaker corpus (speakers.npy, data_input.py:79-83)
            h["speaker"] = host((B,), torch.int32)
        d = {k: torch.empty(v.shape, dtype=v.dtype, device=self.device) for k, v in h.items()}
        out = {"stft": torch.empty(h["stft"].shape, dtype=torch.float32, device=self.device),
               "mel": torch.empty(h["mel"].shape, dtype=torch.float32, device=self.device)}
        return {"h": h, "d": d, "out": out, "ready": torch.cuda.Event() if self.cuda else None,
                "free": torch.cuda.Event() if self.cuda else None, "used": False}

    def _next_indices(self):
        # every rank advances the common stream by world*B and keeps its own slice -> disjoint batches
        take = [next(self.idx) for _ in range(self.B * self.world)]
        return np.sort(np.asarray(take[self.rank * self.B:(self.rank + 1) * self.B]))

    def _fill(self, slot):
        """background thread: gather the batch into (pinned) staging buffers, then H2D + device normalisation"""
        s = self.slots[slot]
        if self.cuda:
            torch.cuda.set_device(self.dev_index)
            if s["used"]:
                s["ready"].synchronize()              # the previous H2D out of these pinned buffers has completed
        ids = self._next_indices()
        for k in s["h"]:
            s["h"][k].copy_(torch.from_numpy(np.ascontiguousarray(self.a[k][ids])))
        ctx = torch.cuda.stream(self.stream) if self.cuda else _null()
        with ctx:
            if self.cuda and s["used"]:
                self.stream.wait_event(s["free"])     # the consumer has finished with this slot's device buffers
            for k in s["h"]:
                s["d"][k].copy_(s["h"][k], non_blocking=True)
            for k in ("stft", "mel"):
                self.K.normalize_f16(s["out"][k], s["d"][k], self.stats[f"{k}_mean"], self.stats[f"{k}_std"])
            if self.cuda:
                s["ready"].record(self.stream)
        s["used"] = True

    def _launch(self, slot):
        self.pending = threading.Thread(target=self._fill, args=(slot,), daemon=True)
        self.pending.start()

    def __iter__(self):
        return self

    def __next__(self):
        self.pending.join()
        slot = self.cur
        s = self.slots[slot]
        if self.cuda:
            torch.cuda.current_stream().wait_event(s["ready"])
        self.cur ^= 1
        if self.cuda and self.slots[self.cur]["used"]:
            self.slots[self.cur]["free"].record()    # everything that reads the previous batch is already enqueued
        self._launch(self.cur)                       # stage the following batch while this one is consumed
        batch = {"text": s["d"]["text"], "text_length": s["d"]["text_length"], "speech_length": s["d"]["speech_length"],
                 "stft": s["out"]["stft"], "mel": s["out"]["mel"]}
        if "speaker" in s["d"]:
            batch["speaker"] = s["d"]["speaker"]
        return batch


class _null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def build_dataset(arrays, names=None, **kw):
    """data_input.build_dataset(sess, inputs, names) (data_input.py:20-40) -> iterator of device batches"""
    return DeviceBatches(arrays, **kw)


def pad(text, max_len, pad_val):
    """data_input.py:87-90"""
    return np.array([np.pad(np.asarray(t, dtype=np.int32), (0, max_len - len(t)), "constant", constant_values=pad_val) for t in text],
                    dtype=np.int32)


def load_prompts(prompts, ivocab, batch_size=32, device="cuda"):
    """data_input.load_prompts (data_input.py:92-108): yields {'text' i32 [b,140], 'text_length' i32 [b]} device batches of
    at most 32 prompts (allow_smaller_final_batch=True, :105-106).  Quirks kept: characters outside the vocabulary are
    dropped from the id sequence, but text_length counts the RAW prompt line (:95-96); ids are padded with 0 to 140 so
    that synthesis sees the padding the model was trained with (:98-99)."""
    vocab = {v: k for k, v in ivocab.items()}
    text = [[vocab[w] for w in p.strip() if w in vocab] for p in prompts]
    text_length = np.array([len(p) for p in prompts], dtype=np.int32)
    text = pad(text, MAX_TEXT_LEN, 0)
    for i in range(0, len(prompts), batch_size):
        yield {"text": torch.from_numpy(text[i:i + batch_size]).to(device),
               "text_length": torch.from_numpy(text_length[i:i + batch_size]).to(device)}
