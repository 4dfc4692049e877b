"""Checkpoint save / resume (SURVEY.md section 8(f) rank 4) -- what ``tf.train.Saver(max_to_keep=3)`` does for the
reference drivers (train.py:47-58, :85-90; test.py:40-48): the model variables, the optimizer slots, ``global_step`` and
the de-normalisation constants ``stft_mean`` / ``stft_std`` that the reference stores as extra TF variables so that they
travel with the weights (train.py:31-33, test.py:27-28).

Format: one ``.npz`` per step, ``<save_path>-<global_step>.npz``, keys = parameter names of tacotron_b200/params.py
(TF layouts), plus ``adam/m``, ``adam/v`` (flat buckets), ``adam/step``, ``global_step``, ``stft_mean``, ``stft_std``.
``import_tf_variables`` maps a {TF-1.2 variable name: array} dict (what ``tf.train.load_checkpoint`` yields on a machine
that has TensorFlow) onto the same store through tacotron_b200/tf_names.py, so the released Nancy weights can be loaded
once they are reachable (download_weights.sh:4).
"""
from __future__ import annotations

import glob
import os
import re

import numpy as np
import torch

from .tf_names import tf_name_to_param

MAX_TO_KEEP = 3            # train.py:47


def save(model, save_path, stft_mean=None, stft_std=None, max_to_keep=MAX_TO_KEEP):
    """saver.save(sess, save_path, global_step=global_step)   (train.py:85-90)"""
    os.makedirs(os.path.dirname(save_path) or ".", exist_ok=True)
    blob = {n: v.detach().cpu().numpy() for n, v in model.store.views.items()}
    blob["global_step"] = np.int64(model.global_step)
    opt = getattr(model, "_opt", None)
    if opt is not None:
        blob["adam/m"] = opt.m.detach().cpu().numpy()
        blob["adam/v"] = opt.v.detach().cpu().numpy()
        blob["adam/step"] = np.int64(opt.step)
    if stft_mean is not None:
        blob["stft_mean"] = np.asarray(stft_mean)
        blob["stft_std"] = np.asarray(stft_std)
    fn = f"{save_path}-{int(model.global_step)}.npz"
    tmp = fn + ".tmp.npz"
    np.savez(tmp, **blob)
    os.replace(tmp, fn)
    old = sorted(_all(save_path), key=lambda t: t[0])[:-max_to_keep]
    for _, f in old:
        os.remove(f)
    return fn


def _all(save_path):
    out = []
    for f in glob.glob(f"{save_path}-*.npz"):
        m = re.search(r"-(\d+)\.npz$", f)
        if m and not f.endswith(".tmp.npz"):
            out.append((int(m.group(1)), f))
    return out


def latest_checkpoint(save_path):
    """tf.train.latest_checkpoint (train.py:51-53, test.py:43-45): newest step, or None"""
    found = _all(save_path)
    return max(found)[1] if found else None


def restore(model, filename):
    """saver.restore(sess, ckpt): parameters, Adam slots, global_step; returns (stft_mean, stft_std) or (None, None)"""
    z = np.load(filename)
    _check_variables(model, z.files, filename)
    model.load_params({n: torch.from_numpy(z[n]) for n in model.store.shapes})
    model.global_step = int(z["global_step"])
    if "adam/m" in z.files:
        model.add_train_op()
        model._opt.m.copy_(torch.from_numpy(z["adam/m"]))
        model._opt.v.copy_(torch.from_numpy(z["adam/v"]))
        model._opt.step = int(z["adam/step"])
    if "stft_mean" in z.files:
        return z["stft_mean"], z["stft_std"]
    return None, None


# entries of a checkpoint written by `save` that are not model variables
_NON_PARAMS = ("global_step", "adam/m", "adam/v", "adam/step", "stft_mean", "stft_std")


def _check_variables(model, names, filename):
    """a checkpoint of a model with the other Config.speaker_decoder setting is refused, naming the variables, instead of
    being loaded partly (or, for the missing ones, from whatever the model was initialised with)"""
    if getattr(model, "store", None) is None:            # (a loader without a parameter list: nothing to compare)
        return
    have = set(names) - set(_NON_PARAMS)
    want = set(model.store.shapes)
    missing, extra = sorted(want - have), sorted(n for n in have - want if n.startswith("dec/spk/"))
    if extra or any(n.startswith("dec/spk/") for n in missing):
        raise ValueError(f"{filename} does not match the model (speaker_decoder = "
                         f"{bool(getattr(getattr(model, 'config', None), 'speaker_decoder', False))}): missing variables {missing}, "
                         f"extra variables {extra}")


def speaker_decoder(filename):
    """whether a checkpoint written by `save` holds a speaker-conditioned decoder (Config.speaker_decoder)"""
    return "dec/spk/attn/W" in np.load(filename).files


def num_speakers(filename):
    """speaker count of a checkpoint written by `save` (rows of its speaker table; 1 for a single-speaker model)"""
    z = np.load(filename)
    return int(z["speaker/embed"].shape[0]) if "speaker/embed" in z.files else 1


def import_tf_variables(model, tf_vars):
    """{TF-1.2 variable name: ndarray} -> parameter store.  Non-model variables (global_step, Adam slots, stft_mean/std,
    beta1_power ...) are returned in a dict instead of being loaded.  A bundle with a speaker table
    (``speaker/speaker_embed``) is read with the multi-speaker name map, one with the decoder's speaker denses
    (``decoder/dense``) with the speaker-conditioned decoder's."""
    params, extra = {}, {}
    strip = lambda n: n[:-2] if n.endswith(":0") else n
    multi = any(strip(n) == "speaker/speaker_embed" for n in tf_vars)
    spk_dec = multi and any(strip(n) == "decoder/dense/kernel" for n in tf_vars)
    for name, arr in tf_vars.items():
        name = strip(name)
        try:
            params[tf_name_to_param(name, multi_speaker=multi, speaker_decoder=spk_dec)] = \
                torch.from_numpy(np.asarray(arr, dtype=np.float32))
        except KeyError:
            extra[name] = arr
    _check_variables(model, params, "the TensorFlow checkpoint")
    model.load_params(params)
    return extra


def import_tf_checkpoint(model, prefix):
    """``saver.restore(sess, prefix)`` for a checkpoint WRITTEN BY TENSORFLOW (V2 format: ``prefix.index`` +
    ``prefix.data-0000N-of-0000M``; train.py:49-58, test.py:40-48, download_weights.sh:4): reads the bundle with
    tacotron_b200/tf_checkpoint.py (no TensorFlow needed), maps the TF-1.2 variable names through tf_names.py and loads
    them.  Returns the non-model variables (global_step, Adam slots, stft_mean / stft_std ...) like import_tf_variables;
    ``global_step`` is applied to the model when present."""
    from . import tf_checkpoint
    tf_vars = tf_checkpoint.read_bundle(prefix)
    extra = import_tf_variables(model, tf_vars)
    if "global_step" in extra:
        model.global_step = int(np.asarray(extra["global_step"]))
    return extra
