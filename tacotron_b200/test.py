"""Synthesis driver -- eager equivalent of the reference's ``test.py`` (test.py:13-88; SURVEY.md section 8(f) rank 2).

    echo "a prompt to say" | python -m tacotron_b200.test -t nancy
    echo "a prompt to say" | python -m tacotron_b200.test -t vctk -s 3      # multi-speaker model: speaker id 3

Prompts come from stdin, one per line (test.py:77-78); they are encoded and padded to 140 characters exactly as
``data_input.load_prompts`` does (quirks included), run through ``Tacotron.inference`` in batches of at most 32, every
output is de-normalised with the checkpoint's ``stft_mean`` / ``stft_std`` and inverted with the GPU Griffin-Lim
(test.py:59-64).  The waveform is written as ``log/<save_path>/test/<n>.wav`` and the alignment as
``<n>_attention.npy``; with ``--summaries`` the reference's TensorBoard audio and image summaries go next to them
(:33, :65-69; tacotron_b200/summary.py).

    echo "a prompt to say" | python -m tacotron_b200.test -t nancy --trim-tail

``--trim-tail`` ends each utterance where its speech ends instead of after ``max_decode_iter * r`` frames: the end is
found on the device (``audio.speech_frames``: the last STFT frame within 60 dB of the utterance's loudest, rounded up to
whole decoder-step blocks) and Griffin-Lim inverts only the frames up to it (``audio.invert_speech``).  The WAV, the
attention array (the first ``frames/r`` decoder steps) and the summaries then end there too.  The rule rests on the
training targets, which end in ``log(1e-8)`` padding frames; it has not been observed on a trained model's output.
Without the flag every file is what the driver writes without it.

    python -m tacotron_b200.test -t nancy --long-form < paragraph.txt

``--long-form`` speaks each stdin line as one clip, whatever its length (without it, a line over 140 vocabulary
characters is an error and a line that takes longer than ``max_decode_iter * r`` frames to say is cut off).  Each line is
split into chunks at sentence ends, clause breaks or spaces (``tacotron_b200/longform.py``); the chunks of all lines are
decoded in batches of at most 32, and ``audio.speech_bounds`` finds where each chunk's speech starts and ends on the
device.  A chunk whose speech reaches its last frame most likely ran out of decoder steps: it is split again at the
break nearest its middle and both halves go to the next round (a chunk with no break left is kept, with one logged
warning).  That rule rests on the training targets, which end in ``log(1e-8)`` padding; it has not been observed on a
trained model.  Each chunk's Griffin-Lim output is cut to its speech (``audio.kept_samples``) and the pieces of a line
are joined with a pause set by the break between them and a 10 ms raised-cosine fade at every cut
(``audio.join_speech``, one launch per batch into one zero-filled device buffer that holds every line).  Per line the
driver writes ``<n>.wav``, ``<n>.txt`` (the whole line), ``<n>_chunks.txt`` (one chunk per line) and
``<n>_attention.npy`` (the block-diagonal stack of the chunk alignments), and with ``--summaries`` one audio and one
image summary.  ``--trim-tail`` changes nothing here: long-form already trims.

    python -m tacotron_b200.test -t nancy --attention-window          # back 2, ahead 5
    python -m tacotron_b200.test -t nancy --attention-window 1,4

``--attention-window [BACK,AHEAD]`` lets each decoder step attend only the characters from BACK behind to AHEAD ahead of
the one the previous step attended most (the first step: the first character), so the alignment cannot jump ahead,
fall far back or stick past the text.  It applies to every decode of the run, with or without ``--long-form``,
``--trim-tail``, ``-s``, ``--max-ctas`` and ``--summaries``; the files written are the same ones.  The default 2,5 is
close to the windows of common open Tacotron implementations and is a starting point only: no value has been tried on
a trained model here.  Without the flag the decoder is the reference's.

    python -m tacotron_b200.test -t nancy --stop-at-end               # hold 4
    python -m tacotron_b200.test -t nancy --stop-at-end 3 --trim-tail

``--stop-at-end [HOLD]`` stops decoding at the end of the text instead of after ``max_decode_iter`` steps: an utterance
ends once HOLD consecutive decoder steps attend most to its last character or past it, each group of 8 utterances stops
decoding a few steps after its last one ends, and the post-net and Griffin-Lim run only on the steps that were decoded.
The WAV, the attention array and the summaries end at the stop (with ``--trim-tail`` also where the speech ends, if
that comes first; with ``--long-form`` a chunk whose rule fired is never split again).  It works with every other flag.
The default hold of 4 steps is a starting point only: no value has been tried on a trained model here.  An utterance
whose attention never reaches the end of its text decodes all ``max_decode_iter`` steps, as without the flag.

    python -m tacotron_b200.test -t nancy --griffin-lim-momentum --griffin-lim-iters 25 --de-emphasis

``--griffin-lim-iters N`` sets the Griffin-Lim iterations (default 50, the reference's).  ``--griffin-lim-momentum [M]``
runs fast Griffin-Lim (Perraudin, Balazs & Sondergaard 2013), which adds a momentum term M in [0, 1] to the phase update
(a bare flag: 0.99, librosa's default; default 0, plain Griffin-Lim).  ``--de-emphasis`` undoes preprocessing's
pre-emphasis ``y[n] - 0.97 y[n-1]`` on every synthesised waveform with the inverse filter ``y[n] = x[n] + 0.97 y[n-1]``;
with ``--long-form`` it runs once over each joined line, through its pauses and fades.  They work with every other flag,
and without them every file is what the driver writes without them.  No value of either has been tried on a trained
model here.
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np
import torch


def test(model_cls, config, prompts, log=print, speaker=0, summary_dir=None, trim_tail=False, long_form=False,
         griffin_lim_iters=50, griffin_lim_momentum=0.0, de_emphasis=False):
    """summary_dir: also write each prompt's audio and attention image as TensorBoard summaries there, at step 0
    (tacotron_b200/summary.py).  trim_tail: end each utterance where its speech ends; long_form: speak each line as one
    clip, whatever its length (module docstring).  config.attention_window (None or (back, ahead)) and
    config.stop_at_end (None or a hold) apply to every decode, plain and long-form.  griffin_lim_iters /
    griffin_lim_momentum: the inversion's iterations and fast Griffin-Lim momentum; de_emphasis: undo preprocessing's
    pre-emphasis on every waveform (module docstring).  Returns one device waveform per prompt."""
    from . import audio, checkpoint, data_input
    from .train import write_wav
    gl = dict(n_iter=griffin_lim_iters, momentum=griffin_lim_momentum)
    audio.gl_check(**gl)                                                                 # before any model is built
    sr = 24000 if "blizzard" in config.data_path else 16000                              # test.py:15
    meta = data_input.load_meta(config.data_path)                                        # :16
    config.r = meta["r"]          # (the reference reads the module constant audio.r here, :17; meta['r'] is the value it was preprocessed with)
    config.max_decode_iter = audio.maximum_audio_length // (config.r * audio.hop_length)  # tacotron.py:13
    ivocab = meta["vocab"]
    config.vocab_size = len(ivocab)                                                      # :19
    config.num_prompts = len(prompts)                                                    # :23
    ck = checkpoint.latest_checkpoint(os.path.join("weights", config.save_path))         # :42-45
    tf_ck = None
    if ck is not None:
        config.num_speakers = checkpoint.num_speakers(ck)
        config.speaker_decoder = checkpoint.speaker_decoder(ck)
    else:
        # no checkpoint of ours: a checkpoint written by the reference itself (TensorFlow V2 format, e.g. the released
        # Nancy weights of download_weights.sh) in the same directory is read directly
        from . import tf_checkpoint
        tf_ck = tf_checkpoint.latest_checkpoint(os.path.dirname(os.path.join("weights", config.save_path)))
        if tf_ck is None:
            raise FileNotFoundError(f"no checkpoint under weights/{config.save_path}")
        spk = tf_checkpoint.read_bundle(tf_ck, names={"speaker/speaker_embed"}).get("speaker/speaker_embed")
        config.num_speakers = 1 if spk is None else int(np.asarray(spk).shape[0])
        config.speaker_decoder = bool(tf_checkpoint.read_bundle(tf_ck, names={"decoder/dense/kernel"}))
    if not 0 <= speaker < config.num_speakers:
        raise ValueError(f"speaker id {speaker} out of range: the checkpoint has {config.num_speakers} speaker(s)")
    model = model_cls(config, None, train=False)                                         # :31
    log("restoring weights")                                                             # :41
    if ck is not None:
        stft_mean, stft_std = checkpoint.restore(model, ck)                              # :46-48
    else:
        extra = checkpoint.import_tf_checkpoint(model, tf_ck)
        stft_mean, stft_std = extra["stft_mean"], extra["stft_std"]
    mean_d = torch.from_numpy(np.asarray(stft_mean, dtype=np.float32)).cuda()
    std_d = torch.from_numpy(np.asarray(stft_std, dtype=np.float32)).cuda()
    out_dir = os.path.join("log", config.save_path, "test")                              # :33
    os.makedirs(out_dir, exist_ok=True)
    writer = None
    if summary_dir is not None:                                                          # :33
        from . import summary
        writer, scopes = summary.EventWriter(summary_dir), summary.NameScopes()
    if long_form:
        try:
            return _long_form(model, config, prompts, ivocab, speaker, mean_d, std_d, out_dir, sr, log, writer,
                              scopes if writer is not None else None, gl, de_emphasis)
        finally:
            if writer is not None:
                writer.close()
    n = 0
    waves = []
    try:
        for inputs in data_input.load_prompts(prompts, ivocab):                          # :21-22, :50-56
            if config.num_speakers > 1:
                inputs["speaker"] = torch.full((inputs["text"].shape[0],), speaker, dtype=torch.int32, device=inputs["text"].device)
            _, outputs = model.inference(inputs, train=False)
            alignments = model.alignments
            log("saving samples")
            steps = None
            if trim_tail or model.end_steps is not None:
                frames = audio.speech_frames(outputs, config.r, stft_mean=mean_d, stft_std=std_d) if trim_tail else None
                if model.end_steps is not None:                                          # the stop rule's frames
                    frames = audio.stop_frames(model.end_steps, config.r, outputs.shape[1], frames)
                y, start = audio.invert_speech_packed(outputs, config.r, frames, stft_mean=mean_d, stft_std=std_d, **gl)
                if de_emphasis:
                    audio.de_emphasis(y, start)
                wav = [y[start[b]:start[b + 1]] for b in range(outputs.shape[0])]
                steps = (frames.cpu() // config.r).tolist()
            else:
                wav = audio.invert_spectrogram(outputs, config.r, stft_mean=mean_d, stft_std=std_d, **gl)   # :64, batched on the device
                if de_emphasis:
                    audio.de_emphasis(wav)
            for b in range(outputs.shape[0]):                                            # :59-70
                text = "".join(ivocab[int(w)] for w in inputs["text"][b].cpu().numpy())
                wave, alignment = wav[b].cpu().numpy(), alignments[b].cpu().numpy()
                if steps is not None:
                    alignment = alignment[:steps[b]]
                write_wav(os.path.join(out_dir, f"{n}.wav"), wave, sr)
                np.save(os.path.join(out_dir, f"{n}_attention.npy"), alignment)
                with open(os.path.join(out_dir, f"{n}.txt"), "w") as f:
                    f.write(text)
                if writer is not None:           # :65-69: audio(text) then image(text), name scopes of one graph
                    tag = summary.clean_tag(text)
                    writer.add(0, [summary.audio_value(scopes.unique(tag) + "/audio/0", wave, sr),
                                   summary.image_value(scopes.unique(tag) + "/image/0", summary.attention_rgba(alignment))])
                waves.append(wav[b])
                n += 1
    finally:
        if writer is not None:
            writer.close()
    return waves


def _long_form(model, config, prompts, ivocab, speaker, mean_d, std_d, out_dir, sr, log, writer, scopes, gl, de_emphasis):
    """test(long_form=True): the rounds of synthesis and re-splitting, then the join (module docstring)"""
    from . import audio, data_input, longform
    from .train import write_wav
    r = config.r
    vocab = set(ivocab.values())
    lines = [longform.split_line(p, vocab, i) for i, p in enumerate(prompts)]
    outs = []                # flat Griffin-Lim output of every synthesised batch
    done = {}                # id(chunk) -> (batch, first sample of the chunk in it, (f0, f1, frames), alignment)
    pending = [c for cs in lines for c in cs]
    while pending:
        again = []
        for i in range(0, len(pending), data_input.BATCH_SIZE):
            group = pending[i:i + data_input.BATCH_SIZE]
            inputs = next(data_input.load_prompts([c.prompt for c in group], ivocab))
            if config.num_speakers > 1:
                inputs["speaker"] = torch.full((len(group),), speaker, dtype=torch.int32, device=inputs["text"].device)
            _, outputs = model.inference(inputs, train=False)
            bounds = audio.speech_bounds(outputs, r, stft_mean=mean_d, stft_std=std_d)
            fired = None
            if model.end_steps is not None:  # stop rule: every chunk's bounds end at its stop (a no-op where it did not fire)
                stop = audio.stop_frames(model.end_steps, r, outputs.shape[1])
                f1 = torch.minimum(bounds[:, 1], stop)
                bounds = torch.stack([torch.minimum(bounds[:, 0], f1), f1, torch.minimum(bounds[:, 2], stop),
                                      (model.end_steps < config.max_decode_iter).to(torch.int32)], dim=1)
            bounds = bounds.cpu().numpy()    # the one read
            if bounds.shape[1] == 4:
                bounds, fired = bounds[:, :3], bounds[:, 3] != 0
            y, start = audio.invert_speech_packed(outputs, r, bounds[:, 2], stft_mean=mean_d, stft_std=std_d, **gl)
            align = model.alignments.cpu().numpy()
            n = 4 * r * (outputs.shape[1] // 4)
            outs.append(y)
            for b, c in enumerate(group):
                f0, f1, frames = (int(v) for v in bounds[b])
                if f1 == n and (fired is None or not fired[b]):    # speech up to the last frame: most likely out of
                                                                   # decoder steps
                    halves = longform.resplit(c)
                    if halves is not None:
                        cs = lines[c.line]
                        k = next(j for j, x in enumerate(cs) if x is c)
                        cs[k:k + 1] = halves
                        again.extend(halves)
                        continue
                    log(f"warning: line {c.line}: chunk {c.text!r} is voiced up to its last decoder step and has no break "
                        f"left to split it at; kept as it is")
                cols = min(len(c.prompt), data_input.MAX_TEXT_LEN)
                done[id(c)] = (len(outs) - 1, int(start[b]), (f0, f1, frames), align[b, :frames // r, :cols])
        pending = again
    log("saving samples")
    segs = {}                # batch -> rows {src_start, dst_start, len} of its join
    spans = []
    total = 0
    for cs in lines:
        kept = [audio.kept_samples(*done[id(c)][2]) for c in cs]
        dst, length = longform.layout([e - a for a, e in kept], [c.brk for c in cs], sr)
        for c, (a, e), d in zip(cs, kept, dst):
            bi, s0 = done[id(c)][:2]
            segs.setdefault(bi, []).append((s0 + a, total + d, e - a))
        spans.append((total, length))
        total += length
    out = torch.zeros(total, dtype=torch.float32, device=mean_d.device)
    for bi, rows in segs.items():
        audio.join_speech(out, outs[bi], np.asarray(rows, dtype=np.int64), sr)
    if de_emphasis:                      # one segment per line: the filter runs through pauses and fades, not across lines
        audio.de_emphasis(out, np.array([o for o, _ in spans] + [total], dtype=np.int64))
    waves = []
    for n, (cs, (o, length)) in enumerate(zip(lines, spans)):
        wave = out[o:o + length]
        w = wave.cpu().numpy()
        alignment = longform.block_diagonal([done[id(c)][3] for c in cs])
        text = prompts[n].rstrip("\r\n")
        write_wav(os.path.join(out_dir, f"{n}.wav"), w, sr)
        np.save(os.path.join(out_dir, f"{n}_attention.npy"), alignment)
        with open(os.path.join(out_dir, f"{n}.txt"), "w") as f:
            f.write(text)
        with open(os.path.join(out_dir, f"{n}_chunks.txt"), "w") as f:
            f.write("".join(c.text + "\n" for c in cs))
        if writer is not None:
            from . import summary
            tag = summary.clean_tag(text)
            writer.add(0, [summary.audio_value(scopes.unique(tag) + "/audio/0", w, sr),
                           summary.image_value(scopes.unique(tag) + "/image/0", summary.attention_rgba(alignment))])
        waves.append(wave)
    return waves


def parse_attention_window(text):
    """'BACK,AHEAD' -> (back, ahead) with back >= 0, ahead >= 1 (the --attention-window value)"""
    parts = text.split(",")
    try:
        if len(parts) != 2:
            raise ValueError
        back, ahead = (int(v) for v in parts)
    except ValueError:
        raise argparse.ArgumentTypeError(f"{text!r}: expected BACK,AHEAD, two integers such as 2,5") from None
    if back < 0 or ahead < 1:
        raise argparse.ArgumentTypeError(f"{text!r}: BACK must be >= 0 and AHEAD >= 1")
    return back, ahead


def parse_stop_hold(text):
    """'HOLD' -> an int >= 1 (the --stop-at-end value)"""
    try:
        hold = int(text)
    except ValueError:
        raise argparse.ArgumentTypeError(f"{text!r}: expected HOLD, an integer number of decoder steps such as 4") from None
    if hold < 1:
        raise argparse.ArgumentTypeError(f"{text!r}: HOLD must be >= 1")
    return hold


def parse_gl_iters(text):
    """'N' -> an int >= 0 (the --griffin-lim-iters value)"""
    try:
        n = int(text)
    except ValueError:
        raise argparse.ArgumentTypeError(f"{text!r}: expected N, an integer number of iterations such as 50") from None
    if n < 0:
        raise argparse.ArgumentTypeError(f"{text!r}: N must be >= 0")
    return n


def parse_gl_momentum(text):
    """'M' -> a float in [0, 1] (the --griffin-lim-momentum value)"""
    try:
        m = float(text)
    except ValueError:
        raise argparse.ArgumentTypeError(f"{text!r}: expected M, a number in [0, 1] such as 0.99") from None
    if not 0.0 <= m <= 1.0:
        raise argparse.ArgumentTypeError(f"{text!r}: M must be in [0, 1]")
    return m


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("-t", "--train-set", default="nancy")
    parser.add_argument("-s", "--speaker", type=int, default=0, help="speaker id of a multi-speaker model")
    parser.add_argument("--summaries", action="store_true", help="write TensorBoard summaries to log/<save_path>/test")
    parser.add_argument("--trim-tail", action="store_true",
                        help="end each utterance where its speech ends and invert only those frames")
    parser.add_argument("--long-form", action="store_true",
                        help="speak each line as one clip, whatever its length: split at sentence and clause breaks, "
                             "decode the pieces as batches and join them")
    parser.add_argument("--max-ctas", type=int, default=None,
                        help="CTAs (SMs) the decoder kernels may occupy, at least 32 (default: all the device holds)")
    parser.add_argument("--attention-window", type=parse_attention_window, nargs="?", const=(2, 5), default=None,
                        metavar="BACK,AHEAD",
                        help="attend only BACK characters behind to AHEAD ahead of the previous step's attention peak "
                             "(a bare flag: 2,5, a starting point only)")
    parser.add_argument("--stop-at-end", type=parse_stop_hold, nargs="?", const=4, default=None, metavar="HOLD",
                        help="stop decoding once HOLD consecutive steps attend to the last character of the text or "
                             "past it (a bare flag: 4, a starting point only)")
    parser.add_argument("--griffin-lim-iters", type=parse_gl_iters, default=50, metavar="N",
                        help="Griffin-Lim iterations (default 50, the reference's)")
    parser.add_argument("--griffin-lim-momentum", type=parse_gl_momentum, nargs="?", const=0.99, default=0.0, metavar="M",
                        help="fast Griffin-Lim with momentum M in [0, 1] (a bare flag: 0.99, librosa's default; "
                             "default 0, the reference's plain Griffin-Lim)")
    parser.add_argument("--de-emphasis", action="store_true",
                        help="undo preprocessing's pre-emphasis (y[n] - 0.97 y[n-1]) on every synthesised waveform")
    args = parser.parse_args(argv)
    prompts = [p for p in sys.stdin.readlines() if len(p) > 0]                           # test.py:77-78
    from .models.tacotron import Config, Tacotron
    config = Config()
    config.data_path = "data/%s/" % args.train_set                                       # :83
    config.save_path = args.train_set + "/tacotron"                                      # :84
    config.max_ctas = args.max_ctas
    config.attention_window = args.attention_window
    config.stop_at_end = args.stop_at_end
    print("Building Tacotron")
    summary_dir = os.path.join("log", config.save_path, "test") if args.summaries else None      # test.py:33
    test(Tacotron, config, prompts, speaker=args.speaker, summary_dir=summary_dir, trim_tail=args.trim_tail,
         long_form=args.long_form, griffin_lim_iters=args.griffin_lim_iters,
         griffin_lim_momentum=args.griffin_lim_momentum, de_emphasis=args.de_emphasis)


if __name__ == "__main__":
    sys.exit(main())
