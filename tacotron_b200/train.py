"""Training driver -- eager equivalent of the reference's ``train.py`` (train.py:16-118; SURVEY.md section 8(f) rank 2).

    python -m tacotron_b200.train -t nancy [-r 1] [--steps N]            (one process)
    torchrun --nproc-per-node 8 -m tacotron_b200.train -t nancy         (data parallel, one process per GPU)

Kept from the reference: data_path / save_path conventions (:107-113), meta.pkl supplies r and the vocabulary (:19-22),
lr fed per step starting at ``init_lr`` and multiplied by ``annealing_rate`` every 1000 steps (:60-61, :79-80), the
explosion guard ``loss > 1e8 and global_step > 500`` (:75-77), a checkpoint + an audio sample every SAVE_EVERY steps
(:82-101; the sample is inverted with the GPU Griffin-Lim and written as .wav next to the checkpoint, the alignment as
.npy).  With ``--summaries`` the reference's TensorBoard summaries are written as well (:41, :64-75, :92-103;
tacotron_b200/summary.py).  Data parallel ranks draw disjoint
batches of 32 and all-reduce the flat gradient bucket inside ``model.train_step`` (tacotron_b200/optim.py).
"""
from __future__ import annotations

import argparse
import math
import os
import sys

import numpy as np
import torch

SAVE_EVERY = 5000          # train.py:13
RESTORE_FROM = None        # train.py:14


def write_wav(path, wave, sr):
    from scipy.io import wavfile
    w = np.asarray(wave, dtype=np.float32)
    peak = float(np.max(np.abs(w))) or 1.0
    wavfile.write(path, sr, (w / peak * 0.95 * 32767).astype(np.int16))


def train(model_cls, config, num_steps=1000000, log=print, save_every=SAVE_EVERY, summary_dir=None, summary_every=1):
    """summary_dir: write TensorBoard summaries there (tacotron_b200/summary.py): the losses, the global gradient norm and
    the histograms of the pre-net output, seq2seq_output and output every `summary_every` steps, the two clips and the
    attention image at every save step.  The histograms are rank 0's batch.
    config.guided_attention > 0 adds the guided attention loss: each batch gets inputs['speech_steps'], the voiced decoder
    steps of its targets (audio.speech_frames), and the loss is summarised and logged as a fourth loss."""
    from . import audio, checkpoint, data_input
    from .utils import dist as D
    world, rank, local = D.world()
    torch.cuda.set_device(local)
    D.init("nccl")
    sr = 24000 if "vctk" in config.data_path else 16000                                   # train.py:18
    meta = data_input.load_meta(config.data_path)                                        # :19
    config.r = meta["r"]                                                                 # :20
    ivocab = meta["vocab"]
    config.vocab_size = len(ivocab)                                                      # :22
    # every rank must normalise with the SAME statistics (the reference is one process: one 100-utterance sample,
    # data_input.py:54): one seeded draw shared by all ranks instead of the unseeded global numpy RNG per rank
    arrays, names, num_speakers, stft_mean, stft_std = data_input.load_from_npy(
        config.data_path, rng=np.random.RandomState(getattr(config, "data_seed", 0)))                # :26-27
    config.num_speakers = num_speakers                                                   # :29
    batches = data_input.build_dataset(arrays, names, seed=0, shard=(rank, world))       # :35
    model = model_cls(config, None, train=True)                                          # :38
    train_op = model.add_train_op()
    weights_dir = os.path.join("weights", config.save_path)
    if getattr(config, "restore", False):                                                # :49-58
        log("restoring weights")
        ck = (checkpoint.latest_checkpoint(weights_dir) if RESTORE_FROM is None else f"{weights_dir}-{RESTORE_FROM}.npz")
        if ck is not None:
            ck_mean, ck_std = checkpoint.restore(model, ck)
            if ck_mean is not None:                  # de-normalise with the statistics the weights were trained on
                stft_mean, stft_std = ck_mean, ck_std
    mean_d = torch.from_numpy(np.asarray(stft_mean, dtype=np.float32)).cuda()
    std_d = torch.from_numpy(np.asarray(stft_std, dtype=np.float32)).cuda()
    lr = model.config.init_lr                                                            # :60
    annealing_rate = model.config.annealing_rate                                         # :61
    # summaries (train.py:41,64-75): rank 0 writes; every rank takes part in the one all-reduce of the three losses
    guided = float(getattr(config, "guided_attention", 0.0) or 0.0) > 0
    summaries = None
    if summary_dir is not None and rank == 0:
        from . import summary
        summaries = summary.TrainSummaries(summary_dir, torch.device("cuda", local), log, guided_attention=guided)
    try:
        for _ in range(num_steps):                                                       # :63
            inputs = next(batches)
            if guided:             # T_b of the guided attention loss: where each target's speech ends, in decoder steps
                inputs["speech_steps"] = audio.speech_frames(inputs["stft"], config.r, mean_d, std_d) // config.r
            loss_t = train_op(inputs, lr).reshape(1).clone()                             # :64-73
            if summary_dir is not None or guided:
                loss_t = torch.stack([model.loss, model.seq2seq_loss, model.output_loss]
                                     + ([model.guided_attention_loss] if guided else []))
            if world > 1:                  # every rank must take the same branch below (a rank that leaves alone hangs the
                torch.distributed.all_reduce(loss_t)   # next gradient all-reduce): the guard and the log use the global loss
            global_step = model.global_step
            if summaries is not None:
                if global_step % summary_every == 0:
                    summaries.enqueue(global_step, (model.saved["enc/prenet/l2"], model.seq2seq_output, model.output), loss_t,
                                      model.grad_sumsq)
                summaries.write_pending()          # the previous step's records, encoded while the GPU runs this step
            loss = float(loss_t[0])                                                      # the only host sync of a step
            if summaries is not None:
                summaries.collect()
            if rank == 0 and global_step % 100 == 0:
                ga = f" guided-attention {float(loss_t[3]):.4g}" if guided else ""
                log(f"step {global_step} loss {loss:.1f}{ga} lr {lr:.3g} grad-norm {float(model.grad_sumsq.sqrt()):.1f}")
            if loss > 1e8 and global_step > 500:                                         # :75-77 detect gradient explosion
                log("loss exploded")
                break
            if global_step % 1000 == 0:                                                  # :79-80
                lr *= annealing_rate
            if global_step % save_every == 0 and global_step != 0 and rank == 0:         # :82
                log("saving weights")
                fn = checkpoint.save(model, weights_dir, stft_mean, stft_std)            # :85-88
                log("saving sample")                                                     # :90-101
                ideal = audio.invert_spectrogram(inputs["stft"][0], config.r, stft_mean=mean_d, stft_std=std_d).cpu().numpy()
                sample = audio.invert_spectrogram(model.output[0], config.r, stft_mean=mean_d, stft_std=std_d).cpu().numpy()
                alignment = model.alignments[0].cpu().numpy()
                base = fn[:-4]
                write_wav(base + "_ideal.wav", ideal, sr)
                write_wav(base + "_sample.wav", sample, sr)
                np.save(base + "_attention.npy", alignment)
                if summaries is not None:
                    summaries.save_step(global_step, ideal, sample, alignment, sr)
    finally:
        if summaries is not None:
            summaries.close()
    return model


def config_from_args(argv=None):
    """(Config, args) of the command line"""
    parser = argparse.ArgumentParser()
    parser.add_argument("-t", "--train-set", default="nancy")
    parser.add_argument("-d", "--debug", type=bool, default=False)
    parser.add_argument("-r", "--restore", type=bool, default=False)
    parser.add_argument("--steps", type=int, default=1000000)
    parser.add_argument("--summaries", action="store_true", help="write TensorBoard summaries to log/<save_path>/train")
    parser.add_argument("--summary-every", type=int, default=1, help="steps between two per-step summaries")
    parser.add_argument("--max-ctas", type=int, default=None,
                        help="CTAs (SMs) the decoder kernels may occupy, at least 32 (default: all the device holds)")
    parser.add_argument("--speaker-decoder", action="store_true",
                        help="multi-speaker data: condition the decoder on the speaker too (initial attention vector and "
                             "GRU states)")
    parser.add_argument("--guided-attention", type=float, default=0.0, metavar="LAMBDA",
                        help="weight of the guided attention loss (Tachibana et al. 2017), a sum like the two L1 losses; "
                             "0 = off (default).  No value has been validated: see README")
    parser.add_argument("--guided-attention-g", type=float, default=0.2, metavar="G",
                        help="width of the guided attention band around the text-speech diagonal (default 0.2)")
    args = parser.parse_args(argv)
    if not (math.isfinite(args.guided_attention) and args.guided_attention >= 0):
        parser.error(f"--guided-attention {args.guided_attention}: must be finite and >= 0")
    if not (math.isfinite(args.guided_attention_g) and args.guided_attention_g > 0):
        parser.error(f"--guided-attention-g {args.guided_attention_g}: must be finite and > 0")
    from .models.tacotron import Config
    config = Config()
    config.data_path = "data/%s/" % args.train_set                                       # train.py:108
    config.restore = args.restore
    config.save_path = "debug" if args.debug else "%s/tacotron" % args.train_set         # :110-113
    config.max_ctas = args.max_ctas
    config.speaker_decoder = args.speaker_decoder
    config.guided_attention = args.guided_attention
    config.guided_attention_g = args.guided_attention_g
    return config, args


def main(argv=None):
    from .models.tacotron import Tacotron
    config, args = config_from_args(argv)
    print("Building Tacotron")
    summary_dir = os.path.join("log", config.save_path, "train") if args.summaries else None     # train.py:41
    train(Tacotron, config, num_steps=args.steps, summary_dir=summary_dir, summary_every=args.summary_every)


if __name__ == "__main__":
    sys.exit(main())
