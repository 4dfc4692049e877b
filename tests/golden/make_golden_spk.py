"""Generates the committed multi-speaker wiring fixtures.  Run IN THE BUILD CONTAINER only (needs /root/reference):

    python tests/golden/make_golden_spk.py

reference_wiring_spk_r{2,5}.npz -- the reference's OWN models/tacotron.py + models/ops.py (unmodified, imported from
/root/reference) with config.num_speakers = 3 (tacotron.py:116-124, ops.py:101-126), executed over oracle/tf12_shim.py
like make_golden.reference_wiring.  The shim's bidirectional_dynamic_rnn takes no initial states, so this script
installs one that does (the speaker-dependent initial_state_fw / initial_state_bw of ops.py:120-126).  Pins the speaker
path of tests/speaker_oracle.py and the multi-speaker variable names against the reference source."""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)


def _bidirectional_dynamic_rnn_h0(shim):
    def rnn(cell_fw, cell_bw, inputs, initial_state_fw=None, initial_state_bw=None, dtype=None, sequence_length=None):
        assert sequence_length is None
        B, T, _ = inputs.shape
        outs = []
        with shim.variable_scope("bidirectional_rnn"):
            for direction, cell, h0 in (("fw", cell_fw, initial_state_fw), ("bw", cell_bw, initial_state_bw)):
                with shim.variable_scope(direction):
                    h = cell.zero_state(B, inputs.dtype) if h0 is None else h0
                    seq = range(T) if direction == "fw" else range(T - 1, -1, -1)
                    o = [None] * T
                    for t in seq:
                        out, h = cell(inputs[:, t], h)
                        o[t] = out
                    outs.append(torch.stack(o, 1))
        return tuple(outs), None
    return rnn


def reference_wiring_spk():
    from oracle import tacotron_oracle as O
    from oracle import tf12_shim as shim
    from tacotron_b200.tf_names import tf_name_to_param
    from tests import speaker_oracle as SO
    for name in ("librosa", "tqdm"):
        m = types.ModuleType(name)
        if name == "tqdm":
            m.tqdm = lambda x, **k: x
        sys.modules[name] = m
    shim.install()
    shim.nn.bidirectional_dynamic_rnn = _bidirectional_dynamic_rnn_h0(shim)
    for k in [k for k in sys.modules if k == "audio" or k == "models" or k.startswith("models.")]:
        del sys.modules[k]
    if "/root/reference" not in sys.path:
        sys.path.insert(0, "/root/reference")
    import models.tacotron as ref_tacotron            # the reference module, unmodified

    nspk = 3
    for r in (2, 5):
        B, Tx, T = 2, 12, 6
        cfg_o = SO.SpkOracleConfig(r=r, max_decode_iter=T, vocab_size=20, num_speakers=nspk)
        params = SO.init_params(cfg_o, seed=1, trained_like=True)
        inp = O.synthetic_inputs(cfg_o, B, Tx, T, seed=0, ragged=True)
        inp["speaker"] = torch.tensor([2, 0], dtype=torch.int32)
        enc_m, dec_m = O.dropout_masks(cfg_o, B, Tx, T, seed=2)
        sm = O.sched_mask(cfg_o, B, T, seed=3)
        used = set()

        def lookup(name, shape):
            on = tf_name_to_param(name, multi_speaker=True)
            used.add(on)
            return params[on]

        out = {"speaker": inp["speaker"].numpy()}
        for mode in ("infer", "teacher", "sched"):
            config = ref_tacotron.Config()
            config.r, config.vocab_size, config.max_decode_iter = r, 20, T
            config.num_speakers = nspk
            config.scheduled_sample = 0.5 if mode == "sched" else 0
            train = mode != "infer"
            drops = []
            if train:                                  # call order: encoder pre-net (2), then 2 per decoder step
                drops = [enc_m[0], enc_m[1]]
                for t in range(T):
                    drops += [dec_m[0][t], dec_m[1][t]]
            shim.S.reset(lookup, dropout_masks=drops, sample_masks=[sm[t] for t in range(T)] if mode == "sched" else None)
            model = ref_tacotron.Tacotron(config, inp, train=train)
            out[f"y_{mode}"] = model.seq2seq_output.numpy()
            out[f"out_{mode}"] = model.output.numpy()
            out[f"align_{mode}"] = model.alignments.numpy()
            if train:
                out[f"loss_{mode}"] = np.array(float(model.loss))
            assert not shim.S.dropout_masks, "dropout masks left over: the reference made fewer dropout calls than assumed"
        assert used == set(params), sorted(set(params) - used)
        out["tf_variable_names"] = np.array(shim.S.created)
        np.savez_compressed(os.path.join(HERE, f"reference_wiring_spk_r{r}.npz"), **out)
        print(f"reference_wiring_spk_r{r}.npz written ({len(shim.S.created)} variables)")


if __name__ == "__main__":
    reference_wiring_spk()
