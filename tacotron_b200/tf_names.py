"""Variable-name map between the reference's TensorFlow-1.2 graph and this package's parameter store.

The names on the left are the ones the reference's graph code creates (variable scopes of models/tacotron.py:107-154
and models/ops.py:48-132 plus tf.layers' default `dense`, `dense_1`, `conv1d_7`, `batch_normalization_2` numbering);
they were obtained by executing the reference's own model code over a TF-API stand-in (tests/golden/make_golden.py,
fixture key `tf_variable_names`).  This is the table a TF-1.2 checkpoint importer needs (SURVEY.md section 8f, row 4);
tensors keep their TF layouts (dense [in,out], conv [k,Cin,Cout], GRU gates/candidate [in+n, 2n|n])."""
import re


def tf_name_to_param(name, multi_speaker=False, speaker_decoder=False):
    """TF-1.2-style variable name -> parameter name of tacotron_b200.params (same layouts, so a checkpoint tensor
    can be copied as is).  Raises KeyError for variables that are not part of the model (global_step, Adam slots,
    stft_mean/std, ...).  multi_speaker: the graph of a model with num_speakers > 1 (tacotron.py:116-124,
    ops.py:101-115), whose encoder highway layers open with a speaker dense and a width-fixing dense.  speaker_decoder: the
    speaker-conditioned decoder as well (Config.speaker_decoder): the dense of the reference's commented-out initial
    attention line (`decoder/dense`, models/tacotron.py:96-97) and one dense per decoder GRU initial state."""
    import re
    if speaker_decoder:
        m = re.match(r"decoder/(?:speaker_state_([123])/)?dense/(kernel|bias)$", name)
        if m:
            return f"dec/spk/{'h' + m.group(1) if m.group(1) else 'attn'}/{'W' if m.group(2) == 'kernel' else 'b'}"
    if name == "embedding/embedding":
        return "embedding"
    if multi_speaker and name == "speaker/speaker_embed":
        return "speaker/embed"
    kb = {"kernel": "W", "bias": "b"}
    m = re.match(r"(encoder|decoder/decoder/attention_wrapper)/pre_net/dense(_1)?/(kernel|bias)$", name)
    if m:
        pre = "enc" if m.group(1) == "encoder" else "dec"
        return f"{pre}/prenet/{kb[m.group(3)]}{2 if m.group(2) else 1}"
    m = re.match(r"(encoder|post-process)/cbhg/(.*)$", name)
    if m:
        pre, K = ("enc/cbhg", 16) if m.group(1) == "encoder" else ("post/cbhg", 8)
        rest = m.group(2)
        mm = re.match(r"conv1d(?:_(\d+))?/(kernel|bias)$", rest)
        if mm:
            i = int(mm.group(1) or 0)
            if i < K:
                return f"{pre}/bank/{kb[mm.group(2)]}{i + 1}"
            return f"{pre}/proj{i - K + 1}/{kb[mm.group(2)]}"
        mm = re.match(r"batch_normalization(?:_(\d+))?/(gamma|beta|moving_mean|moving_variance)$", rest)
        if mm:
            i = int(mm.group(1) or 0)
            where = "bank" if i == 0 else f"proj{i}"
            return f"{pre}/{where}/bn_{ {'gamma': 'gamma', 'beta': 'beta', 'moving_mean': 'mean', 'moving_variance': 'var'}[mm.group(2)] }"
        mm = re.match(r"highway_(\d+)/dense(?:_(\d+))?/(kernel|bias)$", rest)
        if mm:
            l, j = int(mm.group(1)), int(mm.group(2) or 0)
            if multi_speaker and pre == "enc/cbhg":            # speaker dense, then the 256 -> 128 width fix (ops.py:101-107)
                role = ["s", "d", "T", "H"][j]
            else:
                has_fix = (pre == "post/cbhg" and l == 0)      # ops.py:29-30: extra dense when the width != 128
                role = (["d", "T", "H"] if has_fix else ["T", "H"])[j]
            return f"{pre}/highway{l}/{kb[mm.group(3)]}{role}"
        if multi_speaker and pre == "enc/cbhg" and rest in ("dense/kernel", "dense/bias"):   # bi-GRU initial state (ops.py:111-115)
            return f"{pre}/gru_init/{kb[rest.rsplit('/', 1)[1]]}s"
        mm = re.match(r"bidirectional_rnn/(fw|bw)/gru_cell/(gates|candidate)/(kernel|bias)$", rest)
        if mm:
            return f"{pre}/gru_{mm.group(1)}/{kb[mm.group(3)]}{'g' if mm.group(2) == 'gates' else 'c'}"
    if name == "decoder/memory_layer/kernel":
        return "dec/attn/W_mem"
    aw = "decoder/decoder/attention_wrapper/"
    if name.startswith(aw):
        rest = name[len(aw):]
        fixed = {"input_projection_wrapper/kernel": "dec/in_proj/W", "input_projection_wrapper/bias": "dec/in_proj/b",
                 "output_projection_wrapper/kernel": "dec/out_proj/W", "output_projection_wrapper/bias": "dec/out_proj/b",
                 "bahdanau_attention/query_layer/kernel": "dec/attn/W_q", "bahdanau_attention/attention_v": "dec/attn/v",
                 "attention_layer/kernel": "dec/attn/W_a"}
        if rest in fixed:
            return fixed[rest]
        mm = re.match(r"multi_rnn_cell/cell_(\d)/gru_cell/(gates|candidate)/(kernel|bias)$", rest)
        if mm:
            return f"dec/gru{int(mm.group(1)) + 1}/{kb[mm.group(3)]}{'g' if mm.group(2) == 'gates' else 'c'}"
    if name in ("post-process/dense/kernel", "post-process/dense/bias"):
        return "post/dense/" + kb[name.rsplit("/", 1)[1]]
    raise KeyError(name)
