"""Host-side mirror of the reference's ``models/tacotron.py`` (Config, Tacotron) over the sm_90a
C-ABI.  Eager equivalent of the TF-1.2 graph: ``Tacotron(config, inputs, train)`` owns the
variables (one flat device buffer, TF layouts) and ``inference`` / ``add_loss_op`` run the hand
written kernels; the attribute names the reference drivers fetch (``seq2seq_output``, ``output``,
``alignments``, ``loss``) are kept (models/tacotron.py:187-195, train.py:60-72, test.py:52-56).
"""
from __future__ import annotations

import math

import torch

from .. import _lib as L
from ..params import ParamStore, model_shapes
from . import ops


class Config(object):
    """models/tacotron.py:12-33, with the values the reference derives from module globals or
    injects at run time (r, vocab_size, max_decode_iter: train.py:20-22, tacotron.py:13) explicit."""
    max_decode_iter = 108000 // (2 * 300)      # audio.maximum_audio_length // (audio.r * audio.hop_length)
    attention_units = 256
    decoder_units = 256
    mel_features = 80
    embed_dim = 256
    fft_size = 1025

    char_dropout_prob = 0.5
    audio_dropout_prob = 0.5

    num_speakers = 1
    speaker_embed_dim = 16

    scheduled_sample = 0.5

    cap_grads = 5

    init_lr = 0.0005
    annealing_rate = 1

    batch_size = 32

    # injected by the drivers in the reference
    r = 2
    vocab_size = 64

    # H100 path, feed-forward contractions (the recurrent kernels are fp32-grade in every mode):
    #   'fp32x3' (default) = wgmma tensor cores with the error-compensated 3xTF32 split: fp32-grade products
    #                        (~1e-6 relative), the reference's own arithmetic class;
    #   'tf32'             = single-pass TF32 products (10-bit mantissa), fp32 accumulate: faster, stated looser tolerance;
    #   'fp32'             = exact-product fp32 FFMA kernel (on-GPU cross-check of the tensor-core paths).
    precision = "fp32x3"
    # replay inference-mode calls from CUDA graphs (captured per input shape)
    cuda_graph = False
    # CTAs (SMs) the persistent decoder kernels may occupy, at least 32; None = what the device holds.  The forward decodes
    # 8 x (max_ctas // 32) utterances per launch (up to 32), the backward runs on min(max_ctas, 128) CTAs.
    max_ctas = None
    # multi-speaker models: condition the decoder on the speaker too (initial attention vector and GRU states, DESIGN.md §7)
    speaker_decoder = False
    # guided attention loss (Tachibana et al. 2017, arXiv:1710.08969): lambda (0 = off) and the width g of the band around
    # the text-speech diagonal outside which attention weight is penalised.  Training only; needs inputs['speech_steps'].
    guided_attention = 0.0
    guided_attention_g = 0.2
    # attention window at synthesis (free-running decoding; training never uses it): None = off, or (back, ahead) with
    # back >= 0, ahead >= 1: step t attends only positions p(t-1) - back .. p(t-1) + ahead around the previous step's
    # attention peak p(t-1) (p(-1) = 0).  Off by default, as in the reference; each call also sets attention_peaks.
    attention_window = None
    # end-of-text stop rule at synthesis (free-running decoding; training never uses it): None = off, or hold >= 1: a row
    # ends once `hold` consecutive steps have their attention peak at or past its last real character; each row group of
    # 8 stops decoding soon after its last row ends, and inference returns only the steps the batch needed (end_steps).
    # 4 steps is a starting point only: no value has been validated on a trained model.
    stop_at_end = None

    def __init__(self, **kw):
        for k, v in kw.items():
            setattr(self, k, v)


class Tacotron(object):
    def __init__(self, config, inputs=None, train=True, device="cuda", seed=1):
        """Reference signature ``Tacotron(config, inputs, train)`` (tacotron.py:187).  `inputs` may be
        None (build only) or the input dict of tensors; when given the forward (and loss, if train)
        is evaluated immediately so the result attributes exist as they do after a sess.run."""
        if config.num_speakers > 1 and getattr(config, "speaker_embed_dim", 16) != 16:
            raise ValueError("speaker_embed_dim must be 16 (models/tacotron.py:30)")
        if not torch.cuda.is_available():
            raise RuntimeError("tacotron_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        L.lib()                                   # fail loudly if the extension is missing
        max_ctas = getattr(config, "max_ctas", None)
        if max_ctas is not None:                  # a budget below one decoder row group fails here, before any launch
            from .. import kernels as K
            ops.decoder_budget(K.decoder_capacity()[0], max_ctas)
        ops.attention_window(getattr(config, "attention_window", None))     # a malformed window fails here too
        ops.stop_rule_hold(getattr(config, "stop_at_end", None))            # and a malformed stop rule hold
        self.config = config
        self.train = train
        self.device = torch.device(device)
        self.store = ParamStore(model_shapes(config), self.device)
        self.store.init_tf_default(seed)
        self.runtime = ops.runtime(self.store, config.precision)
        self.lr = config.init_lr
        self.global_step = 0
        self.seq2seq_output = self.output = self.alignments = self.loss = None
        self.attention_peaks = None               # int32 [B, T] peak position of each decoder step (attention window on)
        self.end_steps = None                     # int32 [B] end_step of each row (stop rule on), on the device
        self.guided_attention_loss = None
        self.step_ns = None
        self.section_wait = None
        self.last_graph_kernels = 0                # kernels inside the CUDA graphs replayed by the last call
        self._marks = None                        # bench.py: list of (name, cuda event) section boundaries
        if inputs is not None:
            self(inputs)

    def _mark(self, name):
        if self._marks is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self._marks.append((name, ev))

    # -- parameters ---------------------------------------------------------------------------
    def load_params(self, params):
        self.store.load(params)

    def state_dict(self):
        return self.store.state_dict()

    # -- Tacotron.pre_net (tacotron.py:38-44) ---------------------------------------------------
    def pre_net(self, inputs, units=[256, 128], dropout=0.5, train=True, masks=None, scope=None, ids=None):
        return ops.pre_net(inputs, units=tuple(units), dropout=dropout, train=train, masks=masks, scope=scope, ids=ids)

    # -- create_decoder + dynamic_decode (tacotron.py:46-105, 136-138) ---------------------------
    def create_decoder(self, encoded, inputs, speaker_embed=None, train=True, T=None, dec_drop_masks=None,
                       sample_mask=None):
        """Returns a zero-argument callable that runs the whole decode (the BasicDecoder +
        dynamic_decode pair of the reference) as one persistent kernel: (seq2seq_output, alignments), and the step
        peaks int32 [B, T] third when config.attention_window or config.stop_at_end is set and train is False, and
        end_step int32 [B] fourth when config.stop_at_end is set (ops.attention_decoder)."""
        cfg = self.config
        if train:
            mel = inputs["mel"]
            T = mel.shape[1] if T is None else T
            if cfg.scheduled_sample:                          # ScheduledOutputTrainingHelper (tacotron.py:83-85)
                mode = L.DEC_SCHED
                if sample_mask is None:
                    sample_mask = (torch.rand(T, mel.shape[0], device=mel.device) < cfg.scheduled_sample).to(torch.uint8)
            else:                                             # TrainingHelper (tacotron.py:87)
                mode = L.DEC_TEACHER
            if dec_drop_masks is None:
                B = mel.shape[0]
                dec_drop_masks = ((torch.rand(T, B, 256, device=mel.device) >= cfg.audio_dropout_prob).to(torch.uint8),
                                  (torch.rand(T, B, 128, device=mel.device) >= cfg.audio_dropout_prob).to(torch.uint8))
        else:
            helper = ops.InferenceHelper(inputs["text"].shape[0], cfg.mel_features * cfg.r)   # tacotron.py:89-92
            mode = helper.decoder_mode
            mel = None
            T = cfg.max_decode_iter if T is None else T
            dec_drop_masks = None
            sample_mask = None
        window = None if train else ops.attention_window(getattr(cfg, "attention_window", None))
        hold = None if train else ops.stop_rule_hold(getattr(cfg, "stop_at_end", None))
        sc = ops.Scope(self.store, "dec")
        step_ns = self.step_ns
        if speaker_embed is not None and not getattr(cfg, "speaker_decoder", False):
            raise ValueError("speaker_embed given to create_decoder of a model without speaker_decoder")

        def run():
            h0 = att0 = None
            if speaker_embed is not None:                     # initial attention vector and GRU states (tacotron.py:96-97)
                _, h0, att0 = ops.decoder_speaker_state(sc, speaker_embed)
            stop_at = None if hold is None else ops.stop_positions(inputs["text"], inputs["text_length"])
            return ops.attention_decoder(encoded, inputs["text_length"], cfg.r, T, mode=mode, mel=mel,
                                         sample_mask=sample_mask, drop_masks=dec_drop_masks,
                                         dropout=cfg.audio_dropout_prob, scope=sc, step_ns=step_ns,
                                         max_ctas=getattr(cfg, "max_ctas", None), h0=h0, att0=att0, window=window,
                                         stop_hold=hold, stop_at=stop_at)
        return run

    # -- inference (tacotron.py:107-154) --------------------------------------------------------
    def _speaker_embed(self, inputs):
        """e [B,16] = speaker table rows of inputs['speaker'] (tacotron.py:116-124), or None for a single-speaker model
        (which ignores a 'speaker' key, as the reference does)"""
        if self.config.num_speakers <= 1:
            return None
        spk = inputs.get("speaker")
        if spk is None:
            raise ValueError(f"a model with num_speakers = {self.config.num_speakers} needs inputs['speaker'] (int32 [B])")
        B = inputs["text"].shape[0]
        if not (spk.dtype == torch.int32 and spk.is_cuda and spk.is_contiguous() and tuple(spk.shape) == (B,)):
            raise ValueError(f"inputs['speaker'] must be a contiguous int32 CUDA tensor of shape [{B}], got "
                             f"{spk.dtype} {spk.device} {tuple(spk.shape)}")
        table = self.store["speaker/embed"]
        e = self.runtime.buf("speaker/e", (B, table.shape[1]))
        L.check(L.lib().taco_gather_rows(L.ptr(table), L.ptr(spk), B, table.shape[1], table.shape[0], None, 1.0, L.ptr(e),
                                         L.current_stream()), "taco_gather_rows")
        return e

    def _decoder_speaker_embed(self, B):
        """e [B,16] for a speaker-conditioned decoder: the rows the encoder gathered in this call (_speaker_embed's buffer,
        also the CUDA-graph path's static one), or None"""
        if not getattr(self.config, "speaker_decoder", False):
            return None
        return self.runtime.buf("speaker/e", (B, self.store["speaker/embed"].shape[1]))

    def _encoder(self, inputs, train, enc_drop_masks, trace):
        cfg, store = self.config, self.store
        speaker_embed = self._speaker_embed(inputs)
        # embedding lookup fused with the first pre-net layer (tacotron.py:111-114, :128)
        with ops.variable_scope(store, "enc"):
            pre_out = self.pre_net(store["embedding"], dropout=cfg.char_dropout_prob, train=train, masks=enc_drop_masks,
                                   ids=inputs["text"])
            encoded = ops.CBHG(pre_out, speaker_embed, K=16, c=[128, 128, 128], gru_units=128, trace=trace)   # :131
        if trace is not None:
            trace["enc/prenet_out"] = pre_out
            trace["encoded"] = encoded
        return encoded

    def _postnet(self, seq2seq_output, trace):
        cfg, store = self.config, self.store
        B = seq2seq_output.shape[0]
        # post-processing CBHG + linear-spectrogram dense (:144-151); the reshapes are views
        with ops.variable_scope(store, "post"):
            post_input = seq2seq_output.view(B, -1, cfg.mel_features)
            post = ops.CBHG(post_input, None, K=8, c=[128, 256, 80], gru_units=128, trace=trace)
            W, b = store["post/dense/W"], store["post/dense/b"]
            rt = self.runtime
            dense = ops.linear(rt, post, W, ops.packed_weight(rt, "post/dense/W", W, 1, 256, cfg.fft_size), cfg.fft_size,
                               bias=b, tag="post/dense/out")
        return dense.view(B, -1, cfg.fft_size * cfg.r)

    def inference(self, inputs, train=True, T=None, enc_drop_masks=None, dec_drop_masks=None, sample_mask=None,
                  trace=None):
        """inputs: dict of CUDA tensors: 'text' int32 [B,Tx], 'text_length' int32 [B]; train adds
        'mel' fp32 [B,T,80r] (and 'stft' for the loss).  Returns (seq2seq_output, output).
        With config.stop_at_end (not train) the decode stops at the end of the text: end_step is read once, the call
        keeps T' = min(T, 4 ceil(max_b end_step / 4)) steps (ops.stopped_steps), runs the post-net on those only and
        returns [B, T', ...] outputs; self.end_steps holds end_step.
        With config.cuda_graph the three sections (encoder / decoder / post-net) of an inference-mode call are
        captured once per input shape and replayed: ~26 launches collapse into 3 graph launches."""
        text = inputs["text"]
        assert text.dtype == torch.int32 and text.is_cuda and text.is_contiguous()
        B, Tx = text.shape
        if not 1 <= Tx <= 256:
            raise ValueError(f"text width {Tx} out of range: the persistent decoder keeps keys/values in shared memory, Tx <= 256")
        if getattr(self.config, "cuda_graph", False) and not train and trace is None:
            return self._inference_graphed(inputs, T)
        self._mark("start")
        encoded = self._encoder(inputs, train, enc_drop_masks, trace)
        self._mark("encoder")
        # attention decoder (:135-138)
        dec = self.create_decoder(encoded, inputs, self._decoder_speaker_embed(B), train, T=T, dec_drop_masks=dec_drop_masks,
                                  sample_mask=sample_mask)
        res = dec()
        seq2seq_output, self.alignments = res[:2]
        self.attention_peaks = res[2] if len(res) > 2 else None
        self.end_steps = res[3] if len(res) > 3 else None
        self._mark("decoder")
        if self.end_steps is not None:                            # stop rule: the steps the batch needed
            Tp = ops.stopped_steps(self.end_steps, seq2seq_output.shape[1])
            seq2seq_output = seq2seq_output[:, :Tp].contiguous()
            self.alignments, self.attention_peaks = self.alignments[:, :Tp], self.attention_peaks[:, :Tp]
        output = self._postnet(seq2seq_output, trace)
        self._mark("postnet")
        return seq2seq_output, output

    def _inference_graphed(self, inputs, T):
        T = self.config.max_decode_iter if T is None else T
        hold = ops.stop_rule_hold(getattr(self.config, "stop_at_end", None))
        key = (tuple(inputs["text"].shape), T, self.store.version, getattr(self.config, "max_ctas", None),
               ops.attention_window(getattr(self.config, "attention_window", None)), hold)
        g = self._graphs.get(key) if hasattr(self, "_graphs") else None
        if g is None:
            if not hasattr(self, "_graphs"):
                self._graphs = {}
            static = {"text": inputs["text"].clone(), "text_length": inputs["text_length"].clone()}
            if self.config.num_speakers > 1:
                self._speaker_embed(inputs)                         # validates the ids before they are captured
                static["speaker"] = inputs["speaker"].clone()
            marks, self._marks = self._marks, None
            cg_flag, self.config.cuda_graph = self.config.cuda_graph, False
            try:
                for _ in range(2):                                  # eager warm-up: allocates every scratch buffer, packs weights
                    self.inference(static, train=False, T=T)
                torch.cuda.synchronize()
                graphs, outs = [], {}
                n_launch0 = L.lib().taco_launch_count()
                pool = torch.cuda.graph_pool_handle()
                ge = torch.cuda.CUDAGraph()
                with torch.cuda.graph(ge, pool=pool):
                    outs["encoded"] = self._encoder(static, False, None, None)
                gd = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gd, pool=pool):
                    dec = self.create_decoder(outs["encoded"], static, self._decoder_speaker_embed(static["text"].shape[0]),
                                              False, T=T)
                    res = dec()
                    outs["y"], outs["align"] = res[:2]
                    outs["peak"] = res[2] if len(res) > 2 else None
                    outs["end_step"] = res[3] if len(res) > 3 else None
                graphs = [ge, gd]
                if hold is None:
                    gp = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(gp, pool=pool):
                        outs["out"] = self._postnet(outs["y"], None)
                    graphs.append(gp)
                else:                                               # post-net graphs per kept length T', on demand
                    outs["post"] = {}
            finally:
                self._marks = marks
                self.config.cuda_graph = cg_flag
            g = (static, graphs, outs, int(L.lib().taco_launch_count() - n_launch0))
            self._graphs[key] = g
        static, graphs, outs, _ = g
        static["text"].copy_(inputs["text"], non_blocking=True)
        static["text_length"].copy_(inputs["text_length"], non_blocking=True)
        if "speaker" in static:
            if inputs.get("speaker") is None:
                raise ValueError(f"a model with num_speakers = {self.config.num_speakers} needs inputs['speaker'] (int32 [B])")
            static["speaker"].copy_(inputs["speaker"], non_blocking=True)
        # optional events a pipelined caller sets so that a section does not overwrite a result buffer that an
        # asynchronous device->host copy of the PREVIOUS call is still reading (bench.py e2e)
        waits = getattr(self, "section_wait", None) or {}
        cur = torch.cuda.current_stream()
        self._mark("start")
        graphs[0].replay(); self._mark("encoder")
        if waits.get("decoder") is not None:
            cur.wait_event(waits["decoder"])
        graphs[1].replay(); self._mark("decoder")
        if waits.get("postnet") is not None:
            cur.wait_event(waits["postnet"])
        self.alignments = outs["align"]
        self.attention_peaks = outs["peak"]
        self.end_steps = outs["end_step"]
        self.last_graph_kernels = g[3]
        if self.end_steps is None:
            graphs[2].replay(); self._mark("postnet")
            return outs["y"], outs["out"]
        Tp = ops.stopped_steps(self.end_steps, T)
        post = outs["post"].get(Tp)
        if post is None:
            post = outs["post"][Tp] = self._capture_postnet(outs["y"], Tp)
        post[0].replay(); self._mark("postnet")
        self.alignments, self.attention_peaks = self.alignments[:, :Tp], self.attention_peaks[:, :Tp]
        return post[1], post[2]

    def _capture_postnet(self, y, Tp):
        """(graph, seq2seq_output [B, Tp, 80r], output) for the stop rule's graphed path: the first Tp steps of the
        decoder graph's output y, copied to a static buffer, and the post-net on them (warmed up eagerly first, so
        every scratch buffer of that length exists before the capture)"""
        marks, self._marks = self._marks, None
        try:
            self._postnet(y[:, :Tp].contiguous(), None)
            torch.cuda.synchronize()
            gp = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gp):
                ys = y[:, :Tp].contiguous()
                out = self._postnet(ys, None)
        finally:
            self._marks = marks
        return gp, ys, out

    # -- add_loss_op (tacotron.py:156-165) -------------------------------------------------------
    def add_loss_op(self, seq2seq_output, output, mel, linear):
        lib = L.lib()
        rt = self.runtime
        part = rt.buf("loss/partial", (lib.taco_l1_partial_count(),))
        res = rt.buf("loss/out", (2,))
        L.check(lib.taco_l1_loss_fwd(L.ptr(seq2seq_output), L.ptr(mel), seq2seq_output.numel(), L.ptr(part),
                                     L.ptr(res[0:1]), L.current_stream()), "taco_l1_loss_fwd")
        part2 = rt.buf("loss/partial2", (lib.taco_l1_partial_count(),))
        L.check(lib.taco_l1_loss_fwd(L.ptr(output), L.ptr(linear), output.numel(), L.ptr(part2), L.ptr(res[1:2]),
                                     L.current_stream()), "taco_l1_loss_fwd")
        self.seq2seq_loss = res[0]
        self.output_loss = res[1]
        return res[0] + res[1]

    # -- add_train_op (tacotron.py:167-185) -------------------------------------------------------
    def add_train_op(self, loss=None):
        """Creates the optimizer state (Adam moments + flat gradient bucket) and returns the callable that plays the
        role of `train_op`: ``train_op(inputs, lr)`` = one ``sess.run([train_op, loss, global_step], {lr})``."""
        from ..optim import FlatAdam
        if getattr(self, "_opt", None) is None:
            self._opt = FlatAdam(self.store.flat)
            self._gviews = self._opt.views(self.store)
        return self.train_step

    def backward(self, S):
        """d(loss)/d(parameters) into the flat gradient bucket (zeroed first): the hand-written reverse of
        inference + add_loss_op (models/grad.py) over the saved activations S of a train-mode forward."""
        from .. import kernels as K
        from . import grad
        self.add_train_op()
        self._opt.zero_grad()
        # GEMM kernel of the backward follows the precision mode: 'tf32' -> 3xTF32 mma.sync tensor cores (fp32-grade,
        # ~1e-6 relative), 'fp32' -> exact-product FFMA.  `self.gemm_impl` (0 / 1) overrides.
        impl = getattr(self, "gemm_impl", None)
        if impl is None:
            impl = 0 if self.config.precision == "fp32" else 1
        prev = K.set_gemm_impl(impl)
        # data gradients of the dense / conv layers run on the wgmma forward kernel (a conv data gradient IS a conv):
        # 3xTF32 (fp32-grade) in 'fp32x3' mode, single-pass TF32 in 'tf32' mode; 'fp32' mode keeps the exact-product GEMM.
        # Config.grad_dx_tc overrides (True / False).
        dx_tc = getattr(self.config, "grad_dx_tc", None)
        if dx_tc is None:
            dx_tc = self.config.precision != "fp32"
        prev_dx, K.DX_TC = K.DX_TC, bool(dx_tc)
        prev_impl, K.DX_TC_IMPL = K.DX_TC_IMPL, (L.IMPL_TC if self.config.precision == "tf32" else L.IMPL_TC3)
        # weight gradients of the dense / conv layers: wgmma 3xTF32 kernel (taco_conv_dw), same switch; Config.grad_dw_tc overrides
        dw_tc = getattr(self.config, "grad_dw_tc", None)
        prev_dw, K.DW_TC = K.DW_TC, bool(dx_tc if dw_tc is None else dw_tc)
        prev_g, K.GEMM_TC = K.GEMM_TC, bool(dx_tc)            # recomputation / data-gradient products on the same kernel
        try:
            grad.model_bwd(K, self.store, self._gviews, S, self.config)
        finally:
            K.set_gemm_impl(prev)
            K.DX_TC = prev_dx
            K.DX_TC_IMPL = prev_impl
            K.DW_TC = prev_dw
            K.GEMM_TC = prev_g
        return self._gviews

    def train_step(self, inputs, lr=None, **kw):
        """forward (train mode, activations saved) -> loss -> backward -> [all-reduce] -> clip -> Adam.
        Returns the loss tensor (device scalar); `self.global_step`, `self.grad_sumsq` are updated."""
        from .. import kernels as K
        self.add_train_op()
        lr = self.lr if lr is None else lr
        lam = self._guided_attention_lambda(inputs)
        S = {}
        with ops.saving(S):
            self.seq2seq_output, self.output = self.inference(inputs, True, **kw)
        self.loss = self.add_loss_op(self.seq2seq_output, self.output, inputs["mel"], inputs["stft"])
        if lam > 0:                                # + guided attention loss; its score gradient goes to the decoder backward
            align = S["dec/align"]
            dscore = torch.empty_like(align)
            ga = self.runtime.buf("loss/ga", (1,))
            part = self.runtime.buf("loss/ga_partial", (L.lib().taco_guided_attention_partial_count(*align.shape[:2]),))
            K.guided_attention(dscore, ga, align, inputs["text_length"], inputs["speech_steps"],
                               self.config.guided_attention_g, lam, part)
            S["dec/dscore_ga"] = dscore
            self.guided_attention_loss = ga[0]
            self.loss = self.loss + ga[0]
        S.update(text=inputs["text"], text_length=inputs["text_length"], mel=inputs["mel"], stft=inputs["stft"])
        if self.config.num_speakers > 1:
            S["speaker"] = inputs["speaker"]
        S["post/out"] = self.output
        self.saved = S
        self.backward(S)
        # data parallel: one SUM all-reduce of the flat gradient bucket when a process group exists (self.dp = False
        # keeps the step local, e.g. for a per-rank health check before the first collective)
        self.grad_sumsq = self._opt.apply(K, self.store.flat, lr, self.config.cap_grads, allreduce=getattr(self, "dp", True))
        self.store.version += 1                    # derived kernel-layout buffers are refreshed on the next forward
        self.global_step += 1
        return self.loss

    def _guided_attention_lambda(self, inputs):
        """lambda of the guided attention loss (0.0 = off), after checking the settings and inputs['speech_steps'] (int32
        [B]: the voiced decoder steps T_b of each target, in [1, T]; the range check reads them to the host once)"""
        lam = float(getattr(self.config, "guided_attention", 0.0) or 0.0)
        g = float(getattr(self.config, "guided_attention_g", 0.2))
        if not (math.isfinite(lam) and lam >= 0.0):
            raise ValueError(f"Config.guided_attention = {lam}: the loss weight must be finite and >= 0 (0 = off)")
        if lam == 0.0:
            return 0.0
        if not (math.isfinite(g) and g > 0.0):
            raise ValueError(f"Config.guided_attention_g = {g}: the band width must be finite and > 0")
        steps = inputs.get("speech_steps")
        if steps is None:
            raise ValueError("Config.guided_attention > 0 needs inputs['speech_steps'] (int32 [B]): the voiced decoder steps "
                             "of each target, e.g. audio.speech_frames(inputs['stft'], r, stft_mean, stft_std) // r")
        B, T = inputs["mel"].shape[:2]
        if not (steps.dtype == torch.int32 and steps.is_cuda and steps.is_contiguous() and tuple(steps.shape) == (B,)):
            raise ValueError(f"inputs['speech_steps'] must be a contiguous int32 CUDA tensor of shape [{B}], got "
                             f"{steps.dtype} {steps.device} {tuple(steps.shape)}")
        lo, hi = torch.stack([steps.min(), steps.max()]).tolist()
        if lo < 1 or hi > T:
            raise ValueError(f"inputs['speech_steps'] must lie in [1, {T}] (the decoder steps of the batch), got [{lo}, {hi}]")
        return lam

    # -- the eager stand-in for sess.run([...]) ---------------------------------------------------
    def __call__(self, inputs, **kw):
        self.seq2seq_output, self.output = self.inference(inputs, self.train, **kw)
        if self.train and "stft" in inputs:
            self.loss = self.add_loss_op(self.seq2seq_output, self.output, inputs["mel"], inputs["stft"])
        return self.seq2seq_output, self.output
