/*
 * taco_b200.h -- C-ABI of libtaco_b200.so: the H100 (sm_90a) hot path of the Tacotron
 * mel/linear-spectrogram model (reference: barronalex/Tacotron, models/tacotron.py, models/ops.py).
 *
 * The reference has no FFI boundary of its own (it is 100% Python over TensorFlow 1.2); the
 * boundary a maintainer binds is therefore the set of TF-1.2 library calls its hot path makes.
 * Each entry point below names the reference call site(s) it replaces.  The Python host
 * (tacotron_b200/models/{ops,tacotron}.py) reaches these through ctypes -- see INTEGRATION.md.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes; no C++/torch types.
 *   - every function returns 0 on success, non-zero on error; taco_last_error() gives the
 *     message for the calling thread.  Nothing throws across the boundary.
 *   - all tensors are caller-owned DEVICE pointers (fp32 unless noted), contiguous in their
 *     last dimension, 16-byte aligned.  The library allocates nothing on the hot path; the
 *     caller passes workspaces where needed.
 *   - all launches are asynchronous on the caller's stream (cudaStream_t passed as void*).
 *   - activations are NWC: x[B][T][C] (TF layout); dense weights are W[in][out]; conv weights
 *     W[k][Cin][Cout]; GRU weights gates[in+n][2n] (r then u), candidate[in+n][n]  (TF 1.2).
 */
#ifndef TACO_B200_H
#define TACO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TACO_VERSION 100

enum { TACO_ACT_NONE = 0, TACO_ACT_RELU = 1, TACO_ACT_SIGMOID = 2, TACO_ACT_TANH = 3 };
enum { TACO_IMPL_TC = 0,   /* wgmma tensor cores, TF32 multiplies, fp32 accumulate (TMA-fed) */
       TACO_IMPL_SIMT = 1, /* fp32 FFMA, exact fp32 products                                  */
       TACO_IMPL_TC3 = 2   /* wgmma tensor cores, error-compensated 3xTF32 (x = hi + lo; lo.hi + hi.lo + hi.hi,
                              fp32 accumulate): fp32-grade products (~1e-6 relative).  Wp then holds the
                              hi rows [0,N) followed by the lo rows [N,2N) (taco_pack_weight_x3)          */ };
enum { TACO_EPI_NORMAL = 0,
       TACO_EPI_HIGHWAY = 1 /* N = 2U: cols [0,U) = H pre-act, [U,2U) = T pre-act; Y[M][U] =
                               relu(H)*sig(T) + X*(1-sig(T)), X = hx (models/ops.py:32-45)   */ };
enum { TACO_DEC_INFER = 0, TACO_DEC_TEACHER = 1, TACO_DEC_SCHED = 2 };

const char* taco_last_error(void);
int         taco_version(void);
/* Number of SMs of the current device and whether the TMA/wgmma path is usable (cc 9.0). */
int         taco_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ------------------------------------------------------------------------------------------
 * taco_linear_fwd -- one fused contraction + epilogue.  Replaces, depending on the fields:
 *   tf.layers.dense            models/ops.py:30,32,39  models/tacotron.py:40,42,148
 *   tf.layers.conv1d('same')   models/ops.py:54-62 (bank: all K filters in ONE call), :80-85
 *   tf.layers.batch_normalization (inference affine, folded into scale/shift)  ops.py:64,87
 *   tf.layers.dropout          models/tacotron.py:41,43   (explicit keep mask)
 *   residual add               models/ops.py:92
 *   highway gate               models/ops.py:32-45 (TACO_EPI_HIGHWAY)
 * Y[b,t,n] = epi( sum_{j<taps} sum_{c<C} X[b, t+tap0+j, c] * W[j,c,n] ),  zero outside [0,T).
 * epi(v) = (act(v + bias[n] + bias_utt[b*ldbu + n]) * scale[n] + shift[n]) * keep[b,t,n]*keep_scale + residual[b,t,n]
 * (bias_utt: a per-utterance bias, e.g. a speaker-dependent term; the two biases are added to each other first)
 * Bank mode (bank_K > 0): N = bank_K*bank_cout; output columns [(k-1)*cout, k*cout) come from
 * filter k (k taps, tap0 = -(k-1)/2).  W then points at the K filters stored back to back
 * (W1 [1][C][cout], W2 [2][C][cout], ...), Wp at the packed form made by taco_pack_weight.
 * ------------------------------------------------------------------------------------------ */
typedef struct taco_linear_desc {
    const float*   X;        /* [B][T][ldx] activations, C valid channels                    */
    int64_t        ldx;      /* floats between consecutive (b,t) rows                        */
    int32_t        B, T, C;
    int32_t        taps;     /* 1 = dense                                                    */
    int32_t        tap0;     /* -(taps-1)/2 for TF 'same'                                    */
    int32_t        N;        /* output channels (total)                                      */
    int32_t        bank_K;   /* 0, or number of bank filters                                 */
    int32_t        bank_cout;
    const float*   W;        /* TF layout [taps*C][N] row-major (SIMT path)                  */
    const float*   Wp;       /* packed K-major [N][ldwp] TF32-rounded (tensor-core path)     */
    int64_t        ldwp;     /* floats per packed row = max_taps * round_up(C,32)            */
    float*         Y;        /* [B*T][ldy]                                                   */
    int64_t        ldy;
    const float*   bias;     /* [N] or NULL                                                  */
    int32_t        act;      /* TACO_ACT_*                                                   */
    const float*   scale;    /* [N] or NULL   (BN: gamma/sqrt(var+1e-3))                     */
    const float*   shift;    /* [N] or NULL   (BN: beta - mean*scale)                        */
    const uint8_t* keep;     /* [B*T][N] dropout keep mask or NULL                           */
    float          keep_scale;
    const float*   residual; /* [B*T][ldr] or NULL                                           */
    int64_t        ldr;
    int32_t        epilogue; /* TACO_EPI_*                                                   */
    const float*   hx;       /* highway carry input X [B*T][ldhx]                            */
    int64_t        ldhx;
    int32_t        pool;     /* 1: fuse max_pooling1d(2,1,'same') over t after the affine    */
                             /*    (models/ops.py:66-71); tensor-core path only              */
    int32_t        impl;     /* TACO_IMPL_*                                                  */
    const float*   bias_utt; /* [B][ldbu] per-utterance bias or NULL; not with TACO_EPI_HIGHWAY */
    int64_t        ldbu;
} taco_linear_desc;

int taco_linear_fwd(const taco_linear_desc* d, void* stream);
/* The launch taco_linear_fwd makes for descriptor d, decided on the host (no CUDA call, no device needed; pointers are
 * only checked for alignment).  Returns taco_linear_fwd's error, with the same message, for a descriptor it rejects.
 * Tensor-core impls: *bn = n-tile width (32: fp32x3 when at most 33 output tiles and N >= 64; 256: highway; else 128),
 * *stages = k-block ring depth, *mode = 0 normal / 1 highway epilogue, *direct = 1 register-direct epilogue (every row
 * segment it touches 16-byte aligned) / 0 transposing epilogue, *tile_stride = 128, or 127 with the fused max-pool.
 * SIMT: 64 x 64 tiles over the flattened rows (*bn = 64, *stages = 1, *direct = 0, *tile_stride = 64).
 * Any output pointer may be NULL.                                                                                */
int taco_linear_route(const taco_linear_desc* d, int* bn, int* stages, int* mode, int* direct, int* tile_stride);

/* Pack one TF-layout weight W[taps][C][N] into the tensor-core operand layout: row n of dst
 * (dst + (n)*ld_dst) holds, for tap j and channel c, W[j][c][n] at column j*round_up(C,32)+c,
 * rounded to TF32 (round-to-nearest, ties away from zero: cvt.rna); padding channels are zero.  */
int taco_pack_weight(const float* W, int taps, int C, int N, float* dst, int64_t ld_dst, void* stream);
/* 3xTF32 operand pair for TACO_IMPL_TC3: dst_hi rows = TF32 round-to-nearest heads (ties away from zero), dst_lo rows =
 * the remainders W - hi rounded to the nearest TF32 value (ties away from zero), so |hi + lo - W| <= 2^-22 |W|; same
 * layout as taco_pack_weight.  For a bank, call once per filter with the row offsets of that filter in the hi half
 * and in the lo half (lo half starts at row bank_K*bank_cout).                                                    */
int taco_pack_weight_x3(const float* W, int taps, int C, int N, float* dst_hi, float* dst_lo, int64_t ld_dst, void* stream);

/* tf.layers.max_pooling1d(pool 2, stride 1, 'same') over t  (models/ops.py:66-71)            */
int taco_maxpool_fwd(const float* X, float* Y, int B, int T, int C, void* stream);

/* Embedding-style row gather with optional dropout keep mask:
 * Y[i][:] = table[ids[i]][:] * keep[i][:]*keep_scale   (tf.nn.embedding_lookup, tacotron.py:114) */
int taco_gather_rows(const float* table, const int32_t* ids, int rows, int width, int vocab,
                     const uint8_t* keep, float keep_scale, float* Y, void* stream);

/* values[b][j][:] = memory[b][j][:] if j < length[b] else 0   (BahdanauAttention _prepare_memory,
 * tacotron.py:48-52)                                                                          */
int taco_mask_rows(const float* X, const int32_t* length, float* Y, int B, int T, int C, void* stream);

/* ------------------------------------------------------------------------------------------
 * taco_bigru_fwd -- tf.nn.bidirectional_dynamic_rnn(GRUCell(128), GRUCell(128)) without
 * sequence_length (models/ops.py:118-128).  The input-side products are hoisted out of the
 * loop by the caller (one taco_linear_fwd):
 *   xp[b][t][0:256]   = x.Wg_fw[0:128,:] + bg_fw     xp[b][t][256:384] = x.Wc_fw[0:128,:] + bc_fw
 *   xp[b][t][384:640] = x.Wg_bw[0:128,:] + bg_bw     xp[b][t][640:768] = x.Wc_bw[0:128,:] + bc_bw
 * wh_fw / wh_bw point at the h-side rows: Wg[128:256][256] followed by Wc[128:256][128] are
 * passed separately.  out[b][t][0:128] = fw state, [128:256] = bw state.
 * One persistent CTA per (utterance, direction), recurrent weights register-resident.
 * ------------------------------------------------------------------------------------------ */
int taco_bigru_fwd(const float* xp, const float* Wg_h_fw, const float* Wc_h_fw,
                   const float* Wg_h_bw, const float* Wc_h_bw,
                   float* out, int B, int T, void* stream);
/* same, with initial states h0_fw / h0_bw [B][128] (NULL = zero state; initial_state_fw/bw of
 * bidirectional_dynamic_rnn, models/ops.py:111-126: the speaker-dependent state of a multi-speaker model) */
int taco_bigru_fwd_h0(const float* xp, const float* Wg_h_fw, const float* Wc_h_fw,
                      const float* Wg_h_bw, const float* Wc_h_bw, const float* h0_fw, const float* h0_bw,
                      float* out, int B, int T, void* stream);

/* ------------------------------------------------------------------------------------------
 * taco_highway_stack_fwd -- the pointwise tail of a CBHG at inference (models/ops.py:27-46,118-128) in ONE kernel:
 *   h = X (C == 128), or X.Wd + bd (width-fixing dense, C != 128, ops.py:29-30)
 *   L times: h = relu(h.WH + bH) * sig(h.WT + bT) + h * (1 - sig(h.WT + bT))          (highway, ops.py:32-45)
 *   Y = h.Wx + bx: the bi-GRU input products xp, in taco_bigru_fwd's layout           (ops.py:118-128)
 * over M flat rows (every layer is a dense, so utterance boundaries do not matter).  Only Y is written; the
 * activations between layers stay on chip.  TACO_IMPL_TC3 only.  Weights are the buffers taco_pack_weight_x3 makes
 * for the unfused route (hi rows [0,N), lo rows [N,2N)): Wd_p N = 128, hw_p[l] = [WH | WT] with N = 256, xp_p N = 768.
 * Each output element sees the same operations in the same order as that of the unfused sequence
 * (taco_linear_fwd dense + L x TACO_EPI_HIGHWAY + dense 768), so the results are bit-identical to it.
 * ------------------------------------------------------------------------------------------ */
#define TACO_HIGHWAY_STACK_MAX 4
typedef struct taco_highway_stack_desc {
    const float*   X;        /* [M][ldx], C valid channels                                    */
    int64_t        ldx;
    int32_t        M, C;     /* 1 <= C <= 128                                                 */
    const float*   Wd_p;     /* packed [2*128][ldwd] (C != 128), NULL when C == 128           */
    int64_t        ldwd;
    const float*   bd;       /* [128] (C != 128)                                              */
    int32_t        L;        /* highway layers, 1..TACO_HIGHWAY_STACK_MAX                     */
    const float*   hw_p[TACO_HIGHWAY_STACK_MAX];   /* packed [2*256][ldhw]                    */
    int64_t        ldhw;
    const float*   hw_b[TACO_HIGHWAY_STACK_MAX];   /* [bH | bT] (256)                         */
    const float*   xp_p;     /* packed [2*768][ldxp]                                          */
    int64_t        ldxp;
    const float*   xp_b;     /* [768]                                                         */
    float*         Y;        /* [M][ldy], ldy >= 768                                          */
    int64_t        ldy;
    int32_t        impl;     /* TACO_IMPL_TC3                                                 */
} taco_highway_stack_desc;
int taco_highway_stack_fwd(const taco_highway_stack_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------
 * Decoder: tacotron.py:46-105 create_decoder + :136-138 dynamic_decode, i.e. per step
 *   pre_net(last frame) ++ attention -> InputProjection -> 3x GRUCell(256) -> Residual ->
 *   OutputProjection(80r) -> BahdanauAttention(query = cell output) -> attention layer.
 * The whole T-step loop runs in ONE persistent kernel: 32 co-resident CTAs (one per SM) per row group of 8 utterances,
 * min(4, CTA budget / 32) row groups per launch (128 CTAs when the device holds them), activations exchanged as
 * {value, step tag} words through L2, weights in shared memory and L2 (csrc/decoder.cu).  Tx in [1,256], any width (the
 * four attention quarters are ragged when Tx % 4 != 0); B <= 8 * row groups (<= 32) per launch; 80 r <= 512.
 * ------------------------------------------------------------------------------------------ */
typedef struct taco_decoder_weights {   /* all TF layout, device pointers */
    const float *pre_W1, *pre_b1, *pre_W2, *pre_b2;      /* [80][256],[256],[256][128],[128]   */
    const float *in_W, *in_b;                            /* [384][256],[256]                   */
    const float *gru_Wg[3], *gru_bg[3], *gru_Wc[3], *gru_bc[3]; /* [512][512],[512],[512][256],[256] */
    const float *out_W, *out_b;                          /* [256][80r],[80r]                   */
    const float *att_Wq, *att_v, *att_Wa;                /* [80r][256],[256],[80r+256][256]    */
} taco_decoder_weights;

/* bytes of the packed-weight buffer / of the workspace taco_decoder_fwd needs */
size_t taco_decoder_packed_bytes(int r);
size_t taco_decoder_workspace_bytes(int B, int Tx, int T, int r);
/* 64-bit word offset in that workspace of the per-stage trace the TACO_TRACE build writes (scripts/dec_time.py): from
 * there [16 T + 16] words of %globaltimer stamps of CTA 0, one per finished stage, then [4][20][8] clock64 records of
 * the stages of steps 10..13                                                                                          */
int64_t taco_decoder_trace_offset(void);
/* re-lay the weights per CTA column slice (call once per weight update) */
int taco_decoder_pack(const taco_decoder_weights* w, int r, float* packed, void* stream);

typedef struct taco_decoder_args {
    const taco_decoder_weights* weights; /* HOST pointer; biases and attention_v are read from here (in_b and
                                            gru_bg[0] were folded in by taco_decoder_pack)              */
    const float*   packed;       /* from taco_decoder_pack                                    */
    const float*   keys;         /* [B][Tx][256]  values . W_mem                              */
    const float*   values;       /* [B][Tx][256]  length-masked memory                        */
    const int32_t* text_length;  /* [B]                                                       */
    const float*   mel;          /* [B][T][80r] teacher inputs (TEACHER / SCHED) or NULL      */
    const uint8_t* sample_mask;  /* [T][B] 1 = feed own output (SCHED) or NULL                */
    const uint8_t* keep1;        /* [T][B][256] pre-net dropout keep masks or NULL            */
    const uint8_t* keep2;        /* [T][B][128]                                               */
    float          keep_scale;   /* 1/(1-rate)                                                */
    int32_t        mode;         /* TACO_DEC_*                                                */
    int32_t        B, Tx, T, r;
    float*         y;            /* [B][T][80r]   seq2seq_output                              */
    float*         align;        /* [B][T][Tx]    alignment history                           */
    void*          workspace;    /* taco_decoder_workspace_bytes                              */
    uint64_t*      step_ns;      /* [T] device buffer: %globaltimer at the start of each step, or NULL */
    float*         h_save;       /* [3][T][B][256] the three GRU state sequences (training: input of
                                    taco_decoder_bwd's batched recomputation), or NULL          */
    int32_t        row0;         /* the [T][B]-major tensors (sample_mask, keep1, keep2, h_save) have   */
    int32_t        row_stride;   /* row_stride rows per step, this launch's row b is row0 + b (a batch
                                    decoded in several launches); row_stride = 0: B rows, row0 = 0   */
    int32_t        max_ctas;     /* CTA budget (>= 32), 0 = what the device holds (taco_decoder_capacity) */
    const float*   h0;           /* [3][row_stride][256] initial states of the three GRUs (speaker-conditioned decoder;
                                    this launch's row b is row0 + b), or NULL = zero state (cell.zero_state)  */
    const float*   att0;         /* [row_stride][256] initial attention vector, or NULL = zero; needs weights->in_W
                                    (h0 needs weights->gru_Wg): their step-0 products are formed in the workspace */
    int32_t        win_back;     /* attention window (TACO_DEC_INFER only; win_ahead = 0: no window, the default).  With   */
    int32_t        win_ahead;    /* p(-1) = 0 and N_b = min(text_length_b, Tx), step t scores only the positions j with
                                    max(0, p(t-1) - win_back) <= j <= p(t-1) + win_ahead, j < N_b (the others are -inf
                                    before the softmax); p(t) = the lowest j of highest score.  win_back >= 0,
                                    win_ahead >= 1; bounds >= Tx - 1 allow every position and give the unwindowed bits */
    int32_t*       peak;         /* [B][T] p(t) of each step (indexed like align), or NULL; needs the window or the stop
                                    rule (-1 at the steps a stopped row group did not decode)                            */
    const int32_t* stop_at;      /* end-of-text stop rule (TACO_DEC_INFER only; NULL: off, the default).  [B] encoder   */
    int32_t        stop_hold;    /* positions: row b ends after step t when p(t - stop_hold + 1), ..., p(t) are all >=
                                    stop_at[b] (p as for peak, windowed or not), end_step[b] = t + 1 for the first such
                                    t, or T.  stop_hold >= 1.  Each row group of 8 decodes D_g = min(T, max over its
                                    rows of end_step + TACO_DECODER_STOP_LAG) steps (padding rows end at 0); at the
                                    steps t >= D_g, y and align hold 0 and peak -1                                      */
    int32_t*       end_step;     /* [B] out: end_step of each row (set with stop_at, NULL with it)                      */
} taco_decoder_args;

/* Steps a row group decodes past its last row's end_step under the stop rule: the row's end is known at the start of
 * the next step's attention, every CTA of the group reads the group's ended rows one step later, and all of them leave
 * at the top of the step after the next stage barrier (csrc/decoder.cu, DESIGN.md 3.4).                               */
#define TACO_DECODER_STOP_LAG 3

int taco_decoder_fwd(const taco_decoder_args* a, void* stream);
/* co-resident CTAs of the forward (taco_decoder_fwd) and backward (taco_decoder_bwd) decoder kernels on the current
 * device (either pointer may be NULL).  The forward runs 32 CTAs per row group of 8 utterances, the backward at least 32
 * and at most 128 CTAs.                                                                                              */
int taco_decoder_capacity(int* fwd_ctas, int* bwd_ctas);

/* tacotron.py:156-160: partial[0] = sum|a-b| over n elements (deterministic two-stage).       */
int taco_l1_loss_fwd(const float* a, const float* b, int64_t n, float* partial_ws, float* out, void* stream);
int taco_l1_partial_count(void);   /* floats partial_ws must hold */

/* number of kernels this library has launched so far in this process (for bench.py's gpu_launches) */
unsigned long long taco_launch_count(void);

/* ==========================================================================================
 * Training path.  Replaces what `tf.gradients` + `tf.clip_by_global_norm` + `tf.train.AdamOptimizer`
 * build for Tacotron.add_train_op (models/tacotron.py:167-185) over the forward graph
 * (models/tacotron.py:107-165, models/ops.py:27-132).  The host side (tacotron_b200/models/grad.py)
 * is the hand-written reverse of the forward; the entry points below are its arithmetic.
 * The semantics of each are pinned by the function of the same name in tests/mirror_kernels.py.
 * ========================================================================================== */

/* C_z[M][N] = beta*C_z + opA_z[M][K] . opB_z[K][N]  for z < batch  (fp32 FFMA; beta in {0,1}).
 *   ta=0: A stored [M][K]: opA[m][k] = A[m + sh(k)][k mod kper],  sh(k) = shift + z*bshift + (k / kper)*dshift
 *   ta=1: A stored [K][M]: opA[m][k] = A[k + sh][m],              sh    = shift + z*bshift
 *         a shifted stored row that leaves its block of `period` rows (0: one block) reads as zero.
 *   tb=0: B stored [K][N];  tb=1: B stored [N][kper] per K-segment j at offset j*b_tap_stride.
 * This one contraction covers every dense / conv1d('same') data gradient (row shift = tap offset, zero fill =
 * the 'same' padding per utterance), every weight gradient (ta=1, batch = taps, split-K with atomics), the
 * h(t-1) products of the recurrent layers (shift = one step) and the per-utterance attention context GEMMs.  */
typedef struct taco_gemm_desc {
    const float* A; int64_t lda;
    const float* B; int64_t ldb;
    float*       C; int64_t ldc;
    int32_t M, N, K;
    int32_t ta, tb;
    float   beta;
    int32_t shift, period;
    int32_t taps, dshift, kper;
    int64_t b_tap_stride;
    int32_t batch;
    int64_t a_bstride, b_bstride, c_bstride;   /* in elements */
    int32_t bshift;
} taco_gemm_desc;
int taco_gemm(const taco_gemm_desc* d, void* stream);
/* which kernel taco_gemm launches: 0 = exact-product FFMA (default), 1 = 3xTF32 mma.sync tensor cores (fp32-grade,
 * ~1e-6 relative; opt-in until it has had a hardware run).  Returns the previous setting. */
int taco_set_gemm_impl(int impl);
/* Weight gradient of tf.layers.conv1d('same') / tf.layers.dense on the wgmma tensor cores (error-compensated 3xTF32,
 * fp32-grade; models/ops.py:54,80, tacotron.py:40,42,148 under tf.gradients, tacotron.py:170):
 *     dW[j*tap_stride + c*ldw + n] += sum_{b<B, t<T} X[(b*T + t + tap0 + j)*ldx + c] * dZ[(b*T + t)*lddz + n]
 * for j < taps, c < C, n < N; rows outside [0,T) of an utterance read as zero (the 'same' padding).  Accumulates into dW
 * (split-K with atomic adds, like taco_gemm's ta=1 path).  X, dZ 16-byte aligned, ldx and lddz multiples of 4 floats. */
int taco_conv_dw(float* dW, int64_t ldw, int64_t tap_stride, const float* X, int64_t ldx, const float* dZ, int64_t lddz,
                 int32_t B, int32_t T, int32_t C, int32_t N, int32_t taps, int32_t tap0, void* stream);

/* out[n] += sum_m A[m][n] * (Bm ? Bm[m][n] - (R ? R[m][n] : 0) : 1)     (bias / batch-norm gradients) */
int taco_colsum(float* out, const float* A, int64_t lda, const float* Bm, int64_t ldb, const float* R, int64_t ldr,
                int M, int N, void* stream);
/* out[m/period][n] += sum over the `period` rows m of segment m/period of A[m][n]  (per-utterance column sums, e.g. the
 * gradient of a per-utterance bias); deterministic, no atomics.  M % period == 0.                               */
int taco_colsum_seg(float* out, int64_t ldo, const float* A, int64_t lda, int M, int N, int period, void* stream);
/* in place C = act(C + bias) (bias may be NULL); out = X * H[row+shift] (zero outside the period block) */
int taco_bias_act(float* C, int64_t ldc, int M, int N, const float* bias, int act, void* stream);
int taco_mul_shift(float* out, int64_t ldo, const float* X, int64_t ldx, const float* H, int64_t ldh, int M, int N,
                   int shift, int period, void* stream);
/* backward of taco_linear_fwd's epilogue: dZ = dY*gain*scale[n]*mask; relu mask = Y > 0 (no scale) or
 * (Y - R - shift[n])*scale[n] > 0.  dZ may alias dY.                                                       */
int taco_epi_bwd(float* dZ, int64_t lddz, const float* dY, int64_t lddy, const float* Y, int64_t ldy, const float* R,
                 int64_t ldr, int M, int N, int relu, const float* scale, const float* shift, float gain, void* stream);
/* in place dropout with an explicit keep mask [M][N]: X = keep ? X*gain : 0   (tacotron.py:41,43) */
int taco_epi_fwd_keep(float* X, int64_t ldx, const uint8_t* keep, int M, int N, float gain, void* stream);
/* dbeta += S1; dgamma += (S2 - beta*S1)/gamma   (tf.layers.batch_normalization, inference form, ops.py:64,87) */
int taco_bn_param_grad(float* dgamma, float* dbeta, const float* S1, const float* S2, const float* gamma,
                       const float* beta, int N, void* stream);
/* tf.layers.max_pooling1d(2,1,'same') backward (ops.py:66-71); ties go to the first element */
int taco_maxpool_bwd(float* dX, const float* dP, const float* X, int B, int T, int C, void* stream);
/* highway gate (ops.py:32-45) from saved pre-activations P = [h_pre | t_pre] ([M][2U]) and its backward */
int taco_highway_fwd(float* Y, int64_t ldy, const float* P, int64_t ldp, const float* X, int64_t ldx, int M, int U,
                     void* stream);
int taco_highway_bwd(float* dP, int64_t lddp, float* dXd, int64_t lddx, const float* dY, int64_t lddy, const float* P,
                     int64_t ldp, const float* X, int64_t ldx, int M, int U, void* stream);
/* dA = beta*dA + sign(A - B)    (tacotron.py:158-160) */
int taco_l1_bwd(float* dA, const float* A, const float* B, int64_t n, float beta, void* stream);
/* same, A / B as [rows][cols] contiguous and dA with a row pitch of ldd >= cols floats (a 16-byte-aligned pitch for the
 * [M][1025] spectrogram gradient, so that the tensor-core data / weight gradient kernels can read it through TMA) */
int taco_l1_bwd_ld(float* dA, int64_t ldd, const float* A, const float* B, int64_t rows, int64_t cols, float beta, void* stream);
/* dTable[ids[m]][:] += dRows[m][:]   (embedding_lookup backward, tacotron.py:111-114) */
int taco_scatter_add_rows(float* dTable, const int32_t* ids, const float* dRows, int rows, int width, int vocab,
                          void* stream);
/* serial part of the bidirectional-GRU backward (ops.py:118-128): see csrc/gru_bwd.cu */
int taco_bigru_bwd(float* dxp, const float* dOut, const float* out, const float* ACT, const float* Wg_h_fw,
                   const float* Wc_h_fw, const float* Wg_h_bw, const float* Wc_h_bw, int B, int T, void* stream);
/* same, for a forward that started from h0_fw / h0_bw [B][128] (NULL = zero state); dh0 [B][2][128] (or NULL)
 * receives d(loss)/d(initial state) per direction */
int taco_bigru_bwd_h0(float* dxp, const float* dOut, const float* out, const float* ACT, const float* Wg_h_fw,
                      const float* Wc_h_fw, const float* Wg_h_bw, const float* Wc_h_bw, const float* h0_fw,
                      const float* h0_bw, float* dh0, int B, int T, void* stream);
/* decoder step inputs of the Training / ScheduledOutputTraining helpers, time-major: Xin [T][B][80], sel [T][B] */
int taco_dec_inputs(float* Xin, uint8_t* sel, const float* mel, const float* y, const uint8_t* sample_mask, int B, int T,
                    int r, int sched, void* stream);

/* serial part of the attention-decoder backward (tacotron.py:46-105,136-138): see csrc/decoder_bwd.cu.
 * All tensors time-major ([T][B][n]) unless noted; B <= 32.                                               */
typedef struct taco_decoder_bwd_args {
    int32_t B, T, Tx, r;
    float   keep_scale;
    const float *W_a, *W_q, *W_out, *W_in, *W1, *W2, *v;      /* TF layouts (see taco_decoder_weights) */
    const float *Wg[3], *Wc[3];
    const float *dy_ext;                  /* [T][B][80r] gradient arriving at seq2seq_output            */
    const float *RU[3], *C[3], *H[3];     /* [T][B][512] gates, [T][B][256] candidates, states          */
    const float *align;                   /* [B][T][Tx]                                                 */
    const float *values, *keys;           /* [B][Tx][256]                                               */
    const float *PQ, *PN1, *PN2;          /* [T][B][256] y.W_q ; pre-net activations [T][B][256|128]    */
    const uint8_t* sel;                   /* [T][B] 1 = step input was the model's own previous output  */
    float *DATT, *DY, *DPQ;               /* out: pre-activation gradients per step                     */
    float *DSCORE;                        /* out: [B][T][Tx]                                            */
    float *DCTX, *DG[3], *DC[3], *DZ, *DPN2, *DPN1, *DX;
    float *workspace;                     /* taco_decoder_bwd_workspace_bytes                           */
    int32_t max_ctas;                     /* CTA budget (>= 32), 0 = what the device holds; the kernel runs on
                                             min(budget, capacity, 128) CTAs                                */
    const float *H0[3];                   /* [B][256] initial state of GRU i (h_i(-1)), or NULL = zero        */
    float *DH0;                           /* out: [3][B][256] d(loss)/d(h_i(-1)), or NULL = not wanted        */
    const float *dscore_add;              /* [B][T][Tx] added to the softmax backward's dscore of every step
                                             before it feeds dpq and DSCORE (taco_guided_attention's
                                             gradient), or NULL = nothing added, today's arithmetic        */
} taco_decoder_bwd_args;
size_t taco_decoder_bwd_workspace_bytes(void);
int    taco_decoder_bwd(const taco_decoder_bwd_args* a, void* stream);
/* dkeys[b][j][d] = sum_t DSCORE[b][t][j] v[d] (1-e^2); dv[d] += sum DSCORE e; e = tanh(keys + PQ[t][b]) */
int taco_attn_bwd_post(float* dkeys, float* dv, const float* DSCORE, const float* keys, const float* PQ, const float* v,
                       int B, int T, int Tx, void* stream);
/* (new; the reference has no such term) guided attention loss of Tachibana et al. 2017, "Efficiently Trainable
 * Text-to-Speech System Based on Deep Convolutional Networks with Guided Attention", arXiv:1710.08969, on the alignments
 * align [B][T][Tx] the forward saves.  With N_b = min(text_length[b], Tx) and T_b = speech_steps[b] (in [1, T]):
 *     W[b][t][j] = 1 - exp(-(j/N_b - t/T_b)^2 / (2 g^2))  for t < T_b and j < N_b, else 0
 *     loss[0]    = lam * sum_{b,t,j} align W                                   (a sum, like the two L1 losses)
 *     dscore[b][t][j] = lam * align[b][t][j] * (W[b][t][j] - s[b][t]),  s = sum_j align W   (0 outside the mask)
 * dscore is d(loss)/d(attention score): the input taco_decoder_bwd_args.dscore_add takes.  One warp per (b, t) row
 * forms W, s and dscore together; the loss is reduced from per-row partials in a fixed order (double accumulation), so
 * it is bit-identical run to run.  g > 0, lam >= 0, Tx <= 256; no host synchronisation.                          */
int taco_guided_attention(float* dscore, float* loss, const float* align, const int32_t* text_length,
                          const int32_t* speech_steps, int B, int T, int Tx, float g, float lam, float* partial_ws,
                          void* stream);
int taco_guided_attention_partial_count(int B, int T);   /* floats partial_ws must hold (one per row: B*T) */

/* tf.clip_by_global_norm(cap_grads) + tf.train.AdamOptimizer (tacotron.py:170-184; SURVEY A.12) on the flat
 * parameter / gradient buffers: out = sum x^2 (deterministic); g *= clip/max(sqrt(sumsq), clip);
 * m = b1 m + (1-b1) g; v = b2 v + (1-b2) g^2; p -= lr_t m/(sqrt(v)+eps), lr_t = lr sqrt(1-b2^t)/(1-b1^t).   */
/* ==========================================================================================
 * Spectrogram inversion (SURVEY section 8(f) rank 1): the fused steps of audio.griffinlim between the two
 * library FFTs of an iteration (reference audio.py:67-97; reshape_frames inverse audio.py:30-35; librosa
 * stft/istft conventions).  n = frames = 4r*(T/4), F = n_fft/2+1 bins, L = hop*(n-1) samples; complex tensors
 * are interleaved (re, im) fp32.  Semantics: tests/mirror_kernels.py gl_*.
 * ========================================================================================== */
/* mag[b,f,k] = exp(spec[b, t(f), c(f)*F+k]*scale + shift) (scale/shift may be NULL), full = mag*exp(2 pi i u):
 * reshape_frames(forward=False) + the driver's de-normalisation (test.py:64) + np.exp + the random phase (:81) */
int taco_gl_init(float* full_c64, float* mag, const float* spec, const float* phase_u, int B, int T, int n, int r, int F,
                 const float* scale, const float* shift, void* stream);
/* tail of librosa.istft: window, overlap-add, window-sum-square normalisation, centre trim: fr [B][n][n_fft] -> y [B][L] */
int taco_gl_ola(float* y, const float* fr, int B, int n, int hop, int n_fft, int win_length, void* stream);
/* head of librosa.stft: reflect padding, framing, hann window: y [B][L] -> frw [B][n][n_fft] */
int taco_gl_frame(float* frw, const float* y, int B, int n, int hop, int n_fft, int win_length, void* stream);
/* full = mag * rebuilt/|rebuilt|  (audio.py:84,87) over `count` complex elements */
int taco_gl_phase(float* full_c64, const float* mag, const float* rebuilt_c64, int64_t count, void* stream);
/* fast Griffin-Lim's phase update (Perraudin, Balazs & Sondergaard 2013; librosa >= 0.7's griffinlim):
 * full = mag * d/|d|, d = rebuilt - beta*prev, and mag + 0i where d == 0 (as taco_gl_phase does for rebuilt == 0), over
 * `count` complex elements.  prev is the previous iteration's rebuilt spectrum, beta = momentum / (1 + momentum) in
 * [0, 0.5]; beta = 0 gives taco_gl_phase's values.  Element-wise, so the padded and packed layouts both use it.     */
int taco_gl_phase_momentum(float* full_c64, const float* mag, const float* rebuilt_c64, const float* prev_c64, float beta,
                           int64_t count, void* stream);
/* De-emphasis, the inverse of preprocessing's pre-emphasis y[n] - coef*y[n-1]: in place, for each segment s in [0, S),
 * y[i] = x[i] + coef*y[i-1] for i in [start[s], start[s+1]) with zero state before start[s]
 * (scipy.signal.lfilter([1], [1, -coef], x) per segment).  start: device int64 [S+1], non-decreasing (the caller checks
 * it); segments may be empty, nothing at or past start[S] is read.  One launch, one CTA per segment walking it in tiles
 * with a block scan of the recurrence; deterministic.  S >= 0, 0 <= coef < 1.                                        */
int taco_de_emphasis(float* y, const int64_t* start, int S, float coef, void* stream);
/* the two transforms of a Griffin-Lim iteration (librosa.istft / librosa.stft inside audio.griffinlim, audio.py:84-86),
 * n_fft = 2048: X [rows][1025] complex (interleaved re, im) <-> x [rows][2048] real.  rfft is unnormalised, irfft scales
 * by 1/2048 and ignores the imaginary parts of the DC and Nyquist bins (numpy / cuFFT conventions).  Shared-memory
 * radix-2 Stockham transform, one CTA per row: no FFT library on the path.                                          */
int taco_rfft2048(float* X_c64, const float* x, int64_t rows, void* stream);
int taco_irfft2048(float* x, const float* X_c64, int64_t rows, void* stream);
/* Where each utterance's speech ends, for the opt-in tail trim of synthesis (tacotron_b200.audio.speech_frames).  The
 * training targets end in padding frames of log(0 + 1e-8) (preprocessing zero-pads the trimmed waveform,
 * features.cu feature_spec), so a trained model ends each utterance with frames far below its speech.
 * spec [B][T][F*r] is the post-net output in the decoder's layout, scale/shift [F*r] the optional de-normalisation
 * (both or neither, as in taco_gl_init).  Writes frames[b], the number of STFT frames to keep:
 *   - frame space is the one gl_init uses: n = 4r*(T/4) frames, frame f = 4r*q + 4c + l comes from decoder step
 *     t = 4q + l, column block c (reshape_frames(forward=False), audio.py:30-35);
 *   - log magnitude v[f,k] = spec[b, t, c*F + k]*scale + shift, as in gl_init;
 *   - log power e[f] = log sum_k exp(2 v[f,k]), a max-shifted float32 sum in a fixed reduction order;
 *   - E = max_f e[f]; frame f is voiced when e[f] >= E - top_db*ln(10)/10;
 *   - f* = the last voiced frame; frames[b] = 4r * clamp(ceil((f*+1) / 4r), k_min, T/4), k_min = ceil(5 / 4r)
 *     (the inversion's reflect padding needs at least 5 frames: hop*(n-1) > n_fft/2);
 *   - frames[b] = n when any e[f] or E is not finite.
 * Whole blocks of 4r frames are the outputs of decoder steps [0, frames[b]/r).  Two launches (one warp per frame, then
 * one CTA per utterance) and a stream-ordered scratch of B*n floats; no host synchronisation.
 * B >= 1, r >= 1, T >= 4, F >= 1, top_db finite and > 0.  Semantics: tests/mirror_kernels_trim.py speech_frames.     */
int taco_speech_frames(int* frames, const float* spec, int B, int T, int r, int F, const float* scale, const float* shift,
                       float top_db, void* stream);
/* Griffin-Lim over a packed batch (tacotron_b200.audio.invert_speech): utterance b owns rows [off[b], off[b+1]) of
 * mag / full / phase_u [N][F] and of the frame buffer [N][n_fft] (off int64 [B+1], off[0] = 0, N = off[B]), and its
 * L_b = hop*(n_b - 1) samples start at hop*(off[b] - b) of one flat y.  The per-element arithmetic is that of
 * taco_gl_init / taco_gl_ola / taco_gl_frame, so utterance b is bit-identical to those run on it alone; gl_ola clamps
 * its frames to n_b - 1 and gl_frame reflects at L_b.  One launch over the whole batch each (blockIdx.y = utterance);
 * max_frames (the largest n_b) sizes the grid.  Each n_b must lie in [5, 4r*(T/4)] (gl_init reads spec[b, :T]).
 * taco_rfft2048 / taco_irfft2048 / taco_gl_phase run unchanged on the N rows.  Semantics: tests/mirror_kernels_trim.py. */
int taco_gl_init_packed(float* full_c64, float* mag, const float* spec, const float* phase_u, const int64_t* off,
                        int B, int T, int r, int F, int max_frames, const float* scale, const float* shift, void* stream);
int taco_gl_ola_packed(float* y, const float* fr, const int64_t* off, int B, int max_frames, int hop, int n_fft,
                       int win_length, void* stream);
int taco_gl_frame_packed(float* frw, const float* y, const int64_t* off, int B, int max_frames, int hop, int n_fft,
                         int win_length, void* stream);
/* Where each utterance's speech starts and ends, for long-form synthesis (tacotron_b200.audio.speech_bounds): the frame
 * space, log power and voiced rule of taco_speech_frames, and writes bounds[b] = {f0, f1, frames}:
 *   - f0 = the first voiced frame, f1 = the last voiced frame + 1;
 *   - frames = exactly the value taco_speech_frames writes for frames[b] (Griffin-Lim's frame count);
 *   - {0, n, n} when any e[f] or E is not finite.
 * Two launches (taco_speech_frames' per-frame power kernel, then one CTA per utterance) and a stream-ordered scratch of
 * B*n floats; no host synchronisation.  Same argument rules as taco_speech_frames.
 * Semantics: tests/longform_oracle.py speech_bounds.                                                                     */
int taco_speech_bounds(int* bounds, const float* spec, int B, int T, int r, int F, const float* scale, const float* shift,
                       float top_db, void* stream);
/* Join synthesised pieces into one waveform (tacotron_b200.audio.join_speech): seg int64 [S][3], segment s =
 * {src_start, dst_start, len}, sets out[dst_start + i] = src[src_start + i] * w(i), i in [0, len), with
 *   - w(i) = min(1, c(i), c(len-1-i)), c(j) = 0.5 - 0.5 cos(pi (j + 0.5) / fade) for j < fade and 1 otherwise: a
 *     raised-cosine fade-in and fade-out of `fade` samples at every cut (evaluated as sin^2 in double, so the product is
 *     one rounding from the exact value);
 *   - samples of out that no segment covers are not written (the caller zero-fills out, so gaps are silence).
 * One launch (blockIdx.y = segment, x over samples); max_len (the largest len) sizes the grid.  The caller checks that
 * every segment lies inside src and out and that no two overlap in out; a segment outside [0, out_len) is skipped.
 * 1 <= S <= 65535, out_len >= 0, max_len >= 0, fade >= 1.  Semantics: tests/longform_oracle.py join_segments.          */
int taco_join_segments(float* out, int64_t out_len, const float* src, const int64_t* seg, int S, int max_len, int fade,
                       void* stream);

/* Input data format (SURVEY 8(f) rank 3): spectrograms are stored float16 (preprocess.py:179-180) and normalised in
 * that dtype (data_input.py:56-64) before the float32 cast (:38-39).  Bit-exact device version of those statements:
 * out[i][c] = f32( f16( f32( f16( f32(x) - f32(mean[c]) ) ) / std[c] ) ),  x [rows][W] float16, mean float16, std float32. */
int taco_normalize_f16(float* out, const void* x_f16, const void* mean_f16, const float* std_f32, int64_t rows, int W,
                       void* stream);

/* ==========================================================================================
 * Feature extraction (preprocess.py:168-208 / audio.py:38-65): WAV samples -> the float16 training arrays.  The
 * waveforms of a chunk are packed end to end (fp32) with int64 offsets; the transform between the two feature kernels is
 * taco_rfft2048.  Semantics: tests/mirror_kernels_features.py.
 * ========================================================================================== */
/* librosa.effects.trim (audio.py:42): one CTA per utterance b = samples [offsets[b], offsets[b+1]).  Frame f < 1 + len/hop
 * of the signal reflect-padded by frame_length/2 has mean-square energy e_f (fp64); it is non-silent when
 * 10 log10(max(1e-10, e_f)) - 10 log10(max(1e-10, max e)) > -top_db.  bounds[b] = {first*hop, min(len, (last+1)*hop)}
 * relative to offsets[b], {0, 0} if no frame is non-silent.  frame_length an even multiple of hop, at most 16 hops;
 * each utterance longer than frame_length/2.                                                                        */
int taco_trim_bounds(int* bounds, const float* y, const int64_t* offsets, int B, int frame_length, int hop, float top_db,
                     void* stream);
/* head of librosa.stft after trimming (audio.py:47-56): w_b = y[start[b] : start[b]+len[b]] zero-padded to max_len
 * (len[b] <= max_len), pre-emphasis e[0] = w[0], e[i] = w[i] - preemph*w[i-1] (fp32, two roundings), reflect padding by
 * n_fft/2, framing, hann window: frw [B][n_frames][n_fft], n_frames = 1 + max_len/hop.                                 */
int taco_feature_frames(float* frw, const float* y, const int64_t* start, const int* len, int B, int n_frames, int max_len,
                        int hop, int n_fft, int win_length, float preemph, void* stream);
/* audio.py:57-63 from X [B][n_frames][1025] complex (taco_rfft2048): stft = log(|X| + 1e-8), mel[m] = log(|sum_{k in
 * [mel_lo[m], mel_hi[m])} mel_basis[m][k] X[k]| + 1e-8) (mel_basis [n_mels][1025]; 0 <= lo <= hi <= 1025), scattered in
 * the reshape_frames(forward=True) layout: stft_out [B][4*(n_frames/4r)][1025 r], mel_out [B][..][n_mels r], float16
 * (out_f16 = 1) or float32.  Frames beyond 4r*(n_frames/4r) are not written.                                        */
int taco_feature_spec(void* stft_out, void* mel_out, int out_f16, const float* X_c64, const float* mel_basis, const int* mel_lo,
                      const int* mel_hi, int B, int n_frames, int r, int n_mels, void* stream);
/* the resampling of librosa.load(f, sr=sr) (audio.py:39) for files at another rate: librosa 0.6 resample(res_type=
 * 'kaiser_best') over resampy 0.2.2's loop, one ratio = sr_new / sr_orig per call.  Input b = in[in_off[b] : in_off[b+1]]
 * (n_in samples), output b = out[out_off[b] : out_off[b+1]] (librosa's n_fix = ceil(n_in*ratio) samples): the first
 * n_out = int(n_in*ratio) samples are resampy's, the rest zeros.  win_delta [nwin][2] float64 = {win, delta} of the
 * (ratio-scaled) 512-entries-per-crossing table, 16-byte aligned; step = int(min(1, ratio)*512); treg [treg_len] the
 * float64 time register (treg[t] = treg[t-1] + 1/ratio, summed in order), treg_len >= every n_out (an output sample the
 * register does not reach is written as NaN).  Float32 accumulation rounded after every tap, no fused multiply-add:
 * bit-identical to tests/mirror_kernels_resample.py.  B <= 65535.                                                   */
int taco_resample(float* out, const float* in, const int64_t* in_off, const int64_t* out_off, int B, const double* win_delta,
                  int nwin, int step, double ratio, const double* treg, int64_t treg_len, void* stream);

/* ==========================================================================================
 * Training summaries: tf.summary.histogram (models/tacotron.py:129,139,152) = TF 1.2's HistogramSummaryOp /
 * histogram::Histogram::Add over x [n] fp32 (16-byte aligned), reduced on the device.  limits [nlim] float64 = TF's default
 * bucket table (nlim = 1551: -DBL_MAX, the mirrored negatives, 0.0 at 775, the positives 1e-12 * 1.1^k by repeated
 * multiplication while < 1e20, DBL_MAX).  A finite value x goes to counts[upper_bound(limits, (double)x) - limits];
 * stats = {min, max, sum, sum of squares} of the widened finite values (min = DBL_MAX, max = -DBL_MAX when there are none);
 * NaN / Inf elements are counted in nonfinite[0], not binned.  Counts, min and max exact; sum and sum of squares from a
 * fixed grid and reduction order (bit-identical from run to run).  workspace: taco_histogram_workspace_bytes(), 16-byte
 * aligned.  Semantics: tests/mirror_kernels_summary.py.
 * ========================================================================================== */
size_t taco_histogram_workspace_bytes(void);
int    taco_histogram(const float* x, int64_t n, const double* limits, int nlim, void* workspace, int64_t* counts,
                      double* stats, int64_t* nonfinite, void* stream);

int taco_sumsq(const float* x, int64_t n, float* partial_ws, float* out, void* stream);
int taco_adam_step(float* p, const float* g, float* m, float* v, int64_t n, float lr_t, float b1, float b2, float eps,
                   float clip, const float* sumsq, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TACO_B200_H */
