// decoder.cu -- the whole autoregressive attention decoder as ONE persistent dataflow kernel (design v5).
//
// Reference: models/tacotron.py:46-105 (create_decoder) + :136-138 (dynamic_decode) over the
// TF-1.2 contrib.seq2seq / contrib.rnn classes (SURVEY.md A.5-A.10).  Per decoder step t:
//   P1  p1   = relu(x_last . W1 + b1) (*keep1)            x_last = last 80 of the 80r-wide input
//   P2  p2   = relu(p1 . W2 + b2) (*keep2)                 Tacotron.pre_net, tacotron.py:38-44,64-71
//   IN  z    = [p2, attn] . W_in + b_in                    InputProjectionWrapper
//   G_i [r,u]= sigmoid([x_i, h_i] . Wg_i + bg_i)           GRUCell x3 (MultiRNNCell), x_1 = z, x_i = h_{i-1}
//   C_i c    = tanh([x_i, r*h_i] . Wc_i + bc_i); h_i = u*h_i + (1-u)*c
//       s    = z + h_3                                     ResidualWrapper (around the 3-stack)
//   OUT y_t  = s . W_out + b_out                           OutputProjectionWrapper -> seq2seq_output
//   Q   q    = y_t . W_q                                   BahdanauAttention query layer (query = cell OUTPUT)
//   ATT e_j  = sum_d v_d tanh(keys_jd + q_d), j >= text_length masked; softmax; ctx = a . values
//   AL  attn = [y_t, ctx] . W_a                            AttentionWrapper attention_layer (no bias)
//   next input: InferenceHelper -> y_t ; TrainingHelper -> mel[:, t+1] ; ScheduledOutput -> per-row mix
//
// History: v1 grid barrier + FFMA -> v2 flag-in-data exchange -> v3 mma.sync 3xTF32 with 12 dependent slots per step,
// most of each slot spent waiting for / ingesting K=512 operands through L2.  v4 attacks the length of the dependent
// chain and what sits on it:
//
//   * 9 dependent slots per step instead of 12 (weight-only algebra at pack time, exact up to re-association):
//       IN  G1 C1 G2 C2 G3 C3  OQP  A|P2
//     OQP computes, from s(t) alone, y(t) (output), q(t) = s.(W_out W_q) + b_out W_q and the FIRST PRE-NET LAYER OF
//     THE NEXT STEP p1(t+1) = relu(s.(W_out[:,last 80] W1) + b_out[last 80] W1 + b1) (free-running rows); A|P2 runs
//     the attention on warps 0-3 and the second pre-net layer on warps 4-7 concurrently; IN takes y(t-1) through
//     s(t-1).(W_out W_a[:80r] W_in[128:]) so y never travels.  Teacher-forced rows take p1 from a separate
//     off-chain stage PM (mel . W1), selected per row by the consumer.
//   * v5: 8 dependent slots, G1 C1 G2 C2 G3 C3 OQP A|P2.  IN only produced z(t), which the chain needs through z . Wg1_x,
//     z . Wc1_x and the residual s = z + h3 alone: G1 multiplies [ctx(t-1) | p2(t)] and s(t-1) by the pack-time products
//     of IN's weights with Wg1_x and [Wc1_x | I] (fused_tail), into a gate tile and a [C1 x-half | z] tile; the second
//     tile stays in the CTA (cx_loc, z_loc), so C1 has no off-chain half and no stage publishes z.
//   * every K=512 contraction is split into the half that is on the dependent chain (x of the gates, r*h of the
//     candidate, ctx/p2 of the input projection) and the half whose operand has been known for a while (h(t-1), x,
//     s(t-1)).  The known half is multiplied in the shadow of the previous slot's L2 hop into the SAME accumulator
//     registers; only K=256 (16 KB of operand words per CTA) is ingested on the chain.
//   * on-chain weight slices are resident in shared memory (124 KB); the off-chain slices (and, when the keys/values
//     leave too little shared memory, further slices) are read every step from the packed buffer in global memory,
//     which stays in the 50 MB L2.  They are loaded one stage early, together with the off-chain operand words, so
//     they travel while the previous stage's epilogue runs (loaded at the start of their own stage, their L2 latency
//     made the off-chain half ~400 cycles longer than the on-chain operand's hop on an H100, so it sat on the chain).
//     Only the first stage of a step loads them in place.
//   * MMA orientation swapped: M = 16 weight columns of the CTA's slice, N = the 8 utterance rows of the CTA's row
//     group, so the 16-column gate stage has no zero-padded rows (half the MMAs of v3).
//   * attention: the four CTAs that share an utterance (blockIdx / 4) each score a quarter of the memory; partial softmax
//     statistics and partial contexts are exchanged as {value,tag} words through a small per-utterance region of the
//     workspace (L2), each CTA normalises and publishes 64 context columns and its own alignment slice: the consumer
//     ingests 256 context words per row instead of 4 x 256 partials + statistics.  A merging thread requests all of its
//     words (each quarter's adjacent {max, sum} pair with one 16-byte load, its four context partials) before it checks
//     any tag: one L2 round trip on the chain instead of twelve dependent ones.  (No thread-block cluster:
//     cudaOccupancyMaxActiveClusters reported 30 co-resident clusters of four such CTAs on the H100 80GB HBM3 this was
//     built on, fewer than the 32 this grid needs; the count depends on each die's GPC configuration.)
//     tanh(k+q) = 1 - 2/(e^{2k} e^{2q} + 1) with e^{2k} precomputed once and e^{2q} once per step: one MUFU per
//     element instead of two.
//   * attention window (opt-in, free-running decoding; decoder_kernel<.., WIN = true>): the score write masks positions
//     outside [p(t-1) - back, p(t-1) + ahead]; warp 4 publishes its quarter's lowest maximising position as one more
//     {value, tag} word after its partial context, and at the start of step t+1's attention thread 128 combines the
//     four (lowest quarter holding the utterance's max) beside the q(t+1) polls, so no new exchange sits on the chain
//     (the windowed step still measures ~0.3 us longer, DESIGN.md 3.4).  The off instantiation is the plain kernel,
//     instruction for instruction.
//   * end-of-text stop rule (opt-in, free-running decoding; decoder_kernel<.., WIN = true, STOP = true>): thread 128 of
//     each utterance's quarter-0 CTA counts the run of peaks >= stop_at and publishes one tagged status word per step;
//     a step later, lanes 0-7 of warp 5 of every CTA of the row group read the group's 8 words beside the q polls, and
//     all 32 CTAs leave at the top of the same step once every row has ended (TACO_DECODER_STOP_LAG, DESIGN.md 3.4).
//
// Unchanged from v3: grid = 32 co-resident CTAs per row group of 8 utterances (128 = 4 row groups when the device holds
// them), CTA (rg, cs) owns utterance rows 8rg..8rg+7 and the
// cs-th of 32 column slices of every dense stage; NO grid barrier: every exchanged activation is a 64-bit word
// {fp32 value, step tag} written with one st.b64 and read with polling 128-bit loads; 3xTF32 error-compensated
// tensor-core products (fp32-grade); GRU gate columns permuted so r,u of a hidden unit live in one CTA.
#include <stdlib.h>
#include "common.cuh"

namespace {

constexpr int NCTA = 128;
constexpr int NTHR = 512;      // 16 warps: 4 per SM sub-partition (the step is a chain of short dependent instruction sequences:
constexpr int NWARP = 16;      // with 2 warps per scheduler every fixed latency was exposed -- 'wait' was the top stall reason)
constexpr int RPG = 8;         // rows per row group
constexpr int NS = 32;         // column slices
constexpr int BPAD = 32;
constexpr int U = 256;         // decoder units
constexpr int AU = 256;        // attention units
constexpr int ENC = 256;       // memory depth
constexpr int MF = 80;
constexpr int KV_LD = 260;     // padded row stride of e^{2 keys} in smem
constexpr int PPITCH = 132;    // floats between the partial tiles of consecutive warps (128 + 4: cross-warp sums hit different banks)

// ---- weight segments (one K slab of one stage, per CTA column slice) ---------------------------------------------
//      The first GRU's gate and candidate products take the input projection z = [ctx | p2] . W_cpF + s(t-1) . W_sF +
//      b_inF folded in (see fused_tail): G1_* = the gates, Z1_* = [candidate x-half | z] of the same 8 units.
enum SegId {
    SG_G1_CP = 0, SG_Z1_CP, SG_G1_S, SG_Z1_S,
    SG_G_H0, SG_G_H1, SG_G_H2, SG_G_X1, SG_G_X2,
    SG_C_X1, SG_C_X2, SG_C_RH0, SG_C_RH1, SG_C_RH2,
    SG_Y, SG_QP, SG_PM, SG_P2, NSEG
};
// ---- exchange buffers: [4 row groups][nkt k-tiles][8 rows][8 words] of 64-bit {value, tag} words.  One k-tile of one
//      row group (512 B) is written by ONE producer CTA and read by one warp-wide 16-byte load: fully coalesced.
//      B_CP holds ctx (k-tiles 0..31) and p2 (k-tiles 32..47): the on-chain operand of the first GRU stage.
enum BufId { B_S = 0, B_CP, B_H0, B_H1, B_H2, B_RH0, B_RH1, B_RH2, B_Q, B_P1Y, B_P1M, NBUF };
__host__ __device__ inline int buf_nkt(int b) { return b == B_CP ? 48 : 32; }
// ---- stages (what "finish" does) --------------------------------------------------------------------------------
enum StageId { ST_G0 = 0, ST_G1, ST_G2, ST_C0, ST_C1, ST_C2, ST_PM, ST_OQP, ST_AP2, ST_NONE };
// bias rows in smem ([row][16]); BR_G0 / BR_Z1 hold the step t > 0 biases of the first stage, BR_G0T / BR_Z1T those of t = 0
enum BiasRow { BR_G0 = 0, BR_G1, BR_G2, BR_G0T, BR_Z1, BR_Z1T, BR_C0, BR_C1, BR_C2, BR_Y, BR_QP, BR_PM, BR_P2, NBR };
// item kinds: fragment width / tiles / k-tile slots per warp
enum ItemKind { IK_F2 = 0, IK_F4, IK_F4X2, IK_G1, IK_PM, IK_AP2 };   // 8 / 16 / 2x16 columns x 2 k-tile slots; G1: 2x16 x 3 slots
// output slots of the per-CTA output-offset table
enum OutId { O_RH0 = 0, O_RH1, O_RH2, O_H0, O_H1, O_H2, O_S, O_Q, O_P1Y, O_P1M, O_P2, NOUT };

struct SegDesc {
    int K;             // contraction length (multiple of 8)
    int FL;            // floats per lane and k-tile: 4 = 16 weight columns, 2 = 8 weight columns
    int nw;            // warps that split K (16, or 8 for the P2 stage)
    int kpw;           // k-tile slots per warp (2, 3 or 4; padded with zeros)
    int smem_off;      // float offset inside the resident smem region, or -1: read from the packed buffer (L2)
    int slice_floats;  // nw * kpw * 32 * FL
    int64_t g_off;     // float offset of slice 0 in the packed buffer
};

struct Item {          // one stage of the per-step program: [off-chain half] + on-chain half of one contraction, then finish
    int kind;          // ItemKind
    int stage;         // StageId finished after the on-chain half
    int pre_seg, pre_src, pre_tagd, pre_skip0;   // off-chain half: weight segment (-1: none), operand buffer, tag = t + tagd,
                                                 // 1 = operand does not exist at t == 0 (zero initial state)
    int on_seg, on_seg2, on_src, on_tagd, on_s0; // on-chain half; seg2 >= 0: second 16-column tile sharing the operand (OQP);
                                                 // on_s0 = leading k-tile slots that do not exist at t == 0
};

constexpr int MAX_ITEMS = 20;

struct DecParams {
    SegDesc seg[NSEG];
    Item items[MAX_ITEMS];
    int n_items;
    int64_t buf[NBUF];           // word offsets of the exchange buffers
    int64_t att_off;             // word offset of the attention exchange region
    int64_t peak_off;            // word offset of the attention window's peak words
    int64_t stop_off;            // word offset of the stop rule's status words (after the initial-state terms)
    int64_t trace_off;
    taco_decoder_args a;
    const float *gru_bg[3], *gru_bc[3], *out_b, *pre_b1, *pre_b2, *att_v;
    const float *b_qF, *b_p1F;             // fused biases (packed tail)
    const float *b_g1F, *b_g1F0, *b_z1F, *b_z1F0;
    const float *init_z, *init_zg, *init_g;   // step-0 terms of a non-zero initial state (workspace tail), or NULL, with
                                              // iz = att0 . W_in[128:]:  [iz . Wc1_x | iz] [32][512],  iz . Wg1_x [32][512],
                                              // h0_i . Wg_i[256:] [3][32][512]
    int OUT, NCY, Tq;
    int smem_kv_off, smem_res_off, smem_total_floats;
};

// global column computed by weight-column m (0..15) of slice cs for a segment (-1 = padding)
__host__ __device__ inline int seg_col(int sg, int cs, int m, int NCY, int OUT) {
    if (sg <= SG_G_X2) return (m < 8) ? (8 * cs + m) : (U + 8 * cs + (m - 8));     // r | u (Z1: candidate | z) of units 8cs..8cs+7
    if (sg == SG_QP) return (m < 8) ? (8 * cs + m) : (AU + 8 * cs + (m - 8));                       // q | p1' (source = [W_qF | W_p1F])
    if (sg == SG_Y) { const int c = cs * NCY + m; return (m < NCY && c < OUT) ? c : -1; }
    if (sg == SG_P2) return (m < 4) ? (4 * cs + m) : -1;
    return (m < 8) ? (8 * cs + m) : -1;
}

// physical position of logical column k inside an exchange buffer row: within each group of 8,
// k and k+4 are adjacent so that one 16-byte load yields the (b0, b1) pair of an MMA B fragment.
__host__ __device__ inline int perm8(int k) {
    const int kk = k & 7;
    return (k & ~7) | ((kk < 4) ? 2 * kk : 2 * (kk - 4) + 1);
}

// ---------------------------------------------------------------------------------------------
// LL words: {value, tag}
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void ll_store(uint64_t* p, float v, uint32_t tag) {
    const uint64_t w = (uint64_t)__float_as_uint(v) | ((uint64_t)tag << 32);
    asm volatile("st.relaxed.gpu.global.b64 [%0], %1;" ::"l"(p), "l"(w) : "memory");
}
// polling load: ld.volatile always observes L2 (scripts/ubench/latency.cu times it against ld.relaxed.gpu).
__device__ __forceinline__ ulonglong2 ll_load2(const uint64_t* p) {
    ulonglong2 v;
    asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ bool ll_ok(const ulonglong2& v, uint32_t tag) {
    return (((uint32_t)(v.x >> 32) ^ tag) | ((uint32_t)(v.y >> 32) ^ tag)) == 0u;
}
// Spin until both words carry `tag`; bounded so that a protocol bug traps instead of hanging the GPU.
__device__ __forceinline__ void ll_spin(ulonglong2& v, const uint64_t* p, uint32_t tag) {
    uint32_t spins = 0;
    while (!ll_ok(v, tag)) {
        if (++spins > (1u << 24)) __trap();
        v = ll_load2(p);
    }
}
__device__ __forceinline__ float2 ll_wait2(const uint64_t* p, uint32_t tag) {
    ulonglong2 v = ll_load2(p);
    ll_spin(v, p, tag);
    return make_float2(__uint_as_float((uint32_t)v.x), __uint_as_float((uint32_t)v.y));
}
// one {value, tag} word (the attention exchange between the four CTAs of an utterance).  The first load is issued apart
// from the tag check so that a thread can have all the words it needs in flight before it waits for any of them.
__device__ __forceinline__ uint64_t ll_load1(const uint64_t* p) {
    uint64_t v;
    asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float ll_spin1(uint64_t& v, const uint64_t* p, uint32_t tag) {
    uint32_t spins = 0;
    while ((uint32_t)(v >> 32) != tag) {
        if (++spins > (1u << 24)) __trap();
        v = ll_load1(p);
    }
    return __uint_as_float((uint32_t)v);
}
__device__ __forceinline__ float rcp_fast(float x) {       // one MUFU.RCP (<= 1 ulp); rcp(+inf) = 0
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// e^{2x} with the argument clamped to [-60, 60] (|x| > 20.79) so that products of two such factors stay finite.  Exact
// while neither the key nor the query component is clamped.  Saturation is a property of k + q, not of k or q: past the
// clamp e^{2k} e^{2q} no longer gives tanh(k + q) (k = 25, q = -24 would give tanh = 0 where tanh(1) = 0.76), so a step
// whose keys or query reach the clamp is scored with tanhf_acc(k + q) instead (attention(), scores_direct).
__device__ __forceinline__ float exp2x(float x) { return exp2f(fminf(fmaxf(x * 2.885390082f, -60.f), 60.f)); }
__device__ __forceinline__ bool exp2x_clamps(float x) { return fabsf(x * 2.885390082f) > 60.f; }
// bar.sync of `n` threads on barrier `id` that also returns whether any of them passed v = true
__device__ __forceinline__ bool named_bar_or(int id, int n, bool v) {
    int r;
    asm volatile("{\n\t.reg .pred p, q;\n\tsetp.ne.s32 q, %1, 0;\n\tbar.red.or.pred p, %2, %3, q;\n\tselp.s32 %0, 1, 0, p;\n\t}"
                 : "=r"(r) : "r"((int)v), "r"(id), "r"(n) : "memory");
    return r != 0;
}
__device__ __forceinline__ void named_bar(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// Scores of one attention step in the direct form e_j = sum_d v_d tanhf_acc(k_jd + q_d), for a step where exp2x clamps,
// over the same warp / lane / butterfly layout as the product form in attention().  keys = this utterance's [Tx][256]
// keys, qw = its q(t) words in the exchange buffer (k-tile = 8 depths, pairs (p, p + 4) adjacent), positions jg = j0 + j
// outside [lo, hi] are masked.  Out of line: the rare path costs the common one no registers.
__device__ __noinline__ void scores_direct(float* e_s, const float* v_s, const float* keys, const uint64_t* qw, uint32_t tag,
                                           int j0, int Tq, int Tx, int lo, int hi, int warp, int lane) {
    float q[8], vv[8];
#pragma unroll
    for (int p = 0; p < 4; ++p) { const float2 qq = ll_wait2(qw + lane * 64 + 2 * p, tag); q[p] = qq.x; q[p + 4] = qq.y; }
#pragma unroll
    for (int i = 0; i < 8; ++i) vv[i] = v_s[8 * lane + i];
    for (int jb = 0; jb < Tq; jb += 32) {
        float a4[4];
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
            const int j = jb + warp + 8 * jj, jg = j0 + j;
            float a = 0.f;
            if (j < Tq) {                               // keys past Tx are zero, as in e^{2 keys}
#pragma unroll
                for (int i = 0; i < 8; ++i)
                    a = fmaf(vv[i], tanhf_acc((jg < Tx ? __ldg(keys + (int64_t)jg * 256 + 8 * lane + i) : 0.f) + q[i]), a);
            }
            a4[jj] = a;
        }
        float b2[2], b1;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const float send = (lane & 16) ? a4[k] : a4[k + 2];
            const float keep = (lane & 16) ? a4[k + 2] : a4[k];
            b2[k] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
        }
        {
            const float send = (lane & 8) ? b2[0] : b2[1];
            const float keep = (lane & 8) ? b2[1] : b2[0];
            b1 = keep + __shfl_xor_sync(0xffffffffu, send, 8);
        }
        b1 += __shfl_xor_sync(0xffffffffu, b1, 4);
        b1 += __shfl_xor_sync(0xffffffffu, b1, 2);
        b1 += __shfl_xor_sync(0xffffffffu, b1, 1);
        const int jj = ((lane >> 4) & 1) * 2 + ((lane >> 3) & 1);
        const int j = jb + warp + 8 * jj;
        if ((lane & 7) == 0 && j < Tq) e_s[j] = (j0 + j >= lo && j0 + j <= hi) ? b1 : -INFINITY;
    }
}

// ---------------------------------------------------------------------------------------------
// 3xTF32 tensor-core contraction pieces
// ---------------------------------------------------------------------------------------------
// x = hi + lo with hi = the TF32-representable head (low 13 mantissa bits cleared) and lo = the exact
// remainder (the tensor core ignores lo's own low 13 bits: <= 2^-21 |x| dropped).
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
    hi = __float_as_uint(x) & 0xffffe000u;
    lo = __float_as_uint(x - __uint_as_float(hi));
}
// D[16 weight columns x 8 utterance rows] += A[16x8] . B[8x8]
__device__ __forceinline__ void mma_tf32(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
// one k-tile: operand pair (x[row g][8kt+tg], x[row g][8kt+tg+4]) against one weight tile.
//   FL = 4: w = (W[k][m=g], W[k][m=g+8], W[k+4][m=g], W[k+4][m=g+8]);  FL = 2: w = (W[k][m=g], W[k+4][m=g]), rows 8..15 zero.
// The three 3xTF32 products go to three independent accumulators (no serialisation on the accumulator latency).
template <int FL>
__device__ __forceinline__ void ktile_mma(float (&acc)[3][4], uint32_t bh0, uint32_t bl0, uint32_t bh1, uint32_t bl1, const float* w) {
    uint32_t ah[4], al[4];
    if constexpr (FL == 4) {
#pragma unroll
        for (int i = 0; i < 4; ++i) split_tf32(w[i], ah[i], al[i]);
    } else {
        split_tf32(w[0], ah[0], al[0]);
        split_tf32(w[1], ah[2], al[2]);
        ah[1] = al[1] = ah[3] = al[3] = 0u;
    }
    mma_tf32(acc[0], al[0], al[1], al[2], al[3], bh0, bh1);
    mma_tf32(acc[1], ah[0], ah[1], ah[2], ah[3], bl0, bl1);
    mma_tf32(acc[2], ah[0], ah[1], ah[2], ah[3], bh0, bh1);
}

// ---- operand ingest + multiply of one item -------------------------------------------------------------------------
// Slot i of warp-index `widx` (of `nw` warps splitting K) covers k-tile widx + nw*i; its 8 rows x 8 words sit at
// p0 + i*nw*64 (p0 already contains this lane's g*8 + 2*tg).  NS_ = slots per call (2, 3 or 4); s0 = first live slot.
template <int NS_>
__device__ __forceinline__ void issue_loads(ulonglong2 (&v)[4], const uint64_t* p0, int nkt, int widx, int nw, int s0) {
#pragma unroll
    for (int i = 0; i < NS_; ++i)
        if (i >= s0 && widx + nw * i < nkt) v[i] = ll_load2(p0 + (size_t)i * nw * 64);
}
// weight word: bit 31 clear: float offset of the segment in the resident smem region; bit 31 set: float offset of this
// CTA's slice in the packed buffer (global memory, L2-resident).  Both hold the slice in the same [warp][slot][lane][FL]
// order.  wslot = index of the first fragment slot used by this call in the segment's [warp][slot] block.
__device__ __forceinline__ const float* weight_ptr(uint32_t ww, const float* res_s, const float* packed) {
    return (ww & 0x80000000u) ? packed + (ww & 0x7fffffffu) : res_s + ww;
}
__device__ __forceinline__ uint32_t seg_word(const SegDesc& d, int cs) {
    return d.smem_off >= 0 ? (uint32_t)d.smem_off : (0x80000000u | (uint32_t)(d.g_off + (int64_t)cs * d.slice_floats));
}
// weight fragments of one call -> w[(mt * NS_ + i) * FL ..] (tile mt, slot i); w may be longer than MT * NS_ * FL
template <int FL, int MT, int NS_, int N>
__device__ __forceinline__ void load_weights(float (&w)[N], uint32_t w1, uint32_t w2, int wslot, const float* res_s, const float* packed, int lane) {
    static_assert(N >= MT * NS_ * FL, "weight fragment array too short");
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
        const float* wp = weight_ptr(mt ? w2 : w1, res_s, packed) + ((size_t)wslot * 32 + lane) * FL;
        float* wm = w + mt * NS_ * FL;
#pragma unroll
        for (int i = 0; i < NS_; ++i) {
            if constexpr (FL == 4) { const float4 t = *reinterpret_cast<const float4*>(wp + (size_t)i * 32 * FL); wm[4 * i] = t.x; wm[4 * i + 1] = t.y; wm[4 * i + 2] = t.z; wm[4 * i + 3] = t.w; }
            else                   { const float2 t = *reinterpret_cast<const float2*>(wp + (size_t)i * 32 * FL); wm[2 * i] = t.x; wm[2 * i + 1] = t.y; }
        }
    }
}
// wait for the operand words v (loads already in flight) and multiply them into acc with weight fragments w (load_weights order)
// TR: ck = thread 0's stage record (or NULL); wk = this warp's stamp of its last on-chain word (lane 0, or NULL)
template <int FL, int MT, int NS_, bool TR, int N>
__device__ __forceinline__ void multiply(float (&acc)[2][3][4], ulonglong2 (&v)[4], const float (&w)[N], const uint64_t* p0, int nkt, int widx,
                                         int nw, int s0, uint32_t tag, long long* ck, long long* wk = nullptr) {
    if (TR && ck) ck[1] = clock64();
    // three-slot G1 call (re-polling inside the loop below spills there): slot 1's word, stale when its load was issued
    // before G1's off-chain halves, is requested again once, beside slot 0's first re-poll
    if (NS_ == 3 && s0 <= 1 && widx + nw < nkt && !ll_ok(v[1], tag)) v[1] = ll_load2(p0 + (size_t)nw * 64);
#pragma unroll
    for (int i = 0; i < NS_; ++i) {
        if (i >= s0 && widx + nw * i < nkt) {          // warp-uniform
            // two-slot calls: every poll of slot 0 also re-polls slot 1 while its word is stale, so that both are in flight
            // together and slot 1's word is seen within the L2 round trip that finds slot 0's, not one round trip after it
            // (its first load was issued before the producers published)
            uint32_t spins = 0;
            while (!ll_ok(v[i], tag)) {
                if (++spins > (1u << 24)) __trap();
                v[i] = ll_load2(p0 + (size_t)i * nw * 64);
                if (NS_ == 2 && i == 0 && widx + nw < nkt && !ll_ok(v[1], tag)) v[1] = ll_load2(p0 + (size_t)nw * 64);
            }
            uint32_t bh0, bl0, bh1, bl1;
            split_tf32(__uint_as_float((uint32_t)v[i].x), bh0, bl0);
            split_tf32(__uint_as_float((uint32_t)v[i].y), bh1, bl1);
            __syncwarp();                               // lanes arrive from divergent polling loops
            if (TR && wk) *wk = clock64();
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) ktile_mma<FL>(acc[mt], bh0, bl0, bh1, bl1, &w[(mt * NS_ + i) * FL]);
        }
    }
    if (TR && ck) ck[2] = clock64();
}
template <int FL, int MT, int NS_, bool TR>
__device__ __forceinline__ void consume(float (&acc)[2][3][4], ulonglong2 (&v)[4], const uint64_t* p0, int nkt, int widx, int nw, int s0,
                                        uint32_t tag, uint32_t w1, uint32_t w2, int wslot, const float* res_s, const float* packed,
                                        int lane, long long* ck, long long* wk = nullptr) {
    float w[MT * NS_ * FL];
    __syncwarp();
    load_weights<FL, MT, NS_>(w, w1, w2, wslot, res_s, packed, lane);
    multiply<FL, MT, NS_, TR>(acc, v, w, p0, nkt, widx, nw, s0, tag, ck, wk);
}

struct ItemRec { uint32_t flags, pre_base; int pre_tagd; uint32_t pre_w; uint32_t on_base; int on_tagd; uint32_t on_w1, on_w2; int on_nkt;
                 uint32_t s_base, s_w1, s_w2; };   // 48 bytes, in smem
// flags: kind | stage << 8 | has_pre << 16 | pre_skip0 << 17 | on_s0 << 20
// s_*: the second off-chain operand of the G1 item, s(t-1), and its two weight tiles (SG_G1_S, SG_Z1_S)

// TR: per-stage clock64 trace of CTA 0 (thread 0) and, per warp, of CTA 0 and CTA 48 (scripts/dec_time.py); the
// production instantiation has none of it.
// WIN: attention window (taco_decoder_args win_back / win_ahead, free-running decoding only): the scores outside
// [p(t-1) - back, p(t-1) + ahead] are masked and each step's peak p(t) is found; without it the kernel is the plain one.
// STOP (implies WIN): the end-of-text stop rule (taco_decoder_args stop_at / stop_hold / end_step): each row group
// leaves the step loop once every row of it has ended (see stop_poll).
template <bool TR, bool WIN, bool STOP>
__global__ void __launch_bounds__(NTHR, 1) decoder_kernel(const __grid_constant__ DecParams P) {
    static_assert(WIN || !STOP, "the stop rule needs the windowed kernel's peaks");
    extern __shared__ __align__(16) float smem[];
    // smem map (floats): [0,16) reserved | part 6400 | part2 512 | loc 384 | bias 256 | att 704 | itab 256 | kv | weights
    float* part_s = smem + 16;                                    // [3 buffers][16 warps][PPITCH]: two alternate, the third is the
                                                                  // 2nd tile of OQP and G1
    float* part2_s = part_s + 6400;                               // [8 warps][64]   (P2, warps 8-15)
    float* loc_s = part2_s + 512;                                 // h_loc[3][64] | u_loc[64] | z_loc[64] | cx_loc[64]
    float* bias_s = loc_s + 384;                                  // [NBR][16]
    float* att_s = bias_s + 256;                                  // eq[256] | v[256] | e[64] | p[64] | misc[64]
                                                                  // (misc: V0 | p(t-1) of the window | a key of this
                                                                  // CTA's slice reaches exp2x's clamp | stop rule: run
                                                                  // of peaks >= stop_at | end step (0: running) |
                                                                  // step to leave at | stop_at)
    ItemRec* itab = reinterpret_cast<ItemRec*>(att_s + 704);                 // [MAX_ITEMS] resolved stage records (20 x 12 words)
    uint32_t* otab = reinterpret_cast<uint32_t*>(itab + MAX_ITEMS);          // [NOUT] output word offsets of this CTA
    float* ek_s = smem + P.smem_kv_off;
    float* vals_s = ek_s + P.Tq * KV_LD;
    float* res_s = smem + P.smem_res_off;
    float* h_loc = loc_s;             // [3][8 cols][8 rows]
    float* u_loc = loc_s + 192;
    float* z_loc = loc_s + 256;       // z(t): the residual term of s = z + h3
    float* cx_loc = loc_s + 320;      // z(t) . Wc1_x + its bias terms: the x-half of the first candidate, formed by G1
    float* eq_s = att_s;
    float* v_s = att_s + 256;
    float* e_s = att_s + 512;
    float* p_s = att_s + 576;
    float* misc_s = att_s + 640;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, tg = lane & 3;            // MMA fragment coordinates
    const int cta = blockIdx.x;
    // dense stages: row group = the 32 consecutive CTAs that also run the attention of those 8 utterances, so the four
    // row groups are INDEPENDENT 32-CTA machines on (mostly) neighbouring SMs: no exchange crosses a group.  A launch runs
    // gridDim.x / 32 of them (as many as the CTA budget allows, up to 4) over a prefix of the workspace.
    const int rg = cta >> 5, cs = cta & 31;
    const int arow = cta >> 2;                          // attention: utterance, quarter aq of its memory
    const uint32_t aq = (uint32_t)(cta & 3);
    const taco_decoder_args& A = P.a;
    uint64_t* ws = reinterpret_cast<uint64_t*>(A.workspace);
    const int B = A.B, T = A.T, OUT = P.OUT, Tq = P.Tq, Tx = A.Tx, NCY = P.NCY;
    const int RS = A.row_stride, R0 = A.row0;          // [T][B]-major tensors: row r of this launch is full-batch row R0 + r
    const int row0 = rg * RPG;
    const int myrow = row0 + g;                        // the utterance row this lane's B fragments belong to
    const int lane_w = g * 8 + 2 * tg;                  // this lane's word offset inside a k-tile block

    for (int i = tid; i < 384; i += NTHR) {                        // initial GRU states: h0 rows, or zero (cell.zero_state)
        float hv = 0.f;
        if (i < 192 && A.h0 && row0 + (i & 7) < B)                 // h_loc[gi][col][row]: unit 8cs + col of row (i & 7)
            hv = __ldg(A.h0 + ((int64_t)(i >> 6) * RS + R0 + row0 + (i & 7)) * U + 8 * cs + ((i >> 3) & 7));
        loc_s[i] = hv;
    }
    // biases of this CTA's columns -> smem
    if (tid < NBR * 16) {
        const int br = tid >> 4, m = tid & 15;
        float bv = 0.f;
        int col; const float* bp = nullptr;
        switch (br) {
            case BR_G0:  col = seg_col(SG_G1_CP, cs, m, NCY, OUT); bp = P.b_g1F; break;
            case BR_G0T: col = seg_col(SG_G1_CP, cs, m, NCY, OUT); bp = P.b_g1F0; break;
            case BR_Z1:  col = seg_col(SG_Z1_CP, cs, m, NCY, OUT); bp = P.b_z1F; break;
            case BR_Z1T: col = seg_col(SG_Z1_CP, cs, m, NCY, OUT); bp = P.b_z1F0; break;
            case BR_G1: case BR_G2: col = seg_col(SG_G_X1, cs, m, NCY, OUT); bp = P.gru_bg[br - BR_G0]; break;
            case BR_C0: case BR_C1: case BR_C2: col = seg_col(SG_C_X1, cs, m, NCY, OUT); bp = P.gru_bc[br - BR_C0]; break;
            case BR_Y:   col = seg_col(SG_Y, cs, m, NCY, OUT); bp = P.out_b; break;
            case BR_QP:  col = (m < 8) ? 8 * cs + m : 8 * cs + (m - 8); bp = (m < 8) ? P.b_qF : P.b_p1F; break;
            case BR_PM:  col = seg_col(SG_PM, cs, m, NCY, OUT); bp = P.pre_b1; break;
            default:     col = seg_col(SG_P2, cs, m, NCY, OUT); bp = P.pre_b2; break;
        }
        if (bp && col >= 0) bv = __ldg(bp + col);
        bias_s[tid] = bv;
    }
    // resolved item records / output offsets (everything the per-item code would otherwise fetch through dependent
    // constant-bank loads: ~300 cycles per item in the first v4 trace)
    if (tid < P.n_items) {
        const Item& it = P.items[tid];
        ItemRec r;
        memset(&r, 0, sizeof(r));
        auto wword = [&](int sg) { return seg_word(P.seg[sg], cs); };
        r.flags = (uint32_t)it.kind | ((uint32_t)it.stage << 8) | ((it.pre_seg >= 0 ? 1u : 0u) << 16) | ((uint32_t)it.pre_skip0 << 17) | ((uint32_t)it.on_s0 << 20);
        if (it.pre_seg >= 0) {
            r.pre_base = (uint32_t)(P.buf[it.pre_src] + (int64_t)rg * buf_nkt(it.pre_src) * 64);
            r.pre_tagd = it.pre_tagd; r.pre_w = wword(it.pre_seg);
        }
        if (it.on_seg >= 0) {
            r.on_base = (uint32_t)(P.buf[it.on_src] + (int64_t)rg * buf_nkt(it.on_src) * 64);
            r.on_tagd = it.on_tagd; r.on_w1 = wword(it.on_seg); r.on_w2 = it.on_seg2 >= 0 ? wword(it.on_seg2) : 0u;
            r.on_nkt = P.seg[it.on_seg].K >> 3;
        }
        if (it.kind == IK_G1) {
            r.s_base = (uint32_t)(P.buf[B_S] + (int64_t)rg * buf_nkt(B_S) * 64);
            r.s_w1 = wword(SG_G1_S); r.s_w2 = wword(SG_Z1_S);
        }
        itab[tid] = r;
    }
    if (tid < NOUT) {
        const int bmap[NOUT] = {B_RH0, B_RH1, B_RH2, B_H0, B_H1, B_H2, B_S, B_Q, B_P1Y, B_P1M, B_CP};
        const int b = bmap[tid];
        uint32_t o = (uint32_t)(P.buf[b] + (int64_t)rg * buf_nkt(b) * 64);
        if (tid == O_P2) o += (uint32_t)((32 + (cs >> 1)) * 64 + 0);     // p2 columns 4cs..4cs+3 live in k-tile 32 + cs/2 of B_CP
        else o += (uint32_t)(cs * 64);                                    // this CTA's 8 columns are k-tile cs
        otab[tid] = o;
    }
    __syncthreads();
    const float* packed = A.packed;

    // ---- one-time preload of the shared-memory-resident weight slices (coalesced copies) ----
    for (int sg = 0; sg < NSEG; ++sg) {
        const SegDesc& d = P.seg[sg];
        if (d.smem_off >= 0) {
            const float4* s4 = reinterpret_cast<const float4*>(A.packed + d.g_off + (int64_t)cs * d.slice_floats);
            float4* d4 = reinterpret_cast<float4*>(res_s + d.smem_off);
            for (int i = tid; i < d.slice_floats / 4; i += NTHR) d4[i] = __ldg(s4 + i);
        }
    }
    // e^{2 keys} / values slice of (arow, aq) -> smem (padded rows), zero for utterances >= B and positions >= Tx
    int kclamp = 0;                                     // a key of this slice reaches exp2x's clamp
    for (int i = tid; i < Tq * (ENC / 4); i += NTHR) {
        const int j = i / (ENC / 4), d4 = (i % (ENC / 4)) * 4;
        float4 kk = make_float4(0, 0, 0, 0), vv = kk;
        if (arow < B && (int)aq * Tq + j < Tx) {
            const int64_t gi = ((int64_t)arow * Tx + aq * Tq + j) * ENC + d4;
            kk = __ldg(reinterpret_cast<const float4*>(A.keys + gi));
            vv = __ldg(reinterpret_cast<const float4*>(A.values + gi));
        }
        kclamp |= exp2x_clamps(kk.x) | exp2x_clamps(kk.y) | exp2x_clamps(kk.z) | exp2x_clamps(kk.w);
        kk.x = exp2x(kk.x); kk.y = exp2x(kk.y); kk.z = exp2x(kk.z); kk.w = exp2x(kk.w);   // tanh(k+q) = 1 - 2/(e^{2k} e^{2q} + 1)
        *reinterpret_cast<float4*>(ek_s + j * KV_LD + d4) = kk;
        *reinterpret_cast<float4*>(vals_s + j * ENC + d4) = vv;
    }
    for (int i = tid; i < AU; i += NTHR) v_s[i] = __ldg(P.att_v + i);
    const int my_len = (arow < B) ? A.text_length[arow] : 0;
    kclamp = __syncthreads_or(kclamp);
    if (warp == 0) {                                    // V0 = sum_d v_d  (e_j = V0 - 2 sum_d v_d / (E_jd + 1))
        float sv = 0.f;
        for (int i = lane; i < AU; i += 32) sv += v_s[i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sv += __shfl_xor_sync(0xffffffffu, sv, o);
        if (lane == 0) { misc_s[0] = sv; misc_s[2] = kclamp ? 1.f : 0.f; }
        if (STOP && lane == 0) {                        // stop rule state (misc_i[3..6])
            int* mi = reinterpret_cast<int*>(misc_s);
            mi[3] = 0; mi[4] = 0; mi[5] = T;
            mi[6] = arow < B ? A.stop_at[arow] : 0;
        }
    }
    __syncthreads();

    float acc[2][3][4];
#pragma unroll
    for (int a0 = 0; a0 < 2; ++a0)
#pragma unroll
        for (int a1 = 0; a1 < 3; ++a1)
#pragma unroll
            for (int a2 = 0; a2 < 4; ++a2) acc[a0][a1][a2] = 0.f;
    ulonglong2 v[4];                                    // operand words in flight

    int par = 0;                                        // parity of the partial-tile buffer
    const bool tracer = (cta == 0 && tid == 0 && A.step_ns != nullptr);
    int64_t trace_i = 0;
    long long* cktr = nullptr;                          // per-item clock64 trace (CTA 0, thread 0, steps 10..13)
    // per-warp stage records of CTA 0 and of CTA 48 (another row group), steps 10..12: [0, 16) last on-chain word seen,
    // [16, 32) stage barrier reached, [32, 48) barrier passed, [48, 64) epilogue done; wtr = lane 0's word of its warp
    const int trw = (TR && A.step_ns != nullptr) ? (cta == 0 ? 0 : cta == 48 ? 1 : -1) : -1;
    long long* wtr = nullptr;

    // =========================================================================================================
    // finish a stage: per-warp partial tiles -> smem, cross-warp sum, epilogue (one thread per output)
    // =========================================================================================================
    auto store_partials = [&](float* part, float* part_b, int MT, bool full16) {
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            if (mt < MT) {
                float* pw = (mt ? part_b : part) + warp * PPITCH;
                *reinterpret_cast<float2*>(pw + g * 8 + 2 * tg) =
                    make_float2((acc[mt][0][0] + acc[mt][1][0]) + acc[mt][2][0], (acc[mt][0][1] + acc[mt][1][1]) + acc[mt][2][1]);
                if (full16)
                    *reinterpret_cast<float2*>(pw + (g + 8) * 8 + 2 * tg) =
                        make_float2((acc[mt][0][2] + acc[mt][1][2]) + acc[mt][2][2], (acc[mt][0][3] + acc[mt][1][3]) + acc[mt][2][3]);
            }
        }
#pragma unroll
        for (int a0 = 0; a0 < 2; ++a0)
#pragma unroll
            for (int a1 = 0; a1 < 3; ++a1)
#pragma unroll
                for (int a2 = 0; a2 < 4; ++a2) acc[a0][a1][a2] = 0.f;
    };
    // cross-warp sum of one output by one thread.  (Spreading each sum over 2-4 lanes + shuffles so that all 16 warps share
    // the epilogue was tried: the extra shuffles cost more than the shorter chains save.)
    auto sum16 = [&](const float* part, int pidx) {
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int w = 0; w < NWARP; w += 2) { s0 += part[w * PPITCH + pidx]; s1 += part[(w + 1) * PPITCH + pidx]; }
        return s0 + s1;
    };
    // epilogue thread mapping: lanes run over the 8 weight columns first (8-byte words of one row are then
    // contiguous: a warp writes two full 128-byte lines), rows next, the second 8 columns (G: u gates) last.
    const int e_brow = (tid >> 3) & 7, e_wc = tid & 7, e_hi = (tid >> 6) & 1;
    const int e_pidx = (e_wc + 8 * e_hi) * 8 + e_brow;       // index into a [16 cols][8 rows] partial tile
    const int e_loc = e_wc * 8 + e_brow;                     // index into the [8 cols][8 rows] local state arrays
    const int e_row = row0 + e_brow;
    const int e_word = e_brow * 8 + perm8(e_wc);             // word inside this CTA's k-tile block of an exchange buffer

    // ---- attention window: the peak p(ts) of step ts from the four quarters' {max, sum} and peak words (the lowest
    //      quarter whose max is the utterance's, then that quarter's lowest maximising position; p(ts - 1) when every
    //      score is masked).  Read a whole step after they were published, so the poll normally finds them there ----
    // this utterance's peak words [2 parity][4 quarters] {position, tag} (formed at each use: a pointer kept live across
    // the kernel costs the windowed instantiation a spill)
    auto xpeak = [&]() { return ws + P.peak_off + (int64_t)arow * (2 * 4); };
    auto window_peak = [&](int ts, int pprev) {
        const uint32_t tag = (uint32_t)ts + 1;
        const uint64_t* xs = ws + P.att_off + (int64_t)arow * (2 * 4 * 2) + (ts & 1) * 4 * 2;
        const uint64_t* xk = xpeak() + (ts & 1) * 4;
        ulonglong2 sw[4];
        uint64_t kw[4];
#pragma unroll
        for (int qd = 0; qd < 4; ++qd) { sw[qd] = ll_load2(xs + qd * 2); kw[qd] = ll_load1(xk + qd); }
        float mq[4], M = -INFINITY;
#pragma unroll
        for (int qd = 0; qd < 4; ++qd) {
            ll_spin(sw[qd], xs + qd * 2, tag);
            mq[qd] = __uint_as_float((uint32_t)sw[qd].x);
            M = fmaxf(M, mq[qd]);
        }
        int p = pprev;
        bool found = false;
#pragma unroll
        for (int qd = 0; qd < 4; ++qd) {
            const int pk = __float_as_int(ll_spin1(kw[qd], xk + qd, tag));
            if (!found && M > -INFINITY && mq[qd] == M) { p = pk; found = true; }
        }
        return p;
    };

    // ---- stop rule (STOP instantiation): thread 128 of the quarter-0 CTA of each
    //      utterance counts the run of peaks >= stop_at and publishes one status word per step, {end step or 0, tag};
    //      thread 160 of every CTA of the row group reads its group's words a step later and sets the step all of them
    //      leave at.  Every CTA reads the same published words, so every CTA picks the same step ----
    //      Status words: [32 utterances][2 parity] {end step or 0 = running, tag t + 1}.  misc_i[3] = the run of peaks
    //      >= stop_at, [4] = the end step, [5] = the step to leave at, [6] = stop_at ----
    auto xstop = [&](int row, int ts) { return ws + P.stop_off + (int64_t)row * 2 + (ts & 1); };
    auto stop_publish = [&](int t, int pp) {            // at step t, with pp = p(t - 1)
        int* mi = reinterpret_cast<int*>(misc_s);
        int end = mi[4];
        if (t > 0 && end == 0) {
            const int run = pp >= mi[6] ? mi[3] + 1 : 0;
            mi[3] = run;
            if (run >= A.stop_hold) { end = t; mi[4] = end; }
        }
        ll_store(xstop(arow, t), __int_as_float(end), (uint32_t)t + 1);
    };
    // at step t >= 1 on lanes 0..7 of warp 5 (one row each): the words of step t - 1, a step old.  Once every row has
    // ended (padding rows have) the CTA leaves at the top of step t + 2: G1(t + 1)'s __syncthreads lies between this
    // store and every thread's read
    auto stop_poll = [&](int t) {
        const int i = tid - 160;
        bool ended = true;
        if (row0 + i < B) {
            uint64_t w = ll_load1(xstop(row0 + i, t - 1));
            ended = __float_as_int(ll_spin1(w, xstop(row0 + i, t - 1), (uint32_t)t)) != 0;
        }
        volatile int* mi = reinterpret_cast<volatile int*>(misc_s);
        if (__all_sync(0xffu, ended) && i == 0 && mi[5] > t + 2) mi[5] = t + 2;
    };

    // ---- attention of step t on warps 0..7 (256 threads): scores, partial softmax / context, merge of the quarters ----
    auto attention = [&](int t) {
        const uint32_t tag = (uint32_t)t + 1;
        const int xp = t & 1;
        uint64_t* ctx_out = ws + P.buf[B_CP] + (int64_t)(arow >> 3) * 48 * 64 + (8 * (int)aq + ((tid & 63) >> 3)) * 64 + (arow & 7) * 8 + perm8(tid & 7);
        if (STOP && tid >= 160 && tid < 160 + RPG && t > 0) stop_poll(t);   // (idle during the q(t) polls;
                                                                                          // also in padding CTAs)
        if (arow >= B) {                                // padding utterance: publish a zero context (consumers poll every row)
            if (tid < 64) ll_store(ctx_out, 0.f, tag + 1);
            return;
        }
        bool clamp = false;                             // q(t) or a key of this slice reaches exp2x's clamp
        if (tid < 128) {   // q(t) of this utterance -> e^{2q}
            const float2 qq = ll_wait2(ws + P.buf[B_Q] + (int64_t)(arow >> 3) * 2048 + (tid >> 2) * 64 + (arow & 7) * 8 + 2 * (tid & 3), tag);
            const int k0 = ((tid >> 2) << 3) + (tid & 3);        // physical pair (2p, 2p+1) = logical k0, k0+4
            eq_s[k0] = exp2x(qq.x);
            eq_s[k0 + 4] = exp2x(qq.y);
            clamp = exp2x_clamps(qq.x) | exp2x_clamps(qq.y) | (tid == 0 && misc_s[2] != 0.f);
        } else if (WIN && tid == 128) {   // p(t-1), off the chain: its words are a step old, the poll runs beside q(t)'s
            const int pp = (t > 0) ? window_peak(t - 1, __float_as_int(misc_s[1])) : 0;
            misc_s[1] = __int_as_float(pp);
            if (t > 0 && aq == 0 && A.peak) A.peak[(int64_t)arow * T + t - 1] = pp;
            if (STOP && aq == 0) stop_publish(t, pp);
        }
        if (TR && cktr) cktr[0] = clock64();
        clamp = named_bar_or(1, 256, clamp);            // (CTA-uniform; trained-like keys and queries never get there)
        if (TR && cktr) cktr[1] = clock64();
        if (clamp) scores_direct(e_s, v_s, A.keys + (int64_t)arow * Tx * ENC,
                                 ws + P.buf[B_Q] + (int64_t)(arow >> 3) * 2048 + (arow & 7) * 8, tag, (int)aq * Tq, Tq, Tx,
                                 WIN ? max(__float_as_int(misc_s[1]) - A.win_back, 0) : 0,
                                 WIN ? min(__float_as_int(misc_s[1]) + A.win_ahead, min(my_len, Tx) - 1) : my_len - 1,
                                 warp, lane);
        else {   // scores: lane owns 8 consecutive depth indices (its e^{2q}, v slices stay in registers), warp w owns
            // positions j = w, w+8, ...; four positions are reduced over the warp with one transposing butterfly
            float eq[8], vv[8];
            {
                const float4 q0 = *reinterpret_cast<const float4*>(eq_s + 8 * lane), q1 = *reinterpret_cast<const float4*>(eq_s + 8 * lane + 4);
                const float4 v0 = *reinterpret_cast<const float4*>(v_s + 8 * lane), v1 = *reinterpret_cast<const float4*>(v_s + 8 * lane + 4);
                eq[0] = q0.x; eq[1] = q0.y; eq[2] = q0.z; eq[3] = q0.w; eq[4] = q1.x; eq[5] = q1.y; eq[6] = q1.z; eq[7] = q1.w;
                vv[0] = v0.x; vv[1] = v0.y; vv[2] = v0.z; vv[3] = v0.w; vv[4] = v1.x; vv[5] = v1.y; vv[6] = v1.z; vv[7] = v1.w;
            }
            const float V0 = misc_s[0];
            int wlo = 0, whi = my_len - 1;              // allowed positions (WIN); the host keeps back, ahead <= Tx
            if (WIN) {
                const int pp = __float_as_int(misc_s[1]);
                wlo = max(pp - A.win_back, 0);
                whi = min(pp + A.win_ahead, min(my_len, Tx) - 1);
            }
            for (int jb = 0; jb < Tq; jb += 32) {       // 4 positions per warp and round
                float a4[4];
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) {
                    const int j = jb + warp + 8 * jj;
                    float a = 0.f;
                    if (j < Tq) {                       // warp-uniform
                        const float4 k0 = *reinterpret_cast<const float4*>(ek_s + j * KV_LD + 8 * lane);
                        const float4 k1 = *reinterpret_cast<const float4*>(ek_s + j * KV_LD + 8 * lane + 4);
                        a = fmaf(vv[0], rcp_fast(fmaf(k0.x, eq[0], 1.0f)), a);
                        a = fmaf(vv[1], rcp_fast(fmaf(k0.y, eq[1], 1.0f)), a);
                        a = fmaf(vv[2], rcp_fast(fmaf(k0.z, eq[2], 1.0f)), a);
                        a = fmaf(vv[3], rcp_fast(fmaf(k0.w, eq[3], 1.0f)), a);
                        a = fmaf(vv[4], rcp_fast(fmaf(k1.x, eq[4], 1.0f)), a);
                        a = fmaf(vv[5], rcp_fast(fmaf(k1.y, eq[5], 1.0f)), a);
                        a = fmaf(vv[6], rcp_fast(fmaf(k1.z, eq[6], 1.0f)), a);
                        a = fmaf(vv[7], rcp_fast(fmaf(k1.w, eq[7], 1.0f)), a);
                    }
                    a4[jj] = a;
                }
                // transposing butterfly: after the two halving steps lane group (lane>>3) holds position jj = lane>>3
                float b2[2], b1;
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                    const float send = (lane & 16) ? a4[k] : a4[k + 2];
                    const float keep = (lane & 16) ? a4[k + 2] : a4[k];
                    b2[k] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
                }
                {
                    const float send = (lane & 8) ? b2[0] : b2[1];
                    const float keep = (lane & 8) ? b2[1] : b2[0];
                    b1 = keep + __shfl_xor_sync(0xffffffffu, send, 8);
                }
                b1 += __shfl_xor_sync(0xffffffffu, b1, 4);
                b1 += __shfl_xor_sync(0xffffffffu, b1, 2);
                b1 += __shfl_xor_sync(0xffffffffu, b1, 1);
                const int jj = ((lane >> 4) & 1) * 2 + ((lane >> 3) & 1);
                const int j = jb + warp + 8 * jj;
                if ((lane & 7) == 0 && j < Tq) {
                    const int jg = (int)aq * Tq + j;
                    e_s[j] = (WIN ? (jg >= wlo && jg <= whi) : jg < my_len) ? fmaf(-2.0f, b1, V0) : -INFINITY;
                }
            }
        }
        if (TR && cktr) cktr[2] = clock64();
        named_bar(1, 256);
        if (TR && cktr) cktr[4] = clock64();
        // quarter statistics (every warp redundantly; Tq <= 64)
        const float e0 = (lane < Tq) ? e_s[lane] : -INFINITY;
        const float e1 = (lane + 32 < Tq) ? e_s[lane + 32] : -INFINITY;
        float m = fmaxf(e0, e1);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        const float p0 = (e0 == -INFINITY) ? 0.f : __expf(e0 - m);
        const float p1 = (e1 == -INFINITY) ? 0.f : __expf(e1 - m);
        float ssum = p0 + p1;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ssum += __shfl_xor_sync(0xffffffffu, ssum, o);
        if (warp == 0) {
            if (lane < Tq) p_s[lane] = p0;
            if (lane + 32 < Tq) p_s[lane + 32] = p1;
        }
        uint64_t* xstat = ws + P.att_off + (int64_t)arow * (2 * 4 * 2);                   // [2 parity][4 quarters][max, sum]
        uint64_t* xctx = ws + P.att_off + (NCTA / 4) * (2 * 4 * 2) + (int64_t)arow * (2 * 4 * ENC);   // [2 parity][4 quarters][256]
        if (tid == 0) {                                  // statistics of this quarter -> the utterance's four CTAs
            ll_store(xstat + (xp * 4 + aq) * 2, m, tag);
            ll_store(xstat + (xp * 4 + aq) * 2 + 1, ssum, tag);
        }
        named_bar(1, 256);
        if (TR && cktr) cktr[5] = clock64();
        {   // partial context: column tid (the CTA owning columns 64 q .. 64 q + 63 merges them)
            float c0 = 0.f, c1 = 0.f;
#pragma unroll 4
            for (int j = 0; j + 1 < Tq; j += 2) {
                c0 = fmaf(p_s[j], vals_s[j * ENC + tid], c0);
                c1 = fmaf(p_s[j + 1], vals_s[(j + 1) * ENC + tid], c1);
            }
            if (Tq & 1) c0 = fmaf(p_s[Tq - 1], vals_s[(Tq - 1) * ENC + tid], c0);
            ll_store(xctx + (xp * 4 + aq) * ENC + tid, c0 + c1, tag);
        }
        if (WIN && warp == 4) {                          // this quarter's peak: its lowest position holding the max (done
            const bool h0 = lane < Tq && e_s[lane] == m;  // after warp 4's partial context, so nothing waits for it)
            const bool h1 = lane + 32 < Tq && e_s[lane + 32] == m;
            const uint32_t b0 = __ballot_sync(0xffffffffu, h0), b1 = __ballot_sync(0xffffffffu, h1);
            const int li = b0 ? __ffs(b0) - 1 : (b1 ? 31 + __ffs(b1) : 0);
            if (lane == 0) ll_store(xpeak() + xp * 4 + aq, __int_as_float((int)aq * Tq + li), tag);
        }
        if (TR && cktr) cktr[6] = clock64();
        if (tid >= 128) return;
        // merge: global max / sum from the four quarter statistics.  Every exchange word this thread needs ({max, sum} of
        // each quarter: one 16-byte load; its context partials) is requested before any tag is checked, so the merge waits
        // for one L2 round trip instead of one per word; only words that were not yet published are polled again.
        const uint64_t* xs = xstat + xp * 4 * 2;
        const uint64_t* xc = xctx + xp * 4 * ENC + 64 * aq + tid;
        ulonglong2 sw[4];
        uint64_t cw[4];
#pragma unroll
        for (int qd = 0; qd < 4; ++qd) sw[qd] = ll_load2(xs + qd * 2);
        if (tid < 64) {
#pragma unroll
            for (int qd = 0; qd < 4; ++qd) cw[qd] = ll_load1(xc + qd * ENC);
        }
        float mq[4], wq[4], M = -INFINITY, S = 0.f, w_own = 0.f;
#pragma unroll
        for (int qd = 0; qd < 4; ++qd) {
            ll_spin(sw[qd], xs + qd * 2, tag);
            mq[qd] = __uint_as_float((uint32_t)sw[qd].x);
            M = fmaxf(M, mq[qd]);
        }
#pragma unroll
        for (int qd = 0; qd < 4; ++qd) {
            const float sq = __uint_as_float((uint32_t)sw[qd].y);
            wq[qd] = (mq[qd] == -INFINITY) ? 0.f : __expf(mq[qd] - M);
            S = fmaf(wq[qd], sq, S);
            if (qd == (int)aq) w_own = wq[qd];
        }
        const float inv = (S > 0.f) ? 1.0f / S : 0.f;
        if (tid < 64) {                                  // final context column 64 aq + tid  (tag of the step that consumes it)
            float c = 0.f;
#pragma unroll
            for (int qd = 0; qd < 4; ++qd) c = fmaf(wq[qd], ll_spin1(cw[qd], xc + qd * ENC, tag), c);
            ll_store(ctx_out, c * inv, tag + 1);
            if (TR && cktr) cktr[7] = clock64();
        } else {                                         // alignments of this quarter (AttentionWrapper alignment_history)
            const int j = tid - 64;
            if (j < Tq && (int)aq * Tq + j < Tx) A.align[((int64_t)arow * T + t) * Tx + aq * Tq + j] = p_s[j] * (w_own * inv);
        }
    };

    // ---- second pre-net layer of step tb on warps 8..15: p2(tb) = relu(p1(tb) . W2 + b2) ----
    auto prenet2 = [&](int tb) {
        const uint32_t tag = (uint32_t)tb + 1;
        const int widx = warp - 8;
        bool from_y = (tb > 0);
        if (A.mode == TACO_DEC_TEACHER) from_y = false;
        else if (A.mode == TACO_DEC_SCHED) from_y = (tb > 0) && (myrow < B) && (A.sample_mask[(int64_t)(tb - 1) * RS + R0 + myrow] != 0);
        const uint64_t* p0 = ws + P.buf[from_y ? B_P1Y : B_P1M] + (int64_t)rg * 2048 + widx * 64 + lane_w;
        const uint32_t w1 = seg_word(P.seg[SG_P2], cs);
        issue_loads<4>(v, p0, 32, widx, 8, 0);
        consume<2, 1, 4, false>(acc, v, p0, 32, widx, 8, 0, tag, w1, w1, widx * 4, res_s, packed, lane, nullptr);
        float* pw = part2_s + widx * 64;
        *reinterpret_cast<float2*>(pw + g * 8 + 2 * tg) =
            make_float2((acc[0][0][0] + acc[0][1][0]) + acc[0][2][0], (acc[0][0][1] + acc[0][1][1]) + acc[0][2][1]);
#pragma unroll
        for (int a1 = 0; a1 < 3; ++a1)
#pragma unroll
            for (int a2 = 0; a2 < 4; ++a2) acc[0][a1][a2] = 0.f;
        named_bar(2, 256);
        const int e = tid - 256;
        if (e < 32) {                                    // 8 rows x 4 columns, columns fastest
            const int wcol = e & 3, brow = e >> 2, row = row0 + brow, col = 4 * cs + wcol, pi = wcol * 8 + brow;
            float pv = bias_s[BR_P2 * 16 + wcol];
#pragma unroll
            for (int w = 0; w < 8; ++w) pv += part2_s[w * 64 + pi];
            pv = fmaxf(pv, 0.f);
            if (A.keep2 && row < B && tb < T) pv = A.keep2[((int64_t)tb * RS + R0 + row) * 128 + col] ? pv * A.keep_scale : 0.f;
            ll_store(ws + otab[O_P2] + brow * 8 + perm8(4 * (cs & 1) + wcol), pv, tag);
        }
        named_bar(2, 256);                               // part2_s may be rewritten
    };

    // ---- first pre-net layer of step tb from the teacher frame (or zeros): p1m(tb) = relu(x . W1 + b1) ----
    auto prenet1_teacher = [&](int tb) {
        const bool have = (A.mode != TACO_DEC_INFER) && (myrow < B) && (tb < T);
        const SegDesc& sd = P.seg[SG_PM];
        float w[4];
        {
            const float2 t2 = *reinterpret_cast<const float2*>(weight_ptr(seg_word(sd, cs), res_s, packed) + ((size_t)(warp * sd.kpw) * 32 + lane) * 2);
            w[0] = t2.x; w[1] = t2.y; w[2] = w[3] = 0.f;
        }
        if (warp < MF / 8) {                             // k-tile = warp (10 k-tiles); warp-uniform
            float xa = 0.f, xb = 0.f;
            if (have) {
                const float* mp = A.mel + ((int64_t)myrow * T + tb) * OUT + (OUT - MF) + warp * 8 + tg;
                xa = __ldg(mp); xb = __ldg(mp + 4);
            }
            uint32_t bh0, bl0, bh1, bl1;
            split_tf32(xa, bh0, bl0);
            split_tf32(xb, bh1, bl1);
            __syncwarp();
            ktile_mma<2>(acc[0], bh0, bl0, bh1, bl1, &w[0]);
        }
    };

    auto finish = [&](int stage, int t) {
        float* part = part_s + par * (NWARP * PPITCH);
        float* part_b = part_s + 2 * (NWARP * PPITCH);               // second tile of OQP and G1
        par ^= 1;
        const bool full16 = (stage >= ST_G0 && stage <= ST_G2) || stage == ST_OQP;
        // part_b was last read by the OQP epilogue just before; the attention and pre-net warps in between do not wait
        // for each other, so every warp must be past that epilogue before G1 overwrites it
        if (stage == ST_G0) __syncthreads();
        store_partials(part, part_b, (stage == ST_OQP || stage == ST_G0) ? 2 : 1, full16);
        if (TR && cktr) cktr[4] = clock64();
        if (TR && wtr) wtr[16] = clock64();
        __syncthreads();
        if (TR && cktr) cktr[5] = clock64();
        if (TR && wtr) wtr[32] = clock64();
        const uint32_t tag = (uint32_t)t + 1;
        switch (stage) {
            case ST_G0: case ST_G1: case ST_G2:
                if (tid < 128) {
                    const int gi = stage - ST_G0;
                    const int br = (gi == 0 && t == 0) ? BR_G0T : BR_G0 + gi;
                    float gp = sum16(part, e_pidx) + bias_s[br * 16 + e_wc + 8 * e_hi];
                    if (t == 0 && e_row < B) {
                        const int64_t ci = (int64_t)e_row * 2 * U + U * e_hi + 8 * cs + e_wc;
                        if (P.init_g) gp += P.init_g[(int64_t)gi * BPAD * 2 * U + ci];             // h0_i . Wg_i[256:]
                        if (gi == 0 && P.init_zg) gp += P.init_zg[ci];                         // att0 . W_in[128:] . Wg1_x
                    }
                    const float gt = sigmoidf_acc(gp);
                    if (!e_hi) ll_store(ws + otab[O_RH0 + gi] + e_word, gt * h_loc[gi * 64 + e_loc], tag);   // r * h
                    else u_loc[e_loc] = gt;                                                                // u stays local
                } else if (stage == ST_G0 && tid < 256) {                 // second tile: candidate x-half (e_hi = 0) | z (e_hi = 1)
                    float zv = sum16(part_b, e_pidx) + bias_s[(t == 0 ? BR_Z1T : BR_Z1) * 16 + e_wc + 8 * e_hi];
                    if (t == 0 && P.init_z && e_row < B) zv += P.init_z[(int64_t)e_row * 2 * U + U * e_hi + 8 * cs + e_wc];
                    (e_hi ? z_loc : cx_loc)[e_loc] = zv;
                }
                break;
            case ST_C0: case ST_C1: case ST_C2:
                if (tid < 64) {
                    const int gi = stage - ST_C0;
                    float cp = sum16(part, e_pidx) + bias_s[(BR_C0 + gi) * 16 + e_wc];
                    if (gi == 0) cp += cx_loc[e_loc];
                    const float cnd = tanhf_acc(cp);
                    const float uu = u_loc[e_loc];
                    const float hn = uu * h_loc[gi * 64 + e_loc] + (1.0f - uu) * cnd;
                    h_loc[gi * 64 + e_loc] = hn;
                    ll_store(ws + otab[O_H0 + gi] + e_word, hn, tag);
                    if (gi == 2) ll_store(ws + otab[O_S] + e_word, z_loc[e_loc] + hn, tag);
                    if (A.h_save && e_row < B) A.h_save[(((int64_t)gi * T + t) * RS + R0 + e_row) * U + 8 * cs + e_wc] = hn;   // training: BPTT input
                }
                break;
            case ST_PM:
                if (tid < 64) {                              // here t = tb, the step the pre-net output belongs to
                    const int col = 8 * cs + e_wc;
                    float pv = fmaxf(sum16(part, e_pidx) + bias_s[BR_PM * 16 + e_wc], 0.f);
                    if (A.keep1 && e_row < B && t < T) pv = A.keep1[((int64_t)t * RS + R0 + e_row) * 256 + col] ? pv * A.keep_scale : 0.f;
                    ll_store(ws + otab[O_P1M] + e_word, pv, tag);
                }
                break;
            case ST_OQP: if (tid < 256) {
                const int mt = tid >> 7;
                const float v0 = sum16(mt ? part_b : part, e_pidx) + bias_s[(BR_Y + mt) * 16 + e_wc + 8 * e_hi];
                if (mt == 0) {                               // y(t): the output itself (nothing downstream reads it)
                    const int wcol = e_wc + 8 * e_hi, col = cs * NCY + wcol;
                    if (wcol < NCY && col < OUT && e_row < B) A.y[((int64_t)e_row * T + t) * OUT + col] = v0;
                } else if (!e_hi) {                          // q(t)
                    ll_store(ws + otab[O_Q] + e_word, v0, tag);
                } else {                                     // p1(t+1) of free-running rows
                    const int col = 8 * cs + e_wc, tb = t + 1;
                    float pv = fmaxf(v0, 0.f);
                    if (A.keep1 && e_row < B && tb < T) pv = A.keep1[((int64_t)tb * RS + R0 + e_row) * 256 + col] ? pv * A.keep_scale : 0.f;
                    ll_store(ws + otab[O_P1Y] + e_word, pv, tag + 1);
                }
            } break;
            default: break;
        }
        if (TR && cktr) cktr[6] = clock64();
        if (TR && wtr) wtr[48] = clock64();
        if (TR && tracer) ws[P.trace_off + (trace_i++)] = globaltimer_ns();
    };

    // =========================================================================================================
    // prologue: p1(0) (teacher frame 0 or zeros), p2(0)
    // =========================================================================================================
    prenet1_teacher(0);
    finish(ST_PM, 0);
    if (warp >= 8) prenet2(0);

    // =========================================================================================================
    // T decoder steps x the item program
    // =========================================================================================================
    const int n_items = P.n_items;
    const uint32_t itab_a = smem_u32(itab);
    ulonglong2 vp[4];                                   // operand words of the off-chain half (prefetched one finish() early)
    float wpre[8];                                      // and its weight fragments (FL = 4: 2 slots x 4 floats; FL = 2: the first 4)
    bool pref = false;                                  // vp[] / wpre[] already hold the loads of the current stage's off-chain half
    auto load_pre_weights = [&](int knd, uint32_t ww) {
        if (knd == IK_F4 || knd == IK_G1) load_weights<4, 1, 2>(wpre, ww, 0u, warp * 2, res_s, packed, lane);
        else              load_weights<2, 1, 2>(wpre, ww, 0u, warp * 2, res_s, packed, lane);
    };
    auto ld_rec = [&](int ii, uint4& r0, uint4& r1, uint32_t& nkt) {
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r0.x), "=r"(r0.y), "=r"(r0.z), "=r"(r0.w) : "r"(itab_a + ii * 48));
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r1.x), "=r"(r1.y), "=r"(r1.z), "=r"(r1.w) : "r"(itab_a + ii * 48 + 16));
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(nkt) : "r"(itab_a + ii * 48 + 32));
    };
    uint4 nr0, nr1; uint32_t nnkt;
    ld_rec(0, nr0, nr1, nnkt);
    for (int t = 0; t < T; ++t) {
        if (STOP && t >= reinterpret_cast<volatile int*>(misc_s)[5]) break;   // CTA-uniform and group-uniform
        if (tracer) A.step_ns[t] = globaltimer_ns();
        for (int ii = 0; ii < n_items; ++ii) {
            // r0 = flags, pre_base, pre_tagd, pre_w;  r1 = on_base, on_tagd, on_w1, on_w2 -- fetched one stage ahead
            const uint4 r0 = nr0, r1 = nr1; const uint32_t on_nkt = nnkt;
            ld_rec(ii + 1 < n_items ? ii + 1 : 0, nr0, nr1, nnkt);
            const int kind = r0.x & 0xff, stage = (r0.x >> 8) & 0xff;
            long long* ck = nullptr;
            if (TR && tracer && t >= 10 && t < 14) { ck = reinterpret_cast<long long*>(ws + P.trace_off + 16 * T + 16 + ((t - 10) * MAX_ITEMS + ii) * 8); ck[3] = clock64(); }
            cktr = ck;
            wtr = (TR && trw >= 0 && lane == 0 && t >= 10 && t < 13)
                ? reinterpret_cast<long long*>(ws + P.trace_off + 16 * T + 16 + 4 * MAX_ITEMS * 8 + 16 + ((trw * 3 + t - 10) * MAX_ITEMS + ii) * 64 + warp)
                : nullptr;
            if (kind == IK_AP2) {
                if (warp < 8) attention(t);
                else if (t + 1 < T) prenet2(t + 1);
                if (TR && tracer) ws[P.trace_off + (trace_i++)] = globaltimer_ns();
                continue;
            }
            if (kind == IK_PM) {
                if (t + 1 < T) { prenet1_teacher(t + 1); finish(ST_PM, t + 1); }
                continue;
            }
            // ---- on-chain operand: loads in flight first, they travel while the off-chain half is multiplied ----
            const uint64_t* pon = ws + r1.x + warp * 64 + lane_w;
            const int s0 = (t == 0) ? (int)((r0.x >> 20) & 0xf) : 0;
            if (kind == IK_G1) issue_loads<3>(v, pon, (int)on_nkt, warp, NWARP, s0);
            else               issue_loads<2>(v, pon, (int)on_nkt, warp, NWARP, 0);
            if (TR && ck) ck[0] = clock64();
            const bool has_pre = ((r0.x >> 16) & 1) && !(t == 0 && ((r0.x >> 17) & 1));
            const uint64_t* ppre = ws + r0.y + warp * 64 + lane_w;
            const uint32_t ptag = (uint32_t)(t + (int)r0.z), otag = (uint32_t)(t + (int)r1.y);
            if (kind == IK_G1) {
                // first stage of a step: [ctx(t-1) | p2(t)] against the gate tile and the [candidate x-half | z] tile.
                // Off-chain, loaded here and one after the other (both in flight at once spill registers; prefetched before
                // A|P2 they delayed OQP's epilogue and the q(t) polls of the attention, H100 80GB HBM3, 700 W): h1(t-1) .
                // Wg1_h into the gates, then s(t-1) against both tiles.  Both end well before the merged context arrives.
                if (has_pre) {
                    issue_loads<2>(vp, ppre, 32, warp, NWARP, 0);
                    __syncwarp();
                    load_pre_weights(kind, r0.w);
                    multiply<4, 1, 2, false>(acc, vp, wpre, ppre, 32, warp, NWARP, 0, ptag, nullptr);
                    const ItemRec& rec = itab[ii];
                    const uint64_t* psv = ws + rec.s_base + warp * 64 + lane_w;
                    issue_loads<2>(vp, psv, 32, warp, NWARP, 0);
                    __syncwarp();
                    float wsx[16];
                    load_weights<4, 2, 2>(wsx, rec.s_w1, rec.s_w2, warp * 2, res_s, packed, lane);
                    multiply<4, 2, 2, false>(acc, vp, wsx, psv, 32, warp, NWARP, 0, ptag, nullptr);
                }
                consume<4, 2, 3, TR>(acc, v, pon, (int)on_nkt, warp, NWARP, s0, otag, r1.z, r1.w, warp * 3, res_s, packed, lane, ck, wtr);
            } else {
                if (has_pre && !pref) {
                    issue_loads<2>(vp, ppre, 32, warp, NWARP, 0);
                    __syncwarp();
                    load_pre_weights(kind, r0.w);
                }
                if (kind == IK_F4) {
                    if (has_pre) multiply<4, 1, 2, false>(acc, vp, wpre, ppre, 32, warp, NWARP, 0, ptag, nullptr);
                    consume<4, 1, 2, TR>(acc, v, pon, 32, warp, NWARP, 0, otag, r1.z, 0u, warp * 2, res_s, packed, lane, ck, wtr);
                } else if (kind == IK_F2) {
                    if (has_pre) multiply<2, 1, 2, false>(acc, vp, wpre, ppre, 32, warp, NWARP, 0, ptag, nullptr);
                    consume<2, 1, 2, TR>(acc, v, pon, 32, warp, NWARP, 0, otag, r1.z, 0u, warp * 2, res_s, packed, lane, ck, wtr);
                } else {
                    consume<4, 2, 2, TR>(acc, v, pon, 32, warp, NWARP, 0, otag, r1.z, r1.w, warp * 2, res_s, packed, lane, ck, wtr);
                }
            }
            pref = false;
            // the next stage's off-chain operand is already known: put its loads in flight now, together with those of its
            // weight fragments; they travel while this stage's epilogue runs
            if (ii + 1 < n_items && ((nr0.x >> 16) & 1)) {
                issue_loads<2>(vp, ws + nr0.y + warp * 64 + lane_w, 32, warp, NWARP, 0);
                load_pre_weights(nr0.x & 0xff, nr0.w);
                pref = true;
            }
            finish(stage, t);
        }
    }
    // steps decoded: T, or the step the stop rule left at (a later write of misc_i[5] by stop_poll can only be >= T)
    const int t_end = STOP ? min(reinterpret_cast<volatile int*>(misc_s)[5], T) : T;
    if (WIN && tid == 128 && aq == 0 && arow < B && A.peak)
        A.peak[(int64_t)arow * T + t_end - 1] = window_peak(t_end - 1, __float_as_int(misc_s[1]));
    if (STOP) {
        if (tid == 128 && aq == 0 && arow < B) {
            const int end = reinterpret_cast<int*>(misc_s)[4];
            A.end_step[arow] = end > 0 ? end : T;
        }
        // the steps the group did not decode: y and align 0, peak -1 (this CTA's columns / quarter / row)
        const int nt = T - t_end;
        for (int i = tid; i < nt * RPG * NCY; i += NTHR) {
            const int tt = t_end + i / (RPG * NCY), br = (i / NCY) % RPG, wc = i % NCY, col = cs * NCY + wc;
            if (row0 + br < B && col < OUT) A.y[((int64_t)(row0 + br) * T + tt) * OUT + col] = 0.f;
        }
        if (arow < B) {
            for (int i = tid; i < nt * Tq; i += NTHR) {
                const int tt = t_end + i / Tq, j = (int)aq * Tq + i % Tq;
                if (j < Tx) A.align[((int64_t)arow * T + tt) * Tx + j] = 0.f;
            }
            if (aq == 0 && A.peak)
                for (int i = tid; i < nt; i += NTHR) A.peak[(int64_t)arow * T + t_end + i] = -1;
        }
    }
}

// ---- packing: TF [K][N] -> per-slice MMA A fragments [cs][warp][k-tile slot][lane][FL] ----
__global__ void pack_seg_kernel(const float* __restrict__ W, int ldw, int k0, int K, int FL, int nw, int kpw, int sg, int NCY, int OUT,
                                float* __restrict__ dst) {
    const int slice = nw * kpw * 32 * FL;
    const int64_t total = (int64_t)NS * slice;
    const int nkt = K / 8;
    for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int cs = (int)(idx / slice);
        int r = (int)(idx % slice);
        const int e = r % FL; r /= FL;
        const int lane = r & 31; r >>= 5;
        const int i = r % kpw;
        const int widx = r / kpw;
        const int kt = widx + nw * i;
        const int g = lane >> 2, tg = lane & 3;
        // FL = 4: e = (k, m=g), (k, m=g+8), (k+4, m=g), (k+4, m=g+8);  FL = 2: e = (k, m=g), (k+4, m=g)
        const int m = (FL == 4) ? g + 8 * (e & 1) : g;
        const int k = kt * 8 + tg + 4 * ((FL == 4) ? (e >> 1) : e);
        float v = 0.f;
        if (kt < nkt) {
            const int col = seg_col(sg, cs, m, NCY, OUT);
            if (col >= 0) v = W[(int64_t)(k0 + k) * ldw + col];
        }
        dst[idx] = v;
    }
}

// weight-only precompute (double accumulation in k order): C = A . B (+ addv).  One 16 x 16 output tile per 256-thread
// block, its A and B k-slabs staged in shared memory (the pack runs after every weight update, i.e. every training step)
__global__ void matmul_f64_kernel(const float* __restrict__ Amat, int lda, const float* __restrict__ Bmat, int ldb,
                                  float* __restrict__ Cmat, int ldc, int M, int N, int K, const float* __restrict__ addv) {
    __shared__ float As[16][17], Bs[16][17];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int tiles_n = (N + 15) / 16;
    const int m = blockIdx.x / tiles_n * 16 + ty, n = blockIdx.x % tiles_n * 16 + tx;
    double a = (addv && n < N) ? (double)addv[n] : 0.0;
    for (int k0 = 0; k0 < K; k0 += 16) {
        As[ty][tx] = (m < M && k0 + tx < K) ? Amat[(int64_t)m * lda + k0 + tx] : 0.f;
        Bs[ty][tx] = (k0 + ty < K && n < N) ? Bmat[(int64_t)(k0 + ty) * ldb + n] : 0.f;
        __syncthreads();
        const int kn = K - k0 < 16 ? K - k0 : 16;
        for (int k = 0; k < kn; ++k) a += (double)As[ty][k] * (double)Bs[k][tx];
        __syncthreads();
    }
    if (m < M && n < N) Cmat[(int64_t)m * ldc + n] = (float)a;
}
void matmul_f64(cudaStream_t st, const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N, int K,
                const float* addv) {
    matmul_f64_kernel<<<(M + 15) / 16 * ((N + 15) / 16), 256, 0, st>>>(A, lda, B, ldb, C, ldc, M, N, K, addv);
}

// ---- fused linear stages (weight-only algebra; sums are re-associated, ~1e-6 relative) --------------------------
//   W_cpF  = [ W_a[80r:80r+256] . W_in[128:384] ; W_in[0:128] ]    [ctx(t-1) | p2(t)] -> z(t)
//   M1     = W_a[0:80r] . W_in[128:384];  W_sF = W_out . M1;  b_inF = b_in + b_out . M1   y(t-1) = s(t-1).W_out + b_out -> z(t)
//   W_qp   = [ W_out . W_q | W_out[:, last 80] . W1 ];  b_qF = b_out . W_q;  b_p1F = b_out[last 80] . W1 + b1
// z(t) itself is never formed on the chain: the first GRU takes it through
//   W_g1cp = W_cpF . Wg1_x,  W_g1s = W_sF . Wg1_x           (gates;                       Wg1_x = Wg1[0:256])
//   W_z1cp = [ W_cpF . Wc1_x | W_cpF ],  W_z1s = [ W_sF . Wc1_x | W_sF ]   ([candidate x-half | z]; Wc1_x = Wc1[0:256])
// with the biases b_g1F = b_inF . Wg1_x + bg1,  b_z1F = [ b_inF . Wc1_x | b_inF ]  (t > 0) and b_g1F0, b_z1F0: the same with
// b_in in place of b_inF (t = 0: there is no s(t-1)).  Every product is accumulated in float64 (matmul_f64_kernel).
// The packed buffer keeps these products only where the kernel reads them: as the MMA fragments of their segments, and the
// bias vectors in the tail.  The weight products are formed in the regions of the segments whose sources are raw weights
// (SG_G_H0 .. SG_Y), which are packed last (PackScratch); M1 lives in the tail, whose first 4 x 512 floats then receive the
// first GRU's folded biases.
struct FusedTail { int64_t fold, b_qF, b_p1F, b_inF, total; };   // fold: M1 [80r][256], then b_g1F | b_g1F0 | b_z1F | b_z1F0
FusedTail fused_tail(int r, int64_t slices_total) {
    const int OUT = MF * r;
    FusedTail f;
    int64_t o = (slices_total + 63) / 64 * 64;
    f.fold = o;   o += (int64_t)OUT * U;                  // >= 4 x 2U floats for every r >= 1
    f.b_qF = o;   o += AU;
    f.b_p1F = o;  o += 256;
    f.b_inF = o;  o += U;
    f.total = o;
    return f;
}
struct PackScratch { int64_t w_z1cp, w_z1s, w_g1cp, w_g1s, w_qp, end; };
PackScratch pack_scratch(const SegDesc* sd) {
    PackScratch p;
    int64_t o = sd[SG_G_H0].g_off;
    p.w_z1cp = o; o += (int64_t)(ENC + 128) * 2 * U;      // [384][512]; columns 256.. hold W_cpF
    p.w_z1s = o;  o += (int64_t)U * 2 * U;                // [256][512]; columns 256.. hold W_sF
    p.w_g1cp = o; o += (int64_t)(ENC + 128) * 2 * U;
    p.w_g1s = o;  o += (int64_t)U * 2 * U;
    p.w_qp = o;   o += (int64_t)U * 2 * AU;
    p.end = o;
    return p;
}

void build_seg_table(SegDesc* sd, int64_t* total_floats) {
    auto set = [&](int id, int K, int FL, int nw, int kpw) { sd[id].K = K; sd[id].FL = FL; sd[id].nw = nw; sd[id].kpw = kpw; };
    set(SG_G1_CP, ENC + 128, 4, 16, 3); set(SG_Z1_CP, ENC + 128, 4, 16, 3); set(SG_G1_S, 256, 4, 16, 2); set(SG_Z1_S, 256, 4, 16, 2);
    for (int i = 0; i < 3; ++i) { set(SG_G_H0 + i, 256, 4, 16, 2); set(SG_C_RH0 + i, 256, 2, 16, 2); }
    for (int i = 0; i < 2; ++i) { set(SG_G_X1 + i, 256, 4, 16, 2); set(SG_C_X1 + i, 256, 2, 16, 2); }
    set(SG_Y, 256, 4, 16, 2); set(SG_QP, 256, 4, 16, 2); set(SG_PM, MF, 2, 16, 2); set(SG_P2, 256, 2, 8, 4);
    int64_t off = 0;
    for (int s = 0; s < NSEG; ++s) {
        sd[s].slice_floats = sd[s].nw * sd[s].kpw * 32 * sd[s].FL;
        sd[s].g_off = off; sd[s].smem_off = -1;
        off += (int64_t)NS * sd[s].slice_floats;
    }
    *total_floats = off;
}

// word offsets of the exchange buffers, the attention exchange and the attention window's peak words; total = the end of
// what each launch zeroes, where the per-stage trace of the TR instantiation starts (taco_decoder_trace_offset)
void build_ws_layout(int64_t* buf, int64_t* att, int64_t* peak, int64_t* total) {
    int64_t o = 0;
    for (int b = 0; b < NBUF; ++b) { buf[b] = o; o += (int64_t)4 * buf_nkt(b) * 64; }
    *att = o;                                                    // [32 utterances][2][4] x (2 statistics + 256 context words)
    o += (int64_t)(NCTA / 4) * 2 * 4 * (2 + ENC);
    *peak = o;                                                   // [32 utterances][2][4] peak words
    o += (int64_t)(NCTA / 4) * 2 * 4;
    *total = o;
}

// [T] step stamps | thread 0's stage records [4 steps][MAX_ITEMS][8] | per-warp records [2 CTAs][3 steps][MAX_ITEMS][64]
inline int trace_words(int T) { return 16 * (T > 0 ? T : 0) + 16 + 4 * MAX_ITEMS * 8 + 16 + 2 * 3 * MAX_ITEMS * 64; }
// after the trace: the step-0 terms of an initial state, [32][512] floats each: init_z, init_zg (attention vector), then
// [3][32][512] init_g (GRU states)
constexpr int64_t INIT_ROWS = (int64_t)BPAD * 2 * U, INIT_FLOATS = 5 * INIT_ROWS;
// after those: the stop rule's status words, [32 utterances][2 parity] (zeroed by the launches that use them)
constexpr int64_t STOP_WORDS = (int64_t)(NCTA / 4) * 2;
inline int64_t stop_words_offset(int64_t ws_total, int T) { return ws_total + trace_words(T) + INIT_FLOATS / 2; }

// co-resident CTAs of the forward kernel on the current device (computed once per device; a MIG instance or an H100 PCIe
// has fewer SMs than the 132 of an H100 SXM).  Also opts the kernel into the full 227 KB of shared memory on that device.
constexpr int MAX_DEVICES = 64;
int decoder_fwd_capacity(int* out) {
    static int cap[MAX_DEVICES];
    int dev = 0;
    TACO_CUDA(cudaGetDevice(&dev));
    TACO_CHECK(dev >= 0 && dev < MAX_DEVICES, "taco_decoder: device %d out of range", dev);
    if (cap[dev] == 0) {
        TACO_CUDA(cudaFuncSetAttribute(decoder_kernel<false, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        TACO_CUDA(cudaFuncSetAttribute(decoder_kernel<true, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        TACO_CUDA(cudaFuncSetAttribute(decoder_kernel<false, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        TACO_CUDA(cudaFuncSetAttribute(decoder_kernel<true, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        TACO_CUDA(cudaFuncSetAttribute(decoder_kernel<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        TACO_CUDA(cudaFuncSetAttribute(decoder_kernel<true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        int per_sm = 0, sms = 0, per_sm_w = 0, per_sm_s = 0;
        TACO_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, decoder_kernel<false, false, false>, NTHR, 227 * 1024));
        // the windowed and stopping kernels run on the same grids: they have the same launch bounds and shared memory
        TACO_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_w, decoder_kernel<false, true, false>, NTHR, 227 * 1024));
        TACO_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_s, decoder_kernel<false, true, true>, NTHR, 227 * 1024));
        TACO_CHECK(per_sm_w == per_sm && per_sm_s == per_sm, "taco_decoder: windowed / stopping kernel occupancy %d / %d != %d",
                   per_sm_w, per_sm_s, per_sm);
        TACO_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        cap[dev] = per_sm * sms > 0 ? per_sm * sms : -1;
    }
    *out = cap[dev] > 0 ? cap[dev] : 0;
    return 0;
}

}  // namespace

int decoder_bwd_capacity(int* out);     // decoder_bwd.cu

extern "C" int taco_decoder_capacity(int* fwd_ctas, int* bwd_ctas) {
    int f = 0, b = 0;
    if (decoder_fwd_capacity(&f) || decoder_bwd_capacity(&b)) return 1;
    if (fwd_ctas) *fwd_ctas = f;
    if (bwd_ctas) *bwd_ctas = b;
    return 0;
}

extern "C" size_t taco_decoder_packed_bytes(int r) {
    SegDesc sd[NSEG]; int64_t tot;
    build_seg_table(sd, &tot);
    return (size_t)fused_tail(r, tot).total * 4;
}

extern "C" size_t taco_decoder_workspace_bytes(int B, int Tx, int T, int r) {
    (void)B; (void)Tx; (void)r;
    int64_t buf[NBUF], att, peak, total;
    build_ws_layout(buf, &att, &peak, &total);
    return (size_t)(stop_words_offset(total, T) + STOP_WORDS) * 8;
}

extern "C" int64_t taco_decoder_trace_offset(void) {
    int64_t buf[NBUF], att, peak, total;
    build_ws_layout(buf, &att, &peak, &total);
    return total;
}

extern "C" int taco_decoder_pack(const taco_decoder_weights* w, int r, float* packed, void* stream) {
    TACO_CHECK(w && packed, "taco_decoder_pack: NULL");
    TACO_CHECK(r >= 1 && MF * r <= 512, "taco_decoder_pack: r=%d out of range (80r <= 512)", r);
    TACO_CHECK(w->att_Wa && w->in_W && w->in_b && w->out_W && w->att_Wq && w->out_b && w->pre_W1 && w->pre_b1 && w->pre_W2,
               "taco_decoder_pack: NULL weight");
    for (int i = 0; i < 3; ++i) TACO_CHECK(w->gru_Wg[i] && w->gru_Wc[i], "taco_decoder_pack: NULL GRU weight");
    TACO_CHECK(w->gru_bg[0], "taco_decoder_pack: NULL GRU bias");
    SegDesc sd[NSEG]; int64_t tot;
    build_seg_table(sd, &tot);
    cudaStream_t stm = (cudaStream_t)stream;
    const int OUT = MF * r;
    const int NCY = (OUT + NS - 1) / NS;
    const FusedTail ft = fused_tail(r, tot);
    const PackScratch ps = pack_scratch(sd);
    TACO_CHECK(ps.end <= sd[SG_QP].g_off, "taco_decoder_pack: scratch overlaps a product segment");
    float *w_z1cp = packed + ps.w_z1cp, *w_z1s = packed + ps.w_z1s, *m1 = packed + ft.fold, *w_qp = packed + ps.w_qp;
    float *w_cpF = w_z1cp + U, *w_sF = w_z1s + U, *b_inF = packed + ft.b_inF;      // (row stride 2U)
    const float* w_inA = w->in_W + (int64_t)128 * U;           // W_in[128:384]
    matmul_f64(stm, w->att_Wa + (int64_t)OUT * AU, AU, w_inA, U, w_cpF, 2 * U, ENC, U, AU, nullptr);
    TACO_LAUNCH_CHECK();
    TACO_CUDA(cudaMemcpy2DAsync(w_cpF + (int64_t)ENC * 2 * U, 2 * U * sizeof(float), w->in_W, U * sizeof(float), U * sizeof(float), 128,
                                cudaMemcpyDeviceToDevice, stm));
    matmul_f64(stm, w->att_Wa, AU, w_inA, U, m1, U, OUT, U, AU, nullptr);
    TACO_LAUNCH_CHECK();
    matmul_f64(stm, w->out_W, OUT, m1, U, w_sF, 2 * U, U, U, OUT, nullptr);
    TACO_LAUNCH_CHECK();
    matmul_f64(stm, w->out_b, OUT, m1, U, b_inF, U, 1, U, OUT, w->in_b);
    TACO_LAUNCH_CHECK();
    // the first GRU's products of z: gates (. Wg1_x) and candidate x-half (. Wc1_x), weights and biases
    const float *wg1x = w->gru_Wg[0], *wc1x = w->gru_Wc[0];
    matmul_f64(stm, w_cpF, 2 * U, wg1x, 2 * U, packed + ps.w_g1cp, 2 * U, ENC + 128, 2 * U, U, nullptr);
    TACO_LAUNCH_CHECK();
    matmul_f64(stm, w_sF, 2 * U, wg1x, 2 * U, packed + ps.w_g1s, 2 * U, U, 2 * U, U, nullptr);
    TACO_LAUNCH_CHECK();
    matmul_f64(stm, w_cpF, 2 * U, wc1x, U, w_z1cp, 2 * U, ENC + 128, U, U, nullptr);
    TACO_LAUNCH_CHECK();
    matmul_f64(stm, w_sF, 2 * U, wc1x, U, w_z1s, 2 * U, U, U, U, nullptr);
    TACO_LAUNCH_CHECK();
    const float* zb[2] = {b_inF, w->in_b};                     // z's bias at t > 0 and at t = 0
    const int64_t gdst[2] = {ft.fold, ft.fold + 2 * U}, zdst[2] = {ft.fold + 4 * U, ft.fold + 6 * U};   // M1 is consumed
    for (int i = 0; i < 2; ++i) {
        matmul_f64(stm, zb[i], U, wg1x, 2 * U, packed + gdst[i], 2 * U, 1, 2 * U, U, w->gru_bg[0]);
        TACO_LAUNCH_CHECK();
        matmul_f64(stm, zb[i], U, wc1x, U, packed + zdst[i], U, 1, U, U, nullptr);
        TACO_LAUNCH_CHECK();
        TACO_CUDA(cudaMemcpyAsync(packed + zdst[i] + U, zb[i], U * sizeof(float), cudaMemcpyDeviceToDevice, stm));
    }
    matmul_f64(stm, w->out_W, OUT, w->att_Wq, AU, w_qp, 2 * AU, U, AU, OUT, nullptr);
    TACO_LAUNCH_CHECK();
    matmul_f64(stm, w->out_W + (OUT - MF), OUT, w->pre_W1, 256, w_qp + AU, 2 * AU, U, 256, MF, nullptr);
    TACO_LAUNCH_CHECK();
    matmul_f64(stm, w->out_b, OUT, w->att_Wq, AU, packed + ft.b_qF, AU, 1, AU, OUT, nullptr);
    TACO_LAUNCH_CHECK();
    matmul_f64(stm, w->out_b + (OUT - MF), MF, w->pre_W1, 256, packed + ft.b_p1F, 256, 1, 256, MF, w->pre_b1);
    TACO_LAUNCH_CHECK();

    struct Src { const float* W; int ld; int k0; };
    Src src[NSEG];
    src[SG_G1_CP] = {packed + ps.w_g1cp, 2 * U, 0}; src[SG_Z1_CP] = {w_z1cp, 2 * U, 0};
    src[SG_G1_S] = {packed + ps.w_g1s, 2 * U, 0};   src[SG_Z1_S] = {w_z1s, 2 * U, 0};
    for (int i = 0; i < 3; ++i) {
        src[SG_G_H0 + i] = {w->gru_Wg[i], 2 * U, U};  src[SG_C_RH0 + i] = {w->gru_Wc[i], U, U};    // rows: x then h (TF 1.2 GRUCell)
    }
    for (int i = 1; i < 3; ++i) { src[SG_G_X1 + i - 1] = {w->gru_Wg[i], 2 * U, 0}; src[SG_C_X1 + i - 1] = {w->gru_Wc[i], U, 0}; }
    src[SG_Y] = {w->out_W, OUT, 0}; src[SG_QP] = {w_qp, 2 * AU, 0}; src[SG_PM] = {w->pre_W1, 256, 0}; src[SG_P2] = {w->pre_W2, 128, 0};
    // the segments made from the products first: the others overwrite the scratch the products were formed in
    const int order[NSEG] = {SG_G1_CP, SG_Z1_CP, SG_G1_S, SG_Z1_S, SG_QP, SG_G_H0, SG_G_H1, SG_G_H2, SG_G_X1, SG_G_X2,
                             SG_C_X1, SG_C_X2, SG_C_RH0, SG_C_RH1, SG_C_RH2, SG_Y, SG_PM, SG_P2};
    for (int s : order) {
        const int64_t total = (int64_t)NS * sd[s].slice_floats;
        const int blocks = (int)((total + 255) / 256);
        pack_seg_kernel<<<blocks, 256, 0, stm>>>(src[s].W, src[s].ld, src[s].k0, sd[s].K, sd[s].FL, sd[s].nw, sd[s].kpw, s, NCY, OUT, packed + sd[s].g_off);
        TACO_LAUNCH_CHECK();
    }
    return 0;
}

extern "C" int taco_decoder_fwd(const taco_decoder_args* a, void* stream) {
    TACO_CHECK(a, "taco_decoder_fwd: NULL args");
    TACO_CHECK(a->max_ctas == 0 || a->max_ctas >= NS, "taco_decoder_fwd: max_ctas=%d: the budget must be 0 (the device's capacity) "
               "or at least %d CTAs", a->max_ctas, NS);
    TACO_CHECK(a->weights != nullptr, "taco_decoder_fwd: weights (biases, attention_v) is NULL");
    const taco_decoder_weights& W = *a->weights;
    TACO_CHECK(a->B >= 1 && a->B <= BPAD, "taco_decoder_fwd: B=%d must be in [1,%d] per launch", a->B, BPAD);
    TACO_CHECK(a->T >= 1, "taco_decoder_fwd: T=%d", a->T);
    TACO_CHECK(a->Tx >= 1 && a->Tx <= 256, "taco_decoder_fwd: Tx=%d must be in [1, 256]", a->Tx);
    TACO_CHECK(a->r >= 1 && MF * a->r <= 512, "taco_decoder_fwd: r=%d unsupported (80r must be <= 512)", a->r);
    TACO_CHECK(a->packed && a->keys && a->values && a->text_length && a->y && a->align && a->workspace, "taco_decoder_fwd: NULL pointer");
    TACO_CHECK((reinterpret_cast<uintptr_t>(a->workspace) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->packed) & 15) == 0,
               "taco_decoder_fwd: workspace / packed must be 16-byte aligned");
    if (a->mode != TACO_DEC_INFER) TACO_CHECK(a->mel != nullptr, "taco_decoder_fwd: teacher/sched mode needs mel");
    if (a->mode == TACO_DEC_SCHED) TACO_CHECK(a->sample_mask != nullptr, "taco_decoder_fwd: sched mode needs sample_mask");
    TACO_CHECK(a->win_back >= 0 && a->win_ahead >= 0, "taco_decoder_fwd: win_back=%d, win_ahead=%d: the attention window "
               "bounds must be >= 0 (win_ahead = 0: no window)", a->win_back, a->win_ahead);
    const bool win = a->win_ahead > 0;
    TACO_CHECK(win || (a->win_back == 0 && (a->peak == nullptr || a->stop_at != nullptr)), "taco_decoder_fwd: win_ahead=0 "
               "(no window) with win_back=%d and peak %s: a window needs win_ahead >= 1 (peak: or the stop rule)",
               a->win_back, a->peak ? "set" : "NULL");
    TACO_CHECK(!win || a->mode == TACO_DEC_INFER, "taco_decoder_fwd: win_ahead=%d: the attention window applies to "
               "free-running decoding (mode TACO_DEC_INFER) only, mode is %d", a->win_ahead, a->mode);
    const bool stop = a->stop_at != nullptr;
    TACO_CHECK(stop == (a->end_step != nullptr), "taco_decoder_fwd: stop_at %s with end_step %s: the stop rule needs both "
               "(or neither)", a->stop_at ? "set" : "NULL", a->end_step ? "set" : "NULL");
    TACO_CHECK(stop || a->stop_hold == 0, "taco_decoder_fwd: stop_hold=%d without stop_at", a->stop_hold);
    TACO_CHECK(!stop || a->stop_hold >= 1, "taco_decoder_fwd: stop_hold=%d: the stop rule needs a hold of >= 1 step",
               a->stop_hold);
    TACO_CHECK(!stop || a->mode == TACO_DEC_INFER, "taco_decoder_fwd: the stop rule applies to free-running decoding "
               "(mode TACO_DEC_INFER) only, mode is %d", a->mode);
    TACO_CHECK((a->keep1 == nullptr) == (a->keep2 == nullptr), "taco_decoder_fwd: keep1/keep2 must both be set or both NULL");
    TACO_CHECK(a->row0 >= 0 && (a->row_stride == 0 ? a->row0 == 0 : a->row0 + a->B <= a->row_stride),
               "taco_decoder_fwd: rows [%d, %d) outside a row stride of %d", a->row0, a->row0 + a->B, a->row_stride);
    cudaStream_t st = (cudaStream_t)stream;

    static DecParams P;                                  // (kept off the stack; a decoder launch is not re-entrant)
    memset(&P, 0, sizeof(P));
    int64_t tot, ws_total;
    build_seg_table(P.seg, &tot);
    build_ws_layout(P.buf, &P.att_off, &P.peak_off, &ws_total);
    P.trace_off = ws_total;
    P.a = *a;
    if (P.a.row_stride == 0) P.a.row_stride = a->B;
    if (win) {                          // a bound >= Tx allows every position already; p + ahead cannot overflow
        P.a.win_back = a->win_back < a->Tx ? a->win_back : a->Tx;
        P.a.win_ahead = a->win_ahead < a->Tx ? a->win_ahead : a->Tx;
    } else if (stop) {                  // the stop rule needs the peaks: the windowed kernel, with bounds that cover every
        P.a.win_back = a->Tx;           // position (the unwindowed bits)
        P.a.win_ahead = a->Tx;
    }
    P.stop_off = stop_words_offset(ws_total, a->T);
    P.OUT = MF * a->r;
    P.NCY = (P.OUT + NS - 1) / NS;
    P.Tq = (a->Tx + 3) / 4;            // quarter width; the last quarter is ragged when Tx % 4 != 0
    TACO_CHECK(P.Tq <= 64 && P.NCY <= 16, "taco_decoder_fwd: Tx/4 = %d > 64 or 80r/32 > 16", P.Tq);
    P.out_b = W.out_b; P.pre_b1 = W.pre_b1; P.pre_b2 = W.pre_b2; P.att_v = W.att_v;
    for (int i = 0; i < 3; ++i) { P.gru_bg[i] = W.gru_bg[i]; P.gru_bc[i] = W.gru_bc[i]; }
    const FusedTail ft = fused_tail(a->r, tot);
    P.b_qF = a->packed + ft.b_qF; P.b_p1F = a->packed + ft.b_p1F;
    P.b_g1F = a->packed + ft.fold; P.b_g1F0 = P.b_g1F + 2 * U; P.b_z1F = P.b_g1F + 4 * U; P.b_z1F0 = P.b_g1F + 6 * U;

    // ---- the per-step program: one record per stage ----
    int n = 0;
    auto stage = [&](int kind, int st_id, int pre_seg, int pre_src, int pre_tagd, int pre_skip0, int on_seg, int on_seg2, int on_src, int on_tagd, int on_s0) {
        P.items[n++] = Item{kind, st_id, pre_seg, pre_src, pre_tagd, pre_skip0, on_seg, on_seg2, on_src, on_tagd, on_s0};
    };
    // G1: h1(t-1) (and s(t-1), see ItemRec) | [ctx(t-1) | p2(t)] against the gate and [candidate x-half | z] tiles (no h, no
    // s, no context at t = 0); C1: r*h only, its x-half came with G1
    stage(IK_G1, ST_G0, SG_G_H0, B_H0, 0, 1, SG_G1_CP, SG_Z1_CP, B_CP, 1, 2);
    stage(IK_F2, ST_C0, -1, 0, 0, 0, SG_C_RH0, -1, B_RH0, 1, 0);
    for (int i = 1; i < 3; ++i) {
        const int x = B_H0 + (i - 1);
        stage(IK_F4, ST_G0 + i, SG_G_H0 + i, B_H0 + i, 0, 1, SG_G_X1 + i - 1, -1, x, 1, 0);       // h_i(t-1) | x
        stage(IK_F2, ST_C0 + i, SG_C_X1 + i - 1, x, 1, 0, SG_C_RH0 + i, -1, B_RH0 + i, 1, 0);     // x (already consumed by the gates) | r*h
    }
    if (a->mode != TACO_DEC_INFER) stage(IK_PM, ST_PM, -1, 0, 0, 0, -1, -1, 0, 0, 0);             // teacher frame t+1 -> p1m(t+1), off-chain
    stage(IK_F4X2, ST_OQP, -1, 0, 0, 0, SG_Y, SG_QP, B_S, 1, 0);
    stage(IK_AP2, ST_AP2, -1, 0, 0, 0, -1, -1, 0, 0, 0);
    P.n_items = n;

    // ---- residency: on-chain segments in shared memory, off-chain segments read from the packed buffer (L2); when the
    //      keys/values leave too little shared memory (large Tx) further segments are read from L2 as well ----
    int off = 16 + 6400 + 512 + 384 + 256 + 704 + 256;
    off = (off + 31) / 32 * 32;
    P.smem_kv_off = off;
    off += P.Tq * KV_LD + P.Tq * ENC;
    off = (off + 31) / 32 * 32;
    P.smem_res_off = off;
    const int budget = (227 * 1024) / 4 - off;
    // (build_seg_table leaves every segment in L2; the packed buffer is far below the 2^31 floats a weight word can address)
    // (at Tx = 128 every slice but the output tile SG_Y fits; SG_Y is loaded with OQP's operand, in the shadow of its hop)
    const int sm_order[] = {SG_G1_CP, SG_Z1_CP, SG_C_RH0, SG_G_X1, SG_C_RH1, SG_G_X2, SG_C_RH2, SG_QP, SG_Y, SG_P2};
    int res = 0;
    for (int s : sm_order) {
        if (P.seg[s].slice_floats <= budget - res) { P.seg[s].smem_off = res; res += P.seg[s].slice_floats; }
    }
    P.smem_total_floats = off + res;
    const size_t smem_bytes = (size_t)P.smem_total_floats * 4;

    // ---- launch geometry: 32 CTAs per row group, as many row groups as the CTA budget allows (at most 4); rows past B are
    //      padding.  (Sizing the grid to ceil(B/8) row groups instead was measured slower: at B = 1, T = 100 the decoder
    //      took 1.86 ms on 32 CTAs against 1.82 ms on 128, H100 80GB HBM3 at 400 W.)  Every CTA polls its row group's peers
    //      (a peer that never runs ends in __trap), so a grid that does not cover the row groups of the launch's
    //      utterances is refused here ----
    int capacity = 0;
    if (decoder_fwd_capacity(&capacity)) return 1;
    TACO_CHECK(capacity >= NS, "taco_decoder_fwd: only %d CTAs can be co-resident on this device (need %d)", capacity, NS);
    const int ctas = a->max_ctas > 0 && a->max_ctas < capacity ? a->max_ctas : capacity;
    const int groups = ctas / NS < NCTA / NS ? ctas / NS : NCTA / NS;
    TACO_CHECK(groups * RPG >= a->B,
               "taco_decoder_fwd: B=%d needs %d CTAs (%d row groups of 8 utterances), the budget allows %d: split the batch",
               a->B, (a->B + RPG - 1) / RPG * NS, (a->B + RPG - 1) / RPG, ctas);
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(groups * NS); cfg.blockDim = dim3(NTHR); cfg.dynamicSmemBytes = smem_bytes; cfg.stream = st;
    // all CTAs must be co-resident (one per SM): the kernel is a dataflow machine without a grid barrier.  A cooperative
    // launch makes that a guarantee (the launch fails instead of leaving CTAs to spin on peers that never start).
    cudaLaunchAttribute coop;
    coop.id = cudaLaunchAttributeCooperative;
    coop.val.cooperative = 1;
    cfg.attrs = &coop; cfg.numAttrs = 1;
    TACO_CUDA(cudaMemsetAsync(a->workspace, 0, (size_t)ws_total * 8, st));
    if (stop) TACO_CUDA(cudaMemsetAsync(reinterpret_cast<uint64_t*>(a->workspace) + P.stop_off, 0, STOP_WORDS * 8, st));
    // initial state (speaker-conditioned decoder): the kernel skips the h(t-1) and attention products at t = 0, so their
    // step-0 values are formed here, per row of this launch, and added by the G1 and G epilogues of step 0 (the C stage
    // sees h0 through r * h and the state update): with iz = att0 . W_in[128:], init_z = [iz . Wc1_x | iz] and
    // init_zg = iz . Wg1_x (z and the first GRU's products of it), init_g = h0_i . Wg_i[256:]
    if (a->att0 || a->h0) {
        float* init = reinterpret_cast<float*>(reinterpret_cast<uint64_t*>(a->workspace) + ws_total + trace_words(a->T));
        const int RS = P.a.row_stride;
        // dst[b][n] = X[b] . Wm[:, n], b < B (the library's own GEMM)
        auto term = [&](const float* X, int64_t ldx, const float* Wm, int N, float* dst) {
            taco_gemm_desc g;
            memset(&g, 0, sizeof(g));
            g.A = X; g.lda = ldx; g.B = Wm; g.ldb = N; g.C = dst; g.ldc = 2 * U; g.M = a->B; g.N = N; g.K = U;
            g.taps = 1; g.batch = 1;
            return taco_gemm(&g, stream);
        };
        if (a->att0) {
            TACO_CHECK(W.in_W != nullptr && W.gru_Wg[0] != nullptr && W.gru_Wc[0] != nullptr,
                       "taco_decoder_fwd: att0 needs weights->in_W, gru_Wg[0] and gru_Wc[0]");
            float *iz = init + U, *izg = init + INIT_ROWS;
            if (term(a->att0 + (int64_t)a->row0 * U, U, W.in_W + (int64_t)128 * U, U, iz)) return 1;
            if (term(iz, 2 * U, W.gru_Wc[0], U, init)) return 1;
            if (term(iz, 2 * U, W.gru_Wg[0], 2 * U, izg)) return 1;
            P.init_z = init; P.init_zg = izg;
        }
        if (a->h0) {
            for (int i = 0; i < 3; ++i) {
                TACO_CHECK(W.gru_Wg[i] != nullptr, "taco_decoder_fwd: h0 needs weights->gru_Wg");
                if (term(a->h0 + ((int64_t)i * RS + a->row0) * U, U, W.gru_Wg[i] + (int64_t)U * 2 * U, 2 * U,
                         init + (2 + i) * INIT_ROWS)) return 1;
            }
            P.init_g = init + 2 * INIT_ROWS;
        }
    }
    static const bool trace_build = getenv("TACO_TRACE") != nullptr;     // per-stage clock trace (scripts/dec_time.py)
    const bool trace = trace_build && a->step_ns;
    if (stop)     TACO_CUDA(cudaLaunchKernelEx(&cfg, trace ? decoder_kernel<true, true, true> : decoder_kernel<false, true, true>, P));
    else if (win) TACO_CUDA(cudaLaunchKernelEx(&cfg, trace ? decoder_kernel<true, true, false> : decoder_kernel<false, true, false>, P));
    else          TACO_CUDA(cudaLaunchKernelEx(&cfg, trace ? decoder_kernel<true, false, false> : decoder_kernel<false, false, false>, P));
    ++g_taco_launches;
    return 0;
}
