// gru.cu -- persistent bidirectional GRU (TF-1.2 GRUCell form), hidden size 128.
//
// Reference: tf.nn.bidirectional_dynamic_rnn(GRUCell(128), GRUCell(128), h) without
// sequence_length, models/ops.py:118-128; cell arithmetic SURVEY.md A.5:
//     [r,u] = sigmoid([x,h].Wg + bg)   c = tanh([x, r*h].Wc + bc)   h' = u*h + (1-u)*c
// (reset gate applied BEFORE the candidate product -- not the cuDNN form.)
//
// Design: the input-side products x.Wg[0:128], x.Wc[0:128] (+ biases) for all T steps are one
// big tensor-core GEMM done by the caller (xp, 768 columns = fw gates|fw cand|bw gates|bw cand).
// The serial part is one CTA per (utterance, direction): 64 CTAs at B=32, no inter-CTA
// communication at all.  The recurrent weights (128x256 + 128x128 fp32 = 192 KB) live in the
// REGISTER FILE of the CTA's 256 threads (192 floats each) for the whole sequence.
//
// Thread mapping (v5).  History: v1 one thread per column, every thread re-reading all of h: shared-memory -> register
// bandwidth bound; v2 lanes split K 32 ways, 16-to-1 halving butterfly: issue bound (half the instructions butterfly);
// v3 4 lanes per hidden unit: bandwidth bound again (128 B of h per thread and mat-vec); v4 512 threads, a group of 8
// lanes owning two hidden units: on Hopper (no packed fp32 FMA) only 96 of ~220 instructions per thread and step were
// FFMA, the rest select-heavy butterflies, divergent owner branches and per-thread address work of 16 warps.
// v5 halves the threads and doubles the work per thread: a GROUP OF 8 LANES owns four hidden units (their r, u and
// candidate columns: 12 columns), the 8 lanes split K (16 rows each: the 16-byte chunks 8i + l3 of h, so a group reads
// 128 contiguous bytes per load and the 4 groups of a warp read the same bytes, one broadcast), and each 8-lane
// reduction is a transposing butterfly without selects (group_sum): slot s of a lane's accumulators holds unit
// s ^ (l3 >> 1), so every lane keeps the low half of its slots and sends the high half.  After 4 shuffles both lanes of
// a pair hold the sum of unit l3 >> 1; the odd lane stores the new state.  r is reduced first and alone gates the first
// barrier; u's products follow it and u's reduction and sigmoid run beside the candidate products.  Per thread and
// step: 192 FFMA of ~301 instructions, 8 warps per CTA instead of 16.  The products keep v4's summation order (even
// and odd rows in two chains), so the outputs are bit-identical to v4's.  Reducing u before the barrier as well (so that
// its products cannot sink past it) measured slower, as did one sigmoid per lane after a 7-shuffle butterfly over all
// 8 gate columns with a 3-step prefetch (DESIGN 3.2).
#include "common.cuh"

namespace {

constexpr int H = 128;
constexpr int NT = 256;

#ifdef TACO_BIGRU_TRACE
// Per-phase clock trace (scripts/bigru_time.py builds a separate library with -DTACO_BIGRU_TRACE): %clock64 of thread 0
// of CTA (utterance 0, forward) at the start of each of the first TRACE_STEPS steps and after each phase of it.
constexpr int TRACE_STEPS = 16, TRACE_MARKS = 6;   // step start | r products | r*h stored | barrier | h stored | barrier
__device__ long long g_bigru_trace[TRACE_STEPS * TRACE_MARKS];
#define BIGRU_MARK(m) do { if (trace_on && trace_step < TRACE_STEPS) g_bigru_trace[trace_step * TRACE_MARKS + (m)] = clock64(); } while (0)
#else
#define BIGRU_MARK(m) do {} while (0)
#endif

// acc[s] = sum over this lane's 16 rows of v[k] * w[s][k] (v: the lane's four 16-byte chunks of a shared vector),
// even and odd rows in two chains that are added at the end: the summation order of v4, so that the results are
// bit-identical to it
__device__ __forceinline__ void matvec16x4(const float4 (&v)[4], const float (&w)[4][16], float (&acc)[4]) {
    float ev[4], od[4];
#pragma unroll
    for (int s = 0; s < 4; ++s) ev[s] = od[s] = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            ev[s] = fmaf(v[i].x, w[s][4 * i], ev[s]);
            od[s] = fmaf(v[i].y, w[s][4 * i + 1], od[s]);
            ev[s] = fmaf(v[i].z, w[s][4 * i + 2], ev[s]);
            od[s] = fmaf(v[i].w, w[s][4 * i + 3], od[s]);
        }
    }
#pragma unroll
    for (int s = 0; s < 4; ++s) acc[s] = ev[s] + od[s];
}

// the 8-lane group's sum of unit l3 >> 1, where slot s of each lane holds unit s ^ (l3 >> 1): every lane keeps the low
// half of its slots and sends the high half (the partner's high slots hold this lane's low units), so the transposing
// butterfly needs no selects; the last level sums the pair (both lanes get the result)
__device__ __forceinline__ float group_sum(const float (&v)[4]) {
    const float q0 = v[0] + __shfl_xor_sync(0xffffffffu, v[2], 4);
    const float q1 = v[1] + __shfl_xor_sync(0xffffffffu, v[3], 4);
    const float p = q0 + __shfl_xor_sync(0xffffffffu, q1, 2);
    return p + __shfl_xor_sync(0xffffffffu, p, 1);
}

__global__ void __launch_bounds__(NT, 1)
bigru_kernel(const float* __restrict__ xp, const float* __restrict__ Wg_fw, const float* __restrict__ Wc_fw,
             const float* __restrict__ Wg_bw, const float* __restrict__ Wc_bw, const float* __restrict__ h0_fw,
             const float* __restrict__ h0_bw, float* __restrict__ out, int T) {
    const int b = blockIdx.x;
    const int dir = blockIdx.y;
    const int tid = threadIdx.x;
    const int grp = tid >> 3;                  // 8-lane group: hidden units 4*grp .. 4*grp + 3
    const int l3 = tid & 7;                    // K slice: rows 4*(8i + l3) + e, i, e = 0..3
    const float* Wg = dir ? Wg_bw : Wg_fw;     // [128][256]  h-side rows of the gates kernel (columns: r then u)
    const float* Wc = dir ? Wc_bw : Wc_fw;     // [128][128]  (r*h)-side rows of the candidate kernel

    __shared__ __align__(16) float h_s[H];
    __shared__ __align__(16) float rh_s[H];

    // rows k = 4*(8i + l3) + e; slot s holds unit 4*grp + (s ^ (l3 >> 1)) in all three:
    // wr[s][4i + e] = Wg[k][unit] (r), wu[s][4i + e] = Wg[k][128 + unit] (u), wc[s][4i + e] = Wc[k][unit]
    float wr[4][16], wu[4][16], wc[4][16];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int k = 4 * (8 * i + l3) + e;
#pragma unroll
            for (int s = 0; s < 4; ++s) {
                const int unit = 4 * grp + (s ^ (l3 >> 1));
                wr[s][4 * i + e] = __ldg(Wg + k * 256 + unit);
                wu[s][4 * i + e] = __ldg(Wg + k * 256 + H + unit);
                wc[s][4 * i + e] = __ldg(Wc + k * 128 + unit);
            }
        }
    }
    const int j = 4 * grp + (l3 >> 1);         // this lane's unit after the reductions (both lanes of a pair)
    const bool owner = l3 & 1;                 // the odd lane of the pair stores the unit's new state

    const float* h0 = dir ? h0_bw : h0_fw;     // initial state (ops.py:111-126): speaker-dependent, or NULL = zero state
    if (tid < H) h_s[tid] = h0 ? __ldg(h0 + b * H + tid) : 0.0f;
    __syncthreads();

    // pointers advance by one time step per iteration (no per-step index arithmetic); the input products are prefetched
    // two steps ahead (they do not depend on h and stream from HBM), alternating between two named register triples
    // (32-bit element offsets: the host checks B*T*768 < 2^31)
    const int seq = b * T;
    const int t_first = dir ? (T - 1) : 0;
    const int xs = dir ? -768 : 768, os = dir ? -256 : 256;
    int xpp = (seq + t_first) * 768 + dir * 384 + j;      // hoisted products of unit j: r at +0, u at +128, candidate at +256
    int outp = (seq + t_first) * 256 + dir * H + j;

    auto load_x = [&](int off) { return make_float3(__ldg(xp + off), __ldg(xp + off + H), __ldg(xp + off + 2 * H)); };
    float3 x0 = make_float3(0.f, 0.f, 0.f), x1 = x0;
    if (T > 0) x0 = load_x(xpp);
    if (T > 1) x1 = load_x(xpp + xs);
    xpp += 2 * xs;                             // -> the row of step + 2

    const float4* h4 = reinterpret_cast<const float4*>(h_s) + l3;
    const float4* rh4 = reinterpret_cast<const float4*>(rh_s) + l3;
#ifdef TACO_BIGRU_TRACE
    const bool trace_on = b == 0 && dir == 0 && tid == 0;
    int trace_step = 0;
#endif

    // one time step: consumes x, refills it with the products of step + 2 when `more`.  Only r*h gates the first
    // barrier: the u products are issued after the r products and fill the latency of r's reduction and sigmoid, and
    // u's reduction and sigmoid run beside the candidate products.
    auto one_step = [&](float3& x, bool more) {
        BIGRU_MARK(0);
        const float3 xv = x;
        if (more) x = load_x(xpp);
        xpp += xs;
        const float hj = h_s[j];
        // ---- gates: h . Wg_h (this lane: 16 rows x 4 units x r, u) ----
        float4 hv[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) hv[i] = h4[8 * i];
        float ar[4], au[4];
        matvec16x4(hv, wr, ar);
        BIGRU_MARK(1);
        const float r = sigmoidf_acc(group_sum(ar) + xv.x);
        matvec16x4(hv, wu, au);
        if (!owner) rh_s[j] = r * hj;          // r * h
        BIGRU_MARK(2);
        __syncthreads();
        BIGRU_MARK(3);
        // ---- candidate: (r*h) . Wc_h (16 rows x 4 units) ----
        float4 rv[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) rv[i] = rh4[8 * i];
        const float u = sigmoidf_acc(group_sum(au) + xv.y);
        float ac[4];
        matvec16x4(rv, wc, ac);
        const float cn = tanhf_acc(group_sum(ac) + xv.z);
        const float hn = u * hj + (1.0f - u) * cn;
        if (owner) {
            h_s[j] = hn;
            out[outp] = hn;
        }
        outp += os;
        BIGRU_MARK(4);
        __syncthreads();
        BIGRU_MARK(5);
#ifdef TACO_BIGRU_TRACE
        ++trace_step;
#endif
    };

    int step = 0;
    for (; step + 2 <= T; step += 2) {
        one_step(x0, step + 2 < T);
        one_step(x1, step + 3 < T);
    }
    if (step < T) one_step(x0, false);
}

}  // namespace

#ifdef TACO_BIGRU_TRACE
extern "C" int taco_bigru_trace_read(long long* dst) {     // TRACE_STEPS x TRACE_MARKS clocks of the last launch
    TACO_CUDA(cudaMemcpyFromSymbol(dst, g_bigru_trace, sizeof(g_bigru_trace)));
    return 0;
}
#endif

extern "C" int taco_bigru_fwd_h0(const float* xp, const float* Wg_h_fw, const float* Wc_h_fw, const float* Wg_h_bw,
                                 const float* Wc_h_bw, const float* h0_fw, const float* h0_bw, float* out, int B, int T,
                                 void* stream) {
    // the operands of an empty sequence may be NULL (torch's empty tensors have no storage); the weights never may
    TACO_CHECK(Wg_h_fw && Wc_h_fw && Wg_h_bw && Wc_h_bw && ((xp && out) || (int64_t)B * T == 0), "taco_bigru_fwd: NULL pointer");
    TACO_CHECK(B >= 0 && T >= 0, "taco_bigru_fwd: negative size");
    TACO_CHECK((int64_t)B * T * 768 < (int64_t)1 << 31, "taco_bigru_fwd: B*T = %lld too large for 32-bit offsets", (long long)B * T);
    if (B == 0 || T == 0) return 0;
    dim3 grid(B, 2);
    TACO_LAUNCH(bigru_kernel, grid, NT, 0, (cudaStream_t)stream, xp, Wg_h_fw, Wc_h_fw, Wg_h_bw, Wc_h_bw, h0_fw, h0_bw, out, T);
    TACO_LAUNCH_CHECK();
    return 0;
}

extern "C" int taco_bigru_fwd(const float* xp, const float* Wg_h_fw, const float* Wc_h_fw, const float* Wg_h_bw,
                              const float* Wc_h_bw, float* out, int B, int T, void* stream) {
    return taco_bigru_fwd_h0(xp, Wg_h_fw, Wc_h_fw, Wg_h_bw, Wc_h_bw, nullptr, nullptr, out, B, T, stream);
}
