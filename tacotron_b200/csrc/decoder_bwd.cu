// decoder_bwd.cu -- serial part of the attention-decoder backward: back-propagation through the T steps of
// BasicDecoder(OutputProjectionWrapper(InputProjectionWrapper(ResidualWrapper(MultiRNNCell(3 x GRUCell(256))))),
// AttentionWrapper(BahdanauAttention), Training/ScheduledOutputTrainingHelper)   models/tacotron.py:46-105, :136-138.
//
// The caller (tacotron_b200/models/grad.py::decoder_bwd) has already recomputed, in batch, every activation of
// every step from what the forward kernel saved (y, alignments, the three GRU state sequences), and will turn the
// PRE-ACTIVATION gradients this kernel stores per step into all weight gradients with batched GEMMs.  What is left
// here is the data-gradient chain, which really is serial in t.  v3: 9 dependent stages per step instead of 11 -- as in the
// forward kernel, products of WEIGHTS are formed once per call (taco_gemm, a few hundred microseconds of work for 200 steps)
// so that two linear stages with nothing non-linear between them become one:
//
//   A   attention of step t: dalign = dctx.values, softmax backward -> dscore, dpq = sum_j dscore_j v (1-e_j^2)
//                                        (+ pre-net L2 backward of step t+1: dpn1(t+1), and its sel-masked copy)
//   4'  dres = E(t) + [dattn(t) | dpq(t) | sel.dpn1(t+1)] . [M1 | M2 | M4]^T ; GRU3 element-wise part
//          E  = dy_ext . W_out^T                   (all steps at once, before the kernel)
//          M1 = W_out . W_a[:OUT]   (dattn -> dy_att -> dres)     M2 = W_out . W_q   (dpq -> dy -> dres)
//          M4 = W_out[:, mel(r-1)] . W1            (dpn1(t+1) -> dx(t+1) -> dy(t) -> dres; scheduled-sampling rows only)
//   5,6 x3  GRU_i:  [dIN_c | drh] = dc_pre.Wc_i^T ;  [dIN_g | dh_g] = [dr_pre,du_pre].Wg_i^T ; carries
//   7'  [dpn2(t) | dattn(t-1) | dctx(t-1)] = dz . [W_in | Mctx]^T ,  Mctx = W_a[OUT:] . W_in[128:]  (dattn(t-1) -> dctx(t-1))
//
// dy(t) itself (needed only for the weight gradients) and dx are formed for all steps at once after the kernel:
// dy = dy_ext + dattn.W_a[:OUT]^T + dpq.W_q^T + sel(t+1).dx(t+1),  dx = dpn1.W1^T.
//
// One cooperative kernel runs all T steps; stages are separated by grid.sync().  Every stage is a skinny GEMM
// out[32 x N] = in[32 x K] . W^T with W rows contiguous (TF [in,out] layouts make every data-gradient a "NT"
// product).  v2 schedule (v1: one warp per output column, the whole 32 x K input staged in shared memory by every CTA
// and re-read from there once per column: bound by shared-memory traffic and by L2 weight-row loads):
//   * a CTA owns C = ceil(N / grid) CONSECUTIVE output columns of every GEMM; their weight rows (C x K floats, 55 KB in
//     total per CTA at r = 5) are copied into shared memory ONCE and stay there for all T steps;
//   * the 8 warps split K; lane = batch row reads its K/8 slice of the input straight from L2 into registers (every
//     input element is read once per CTA and reused for all C columns), weights are shared-memory broadcasts;
//   * per-warp partial sums are combined through shared memory, one thread per (row, column) runs the stage epilogue.
// Inter-stage data lives in L2 (ld.global.cg; never the non-coherent path).
// Semantics pinned by tests/mirror_kernels.py::decoder_bwd.
#ifndef TACO_HOST_EMU
#include <cooperative_groups.h>
#endif
#include "common.cuh"

#ifndef TACO_HOST_EMU
namespace cg = cooperative_groups;
#endif                              // (the host emulation, tests/cuda_emu/emu.h, provides cg:: for a 1-CTA grid)

namespace {

constexpr int U = 256;        // decoder / attention units
constexpr int RB = 32;        // rows (utterances) per launch
constexpr int NW = 8;         // warps per CTA
constexpr int MAXK = 768;     // widest contraction: stage 4' (dattn | dpq | dpn1)
constexpr int CB = 8;         // output columns processed per pass (register accumulators per lane)
constexpr int NGEMM = 9;      // GEMMs per step (weight-row cache slots)

struct DecBwdP {
    int B, T, Tx, OUT, MF;
    float ks;
    const float *W_a, *W_q, *W_out, *W_in, *W1, *W2, *v, *Wg[3], *Wc[3];
    const float *dy_ext, *RU[3], *C[3], *Hs[3], *align, *values, *keys, *PQ, *PN1, *PN2;
    const uint8_t* sel;
    float *DATT, *DY, *DPQ, *DSCORE, *DCTX, *DG[3], *DC[3], *DZ, *DPN2, *DPN1, *DX;
    const float *M124, *M7, *E;   // fused weights [U][768], [640][U]; E = dy_ext . W_out^T  [T][B][U]   (workspace, see host)
    const float* H0[3];           // [B][U] initial states h_i(-1), or NULL (zero state)
    const float* dscore_add;      // [B][T][Tx] added to the softmax backward's dscore (guided attention), or NULL
    float* ws;
    unsigned int* bar;       // grid-barrier counter (zeroed by the host before the launch)
    int cache_weights;       // 1: this CTA's weight rows fit in shared memory (the normal case); 0: read them from L2
};

// scratch layout (floats): every buffer is [32][ld]
constexpr int WS_XC = 0;                          // [32][768] input of stage 4': dattn(t) | dpq(t) | sel.dpn1(t+1)
constexpr int WS_DRES = WS_XC + RB * 768;         // [32][256]
constexpr int WS_DINC = WS_DRES + RB * U;         // [32][256]
constexpr int WS_DHR = WS_DINC + RB * U;          // [32][256]
constexpr int WS_DHU = WS_DHR + RB * U;           // [3][32][256]
constexpr int WS_DHC = WS_DHU + 3 * RB * U;       // [3][32][256]   carries, zeroed by the host
constexpr int WS_BAR = WS_DHC + 3 * RB * U;       // grid-barrier counter (1 word, padded)
constexpr int WS_ZERO_END = WS_BAR + 32;          // [0, WS_ZERO_END) is zeroed by the host before every launch
constexpr int WS_M124 = WS_ZERO_END;              // [256][768]
constexpr int WS_M7 = WS_M124 + U * 768;          // [640][256]
constexpr int WS_E = WS_M7 + 640 * U;             // [T][B][256], T <= WS_MAXT
constexpr int WS_MAXT = 1024;
constexpr int WS_TOTAL = WS_E + WS_MAXT * RB * U;

// One block of <= CB output columns: res[c][row] = sum_k in[row][k] * W[nb + c][k]  (row = lane), left in part_s + NW*CB*32.
// wc: the block's weight rows [nc][K] in shared memory, or nullptr (rows are then read from global memory).
// NOT inlined: the fully unrolled body is ~1000 instructions and the step has 12 GEMMs -- inlined copies made the kernel
// 255 KB of code and every stage started with a cold instruction cache (ncu: 11 % issue utilisation, 13 K cycles per stage).
#ifdef TACO_HOST_EMU
#define TACO_NOINLINE
static inline float __fadd_rn(float a, float b) { return a + b; }     // (host: one IEEE add, like the device intrinsic)
#else
#define TACO_NOINLINE __noinline__
#endif
__device__ TACO_NOINLINE void gemm_block(float* part_s, const float* in, int ldi, int rows, int K, const float* __restrict__ W, int ldw,
                                         int nb, int nc, const float* wc) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int K4 = K >> 2;
    const int cpw = (K4 + NW - 1) / NW;                  // 16-byte chunks of K per warp
    const int c_lo = warp * cpw, c_hi = (c_lo + cpw < K4) ? c_lo + cpw : K4;
    const float4* arow = reinterpret_cast<const float4*>(in + (int64_t)lane * ldi);
    const bool live = lane < rows;
    // this lane's slice of its input row: up to 24 independent 16-byte L2 loads (K <= 768), all in flight before the first product
    constexpr int MAXC = MAXK / 4 / NW;                  // 24
    float4 av[MAXC];
#pragma unroll
    for (int i = 0; i < MAXC; ++i)
        av[i] = (live && c_lo + i < c_hi) ? __ldcg(arow + c_lo + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    float acc[CB];
#pragma unroll
    for (int c = 0; c < CB; ++c) acc[c] = 0.f;
#pragma unroll
    for (int i = 0; i < MAXC; ++i) {
        const int k4 = c_lo + i;
        if (k4 >= c_hi) break;                           // warp-uniform
        const float4 a = av[i];
#pragma unroll
        for (int c = 0; c < CB; ++c) {
            if (c < nc) {                                // warp-uniform
                const float4 w = wc ? *reinterpret_cast<const float4*>(wc + (size_t)c * K + 4 * k4)
                                    : __ldg(reinterpret_cast<const float4*>(W + (int64_t)(nb + c) * ldw) + k4);
                acc[c] = fmaf(a.x, w.x, acc[c]); acc[c] = fmaf(a.y, w.y, acc[c]);
                acc[c] = fmaf(a.z, w.z, acc[c]); acc[c] = fmaf(a.w, w.w, acc[c]);
            }
        }
    }
#pragma unroll
    for (int c = 0; c < CB; ++c)
        if (c < nc) part_s[(warp * CB + c) * 32 + lane] = acc[c];
    __syncthreads();
    if (tid < nc * 32) {                                 // one thread per (column, row)
        const int c = tid >> 5;
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < NW; ++w) v += part_s[(w * CB + c) * 32 + lane];
        part_s[NW * CB * 32 + tid] = v;
    }
    __syncthreads();
}

// columns of GEMM `N` owned by this CTA: C = ceil(N / grid) consecutive columns; `reverse` deals them from the last CTA
// backwards so that the two GEMMs of one stage land on different CTAs
__host__ __device__ inline void cta_columns(int N, int G, int cta, bool reverse, int& n0, int& n1) {
    const int C = (N + G - 1) / G;
    const int c = reverse ? (G - 1 - cta) : cta;
    n0 = c * C;
    n1 = n0 + C < N ? n0 + C : N;
    if (n0 > N) n0 = N;
}

__host__ __device__ inline int side_gemm_ctas(int G, int B) { return (G >= 2 * B) ? G - B : G; }

// the 9 GEMMs of a step (weight-row cache slots): output columns N and contraction length K
constexpr int GEMM_N[NGEMM] = {256, U, 2 * U, 2 * U, 2 * U, 2 * U, 2 * U, 2 * U, 640};
constexpr int GEMM_K[NGEMM] = {128, 768, U, 2 * U, U, 2 * U, U, 2 * U, U};
constexpr size_t SMEM_LIMIT = 200 * 1024;                 // dynamic shared memory the kernel may take
constexpr size_t SMEM_PARTIALS = ((size_t)NW * CB * 32 + CB * 32) * 4;

// floats of one CTA's weight-row cache on a grid of G CTAs: ceil(N / ctas) rows of K per GEMM (the largest share any CTA
// gets; cta_columns deals the columns of GEMM 0 over the side_gemm_ctas(G, B) CTAs, every other GEMM over all G)
inline size_t cache_floats(int G, int B) {
    size_t f = 0;
    for (int g = 0; g < NGEMM; ++g) {
        const int ctas = (g == 0) ? side_gemm_ctas(G, B) : G;
        f += (size_t)(((GEMM_N[g] + ctas - 1) / ctas) * GEMM_K[g] + 3) & ~(size_t)3;
    }
    return f;
}

// out[row][n] = sum_k in[row][k] * W[n][k] for this CTA's columns, then the stage epilogue per (row, column).
// pre(row, n) runs BEFORE the product and returns the saved activations / carries the epilogue of (row, n) needs: those L2
// loads then travel together with the GEMM's input loads instead of after the reduction.
struct Pre { float x0, x1, x2, x3, x4; };
template <class PreF, class Epi>
__device__ __forceinline__ void skinny_gemm(float* part_s, const float* in, int ldi, int rows, int K, const float* __restrict__ W, int ldw,
                                            int N, int geff, const float* wc, PreF pre, Epi epi) {
    int n0, n1;
    cta_columns(N, geff, (int)blockIdx.x, false, n0, n1);    // geff < grid: only the first geff CTAs take columns
    for (int nb = n0; nb < n1; nb += CB) {               // one block at 128 CTAs (<= 6 columns per CTA), up to three at 32
        const int nc = (n1 - nb < CB) ? n1 - nb : CB;
        const int tid = threadIdx.x;
        Pre pr = {0.f, 0.f, 0.f, 0.f, 0.f};
        if (tid < nc * 32) pr = pre(tid & 31, nb + (tid >> 5));
        gemm_block(part_s, in, ldi, rows, K, W, ldw, nb, nc, wc ? wc + (size_t)(nb - n0) * K : nullptr);
        if (tid < nc * 32) epi(tid & 31, nb + (tid >> 5), part_s[NW * CB * 32 + tid], pr);
        __syncthreads();                                 // part_s is reused
    }
}

// Grid barrier on a monotonically increasing counter (all CTAs are co-resident: cooperative launch).  One release-add and
// an acquire-poll per CTA: cheaper than the cooperative-groups grid.sync() it replaces.
struct GridBar {
    unsigned int* ctr;
    unsigned int target;
    unsigned int G;
#ifdef TACO_HOST_EMU
    __device__ void sync() { __syncthreads(); }
#else
    __device__ __forceinline__ void sync() {
        __syncthreads();
        if (threadIdx.x == 0) {
            target += G;
            red_release_add(ctr, 1u);
            unsigned int spins = 0;
            while (ld_acquire(ctr) < target) { if (++spins > (1u << 26)) __trap(); }
        }
        __syncthreads();
    }
#endif
};

__global__ void __launch_bounds__(256, 1) decoder_bwd_kernel(const DecBwdP p) {
    GridBar grid{p.bar, 0u, gridDim.x};
#ifdef TACO_HOST_EMU
    float* dyn_s = emu::dynamic_smem();
#else
    extern __shared__ __align__(16) float dyn_s[];       // [NW][CB][32] partial sums | cached weight rows of this CTA
#endif
    float* in_s = dyn_s;                                 // (partial-sum scratch of skinny_gemm)
    __shared__ float dctx_s[U], dal_s[256], ds_s[256], red_s[NW];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int B = p.B, T = p.T, Tx = p.Tx, OUT = p.OUT, MF = p.MF;
    const int lo = OUT - MF;
    float* xc = p.ws + WS_XC;
    float* dres = p.ws + WS_DRES;
    float* dINc = p.ws + WS_DINC;
    float* dhr = p.ws + WS_DHR;
    float* dhu = p.ws + WS_DHU;
    float* dhc = p.ws + WS_DHC;
    (void)lo;
    // the attention of stage A runs on the last B CTAs (one utterance each); the side GEMM of that stage goes to the others
    const int side_ctas = side_gemm_ctas((int)gridDim.x, B);

    // ---- weight-row cache: for each of the 9 GEMMs of a step, the rows of this CTA's columns, copied once ----
    const float* wcp[NGEMM];
    {
        const float* Wm[NGEMM] = {p.W2, p.M124, p.Wc[2], p.Wg[2], p.Wc[1], p.Wg[1], p.Wc[0], p.Wg[0], p.M7};
        const int Nn[NGEMM] = {256, U, 2 * U, 2 * U, 2 * U, 2 * U, 2 * U, 2 * U, 640};     // = GEMM_N, GEMM_K (host)
        const int Kk[NGEMM] = {128, 768, U, 2 * U, U, 2 * U, U, 2 * U, U};
        float* cur = dyn_s + NW * CB * 32 + CB * 32;
        for (int g = 0; g < NGEMM; ++g) {
            int n0, n1;
            cta_columns(Nn[g], g == 0 ? side_ctas : (int)gridDim.x, (int)blockIdx.x, false, n0, n1);
            wcp[g] = nullptr;
            if (p.cache_weights && n1 > n0) {
                wcp[g] = cur;
                const int cnt = (n1 - n0) * Kk[g];       // rows are contiguous in W (ldw == K for every GEMM here)
                const float* src = Wm[g] + (int64_t)n0 * Kk[g];
                for (int i = tid; i < cnt; i += blockDim.x) cur[i] = __ldg(src + i);
                cur += (cnt + 3) & ~3;
            }
        }
        __syncthreads();
    }

    // element-wise head of GRU layer i at step t for (row, unit n): consumes the gradient arriving at h_i(t).
    // head_pre loads what it needs (carry, h(t-1), u, c) ahead of the product that delivers dh_in.
    auto head_pre = [&](int i, int t, int row, int n, Pre& q) {
        const int64_t o = (int64_t)t * B + row;
        q.x0 = __ldcg(dhc + (i * RB + row) * U + n);
        q.x1 = (t > 0) ? __ldg(p.Hs[i] + (o - B) * U + n) : (p.H0[i] ? __ldg(p.H0[i] + row * U + n) : 0.f);
        q.x2 = __ldg(p.RU[i] + o * 2 * U + U + n);
        q.x3 = __ldg(p.C[i] + o * U + n);
    };
    auto gru_head = [&](int i, int t, int row, int n, float dh_in, const Pre& q) {
        const int64_t o = (int64_t)t * B + row;
        const float dh = dh_in + q.x0;
        const float hprev = q.x1, u = q.x2, c = q.x3;
        p.DG[i][o * 2 * U + U + n] = dh * (hprev - c) * u * (1.0f - u);     // du_pre
        p.DC[i][o * U + n] = dh * (1.0f - u) * (1.0f - c * c);               // dc_pre
        dhu[(i * RB + row) * U + n] = dh * u;
    };
    const Pre pre0 = {0.f, 0.f, 0.f, 0.f, 0.f};

    for (int t = T - 1; t >= -1; --t) {
        const int tt = t + 1;
        // ================= stage A: attention scores backward of step t  |  pre-net layer 2 backward of step t+1 ==========
        if (t >= 0) {
            for (int b = (int)gridDim.x - 1 - (int)blockIdx.x; b < B; b += gridDim.x) {
                dctx_s[tid] = __ldcg(p.DCTX + ((int64_t)t * B + b) * U + tid);
                __syncthreads();
                // dalign_j = dctx . values_j, four positions per warp and pass: 32 independent L2 loads are in flight before
                // the first product (one position at a time exposed the L2 latency Tx/8 times per step)
                for (int j0 = warp; j0 < Tx; j0 += 4 * NW) {
                    float vv[4][U / 32];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int j = j0 + q * NW;
                        const float* vj = p.values + ((int64_t)b * Tx + (j < Tx ? j : j0)) * U;
#pragma unroll
                        for (int i = 0; i < U / 32; ++i) vv[q][i] = __ldg(vj + lane + 32 * i);
                    }
                    float s4[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        float sq = 0.f;
#pragma unroll
                        for (int i = 0; i < U / 32; ++i) sq = fmaf(dctx_s[lane + 32 * i], vv[q][i], sq);
                        s4[q] = sq;
                    }
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
                        for (int q = 0; q < 4; ++q) s4[q] += __shfl_xor_sync(0xffffffffu, s4[q], o);
                    }
                    if (lane == 0) {
#pragma unroll
                        for (int q = 0; q < 4; ++q) if (j0 + q * NW < Tx) dal_s[j0 + q * NW] = s4[q];
                    }
                }
                __syncthreads();
                const float aj = (tid < Tx) ? __ldg(p.align + ((int64_t)b * T + t) * Tx + tid) : 0.f;
                // issued with the align load, so its L2 latency overlaps the reduction below instead of following it
                const float dsa = (p.dscore_add && tid < Tx) ? __ldg(p.dscore_add + ((int64_t)b * T + t) * Tx + tid) : 0.f;
                float part = (tid < Tx) ? aj * dal_s[tid] : 0.f;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
                if (lane == 0) red_s[warp] = part;
                __syncthreads();
                float tot = 0.f;
#pragma unroll
                for (int w = 0; w < NW; ++w) tot += red_s[w];
                if (tid < Tx) {                                              // softmax backward
                    float ds = aj * (dal_s[tid] - tot);
                    if (p.dscore_add) ds = __fadd_rn(ds, dsa);            // (never fused with the product: NULL keeps it as it was)
                    ds_s[tid] = ds;
                    p.DSCORE[((int64_t)b * T + t) * Tx + tid] = ds;
                }
                __syncthreads();
                {                                                            // dpq_d = v_d sum_j dscore_j (1 - e_jd^2)
                    const int d = tid;
                    const float pq = __ldg(p.PQ + ((int64_t)t * B + b) * U + d);
                    const float* kb = p.keys + (int64_t)b * Tx * U + d;
                    float acc = 0.f;
                    // eight keys in flight per batch, no data-dependent branch (masked positions carry dscore = 0 and
                    // finite keys): the one-at-a-time loop paid one L2 latency per position
                    int j = 0;
                    for (; j + 8 <= Tx; j += 8) {
                        float kk[8];
#pragma unroll
                        for (int q = 0; q < 8; ++q) kk[q] = __ldg(kb + (int64_t)(j + q) * U);
#pragma unroll
                        for (int q = 0; q < 8; ++q) {
                            const float e = tanhf_acc(kk[q] + pq);
                            acc = fmaf(ds_s[j + q], 1.0f - e * e, acc);
                        }
                    }
                    for (; j < Tx; ++j) {
                        const float e = tanhf_acc(__ldg(kb + (int64_t)j * U) + pq);
                        acc = fmaf(ds_s[j], 1.0f - e * e, acc);
                    }
                    const float dpq = acc * __ldg(p.v + d);
                    p.DPQ[((int64_t)t * B + b) * U + d] = dpq;
                    xc[b * 768 + U + d] = dpq;
                }
                __syncthreads();
            }
        }
        if (tt < T) {
            const float* in = p.DPN2 + (int64_t)tt * B * 128;
            skinny_gemm(in_s, in, 128, B, 128, p.W2, 128, 256, side_ctas, wcp[0],
                [&](int row, int n) {
                    Pre q = pre0;
                    if (row < B) { q.x0 = __ldg(p.PN1 + ((int64_t)tt * B + row) * 256 + n); q.x1 = p.sel[(int64_t)tt * B + row] ? 1.f : 0.f; }
                    return q;
                },
                [&](int row, int n, float v, const Pre& q) {
                    if (row >= B) return;
                    const float d1 = (q.x0 > 0.f) ? v * p.ks : 0.f;
                    p.DPN1[((int64_t)tt * B + row) * 256 + n] = d1;
                    xc[row * 768 + 2 * U + n] = (q.x1 != 0.f) ? d1 : 0.f;             // only sampled inputs pass gradient to y(t)
                });
        }
        grid.sync();
        if (t < 0) break;
        // ================= stage 4': everything that arrives at the residual output, GRU3 head ==========================
        {
            skinny_gemm(in_s, xc, 768, B, 768, p.M124, 768, U, (int)gridDim.x, wcp[1],
                [&](int row, int n) {
                    Pre q = pre0;
                    if (row < B) { head_pre(2, t, row, n, q); q.x4 = __ldg(p.E + ((int64_t)t * B + row) * U + n); }
                    return q;
                },
                [&](int row, int n, float v, const Pre& q) {
                    if (row >= B) return;
                    const float dr = q.x4 + v;
                    dres[row * U + n] = dr;
                    gru_head(2, t, row, n, dr, q);
                });
        }
        grid.sync();
        // ================= stages 5/6 x 3: the GRU stack, top to bottom ===============================================
        for (int i = 2; i >= 0; --i) {
            {   // [dIN_c | drh] = dc_pre . Wc_i^T
                const float* in = p.DC[i] + (int64_t)t * B * U;
                skinny_gemm(in_s, in, U, B, U, p.Wc[i], U, 2 * U, (int)gridDim.x, wcp[2 + 2 * (2 - i)],
                    [&](int row, int n) {
                        Pre q = pre0;
                        if (row < B && n >= U) {
                            const int64_t o = (int64_t)t * B + row;
                            q.x0 = (t > 0) ? __ldg(p.Hs[i] + (o - B) * U + (n - U))
                                           : (p.H0[i] ? __ldg(p.H0[i] + row * U + (n - U)) : 0.f);
                            q.x1 = __ldg(p.RU[i] + o * 2 * U + (n - U));
                        }
                        return q;
                    },
                    [&](int row, int n, float v, const Pre& q) {
                        if (row >= B) return;
                        if (n < U) { dINc[row * U + n] = v; return; }
                        const int k = n - U;
                        const int64_t o = (int64_t)t * B + row;
                        const float hprev = q.x0, r = q.x1;
                        p.DG[i][o * 2 * U + k] = v * hprev * r * (1.0f - r);     // dr_pre
                        dhr[row * U + k] = v * r;
                    });
            }
            grid.sync();
            {   // [dIN_g | dh_g] = [dr_pre, du_pre] . Wg_i^T
                const float* in = p.DG[i] + (int64_t)t * B * 2 * U;
                skinny_gemm(in_s, in, 2 * U, B, 2 * U, p.Wg[i], 2 * U, 2 * U, (int)gridDim.x, wcp[3 + 2 * (2 - i)],
                    [&](int row, int n) {                                    // (everything here was written at least one barrier ago)
                        Pre q = pre0;
                        if (row >= B) return q;
                        if (n < U) {
                            q.x4 = __ldcg(dINc + row * U + n);
                            if (i > 0) head_pre(i - 1, t, row, n, q);
                            else q.x0 = __ldcg(dres + row * U + n);
                        } else {
                            q.x0 = __ldcg(dhu + (i * RB + row) * U + (n - U));
                            q.x1 = __ldcg(dhr + row * U + (n - U));
                        }
                        return q;
                    },
                    [&](int row, int n, float v, const Pre& q) {
                        if (row >= B) return;
                        if (n < U) {
                            const float dIN = q.x4 + v;                     // gradient at the layer input
                            if (i > 0) gru_head(i - 1, t, row, n, dIN, q);
                            else p.DZ[((int64_t)t * B + row) * U + n] = q.x0 + dIN;
                        } else {
                            dhc[(i * RB + row) * U + (n - U)] = q.x0 + q.x1 + v;
                        }
                    });
            }
            grid.sync();
        }
        // ================= stage 7': input projection backward, through to the attention context of step t-1 ============
        {
            const float* in = p.DZ + (int64_t)t * B * U;
            skinny_gemm(in_s, in, U, B, U, p.M7, U, 640, (int)gridDim.x, wcp[8],
                [&](int row, int n) {
                    Pre q = pre0;
                    if (row < B && n < 128) q.x0 = __ldg(p.PN2 + ((int64_t)t * B + row) * 128 + n);
                    return q;
                },
                [&](int row, int n, float v, const Pre& q) {
                if (row >= B) return;
                if (n < 128) {
                    const int64_t o = ((int64_t)t * B + row) * 128 + n;
                    p.DPN2[o] = (q.x0 > 0.f) ? v * p.ks : 0.f;
                } else if (t > 0) {
                    if (n < 128 + U) {
                        p.DATT[((int64_t)(t - 1) * B + row) * U + (n - 128)] = v;
                        xc[row * 768 + (n - 128)] = v;
                    } else {
                        p.DCTX[((int64_t)(t - 1) * B + row) * U + (n - 128 - U)] = v;
                    }
                }
            });
        }
        grid.sync();
    }
}

// dy(t)[lo + m] += sel(t+1) * dx(t+1)[m]   (gradient of the sampled step inputs, ScheduledOutputTrainingHelper)
__global__ void dy_tail_kernel(float* DY, const float* __restrict__ DX, const uint8_t* __restrict__ sel, int T, int B, int OUT, int MF) {
    const int64_t total = (int64_t)(T - 1) * B * MF;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t rowi = i / MF;                     // (t, row) with t < T-1
        const int m = (int)(i - rowi * MF);
        if (sel[rowi + B]) DY[rowi * OUT + (OUT - MF) + m] += DX[(rowi + B) * MF + m];
    }
}

}  // namespace

#ifndef TACO_HOST_EMU
// co-resident CTAs of the backward kernel on the current device (computed once per device); also opts the kernel into
// SMEM_LIMIT bytes of dynamic shared memory there.  Used by taco_decoder_capacity (decoder.cu).
int decoder_bwd_capacity(int* out) {
    constexpr int MAX_DEVICES = 64;
    static int cap[MAX_DEVICES];
    int dev = 0;
    TACO_CUDA(cudaGetDevice(&dev));
    TACO_CHECK(dev >= 0 && dev < MAX_DEVICES, "taco_decoder_bwd: device %d out of range", dev);
    if (cap[dev] == 0) {
        TACO_CUDA(cudaFuncSetAttribute(decoder_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_LIMIT));
        int sms = 0, per_sm = 0;
        TACO_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        TACO_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, decoder_bwd_kernel, 256, SMEM_LIMIT));
        cap[dev] = sms * per_sm > 0 ? sms * per_sm : -1;
    }
    *out = cap[dev] > 0 ? cap[dev] : 0;
    return 0;
}
#endif

extern "C" size_t taco_decoder_bwd_workspace_bytes(void) { return (size_t)WS_TOTAL * 4; }

extern "C" int taco_decoder_bwd(const taco_decoder_bwd_args* a, void* stream) {
    TACO_CHECK(a, "taco_decoder_bwd: NULL args");
    TACO_CHECK(a->B >= 1 && a->B <= RB, "taco_decoder_bwd: B=%d must be in [1,%d] per launch", a->B, RB);
    TACO_CHECK(a->max_ctas == 0 || a->max_ctas >= 32, "taco_decoder_bwd: max_ctas=%d: the budget must be 0 (the device's "
               "capacity) or at least 32 CTAs", a->max_ctas);
    TACO_CHECK(a->T >= 1 && a->Tx >= 1 && a->Tx <= 256, "taco_decoder_bwd: T=%d Tx=%d (Tx <= 256)", a->T, a->Tx);
    TACO_CHECK(a->r >= 1 && 80 * a->r <= MAXK && ((80 * a->r) % 4) == 0, "taco_decoder_bwd: r=%d unsupported", a->r);
    TACO_CHECK(a->W_a && a->W_q && a->W_out && a->W_in && a->W1 && a->W2 && a->v, "taco_decoder_bwd: NULL weight");
    TACO_CHECK(a->dy_ext && a->align && a->values && a->keys && a->PQ && a->PN1 && a->PN2 && a->sel, "taco_decoder_bwd: NULL saved tensor");
    TACO_CHECK(a->DATT && a->DY && a->DPQ && a->DSCORE && a->DCTX && a->DZ && a->DPN2 && a->DPN1 && a->DX && a->workspace,
               "taco_decoder_bwd: NULL output");
    DecBwdP p;
    memset(&p, 0, sizeof(p));
    p.B = a->B; p.T = a->T; p.Tx = a->Tx; p.OUT = 80 * a->r; p.MF = 80; p.ks = a->keep_scale;
    p.W_a = a->W_a; p.W_q = a->W_q; p.W_out = a->W_out; p.W_in = a->W_in; p.W1 = a->W1; p.W2 = a->W2; p.v = a->v;
    for (int i = 0; i < 3; ++i) {
        TACO_CHECK(a->Wg[i] && a->Wc[i] && a->RU[i] && a->C[i] && a->H[i] && a->DG[i] && a->DC[i], "taco_decoder_bwd: NULL GRU tensor %d", i);
        p.Wg[i] = a->Wg[i]; p.Wc[i] = a->Wc[i]; p.RU[i] = a->RU[i]; p.C[i] = a->C[i]; p.Hs[i] = a->H[i];
        p.DG[i] = a->DG[i]; p.DC[i] = a->DC[i];
    }
    p.dy_ext = a->dy_ext; p.align = a->align; p.values = a->values; p.keys = a->keys; p.PQ = a->PQ; p.PN1 = a->PN1; p.PN2 = a->PN2;
    p.sel = a->sel;
    for (int i = 0; i < 3; ++i) p.H0[i] = a->H0[i];
    p.dscore_add = a->dscore_add;
    p.DATT = a->DATT; p.DY = a->DY; p.DPQ = a->DPQ; p.DSCORE = a->DSCORE; p.DCTX = a->DCTX; p.DZ = a->DZ; p.DPN2 = a->DPN2;
    p.DPN1 = a->DPN1; p.DX = a->DX;
    p.ws = a->workspace;
    p.bar = reinterpret_cast<unsigned int*>(a->workspace + WS_BAR);
    TACO_CHECK(a->T <= WS_MAXT, "taco_decoder_bwd: T=%d exceeds %d steps per launch", a->T, WS_MAXT);
#ifndef TACO_HOST_EMU
    // grid: G = min(budget, capacity, 128) CTAs; every CTA takes its columns from gridDim, so any G works.  The weight-row
    // cache is kept whenever it fits at that G (about 48 KB at 128 CTAs, 62 KB at 114, 98 KB at 64; not at 32)
    int capacity = 0;
    if (decoder_bwd_capacity(&capacity)) return 1;
    TACO_CHECK(capacity >= 32, "taco_decoder_bwd: only %d CTAs can be co-resident on this device (need 32)", capacity);
    int G = capacity < 128 ? capacity : 128;
    if (a->max_ctas > 0 && a->max_ctas < G) G = a->max_ctas;
    p.cache_weights = (SMEM_PARTIALS + cache_floats(G, a->B) * 4 <= SMEM_LIMIT) ? 1 : 0;
    const size_t smem = SMEM_PARTIALS + (p.cache_weights ? cache_floats(G, a->B) * 4 : 0);
#endif
    const int OUTh = 80 * a->r, MF = 80, lo = OUTh - MF;
    const int M = a->T * a->B;
    float* M124 = a->workspace + WS_M124;
    float* M7 = a->workspace + WS_M7;
    float* E = a->workspace + WS_E;
    p.M124 = M124; p.M7 = M7; p.E = E;
    // C[M x N] (ldc) = beta*C + A[M x K] (lda) . B   (tb: B stored [N][K], else [K][N]) through the library's own GEMM
    auto gemm = [&](float* Cm, int64_t ldc, const float* A, int64_t lda, const float* Bm, int64_t ldb, int Mm, int Nn, int Kk, int tb,
                    float beta) {
        taco_gemm_desc g;
        memset(&g, 0, sizeof(g));
        g.A = A; g.lda = lda; g.B = Bm; g.ldb = ldb; g.C = Cm; g.ldc = ldc; g.M = Mm; g.N = Nn; g.K = Kk; g.tb = tb; g.beta = beta;
        g.taps = 1; g.batch = 1;
        return taco_gemm(&g, stream);
    };
    // ---- weight-only products (once per call) and the part of dres that is known for all steps ----
    if (gemm(M124, 768, a->W_out, OUTh, a->W_a, U, U, U, OUTh, 0, 0.f)) return 1;                           // M1 = W_out . W_a[:OUT]
    if (gemm(M124 + U, 768, a->W_out, OUTh, a->W_q, U, U, U, OUTh, 0, 0.f)) return 1;                       // M2 = W_out . W_q
    if (gemm(M124 + 2 * U, 768, a->W_out + lo, OUTh, a->W1, 256, U, 256, MF, 0, 0.f)) return 1;             // M4 = W_out[:, lo:] . W1
    if (gemm(M7 + 384 * U, U, a->W_a + (int64_t)OUTh * U, U, a->W_in + 128 * U, U, U, U, U, 0, 0.f)) return 1;   // Mctx
    if (gemm(E, U, a->dy_ext, OUTh, a->W_out, OUTh, M, U, OUTh, 1, 0.f)) return 1;                          // E = dy_ext . W_out^T
    // after the serial kernel: dx and dy for all steps (outputs of the ABI; dy feeds the weight gradients)
    auto tail = [&]() -> int {
        if (gemm(a->DX, MF, a->DPN1, 256, a->W1, 256, M, MF, 256, 1, 0.f)) return 1;                        // dx = dpn1 . W1^T
        if (gemm(a->DY, OUTh, a->DATT, U, a->W_a, U, M, OUTh, U, 1, 1.f)) return 1;                         // dy += dattn . W_a[:OUT]^T
        if (gemm(a->DY, OUTh, a->DPQ, U, a->W_q, U, M, OUTh, U, 1, 1.f)) return 1;                          // dy += dpq . W_q^T
        return 0;
    };
#ifdef TACO_HOST_EMU
    // host emulation: one CTA (the kernel is written for any grid size), grid.sync() = block barrier
    p.cache_weights = 0;                                 // one CTA owns every column: rows come from global memory
    memcpy(M7, a->W_in, (size_t)384 * U * 4);
    memset(a->workspace, 0, (size_t)WS_ZERO_END * 4);
    memset(a->DATT + (int64_t)(a->T - 1) * a->B * U, 0, (size_t)a->B * U * 4);
    memset(a->DCTX + (int64_t)(a->T - 1) * a->B * U, 0, (size_t)a->B * U * 4);
    memcpy(a->DY, a->dy_ext, (size_t)M * OUTh * 4);
    emu::launch(dim3(1), dim3(256), [&] { decoder_bwd_kernel(p); });
    ++g_taco_launches;
    if (a->DH0)                                          // after step 0 the GRU carries are d(loss)/d(h_i(-1))
        for (int i = 0; i < 3; ++i) memcpy(a->DH0 + (int64_t)i * a->B * U, a->workspace + WS_DHC + (int64_t)i * RB * U, (size_t)a->B * U * 4);
    if (tail()) return 1;
    {
        float* DY = a->DY; const float* DX = a->DX; const uint8_t* sel = a->sel; const int T = a->T, B = a->B;
        emu::launch(dim3(1), dim3(256), [&] { dy_tail_kernel(DY, DX, sel, T, B, OUTh, MF); });
    }
    ++g_taco_launches;
    return 0;
#else
    cudaStream_t st = (cudaStream_t)stream;
    TACO_CUDA(cudaMemcpyAsync(M7, a->W_in, (size_t)384 * U * 4, cudaMemcpyDeviceToDevice, st));
    // carries and the stage-4' input start at zero; dattn(T-1) = dctx(T-1) = 0 (the last attention state feeds nothing)
    TACO_CUDA(cudaMemsetAsync(a->workspace, 0, (size_t)WS_ZERO_END * 4, st));
    TACO_CUDA(cudaMemsetAsync(a->DATT + (int64_t)(a->T - 1) * a->B * U, 0, (size_t)a->B * U * 4, st));
    TACO_CUDA(cudaMemsetAsync(a->DCTX + (int64_t)(a->T - 1) * a->B * U, 0, (size_t)a->B * U * 4, st));
    TACO_CUDA(cudaMemcpyAsync(a->DY, a->dy_ext, (size_t)M * OUTh * 4, cudaMemcpyDeviceToDevice, st));
    void* args[] = {(void*)&p};
    TACO_CUDA(cudaLaunchCooperativeKernel((void*)decoder_bwd_kernel, dim3(G), dim3(256), args, smem, st));
    ++g_taco_launches;
    if (a->DH0)                                          // after step 0 the GRU carries are d(loss)/d(h_i(-1))
        TACO_CUDA(cudaMemcpy2DAsync(a->DH0, (size_t)a->B * U * 4, a->workspace + WS_DHC, (size_t)RB * U * 4, (size_t)a->B * U * 4, 3,
                                    cudaMemcpyDeviceToDevice, st));
    if (tail()) return 1;
    if (a->T > 1) {
        const int64_t total = (int64_t)(a->T - 1) * a->B * MF;
        int blocks = (int)((total + 255) / 256);
        if (blocks > TACO_SMS * 8) blocks = TACO_SMS * 8;
        dy_tail_kernel<<<blocks, 256, 0, st>>>(a->DY, a->DX, a->sel, a->T, a->B, OUTh, MF);
        TACO_LAUNCH_CHECK();
    }
    return 0;
#endif
}
