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
// REGISTER FILE of the CTA's 512 threads (96 floats each) for the whole sequence.
//
// Thread mapping (v4).  History: v1 one thread per column, every thread re-reading all of h: shared-memory -> register
// bandwidth bound; v2 lanes split K 32 ways, 16-to-1 halving butterfly: issue bound (half the instructions butterfly);
// v3 4 lanes per hidden unit: bandwidth bound again (128 B of h per thread and mat-vec).  v4 sits between: a GROUP OF 8 LANES owns two hidden units
// (their r, u gate columns and candidate columns: 6 columns), the 8 lanes split K (16 rows each: 64 B of h per mat-vec and
// thread = 32 KB per phase), products are taken two k at a time (on the h pair as it comes out of a 16-byte
// shared load) and the 8-lane reduction is a transposing butterfly (4 -> 2 -> 1 values): 7 shuffles per step.
#include "common.cuh"

namespace {

constexpr int H = 128;

// d.x += a.x * b.x ; d.y += a.y * b.y  (Hopper has no packed fp32 FMA: two FFMAs)
__device__ __forceinline__ void ffma2(float2& d, const float2 a, const float2 b) {
    d.x = fmaf(a.x, b.x, d.x);
    d.y = fmaf(a.y, b.y, d.y);
}

__global__ void __launch_bounds__(512, 1)
bigru_kernel(const float* __restrict__ xp, const float* __restrict__ Wg_fw, const float* __restrict__ Wc_fw,
             const float* __restrict__ Wg_bw, const float* __restrict__ Wc_bw, const float* __restrict__ h0_fw,
             const float* __restrict__ h0_bw, float* __restrict__ out, int T) {
    const int b = blockIdx.x;
    const int dir = blockIdx.y;
    const int tid = threadIdx.x, lane = tid & 31;
    const int grp = tid >> 3;                  // 8-lane group: hidden units 2*grp, 2*grp + 1
    const int l3 = tid & 7;                    // K slice: the 16-byte chunks 8i + l3, i = 0..3 (a group reads 128 contiguous bytes)
    const float* Wg = dir ? Wg_bw : Wg_fw;     // [128][256]  h-side rows of the gates kernel (columns: r then u)
    const float* Wc = dir ? Wc_bw : Wc_fw;     // [128][128]  (r*h)-side rows of the candidate kernel

    __shared__ __align__(16) float h_s[H];
    __shared__ __align__(16) float rh_s[H];
    __shared__ float u_s[H];

    // weights as k-pairs: wg[c][2i+p] = (W[k][col_c], W[k+1][col_c]), k = 4*(8i + l3) + 2p;
    // gate columns c = 0..3: r(j0), u(j0), r(j1), u(j1); candidate columns c = 0..1: j0, j1
    const int j0 = 2 * grp;
    float2 wg[4][8], wc[2][8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int p = 0; p < 2; ++p) {
            const int k = 4 * (8 * i + l3) + 2 * p;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int col = (c & 1) * H + j0 + (c >> 1);
                wg[c][2 * i + p] = make_float2(__ldg(Wg + (int64_t)k * 256 + col), __ldg(Wg + (int64_t)(k + 1) * 256 + col));
            }
#pragma unroll
            for (int c = 0; c < 2; ++c)
                wc[c][2 * i + p] = make_float2(__ldg(Wc + (int64_t)k * 128 + j0 + c), __ldg(Wc + (int64_t)(k + 1) * 128 + j0 + c));
        }
    }
    // after the butterflies: lane pair (l3 >> 1) of the group holds gate column gc = 2*bit2 + bit1 -> unit j0 + bit2, gate bit1;
    // lane quad (l3 >> 2) holds the candidate column of unit j0 + bit2
    const int gj = j0 + ((l3 >> 2) & 1);
    const bool g_is_u = (l3 >> 1) & 1;
    const bool g_owner = (l3 & 1) == 0;
    const bool c_owner = (l3 & 3) == 0;

    const float* h0 = dir ? h0_bw : h0_fw;     // initial state (ops.py:111-126): speaker-dependent, or NULL = zero state
    if (tid < H) h_s[tid] = h0 ? __ldg(h0 + b * H + tid) : 0.0f;
    __syncthreads();

    // pointers advance by one time step per iteration (no per-step index arithmetic); the input products are prefetched
    // three steps ahead (they do not depend on h and stream from HBM), rotating through three named registers
    // (32-bit element offsets: the host checks B*T*768 < 2^31)
    const int seq = b * T;
    const int t_first = dir ? (T - 1) : 0;
    const int xs = dir ? -768 : 768, os = dir ? -256 : 256;
    int xgp = (seq + t_first) * 768 + dir * 384 + (g_is_u ? H : 0) + gj;     // this lane's hoisted gate product
    int outp = (seq + t_first) * 256 + dir * H + gj;
    const int xc_off = 256 + gj - ((g_is_u ? H : 0) + gj);                  // candidate product relative to xgp

    float xg0 = 0.f, xg1 = 0.f, xg2 = 0.f, xc0 = 0.f, xc1 = 0.f, xc2 = 0.f;
    if (T > 0) { if (g_owner) xg0 = __ldg(xp + xgp); if (c_owner) xc0 = __ldg(xp + xgp + xc_off); }
    if (T > 1) { if (g_owner) xg1 = __ldg(xp + xgp + xs); if (c_owner) xc1 = __ldg(xp + xgp + xs + xc_off); }
    if (T > 2) { if (g_owner) xg2 = __ldg(xp + xgp + 2 * xs); if (c_owner) xc2 = __ldg(xp + xgp + 2 * xs + xc_off); }
    xgp += 3 * xs;                             // -> the row of step + 3

    const float4* h4 = reinterpret_cast<const float4*>(h_s) + l3;
    const float4* rh4 = reinterpret_cast<const float4*>(rh_s) + l3;
    const bool b2 = (l3 & 4) != 0, b1 = (l3 & 2) != 0;

    // one time step: consumes (xg, xc), refills them with the products of step + 3 when `more`
    auto one_step = [&](float& xg, float& xc, bool more) {
        const float xgv = xg, xcv = xc;
        if (more) {
            if (g_owner) xg = __ldg(xp + xgp);
            if (c_owner) xc = __ldg(xp + xgp + xc_off);
        }
        xgp += xs;
        // ---- gates: h . Wg_h (this lane: 16 rows x 4 columns) ----
        {
            float2 a0 = make_float2(0.f, 0.f), a1 = a0, a2 = a0, a3 = a0;
            float4 hv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) hv[i] = h4[8 * i];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 lo = make_float2(hv[i].x, hv[i].y), hi = make_float2(hv[i].z, hv[i].w);
                ffma2(a0, lo, wg[0][2 * i]); ffma2(a1, lo, wg[1][2 * i]); ffma2(a2, lo, wg[2][2 * i]); ffma2(a3, lo, wg[3][2 * i]);
                ffma2(a0, hi, wg[0][2 * i + 1]); ffma2(a1, hi, wg[1][2 * i + 1]); ffma2(a2, hi, wg[2][2 * i + 1]); ffma2(a3, hi, wg[3][2 * i + 1]);
            }
            const float p0 = a0.x + a0.y, p1 = a1.x + a1.y, p2 = a2.x + a2.y, p3 = a3.x + a3.y;
            // transposing butterfly over the 8 lanes: xor 4 keeps the unit (bit2), xor 2 keeps the gate (bit1), xor 1 sums
            const float q0 = (b2 ? p2 : p0) + __shfl_xor_sync(0xffffffffu, b2 ? p0 : p2, 4);   // r of the kept unit
            const float q1 = (b2 ? p3 : p1) + __shfl_xor_sync(0xffffffffu, b2 ? p1 : p3, 4);   // u of the kept unit
            float g = (b1 ? q1 : q0) + __shfl_xor_sync(0xffffffffu, b1 ? q0 : q1, 2);
            g += __shfl_xor_sync(0xffffffffu, g, 1);
            if (g_owner) {
                const float gt = sigmoidf_acc(g + xgv);
                if (g_is_u) u_s[gj] = gt;
                else rh_s[gj] = gt * h_s[gj];   // r * h
            }
        }
        __syncthreads();
        // ---- candidate: (r*h) . Wc_h (16 rows x 2 columns) ----
        {
            float2 c0 = make_float2(0.f, 0.f), c1 = c0;
            float4 rvv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) rvv[i] = rh4[8 * i];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 lo = make_float2(rvv[i].x, rvv[i].y), hi = make_float2(rvv[i].z, rvv[i].w);
                ffma2(c0, lo, wc[0][2 * i]); ffma2(c1, lo, wc[1][2 * i]);
                ffma2(c0, hi, wc[0][2 * i + 1]); ffma2(c1, hi, wc[1][2 * i + 1]);
            }
            const float p0 = c0.x + c0.y, p1 = c1.x + c1.y;
            float cc = (b2 ? p1 : p0) + __shfl_xor_sync(0xffffffffu, b2 ? p0 : p1, 4);
            cc += __shfl_xor_sync(0xffffffffu, cc, 2);
            cc += __shfl_xor_sync(0xffffffffu, cc, 1);
            if (c_owner) {
                const float cn = tanhf_acc(cc + xcv);
                const float u = u_s[gj];
                const float hn = u * h_s[gj] + (1.0f - u) * cn;
                h_s[gj] = hn;
                out[outp] = hn;
            }
            outp += os;
        }
        __syncthreads();
    };

    int step = 0;
    for (; step + 3 <= T; step += 3) {
        one_step(xg0, xc0, step + 3 < T);
        one_step(xg1, xc1, step + 4 < T);
        one_step(xg2, xc2, step + 5 < T);
    }
    if (step < T) { one_step(xg0, xc0, false); ++step; }
    if (step < T) { one_step(xg1, xc1, false); ++step; }
    (void)lane;
}

}  // namespace

extern "C" int taco_bigru_fwd_h0(const float* xp, const float* Wg_h_fw, const float* Wc_h_fw, const float* Wg_h_bw,
                                 const float* Wc_h_bw, const float* h0_fw, const float* h0_bw, float* out, int B, int T,
                                 void* stream) {
    TACO_CHECK(xp && Wg_h_fw && Wc_h_fw && Wg_h_bw && Wc_h_bw && out, "taco_bigru_fwd: NULL pointer");
    TACO_CHECK(B >= 0 && T >= 0, "taco_bigru_fwd: negative size");
    TACO_CHECK((int64_t)B * T * 768 < (int64_t)1 << 31, "taco_bigru_fwd: B*T = %lld too large for 32-bit offsets", (long long)B * T);
    if (B == 0 || T == 0) return 0;
    dim3 grid(B, 2);
    TACO_LAUNCH(bigru_kernel, grid, 512, 0, (cudaStream_t)stream, xp, Wg_h_fw, Wc_h_fw, Wg_h_bw, Wc_h_bw, h0_fw, h0_bw, out, T);
    TACO_LAUNCH_CHECK();
    return 0;
}

extern "C" int taco_bigru_fwd(const float* xp, const float* Wg_h_fw, const float* Wc_h_fw, const float* Wg_h_bw,
                              const float* Wc_h_bw, float* out, int B, int T, void* stream) {
    return taco_bigru_fwd_h0(xp, Wg_h_fw, Wc_h_fw, Wg_h_bw, Wc_h_bw, nullptr, nullptr, out, B, T, stream);
}
