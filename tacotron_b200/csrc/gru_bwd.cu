// gru_bwd.cu -- serial part of the bidirectional-GRU backward (hidden size 128): back-propagation through time of
// tf.nn.bidirectional_dynamic_rnn(GRUCell(128), GRUCell(128)) (models/ops.py:118-128; cell arithmetic SURVEY A.5).
//
// Everything that is not a recurrence is done by the caller as batched GEMMs (tacotron_b200/models/grad.py):
//   before: gates r,u,c for all steps, recomputed from the saved output sequence (h(t-1) = shifted output row);
//   after : dX = dxp.Wx^T, dWx = X^T.dxp, dW_h = Hprev^T.dxp_g / (r*Hprev)^T.dxp_c, bias column sums.
// This kernel runs the chain   dh(t) -> [dr_pre, du_pre, dc_pre](t), dh(t-1)   for one (utterance, direction) per CTA:
//   dh      = dOut[t] + carry
//   du_pre  = dh (hprev - c) u (1-u)          dc_pre = dh (1-u) (1-c^2)
//   drh     = dc_pre . Wc_h^T                 dr_pre = drh hprev r (1-r)
//   carry   = dh u + drh r + [dr_pre, du_pre] . Wg_h^T
// The two transposed recurrent matrices (128x128 + 256x128 fp32 = 192 KB) stay in the register file of the CTA's
// 512 threads for the whole sequence, exactly like the forward kernel (gru.cu): the 32 lanes of a warp split the
// contraction index, a warp owns 8 outputs, partial sums are combined with the halving butterfly.
// Semantics pinned by tests/mirror_kernels.py::bigru_bwd.
#include "common.cuh"

namespace {

constexpr int H = 128;

// (same reduction as gru.cu) N = 8: after the call p[0] = full sum of column c = 4*b4 + 2*b3 + b2 of the lane id
__device__ __forceinline__ float butterfly8(float (&p)[8], int lane) {
    int n = 8;
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        if (n > 1) {
            const bool hi = (lane & off) != 0;
            n >>= 1;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (j < n) {
                    const float send = hi ? p[j] : p[j + n];
                    const float keep = hi ? p[j + n] : p[j];
                    p[j] = keep + __shfl_xor_sync(0xffffffffu, send, off);
                }
            }
        } else {
            p[0] += __shfl_xor_sync(0xffffffffu, p[0], off);
        }
    }
    return p[0];
}

__global__ void __launch_bounds__(512, 1)
bigru_bwd_kernel(float* __restrict__ dxp, const float* __restrict__ dOut, const float* __restrict__ out, const float* __restrict__ ACT,
                 const float* __restrict__ Wg_fw, const float* __restrict__ Wc_fw, const float* __restrict__ Wg_bw,
                 const float* __restrict__ Wc_bw, const float* __restrict__ h0_fw, const float* __restrict__ h0_bw,
                 float* __restrict__ dh0, int T) {
    const int b = blockIdx.x;
    const int dir = blockIdx.y;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const float* Wg = dir ? Wg_bw : Wg_fw;     // [128][256]  h-side rows of the gates kernel
    const float* Wc = dir ? Wc_bw : Wc_fw;     // [128][128]  (r*h)-side rows of the candidate kernel
    const float* h0 = dir ? h0_bw : h0_fw;     // initial state [B][128] or NULL (zero): hprev of the first processed step

    __shared__ __align__(16) float dc_s[H];        // dc_pre
    __shared__ __align__(16) float dg_s[2 * H];    // [dr_pre | du_pre]
    __shared__ float carry_s[H], dhu_s[H], hprev_s[H], r_s[H], drhr_s[H];

    // transposed weights: warp owns outputs k = 8*warp + kk; lane owns contraction indices 4*lane+i (Wc) / 8*lane+i (Wg)
    float wc[4][8], wg[8][8];
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
        const int k = warp * 8 + kk;
#pragma unroll
        for (int i = 0; i < 4; ++i) wc[i][kk] = __ldg(Wc + (int64_t)k * H + 4 * lane + i);
#pragma unroll
        for (int i = 0; i < 8; ++i) wg[i][kk] = __ldg(Wg + (int64_t)k * 2 * H + 8 * lane + i);
    }
    const int kcol = warp * 8 + (((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1));
    const bool owner = (lane & 3) == 0;

    if (tid < H) carry_s[tid] = 0.f;
    __syncthreads();

    const int64_t seq = (int64_t)b * T;
    for (int step = 0; step < T; ++step) {
        const int t = dir ? step : (T - 1 - step);          // reverse of the forward processing order
        const int tp = dir ? (t + 1) : (t - 1);             // forward predecessor (holds h(t-1) in processing order)
        // ---- phase 0: element-wise part, one thread per hidden unit ----
        if (tid < H) {
            const int n = tid;
            const float* a = ACT + (seq + t) * 768 + dir * 384;
            const float r = a[n], u = a[H + n], c = a[2 * H + n];
            const float hprev = (tp >= 0 && tp < T) ? out[(seq + tp) * 256 + dir * H + n] : (h0 ? h0[b * H + n] : 0.f);
            const float dh = dOut[(seq + t) * 256 + dir * H + n] + carry_s[n];
            const float du_pre = dh * (hprev - c) * u * (1.0f - u);
            const float dc_pre = dh * (1.0f - u) * (1.0f - c * c);
            dc_s[n] = dc_pre;
            dg_s[H + n] = du_pre;
            dhu_s[n] = dh * u;
            hprev_s[n] = hprev;
            r_s[n] = r;
            float* d = dxp + (seq + t) * 768 + dir * 384;
            d[H + n] = du_pre;
            d[2 * H + n] = dc_pre;
        }
        __syncthreads();
        // ---- phase 1: drh = dc_pre . Wc_h^T ----
        {
            const float4 v = *reinterpret_cast<const float4*>(dc_s + 4 * lane);
            float p[8];
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) p[kk] = v.x * wc[0][kk];
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) p[kk] = fmaf(v.y, wc[1][kk], p[kk]);
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) p[kk] = fmaf(v.z, wc[2][kk], p[kk]);
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) p[kk] = fmaf(v.w, wc[3][kk], p[kk]);
            const float drh = butterfly8(p, lane);
            if (owner) {
                const float r = r_s[kcol];
                const float dr_pre = drh * hprev_s[kcol] * r * (1.0f - r);
                dg_s[kcol] = dr_pre;
                drhr_s[kcol] = drh * r;
                dxp[(seq + t) * 768 + dir * 384 + kcol] = dr_pre;
            }
        }
        __syncthreads();
        // ---- phase 2: carry = dh u + drh r + [dr_pre, du_pre] . Wg_h^T ----
        {
            const float4 v0 = *reinterpret_cast<const float4*>(dg_s + 8 * lane);
            const float4 v1 = *reinterpret_cast<const float4*>(dg_s + 8 * lane + 4);
            const float vv[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
            float p[8];
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) p[kk] = vv[0] * wg[0][kk];
#pragma unroll
            for (int i = 1; i < 8; ++i)
#pragma unroll
                for (int kk = 0; kk < 8; ++kk) p[kk] = fmaf(vv[i], wg[i][kk], p[kk]);
            const float dhg = butterfly8(p, lane);
            if (owner) carry_s[kcol] = dhu_s[kcol] + drhr_s[kcol] + dhg;
        }
        __syncthreads();
    }
    if (dh0 && tid < H) dh0[(b * 2 + dir) * H + tid] = carry_s[tid];     // d(loss)/d(initial state)
}

}  // namespace

extern "C" int taco_bigru_bwd_h0(float* dxp, const float* dOut, const float* out, const float* ACT, const float* Wg_h_fw,
                                 const float* Wc_h_fw, const float* Wg_h_bw, const float* Wc_h_bw, const float* h0_fw,
                                 const float* h0_bw, float* dh0, int B, int T, void* stream) {
    // the operands of an empty sequence may be NULL (torch's empty tensors have no storage); the weights never may
    TACO_CHECK(Wg_h_fw && Wc_h_fw && Wg_h_bw && Wc_h_bw && ((dxp && dOut && out && ACT) || (int64_t)B * T == 0),
               "taco_bigru_bwd: NULL pointer");
    TACO_CHECK(B >= 0 && T >= 0, "taco_bigru_bwd: negative size");
    if (B == 0 || (T == 0 && !dh0)) return 0;             // T == 0 with dh0: the kernel only writes dh0 = 0
    TACO_LAUNCH(bigru_bwd_kernel, dim3(B, 2), 512, 0, (cudaStream_t)stream, dxp, dOut, out, ACT, Wg_h_fw, Wc_h_fw, Wg_h_bw, Wc_h_bw,
                h0_fw, h0_bw, dh0, T);
    TACO_LAUNCH_CHECK();
    return 0;
}

extern "C" int taco_bigru_bwd(float* dxp, const float* dOut, const float* out, const float* ACT, const float* Wg_h_fw,
                              const float* Wc_h_fw, const float* Wg_h_bw, const float* Wc_h_bw, int B, int T, void* stream) {
    return taco_bigru_bwd_h0(dxp, dOut, out, ACT, Wg_h_fw, Wc_h_fw, Wg_h_bw, Wc_h_bw, nullptr, nullptr, nullptr, B, T, stream);
}
