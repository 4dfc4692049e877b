// gemm_simt.cu -- exact-fp32 FFMA implementation of taco_linear_fwd (TACO_IMPL_SIMT).
// Same contraction + epilogue as the tensor-core kernel (gemm_tc.cu); used as the full-fp32
// precision mode and as the on-GPU cross-check of the tensor-core path.  64x64x16 tiles,
// 256 threads, 4x4 register micro-tile, implicit-GEMM addressing for conv1d 'same'
// (models/ops.py:54-62, :80-85; TF 'same': pad_left=(k-1)//2, extra pad on the right).
#include "epilogue.cuh"

namespace {

struct SimtArgs {
    const float* X; int64_t ldx; int B, T, C, taps, tap0;
    const float* W; int64_t ldw;   // [taps*C][ldw]; for highway the T-gate columns start at W + U
    int N;                          // columns computed by this launch (highway: U)
    int col0;                       // output / epilogue column offset (bank filter slot)
    int highway;
    EpiParams e;
};

constexpr int BM = 64, BN = 64, BK = 16;

template <bool HW>
__global__ void __launch_bounds__(256) gemm_simt_kernel(SimtArgs a) {
    __shared__ float As[BK][BM + 4];
    __shared__ float Bs[HW ? 2 : 1][BK][BN + 4];

    const int tid = threadIdx.x;
    const int tx = tid % 16, ty = tid / 16;
    const int64_t M = (int64_t)a.B * a.T;
    const int64_t m0 = (int64_t)blockIdx.y * BM;
    const int n0 = blockIdx.x * BN;
    const int Ktot = a.taps * a.C;

    float acc[4][4] = {};
    float acc2[HW ? 4 : 1][HW ? 4 : 1] = {};

    // A-load coordinates: row = tid/4 (0..63), 4 consecutive k at (tid%4)*4
    const int a_row = tid / 4;
    const int a_k = (tid % 4) * 4;
    const int64_t am = m0 + a_row;
    const bool a_row_ok = am < M;
    const int ab = a_row_ok ? (int)(am / a.T) : 0;
    const int at = a_row_ok ? (int)(am % a.T) : 0;
    // B-load coordinates: k = tid/16, 4 consecutive n at (tid%16)*4
    const int b_k = tid / 16;
    const int b_n = (tid % 16) * 4;

    for (int k0 = 0; k0 < Ktot; k0 += BK) {
        // ---- A tile (implicit im2col) ----
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int kk = k0 + a_k + i;
            float v = 0.0f;
            if (a_row_ok && kk < Ktot) {
                int j = kk / a.C;
                int c = kk - j * a.C;
                int ts = at + a.tap0 + j;
                if (ts >= 0 && ts < a.T) v = __ldg(a.X + ((int64_t)ab * a.T + ts) * a.ldx + c);
            }
            As[a_k + i][a_row] = v;
        }
        // ---- B tile ----
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int kk = k0 + b_k;
            int n = n0 + b_n + i;
            float v = 0.0f, v2 = 0.0f;
            if (kk < Ktot && n < a.N) {
                v = __ldg(a.W + (int64_t)kk * a.ldw + n);
                if (HW) v2 = __ldg(a.W + (int64_t)kk * a.ldw + a.N + n);
            }
            Bs[0][b_k][b_n + i] = v;
            if (HW) Bs[HW ? 1 : 0][b_k][b_n + i] = v2;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float av[4], bv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) av[i] = As[k][ty * 4 + i];
#pragma unroll
            for (int j = 0; j < 4; ++j) bv[j] = Bs[0][k][tx * 4 + j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
            if (HW) {
                float cv[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) cv[j] = Bs[HW ? 1 : 0][k][tx * 4 + j];
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc2[HW ? i : 0][HW ? j : 0] = fmaf(av[i], cv[j], acc2[HW ? i : 0][HW ? j : 0]);
            }
        }
        __syncthreads();
    }

#pragma unroll
    for (int i = 0; i < 4; ++i) {
        int64_t row = m0 + ty * 4 + i;
        if (row >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int col = n0 + tx * 4 + j;
            if (col >= a.N) continue;
            float v;
            if (HW) v = epi_highway(a.e, row, col, a.N, acc[i][j], acc2[HW ? i : 0][HW ? j : 0]);
            else    v = epi_value(a.e, row, a.col0 + col, acc[i][j]);
            a.e.Y[row * a.e.ldy + a.col0 + col] = v;
        }
    }
}

}  // namespace

int taco_linear_simt(const taco_linear_desc* d, cudaStream_t st) {
    TACO_CHECK(d->W != nullptr, "taco_linear_fwd(SIMT): W (TF-layout weights) is NULL");
    TACO_CHECK(!d->pool, "taco_linear_fwd(SIMT): fused max-pool is only available on the tensor-core path");
    SimtArgs a;
    a.X = d->X; a.ldx = d->ldx; a.B = d->B; a.T = d->T; a.C = d->C;
    a.e.Y = d->Y; a.e.ldy = d->ldy; a.e.bias = d->bias; a.e.scale = d->scale; a.e.shift = d->shift;
    a.e.keep = d->keep; a.e.keep_scale = d->keep_scale; a.e.residual = d->residual; a.e.ldr = d->ldr;
    a.e.hx = d->hx; a.e.ldhx = d->ldhx; a.e.act = d->act; a.e.N = d->N;
    a.e.bias_utt = d->bias_utt; a.e.ldbu = d->ldbu; a.e.T = d->T;
    const int64_t M = (int64_t)d->B * d->T;
    if (M == 0 || d->N == 0) return 0;
    if (d->epilogue == TACO_EPI_HIGHWAY) {
        TACO_CHECK(d->bank_K == 0 && d->taps == 1 && (d->N % 2) == 0 && d->hx, "highway epilogue needs dense N=2U and hx");
        int U = d->N / 2;
        a.taps = 1; a.tap0 = 0; a.W = d->W; a.ldw = d->N; a.N = U; a.col0 = 0; a.highway = 1;
        a.e.N = U;
        dim3 grid((U + BN - 1) / BN, (unsigned)((M + BM - 1) / BM));
        gemm_simt_kernel<true><<<grid, 256, 0, st>>>(a);
        TACO_LAUNCH_CHECK();
        return 0;
    }
    a.highway = 0;
    if (d->bank_K > 0) {
        TACO_CHECK(d->N == d->bank_K * d->bank_cout, "bank: N must equal bank_K*bank_cout");
        const float* w = d->W;
        for (int k = 1; k <= d->bank_K; ++k) {
            a.taps = k; a.tap0 = -((k - 1) / 2);
            a.W = w; a.ldw = d->bank_cout; a.N = d->bank_cout; a.col0 = (k - 1) * d->bank_cout;
            dim3 grid((a.N + BN - 1) / BN, (unsigned)((M + BM - 1) / BM));
            gemm_simt_kernel<false><<<grid, 256, 0, st>>>(a);
            TACO_LAUNCH_CHECK();
            w += (int64_t)k * d->C * d->bank_cout;
        }
        return 0;
    }
    a.taps = d->taps; a.tap0 = d->tap0; a.W = d->W; a.ldw = d->N; a.N = d->N; a.col0 = 0;
    dim3 grid((d->N + BN - 1) / BN, (unsigned)((M + BM - 1) / BM));
    gemm_simt_kernel<false><<<grid, 256, 0, st>>>(a);
    TACO_LAUNCH_CHECK();
    return 0;
}
