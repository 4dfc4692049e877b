// train.cu -- training-path kernels that are NOT recurrences: the general fp32 GEMM with row shifts (every data /
// weight gradient of a dense or conv1d layer), column reductions (bias / batch-norm gradients), the epilogue,
// max-pool, highway, L1, embedding-gather backward kernels, and the clip + Adam update.
//
// Reference: what tf.gradients + AdamOptimizer + clip_by_global_norm build for Tacotron.add_train_op
// (models/tacotron.py:167-185) over the forward graph (models/tacotron.py:107-165, models/ops.py:27-132).
// Semantics of every kernel are pinned by the function of the same name in tests/mirror_kernels.py.
#include "common.cuh"

namespace {

inline int grid_for(int64_t total, int block) {
    int64_t g = (total + block - 1) / block;
    if (g > TACO_SMS * 16) g = TACO_SMS * 16;
    if (g < 1) g = 1;
    return (int)g;
}

// =============================================================================================================
// general GEMM, fp32 FFMA (exact products), 64x64x16 tiles, 4x4 outputs per thread, optional split-K (atomics)
// =============================================================================================================
constexpr int GBM = 64, GBN = 64, GBK = 16, GLD = 68;   // GLD: padded smem row (multiple of 4 floats)

struct GemmP {
    const float* A; int64_t lda; const float* B; int64_t ldb; float* C; int64_t ldc;
    int M, N, K, ta, tb;
    float beta;
    int shift, period, taps, dshift, kper;
    int64_t b_tap_stride;
    int batch;
    int64_t a_bstride, b_bstride, c_bstride;
    int bshift;
    int splits, kchunk;          // split-K: K range of split s = [s*kchunk, min(K, (s+1)*kchunk))
    int a_rows;                  // number of STORED rows of A (M if !ta, K if ta) -- bound for the shifted row
    int atomic;                  // accumulate with atomicAdd (beta == 1 and (splits > 1 or always, see host))
};

// stored row `row` shifted by sh; valid only inside the same period block and inside [0, a_rows)
__device__ __forceinline__ bool shifted_row(int row, int sh, int period, int a_rows, int& src) {
    src = row + sh;
    if (src < 0 || src >= a_rows) return false;
    if (period > 0 && (row / period) != (src / period)) return false;
    return true;
}

__global__ void __launch_bounds__(256) gemm_kernel(const GemmP p) {
    __shared__ __align__(16) float As[GBK][GLD];
    __shared__ __align__(16) float Bs[GBK][GLD];
    const int tid = threadIdx.x;
    const int z = blockIdx.z / p.splits, split = blockIdx.z % p.splits;
    const int m0 = blockIdx.y * GBM, n0 = blockIdx.x * GBN;
    const float* A = p.A + (int64_t)z * p.a_bstride;
    const float* B = p.B + (int64_t)z * p.b_bstride;
    float* C = p.C + (int64_t)z * p.c_bstride;
    const int sh0 = p.shift + z * p.bshift;
    const int kbeg = split * p.kchunk;
    const int kend = min(p.K, kbeg + p.kchunk);
    const int tx = tid & 15, ty = tid >> 4;

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int k0 = kbeg; k0 < kend; k0 += GBK) {
        // ---- A tile -> As[k][m] ----
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int idx = tid + i * 256;
            int kk, mm;
            if (p.ta) { mm = idx & 63; kk = idx >> 6; } else { kk = idx & 15; mm = idx >> 4; }
            const int k = k0 + kk, m = m0 + mm;
            float v = 0.f;
            if (k < kend && m < p.M) {
                if (p.ta) {                                  // stored [K][M]: row index = k (shifted), column m
                    int src;
                    if (shifted_row(k, sh0, p.period, p.a_rows, src)) v = A[(int64_t)src * p.lda + m];
                } else {                                     // stored [M][Kseg]: row index = m (shifted), column k (mod kper)
                    int sh = sh0, kc = k;
                    if (p.taps > 1) { const int j = k / p.kper; sh += j * p.dshift; kc = k - j * p.kper; }
                    int src;
                    if (shifted_row(m, sh, p.period, p.a_rows, src)) v = A[(int64_t)src * p.lda + kc];
                }
            }
            As[kk][mm] = v;
        }
        // ---- B tile -> Bs[k][n] ----
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int idx = tid + i * 256;
            int kk, nn;
            if (p.tb) { kk = idx & 15; nn = idx >> 4; } else { nn = idx & 63; kk = idx >> 6; }
            const int k = k0 + kk, n = n0 + nn;
            float v = 0.f;
            if (k < kend && n < p.N) {
                if (p.tb) {
                    int64_t off = 0; int kc = k;
                    if (p.taps > 1) { const int j = k / p.kper; off = (int64_t)j * p.b_tap_stride; kc = k - j * p.kper; }
                    v = B[off + (int64_t)n * p.ldb + kc];
                } else {
                    v = B[(int64_t)k * p.ldb + n];
                }
            }
            Bs[kk][nn] = v;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < GBK; ++kk) {
            const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
            const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
            const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
        if (m >= p.M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n >= p.N) continue;
            float* c = C + (int64_t)m * p.ldc + n;
            if (p.atomic) atomicAdd(c, acc[i][j]);
            else if (p.beta != 0.f) *c = fmaf(p.beta, *c, acc[i][j]);
            else *c = acc[i][j];
        }
    }
}

// =============================================================================================================
// The same contraction on the tensor cores: mma.sync m16n8k8 TF32 with the 3xTF32 split (hi*hi + hi*lo + lo*hi,
// fp32 accumulate) -- fp32-grade results (~1e-6 relative, like the forward decoder kernel) at a multiple of the FFMA
// rate.  Tile loaders (transposes, row shifts, K segments, batches, split-K) are the SIMT kernel's, verbatim; only
// the inner product differs.  Shared tiles use a 72-float row so that the fragment reads (bank = 8*tg + g) are
// conflict-free.  8 warps: warp w owns rows [16*(w&3), +16) x columns [32*(w>>2), +32) of the 64x64 tile.
// Opt-in (taco_set_gemm_impl(1)); the FFMA kernel stays the default until this one has had a hardware run.
// Fragment coordinates (PTX m16n8k8 .tf32, g = lane>>2, tg = lane&3):
//   A: a0 (g, tg) a1 (g+8, tg) a2 (g, tg+4) a3 (g+8, tg+4)    B: b0 (k=tg, n=g) b1 (k=tg+4, n=g)
//   C: c0 (g, 2tg) c1 (g, 2tg+1) c2 (g+8, 2tg) c3 (g+8, 2tg+1)
// =============================================================================================================
constexpr int MLD = 72;

__device__ __forceinline__ void split3(float x, uint32_t& hi, uint32_t& lo) {
    hi = __float_as_uint(x) & 0xffffe000u;
    lo = __float_as_uint(x - __uint_as_float(hi));
}
__device__ __forceinline__ void mma16n8k8(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
#ifdef TACO_HOST_EMU
    emu_mma_m16n8k8_tf32(d, a, b0, b1);     // warp-collective emulation of the instruction (tests/cuda_emu/emu.h)
    return;
#else
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
#endif
}

__global__ void __launch_bounds__(256) gemm_mma_kernel(const GemmP p) {
    __shared__ __align__(16) float As[GBK][MLD];
    __shared__ __align__(16) float Bs[GBK][MLD];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, tg = lane & 3;
    const int z = blockIdx.z / p.splits, split = blockIdx.z % p.splits;
    const int m0 = blockIdx.y * GBM, n0 = blockIdx.x * GBN;
    const float* A = p.A + (int64_t)z * p.a_bstride;
    const float* B = p.B + (int64_t)z * p.b_bstride;
    float* C = p.C + (int64_t)z * p.c_bstride;
    const int sh0 = p.shift + z * p.bshift;
    const int kbeg = split * p.kchunk;
    const int kend = min(p.K, kbeg + p.kchunk);
    const int wm = (warp & 3) * 16, wn = (warp >> 2) * 32;

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int k0 = kbeg; k0 < kend; k0 += GBK) {
        // ---- tile loaders: identical to gemm_kernel ----
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int idx = tid + i * 256;
            int kk, mm;
            if (p.ta) { mm = idx & 63; kk = idx >> 6; } else { kk = idx & 15; mm = idx >> 4; }
            const int k = k0 + kk, m = m0 + mm;
            float v = 0.f;
            if (k < kend && m < p.M) {
                if (p.ta) {
                    int src;
                    if (shifted_row(k, sh0, p.period, p.a_rows, src)) v = A[(int64_t)src * p.lda + m];
                } else {
                    int sh = sh0, kc = k;
                    if (p.taps > 1) { const int j = k / p.kper; sh += j * p.dshift; kc = k - j * p.kper; }
                    int src;
                    if (shifted_row(m, sh, p.period, p.a_rows, src)) v = A[(int64_t)src * p.lda + kc];
                }
            }
            As[kk][mm] = v;
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int idx = tid + i * 256;
            int kk, nn;
            if (p.tb) { kk = idx & 15; nn = idx >> 4; } else { nn = idx & 63; kk = idx >> 6; }
            const int k = k0 + kk, n = n0 + nn;
            float v = 0.f;
            if (k < kend && n < p.N) {
                if (p.tb) {
                    int64_t off = 0; int kc = k;
                    if (p.taps > 1) { const int j = k / p.kper; off = (int64_t)j * p.b_tap_stride; kc = k - j * p.kper; }
                    v = B[off + (int64_t)n * p.ldb + kc];
                } else {
                    v = B[(int64_t)k * p.ldb + n];
                }
            }
            Bs[kk][nn] = v;
        }
        __syncthreads();
        // ---- two k8 steps: 1 A fragment (16 rows) x 4 B fragments (4 x 8 columns), 3 MMAs each ----
#pragma unroll
        for (int ks = 0; ks < GBK; ks += 8) {
            uint32_t ah[4], al[4];
            split3(As[ks + tg][wm + g], ah[0], al[0]);
            split3(As[ks + tg][wm + g + 8], ah[1], al[1]);
            split3(As[ks + tg + 4][wm + g], ah[2], al[2]);
            split3(As[ks + tg + 4][wm + g + 8], ah[3], al[3]);
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                uint32_t bh0, bl0, bh1, bl1;
                split3(Bs[ks + tg][wn + nt * 8 + g], bh0, bl0);
                split3(Bs[ks + tg + 4][wn + nt * 8 + g], bh1, bl1);
                mma16n8k8(acc[nt], al, bh0, bh1);          // small terms first
                mma16n8k8(acc[nt], ah, bl0, bl1);
                mma16n8k8(acc[nt], ah, bh0, bh1);
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int m = m0 + wm + g + ((e >> 1) ? 8 : 0);
            const int n = n0 + wn + nt * 8 + 2 * tg + (e & 1);
            if (m >= p.M || n >= p.N) continue;
            float* c = C + (int64_t)m * p.ldc + n;
            if (p.atomic) atomicAdd(c, acc[nt][e]);
            else if (p.beta != 0.f) *c = fmaf(p.beta, *c, acc[nt][e]);
            else *c = acc[nt][e];
        }
    }
}

// =============================================================================================================
// column reductions: out[n] += sum_m A[m,n] * (Bm ? Bm[m,n] - (R ? R[m,n] : 0) : 1)
// =============================================================================================================
__global__ void __launch_bounds__(256) colsum_kernel(float* __restrict__ out, const float* __restrict__ A, int64_t lda,
                                                     const float* __restrict__ Bm, int64_t ldb, const float* __restrict__ R,
                                                     int64_t ldr, int M, int N, int rows_per_block) {
    __shared__ float red[8][33];
    const int x = threadIdx.x & 31, y = threadIdx.x >> 5;
    const int n = blockIdx.x * 32 + x;
    const int r0 = blockIdx.y * rows_per_block;
    const int r1 = min(M, r0 + rows_per_block);
    float acc = 0.f;
    if (n < N) {
        for (int m = r0 + y; m < r1; m += 8) {
            float a = A[(int64_t)m * lda + n];
            if (Bm) {
                float b = Bm[(int64_t)m * ldb + n];
                if (R) b -= R[(int64_t)m * ldr + n];
                a *= b;
            }
            acc += a;
        }
    }
    red[y][x] = acc;
    __syncthreads();
    if (y == 0 && n < N) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) s += red[w][x];
        atomicAdd(out + n, s);
    }
}

// =============================================================================================================
// element-wise kernels over [M][N] views with leading strides
// =============================================================================================================
__global__ void bias_act_kernel(float* C, int64_t ldc, int M, int N, const float* __restrict__ bias, int act) {
    const int64_t total = (int64_t)M * N;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int m = (int)(i / N), n = (int)(i % N);
        float v = C[(int64_t)m * ldc + n];
        if (bias) v += bias[n];
        float o;
        switch (act) {                         // training path: library-accurate transcendental functions
            case TACO_ACT_RELU:    o = fmaxf(v, 0.f); break;
            case TACO_ACT_SIGMOID: o = 1.0f / (1.0f + expf(-v)); break;
            case TACO_ACT_TANH:    o = tanhf(v); break;
            default:               o = v; break;
        }
        C[(int64_t)m * ldc + n] = o;
    }
}

__global__ void mul_shift_kernel(float* out, int64_t ldo, const float* X, int64_t ldx, const float* Hm, int64_t ldh, int M, int N,
                                 int shift, int period) {
    const int64_t total = (int64_t)M * N;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int m = (int)(i / N), n = (int)(i % N);
        int src;
        float h = 0.f;
        if (shifted_row(m, shift, period, M, src)) h = Hm[(int64_t)src * ldh + n];
        out[(int64_t)m * ldo + n] = X[(int64_t)m * ldx + n] * h;
    }
}

__global__ void epi_bwd_kernel(float* dZ, int64_t lddz, const float* dY, int64_t lddy, const float* Y, int64_t ldy,
                               const float* R, int64_t ldr, int M, int N, int relu, const float* __restrict__ scale,
                               const float* __restrict__ shift, float gain) {
    const int64_t total = (int64_t)M * N;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int m = (int)(i / N), n = (int)(i % N);
        float g = dY[(int64_t)m * lddy + n] * gain;
        const float sc = scale ? scale[n] : 1.0f;
        if (scale) g *= sc;
        if (relu) {
            float y = Y[(int64_t)m * ldy + n];
            bool on;
            if (scale) {
                if (R) y -= R[(int64_t)m * ldr + n];
                on = (y - shift[n]) * sc > 0.f;
            } else {
                on = y > 0.f;
            }
            if (!on) g = 0.f;
        }
        dZ[(int64_t)m * lddz + n] = g;
    }
}

__global__ void epi_fwd_keep_kernel(float* X, int64_t ldx, const uint8_t* __restrict__ keep, int M, int N, float gain) {
    const int64_t total = (int64_t)M * N;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int m = (int)(i / N), n = (int)(i % N);
        float* x = X + (int64_t)m * ldx + n;
        *x = keep[i] ? *x * gain : 0.f;
    }
}

__global__ void bn_param_grad_kernel(float* dgamma, float* dbeta, const float* S1, const float* S2, const float* gamma,
                                     const float* beta, int N) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n < N) {
        dbeta[n] += S1[n];
        dgamma[n] += (S2[n] - beta[n] * S1[n]) / gamma[n];
    }
}

// max-pool(2,1,'same') backward; ties go to the first element of the window
__global__ void maxpool_bwd_kernel(float* __restrict__ dX, const float* __restrict__ dP, const float* __restrict__ X, int T, int C,
                                   int64_t total) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = i / C;
        const int t = (int)(row % T);
        const float x = X[i];
        float g = 0.f;
        if (t == T - 1) g += dP[i];                                   // P[T-1] = X[T-1]
        else if (x >= X[i + C]) g += dP[i];                            // window t: (X[t], X[t+1]), first wins ties
        if (t > 0 && x > X[i - C]) g += dP[i - C];                     // window t-1: second element wins only if strictly larger
        dX[i] = g;
    }
}

__global__ void highway_fwd_kernel(float* Y, int64_t ldy, const float* Pm, int64_t ldp, const float* X, int64_t ldx, int M, int U) {
    const int64_t total = (int64_t)M * U;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int m = (int)(i / U), n = (int)(i % U);
        const float h = fmaxf(Pm[(int64_t)m * ldp + n], 0.f);
        const float t = 1.0f / (1.0f + expf(-Pm[(int64_t)m * ldp + U + n]));
        const float x = X[(int64_t)m * ldx + n];
        Y[(int64_t)m * ldy + n] = h * t + x * (1.0f - t);
    }
}

__global__ void highway_bwd_kernel(float* dP, int64_t lddp, float* dXd, int64_t lddx, const float* dY, int64_t lddy, const float* Pm,
                                   int64_t ldp, const float* X, int64_t ldx, int M, int U) {
    const int64_t total = (int64_t)M * U;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int m = (int)(i / U), n = (int)(i % U);
        const float hp = Pm[(int64_t)m * ldp + n];
        const float h = fmaxf(hp, 0.f);
        const float t = 1.0f / (1.0f + expf(-Pm[(int64_t)m * ldp + U + n]));
        const float x = X[(int64_t)m * ldx + n];
        const float g = dY[(int64_t)m * lddy + n];
        dP[(int64_t)m * lddp + n] = (hp > 0.f) ? g * t : 0.f;
        dP[(int64_t)m * lddp + U + n] = g * (h - x) * t * (1.0f - t);
        dXd[(int64_t)m * lddx + n] = g * (1.0f - t);
    }
}

__global__ void l1_bwd_kernel(float* dA, const float* __restrict__ A, const float* __restrict__ Bt, int64_t n, float beta) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float d = A[i] - Bt[i];
        const float s = (d > 0.f) ? 1.f : ((d < 0.f) ? -1.f : 0.f);
        dA[i] = (beta != 0.f) ? fmaf(beta, dA[i], s) : s;
    }
}

// same with a row-padded gradient buffer (rows of `cols` values, `ldd` floats apart): lets the [M][1025] spectrogram gradient
// live in a 16-byte-aligned row pitch so that the tensor-core dX / dW kernels can TMA it
__global__ void l1_bwd_ld_kernel(float* dA, int64_t ldd, const float* __restrict__ A, const float* __restrict__ Bt, int64_t rows,
                                 int64_t cols, float beta) {
    const int64_t n = rows * cols;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / cols, c = i - r * cols;
        const float d = A[i] - Bt[i];
        const float s = (d > 0.f) ? 1.f : ((d < 0.f) ? -1.f : 0.f);
        float* o = dA + r * ldd + c;
        *o = (beta != 0.f) ? fmaf(beta, *o, s) : s;
    }
}

__global__ void scatter_add_rows_kernel(float* dTable, const int32_t* __restrict__ ids, const float* __restrict__ dRows, int rows,
                                        int width, int vocab) {
    const int64_t total = (int64_t)rows * width;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int row = (int)(i / width), c = (int)(i % width);
        int id = ids[row];
        id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
        const float v = dRows[i];
        if (v != 0.f) atomicAdd(dTable + (int64_t)id * width + c, v);
    }
}

// decoder step inputs (helper.next_inputs of TrainingHelper / ScheduledOutputTrainingHelper, SURVEY A.8/A.9), time-major
__global__ void dec_inputs_kernel(float* Xin, uint8_t* sel, const float* __restrict__ mel, const float* __restrict__ y,
                                  const uint8_t* __restrict__ sample_mask, int B, int T, int r, int mf, int sched) {
    const int64_t total = (int64_t)T * B * mf;
    const int OUT = mf * r, lo = (r - 1) * mf;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % mf);
        const int b = (int)((i / mf) % B);
        const int t = (int)(i / ((int64_t)mf * B));
        const bool s = sched && t > 0 && sample_mask[(int64_t)(t - 1) * B + b] != 0;
        const float v = s ? y[((int64_t)b * T + (t - 1)) * OUT + lo + c] : mel[((int64_t)b * T + t) * OUT + lo + c];
        Xin[i] = v;
        if (c == 0) sel[(int64_t)t * B + b] = s ? 1 : 0;
    }
}

// dkeys[b,j,d] = sum_t DSCORE[b,t,j] v[d] (1-e^2);  dv[d] += sum_{b,t,j} DSCORE[b,t,j] e;  e = tanh(keys[b,j,d] + PQ[t,b,d])
__global__ void __launch_bounds__(256) attn_bwd_post_kernel(float* __restrict__ dkeys, float* dv, const float* __restrict__ DSCORE,
                                                            const float* __restrict__ keys, const float* __restrict__ PQ,
                                                            const float* __restrict__ v, int B, int T, int Tx) {
    const int bj = blockIdx.x;                 // b*Tx + j
    const int b = bj / Tx, j = bj % Tx;
    const int d = threadIdx.x;                 // 256 attention units
    const float k = keys[(int64_t)bj * 256 + d];
    const float vd = v[d];
    float ak = 0.f, av = 0.f;
    for (int t = 0; t < T; ++t) {
        const float ds = DSCORE[((int64_t)b * T + t) * Tx + j];
        if (ds == 0.f) continue;               // masked positions / exact zeros contribute nothing
        const float e = tanhf(k + PQ[((int64_t)t * B + b) * 256 + d]);
        ak = fmaf(ds * vd, 1.0f - e * e, ak);
        av = fmaf(ds, e, av);
    }
    dkeys[(int64_t)bj * 256 + d] = ak;
    if (av != 0.f) atomicAdd(dv + d, av);
}

// deterministic sum of squares (two stages, double accumulation in stage 2)
constexpr int SS_BLOCKS = 1184;
__global__ void sumsq_stage1(const float* __restrict__ x, int64_t n, float* __restrict__ partial) {
    __shared__ float red[8];
    float acc = 0.f;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float v = x[i];
        acc = fmaf(v, v, acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < 8; ++w) s += red[w];
        partial[blockIdx.x] = s;
    }
}
__global__ void sumsq_stage2(const float* __restrict__ partial, int n, float* __restrict__ out) {
    __shared__ double red[32];
    double acc = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) acc += (double)partial[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
        out[0] = (float)s;
    }
}

// clip_by_global_norm + TF Adam (SURVEY A.12): g *= clip/max(norm, clip); m,v update; p -= lr_t * m / (sqrt(v) + eps)
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, int64_t n,
                            float lr_t, float b1, float b2, float eps, float clip, const float* __restrict__ sumsq) {
    const float norm = sqrtf(sumsq[0]);
    const float scale = (clip > 0.f) ? clip / fmaxf(norm, clip) : 1.0f;   // cap_grads <= 0: no clipping (tacotron.py:179)
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float gc = g[i] * scale;
        const float mi = b1 * m[i] + (1.0f - b1) * gc;
        const float vi = b2 * v[i] + (1.0f - b2) * gc * gc;
        m[i] = mi;
        v[i] = vi;
        p[i] -= lr_t * mi / (sqrtf(vi) + eps);
    }
}

// per-segment column sums: block (column chunk, segment) reduces the `period` rows of its segment in a fixed order and is the
// only writer of its 32 outputs -- deterministic without atomics
__global__ void __launch_bounds__(256) colsum_seg_kernel(float* __restrict__ out, int64_t ldo, const float* __restrict__ A,
                                                         int64_t lda, int N, int period) {
    __shared__ float red[8][33];
    const int x = threadIdx.x & 31, y = threadIdx.x >> 5;
    const int n = blockIdx.x * 32 + x;
    const int64_t r0 = (int64_t)blockIdx.y * period;
    float acc = 0.f;
    if (n < N)
        for (int m = y; m < period; m += 8) acc += A[(r0 + m) * lda + n];
    red[y][x] = acc;
    __syncthreads();
    if (y == 0 && n < N) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) s += red[w][x];
        out[(int64_t)blockIdx.y * ldo + n] += s;
    }
}

// guided attention (Tachibana et al. 2017): one warp per (b, t) row of the alignments.  The lane's up-to-8 positions
// j = lane + 32 i are loaded at once; W, s = sum_j align W and the gradient lam align (W - s) are formed from the same
// registers, so the loss and its gradient see the same W.  row_s[row] = s (the loss' per-row partial).
constexpr int GA_WARPS = 8;
constexpr int GA_PER_LANE = 256 / 32;        // Tx <= 256
__global__ void __launch_bounds__(256) guided_attention_kernel(float* __restrict__ dscore, float* __restrict__ row_s,
                                                               const float* __restrict__ align,
                                                               const int32_t* __restrict__ text_length,
                                                               const int32_t* __restrict__ speech_steps, int B, int T,
                                                               int Tx, float inv_2g2, float lam) {
    const int lane = threadIdx.x & 31;
    const int64_t rows = (int64_t)B * T;
    for (int64_t row = (int64_t)blockIdx.x * GA_WARPS + (threadIdx.x >> 5); row < rows; row += (int64_t)gridDim.x * GA_WARPS) {
        const int b = (int)(row / T), t = (int)(row - (int64_t)b * T);
        const int n = min(text_length[b], Tx);
        const int tb = speech_steps[b];
        const int nlive = (t < tb && n > 0) ? n : 0;     // positions j < nlive are inside the mask
        const float* a = align + row * Tx;
        float al[GA_PER_LANE], w[GA_PER_LANE];
#pragma unroll
        for (int i = 0; i < GA_PER_LANE; ++i) {
            const int j = lane + 32 * i;
            al[i] = (j < nlive) ? a[j] : 0.f;
        }
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < GA_PER_LANE; ++i) {
            const int j = lane + 32 * i;
            w[i] = 0.f;
            if (j < nlive) {
                const float d = (float)j / (float)n - (float)t / (float)tb;
                w[i] = -expm1f(-d * d * inv_2g2);        // 1 - exp(-x), accurate near the diagonal where W -> 0
            }
            s = fmaf(al[i], w[i], s);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
#pragma unroll
        for (int i = 0; i < GA_PER_LANE; ++i) {
            const int j = lane + 32 * i;
            if (j < Tx) dscore[row * Tx + j] = (j < nlive) ? lam * al[i] * (w[i] - s) : 0.f;
        }
        if (lane == 0) row_s[row] = s;
    }
}
// loss = lam * sum of the row partials: fixed per-thread strides, then thread 0 adds the 256 double sums in order
__global__ void __launch_bounds__(256) guided_attention_sum_kernel(const float* __restrict__ row_s, int64_t rows, double lam,
                                                                   float* __restrict__ loss) {
    __shared__ double red[256];
    double acc = 0.0;
    for (int64_t i = threadIdx.x; i < rows; i += 256) acc += (double)row_s[i];
    red[threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double tot = 0.0;
        for (int k = 0; k < 256; ++k) tot += red[k];
        loss[0] = (float)(lam * tot);
    }
}

}  // namespace

static int g_gemm_impl = 0;        // taco_set_gemm_impl

extern "C" {

int taco_gemm(const taco_gemm_desc* d, void* stream) {
    TACO_CHECK(d && d->A && d->B && d->C, "taco_gemm: NULL pointer");
    TACO_CHECK(d->M >= 0 && d->N >= 0 && d->K >= 0 && d->batch >= 1, "taco_gemm: bad sizes M=%d N=%d K=%d batch=%d", d->M, d->N, d->K, d->batch);
    TACO_CHECK(d->beta == 0.f || d->beta == 1.f, "taco_gemm: beta must be 0 or 1");
    TACO_CHECK(d->taps >= 1, "taco_gemm: taps must be >= 1");
    if (d->taps > 1) TACO_CHECK(!d->ta && d->tb && d->kper > 0 && d->K == d->taps * d->kper, "taco_gemm: K-segmented form needs ta=0, tb=1, K = taps*kper");
    if (d->M == 0 || d->N == 0) return 0;
    GemmP p;
    p.A = d->A; p.lda = d->lda; p.B = d->B; p.ldb = d->ldb; p.C = d->C; p.ldc = d->ldc;
    p.M = d->M; p.N = d->N; p.K = d->K; p.ta = d->ta; p.tb = d->tb; p.beta = d->beta;
    p.shift = d->shift; p.period = d->period; p.taps = d->taps; p.dshift = d->dshift; p.kper = d->kper;
    p.b_tap_stride = d->b_tap_stride; p.batch = d->batch; p.a_bstride = d->a_bstride; p.b_bstride = d->b_bstride;
    p.c_bstride = d->c_bstride; p.bshift = d->bshift;
    p.a_rows = d->ta ? d->K : d->M;
    const int tiles_m = (d->M + GBM - 1) / GBM, tiles_n = (d->N + GBN - 1) / GBN;
    const int64_t tiles = (int64_t)tiles_m * tiles_n * d->batch;
    int splits = 1;
    if (d->beta == 1.f && d->K > 512) {            // split-K only when accumulating (atomics); target ~3 CTAs per SM
        const int want = (int)((444 + tiles - 1) / tiles);
        const int maxs = (d->K + 255) / 256;
        splits = want < 1 ? 1 : (want > maxs ? maxs : want);
    }
    int kchunk = (d->K + splits - 1) / splits;
    kchunk = (kchunk + GBK - 1) / GBK * GBK;
    if (kchunk < GBK) kchunk = GBK;
    splits = d->K > 0 ? (d->K + kchunk - 1) / kchunk : 1;
    p.splits = splits; p.kchunk = kchunk;
    p.atomic = (d->beta == 1.f) ? 1 : 0;             // several launches may accumulate into the same C concurrently-in-order; atomics keep split-K safe
    TACO_CHECK((int64_t)splits * d->batch <= 65535 && tiles_m <= 65535, "taco_gemm: grid too large");
    dim3 grid(tiles_n, tiles_m, splits * d->batch);
    if (g_gemm_impl == 1) TACO_LAUNCH(gemm_mma_kernel, grid, 256, 0, (cudaStream_t)stream, p);
    else TACO_LAUNCH(gemm_kernel, grid, 256, 0, (cudaStream_t)stream, p);
    TACO_LAUNCH_CHECK();
    return 0;
}

/* 0 = exact-product FFMA kernel (default), 1 = 3xTF32 mma.sync tensor-core kernel; returns the previous setting */
int taco_set_gemm_impl(int impl) {
    const int prev = g_gemm_impl;
    if (impl == 0 || impl == 1) g_gemm_impl = impl;
    return prev;
}

int taco_colsum_seg(float* out, int64_t ldo, const float* A, int64_t lda, int M, int N, int period, void* stream) {
    TACO_CHECK(out && A && M >= 0 && N >= 0 && period >= 1 && M % period == 0 && ldo >= N,
               "taco_colsum_seg: bad arguments (M=%d N=%d period=%d)", M, N, period);
    if (M == 0 || N == 0) return 0;
    TACO_LAUNCH(colsum_seg_kernel, dim3((N + 31) / 32, M / period), 256, 0, (cudaStream_t)stream, out, ldo, A, lda, N, period);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_guided_attention_partial_count(int B, int T) { return (B > 0 && T > 0) ? B * T : 0; }

int taco_guided_attention(float* dscore, float* loss, const float* align, const int32_t* text_length,
                          const int32_t* speech_steps, int B, int T, int Tx, float g, float lam, float* partial_ws,
                          void* stream) {
    TACO_CHECK(dscore && loss && align && text_length && speech_steps && partial_ws, "taco_guided_attention: NULL");
    TACO_CHECK(B >= 1 && T >= 1 && Tx >= 1 && Tx <= 256 && (int64_t)B * T <= INT32_MAX,
               "taco_guided_attention: bad sizes (B=%d, T=%d, Tx=%d; Tx <= 256)", B, T, Tx);
    TACO_CHECK(g > 0.f && g <= 3.0e38f, "taco_guided_attention: g=%g must be finite and positive", (double)g);
    TACO_CHECK(lam >= 0.f && lam <= 3.0e38f, "taco_guided_attention: lam=%g must be finite and >= 0", (double)lam);
    const int64_t rows = (int64_t)B * T;
    // the grid only sets how rows are dealt to warps: every row's arithmetic, and the reduction, are independent of it
    int blocks = (int)((rows + GA_WARPS - 1) / GA_WARPS);
    if (blocks > TACO_SMS * 8) blocks = TACO_SMS * 8;
    const float inv_2g2 = (float)(0.5 / ((double)g * (double)g));
    TACO_LAUNCH(guided_attention_kernel, blocks, 256, 0, (cudaStream_t)stream, dscore, partial_ws, align, text_length,
                speech_steps, B, T, Tx, inv_2g2, lam);
    TACO_LAUNCH_CHECK();
    TACO_LAUNCH(guided_attention_sum_kernel, 1, 256, 0, (cudaStream_t)stream, partial_ws, rows, (double)lam, loss);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_colsum(float* out, const float* A, int64_t lda, const float* Bm, int64_t ldb, const float* R, int64_t ldr, int M, int N,
                void* stream) {
    TACO_CHECK(out && A && M >= 0 && N >= 0, "taco_colsum: bad arguments");
    if (M == 0 || N == 0) return 0;
    const int colblocks = (N + 31) / 32;
    int rowblocks = (592 + colblocks - 1) / colblocks;
    const int maxrb = (M + 63) / 64;
    if (rowblocks > maxrb) rowblocks = maxrb;
    if (rowblocks < 1) rowblocks = 1;
    const int rpb = (M + rowblocks - 1) / rowblocks;
    rowblocks = (M + rpb - 1) / rpb;
    TACO_LAUNCH(colsum_kernel, dim3(colblocks, rowblocks), 256, 0, (cudaStream_t)stream, out, A, lda, Bm, ldb, R, ldr, M, N, rpb);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_bias_act(float* C, int64_t ldc, int M, int N, const float* bias, int act, void* stream) {
    TACO_CHECK(C && M >= 0 && N >= 0, "taco_bias_act: bad arguments");
    const int64_t total = (int64_t)M * N;
    if (total == 0) return 0;
    TACO_LAUNCH(bias_act_kernel, grid_for(total, 256), 256, 0, (cudaStream_t)stream, C, ldc, M, N, bias, act);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_mul_shift(float* out, int64_t ldo, const float* X, int64_t ldx, const float* Hm, int64_t ldh, int M, int N, int shift,
                   int period, void* stream) {
    TACO_CHECK(out && X && Hm, "taco_mul_shift: NULL");
    const int64_t total = (int64_t)M * N;
    if (total == 0) return 0;
    TACO_LAUNCH(mul_shift_kernel, grid_for(total, 256), 256, 0, (cudaStream_t)stream, out, ldo, X, ldx, Hm, ldh, M, N, shift, period);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_epi_bwd(float* dZ, int64_t lddz, const float* dY, int64_t lddy, const float* Y, int64_t ldy, const float* R, int64_t ldr,
                 int M, int N, int relu, const float* scale, const float* shift, float gain, void* stream) {
    TACO_CHECK(dZ && dY, "taco_epi_bwd: NULL");
    TACO_CHECK(!relu || Y, "taco_epi_bwd: relu needs the saved output Y");
    TACO_CHECK((scale == nullptr) == (shift == nullptr), "taco_epi_bwd: scale and shift go together");
    const int64_t total = (int64_t)M * N;
    if (total == 0) return 0;
    TACO_LAUNCH(epi_bwd_kernel, grid_for(total, 256), 256, 0, (cudaStream_t)stream, dZ, lddz, dY, lddy, Y, ldy, R, ldr, M, N, relu,
                scale, shift, gain);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_epi_fwd_keep(float* X, int64_t ldx, const uint8_t* keep, int M, int N, float gain, void* stream) {
    TACO_CHECK(X && keep, "taco_epi_fwd_keep: NULL");
    const int64_t total = (int64_t)M * N;
    if (total == 0) return 0;
    TACO_LAUNCH(epi_fwd_keep_kernel, grid_for(total, 256), 256, 0, (cudaStream_t)stream, X, ldx, keep, M, N, gain);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_bn_param_grad(float* dgamma, float* dbeta, const float* S1, const float* S2, const float* gamma, const float* beta, int N,
                       void* stream) {
    TACO_CHECK(dgamma && dbeta && S1 && S2 && gamma && beta, "taco_bn_param_grad: NULL");
    if (N == 0) return 0;
    TACO_LAUNCH(bn_param_grad_kernel, (N + 255) / 256, 256, 0, (cudaStream_t)stream, dgamma, dbeta, S1, S2, gamma, beta, N);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_maxpool_bwd(float* dX, const float* dP, const float* X, int B, int T, int C, void* stream) {
    TACO_CHECK(dX && dP && X, "taco_maxpool_bwd: NULL");
    const int64_t total = (int64_t)B * T * C;
    if (total == 0) return 0;
    TACO_LAUNCH(maxpool_bwd_kernel, grid_for(total, 256), 256, 0, (cudaStream_t)stream, dX, dP, X, T, C, total);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_highway_fwd(float* Y, int64_t ldy, const float* Pm, int64_t ldp, const float* X, int64_t ldx, int M, int U, void* stream) {
    TACO_CHECK(Y && Pm && X, "taco_highway_fwd: NULL");
    const int64_t total = (int64_t)M * U;
    if (total == 0) return 0;
    TACO_LAUNCH(highway_fwd_kernel, grid_for(total, 256), 256, 0, (cudaStream_t)stream, Y, ldy, Pm, ldp, X, ldx, M, U);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_highway_bwd(float* dP, int64_t lddp, float* dXd, int64_t lddx, const float* dY, int64_t lddy, const float* Pm, int64_t ldp,
                     const float* X, int64_t ldx, int M, int U, void* stream) {
    TACO_CHECK(dP && dXd && dY && Pm && X, "taco_highway_bwd: NULL");
    const int64_t total = (int64_t)M * U;
    if (total == 0) return 0;
    TACO_LAUNCH(highway_bwd_kernel, grid_for(total, 256), 256, 0, (cudaStream_t)stream, dP, lddp, dXd, lddx, dY, lddy, Pm, ldp, X,
                ldx, M, U);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_l1_bwd(float* dA, const float* A, const float* Bt, int64_t n, float beta, void* stream) {
    TACO_CHECK(dA && A && Bt && n >= 0, "taco_l1_bwd: bad arguments");
    if (n == 0) return 0;
    TACO_LAUNCH(l1_bwd_kernel, grid_for(n, 256), 256, 0, (cudaStream_t)stream, dA, A, Bt, n, beta);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_l1_bwd_ld(float* dA, int64_t ldd, const float* A, const float* Bt, int64_t rows, int64_t cols, float beta, void* stream) {
    TACO_CHECK(dA && A && Bt && rows >= 0 && cols >= 0 && ldd >= cols, "taco_l1_bwd_ld: bad arguments");
    if (rows * cols == 0) return 0;
    TACO_LAUNCH(l1_bwd_ld_kernel, grid_for(rows * cols, 256), 256, 0, (cudaStream_t)stream, dA, ldd, A, Bt, rows, cols, beta);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_scatter_add_rows(float* dTable, const int32_t* ids, const float* dRows, int rows, int width, int vocab, void* stream) {
    TACO_CHECK(dTable && ids && dRows && vocab > 0, "taco_scatter_add_rows: bad arguments");
    const int64_t total = (int64_t)rows * width;
    if (total == 0) return 0;
    TACO_LAUNCH(scatter_add_rows_kernel, grid_for(total, 256), 256, 0, (cudaStream_t)stream, dTable, ids, dRows, rows, width, vocab);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_dec_inputs(float* Xin, uint8_t* sel, const float* mel, const float* y, const uint8_t* sample_mask, int B, int T, int r,
                    int sched, void* stream) {
    TACO_CHECK(Xin && sel && mel, "taco_dec_inputs: NULL");
    TACO_CHECK(!sched || (y && sample_mask), "taco_dec_inputs: scheduled sampling needs y and sample_mask");
    const int64_t total = (int64_t)T * B * 80;
    if (total == 0) return 0;
    TACO_LAUNCH(dec_inputs_kernel, grid_for(total, 256), 256, 0, (cudaStream_t)stream, Xin, sel, mel, y, sample_mask, B, T, r, 80, sched);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_attn_bwd_post(float* dkeys, float* dv, const float* DSCORE, const float* keys, const float* PQ, const float* v, int B, int T,
                       int Tx, void* stream) {
    TACO_CHECK(dkeys && dv && DSCORE && keys && PQ && v, "taco_attn_bwd_post: NULL");
    if (B * Tx == 0) return 0;
    TACO_LAUNCH(attn_bwd_post_kernel, B * Tx, 256, 0, (cudaStream_t)stream, dkeys, dv, DSCORE, keys, PQ, v, B, T, Tx);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_sumsq(const float* x, int64_t n, float* partial_ws, float* out, void* stream) {
    TACO_CHECK((x || n == 0) && partial_ws && out && n >= 0, "taco_sumsq: bad arguments");   // an empty x may be NULL
    TACO_LAUNCH(sumsq_stage1, SS_BLOCKS, 256, 0, (cudaStream_t)stream, x, n, partial_ws);
    TACO_LAUNCH_CHECK();
    TACO_LAUNCH(sumsq_stage2, 1, 1024, 0, (cudaStream_t)stream, partial_ws, SS_BLOCKS, out);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_adam_step(float* p, const float* g, float* m, float* v, int64_t n, float lr_t, float b1, float b2, float eps, float clip,
                   const float* sumsq, void* stream) {
    TACO_CHECK(p && g && m && v && sumsq && n >= 0, "taco_adam_step: bad arguments");
    if (n == 0) return 0;
    TACO_LAUNCH(adam_kernel, grid_for(n, 256), 256, 0, (cudaStream_t)stream, p, g, m, v, n, lr_t, b1, b2, eps, clip, sumsq);
    TACO_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
