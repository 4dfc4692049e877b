// api.cu -- C-ABI glue: error strings, device query, dispatch, and the small bandwidth-bound
// kernels (max-pool, row gather, length mask, L1 loss).  See include/taco_b200.h.
#include <stdarg.h>
#include "common.cuh"

static thread_local char g_err[1024] = "";
unsigned long long g_taco_launches = 0;

void taco_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int taco_linear_simt(const taco_linear_desc* d, cudaStream_t st);
int taco_linear_tc(const taco_linear_desc* d, cudaStream_t st);
int taco_linear_tc_route(const taco_linear_desc* d, TcRoute* r);
int taco_pack_weight_impl(const float* W, int taps, int C, int N, float* dst, int64_t ld_dst, cudaStream_t st);
int taco_pack_weight_x3_impl(const float* W, int taps, int C, int N, float* dst_hi, float* dst_lo, int64_t ld_dst, cudaStream_t st);
int taco_conv_dw_tc_impl(float* dW, int64_t ldw, int64_t tap_stride, const float* X, int64_t ldx, const float* dZ, int64_t lddz,
                         int B, int T, int C, int N, int taps, int tap0, cudaStream_t st);
int taco_highway_stack(const taco_highway_stack_desc* d, cudaStream_t st);

namespace {

// tf.layers.max_pooling1d(pool_size=2, strides=1, padding='same')  models/ops.py:66-71
__global__ void maxpool_kernel(const float4* __restrict__ X, float4* __restrict__ Y, int T, int C4, int64_t total) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t row = i / C4;
        int t = (int)(row % T);
        float4 a = X[i];
        if (t + 1 < T) {
            float4 b = X[i + C4];
            a.x = fmaxf(a.x, b.x); a.y = fmaxf(a.y, b.y); a.z = fmaxf(a.z, b.z); a.w = fmaxf(a.w, b.w);
        }
        Y[i] = a;
    }
}

__global__ void gather_rows_kernel(const float* __restrict__ table, const int32_t* __restrict__ ids, int rows, int width,
                                   int vocab, const uint8_t* __restrict__ keep, float keep_scale, float* __restrict__ Y) {
    int64_t total = (int64_t)rows * width;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int row = (int)(i / width), c = (int)(i % width);
        int id = ids[row];
        id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
        float v = table[(int64_t)id * width + c];
        if (keep) v = keep[i] ? v * keep_scale : 0.0f;
        Y[i] = v;
    }
}

__global__ void mask_rows_kernel(const float4* __restrict__ X, const int32_t* __restrict__ len, float4* __restrict__ Y,
                                 int T, int C4, int64_t total) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t row = i / C4;
        int t = (int)(row % T);
        int b = (int)(row / T);
        float4 v = X[i];
        if (t >= len[b]) v = make_float4(0.f, 0.f, 0.f, 0.f);
        Y[i] = v;
    }
}

// deterministic two-stage sum |a-b|: fixed grid, fixed per-block order, double accumulation in stage 2
constexpr int L1_BLOCKS = TACO_SMS * 8;
__global__ void l1_stage1(const float* __restrict__ a, const float* __restrict__ b, int64_t n, float* __restrict__ partial) {
    __shared__ float red[8];
    float acc = 0.f;
    const int64_t n4 = n / 4;
    const float4* a4 = reinterpret_cast<const float4*>(a);
    const float4* b4 = reinterpret_cast<const float4*>(b);
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 x = __ldcs(a4 + i), y = __ldcs(b4 + i);
        acc += fabsf(x.x - y.x) + fabsf(x.y - y.y) + fabsf(x.z - y.z) + fabsf(x.w - y.w);
    }
    if (blockIdx.x == 0) for (int64_t i = n4 * 4 + threadIdx.x; i < n; i += blockDim.x) acc += fabsf(a[i] - b[i]);
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
__global__ void l1_stage2(const float* __restrict__ partial, int n, float* __restrict__ out) {
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

// the checks every taco_linear_fwd descriptor passes, whichever kernel runs it
int linear_check(const taco_linear_desc* d) {
    TACO_CHECK(d != nullptr, "taco_linear_fwd: NULL descriptor");
    TACO_CHECK(d->X && d->Y, "taco_linear_fwd: X or Y is NULL");
    TACO_CHECK(d->B >= 0 && d->T >= 0 && d->C > 0 && d->N > 0, "taco_linear_fwd: bad sizes B=%d T=%d C=%d N=%d", d->B, d->T, d->C, d->N);
    TACO_CHECK(d->bank_K > 0 || d->taps >= 1, "taco_linear_fwd: taps must be >= 1");
    TACO_CHECK(d->ldx >= d->C, "taco_linear_fwd: ldx < C");
    const bool highway = d->epilogue == TACO_EPI_HIGHWAY;
    const int nout = highway ? d->N / 2 : d->N;
    TACO_CHECK(d->ldy >= nout, "taco_linear_fwd: ldy %lld < %d output columns (N, or N/2 for highway)", (long long)d->ldy, nout);
    TACO_CHECK(!d->residual || d->ldr >= d->N, "taco_linear_fwd: ldr %lld < N %d", (long long)d->ldr, d->N);
    TACO_CHECK(!highway || !d->hx || d->ldhx >= nout, "taco_linear_fwd: ldhx %lld < U %d", (long long)d->ldhx, nout);
    // both highway epilogues compute relu(H)*sig(T) + hx*(1-sig(T)) and nothing else: refuse fields they would ignore
    TACO_CHECK(!highway || (d->act == TACO_ACT_NONE && !d->scale && !d->shift && !d->keep && !d->residual && !d->pool),
               "taco_linear_fwd: the highway epilogue takes only bias and hx (act, scale, shift, keep, residual, pool are not applied)");
    TACO_CHECK(!d->bias_utt || (!highway && d->ldbu >= d->N),
               "taco_linear_fwd: bias_utt needs the normal epilogue and ldbu >= N");
    return 0;
}

inline int grid_for(int64_t total, int block) {
    int64_t g = (total + block - 1) / block;
    if (g > TACO_SMS * 16) g = TACO_SMS * 16;
    if (g < 1) g = 1;
    return (int)g;
}

}  // namespace

extern "C" {

const char* taco_last_error(void) { return g_err; }
int taco_version(void) { return TACO_VERSION; }

int taco_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    int dev = 0;
    TACO_CUDA(cudaGetDevice(&dev));
    cudaDeviceProp p;
    TACO_CUDA(cudaGetDeviceProperties(&p, dev));
    if (sm_count) *sm_count = p.multiProcessorCount;
    if (cc_major) *cc_major = p.major;
    if (cc_minor) *cc_minor = p.minor;
    return 0;
}

int taco_linear_fwd(const taco_linear_desc* d, void* stream) {
    if (int rc = linear_check(d)) return rc;
    if (d->impl == TACO_IMPL_SIMT) return taco_linear_simt(d, (cudaStream_t)stream);
    if (d->impl == TACO_IMPL_TC || d->impl == TACO_IMPL_TC3) return taco_linear_tc(d, (cudaStream_t)stream);
    taco_set_error("taco_linear_fwd: unknown impl %d", d->impl);
    return 1;
}

int taco_linear_route(const taco_linear_desc* d, int* bn, int* stages, int* mode, int* direct, int* tile_stride) {
    if (int rc = linear_check(d)) return rc;
    TcRoute r;
    if (d->impl == TACO_IMPL_SIMT) {
        // gemm_simt.cu: 64 x 64 tiles over the flattened rows, one k-block in shared memory, element-wise epilogue
        TACO_CHECK(!d->pool, "taco_linear_fwd(SIMT): fused max-pool is only available on the tensor-core path");
        r.bn = 64; r.stages = 1; r.mode = d->epilogue == TACO_EPI_HIGHWAY ? 1 : 0; r.direct = 0; r.tile_stride = 64;
    } else if (d->impl == TACO_IMPL_TC || d->impl == TACO_IMPL_TC3) {
        if (int rc = taco_linear_tc_route(d, &r)) return rc;
    } else {
        taco_set_error("taco_linear_fwd: unknown impl %d", d->impl);
        return 1;
    }
    if (bn) *bn = r.bn;
    if (stages) *stages = r.stages;
    if (mode) *mode = r.mode;
    if (direct) *direct = r.direct;
    if (tile_stride) *tile_stride = r.tile_stride;
    return 0;
}

int taco_highway_stack_fwd(const taco_highway_stack_desc* d, void* stream) {
    return taco_highway_stack(d, (cudaStream_t)stream);
}

int taco_pack_weight_x3(const float* W, int taps, int C, int N, float* dst_hi, float* dst_lo, int64_t ld_dst, void* stream) {
    TACO_CHECK(W && dst_hi && dst_lo && taps >= 1 && C >= 1 && N >= 1, "taco_pack_weight_x3: bad arguments");
    return taco_pack_weight_x3_impl(W, taps, C, N, dst_hi, dst_lo, ld_dst, (cudaStream_t)stream);
}

int taco_conv_dw(float* dW, int64_t ldw, int64_t tap_stride, const float* X, int64_t ldx, const float* dZ, int64_t lddz,
                 int B, int T, int C, int N, int taps, int tap0, void* stream) {
    TACO_CHECK(dW && X && dZ, "taco_conv_dw: NULL");
    return taco_conv_dw_tc_impl(dW, ldw, tap_stride, X, ldx, dZ, lddz, B, T, C, N, taps, tap0, (cudaStream_t)stream);
}

int taco_pack_weight(const float* W, int taps, int C, int N, float* dst, int64_t ld_dst, void* stream) {
    TACO_CHECK(W && dst && taps >= 1 && C >= 1 && N >= 1, "taco_pack_weight: bad arguments");
    return taco_pack_weight_impl(W, taps, C, N, dst, ld_dst, (cudaStream_t)stream);
}

int taco_maxpool_fwd(const float* X, float* Y, int B, int T, int C, void* stream) {
    TACO_CHECK(X && Y, "taco_maxpool_fwd: NULL");
    TACO_CHECK((C % 4) == 0 && taco_aligned16(X) && taco_aligned16(Y), "taco_maxpool_fwd: C %% 4 != 0 or unaligned");
    int64_t total = (int64_t)B * T * (C / 4);
    if (total == 0) return 0;
    maxpool_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(X),
                                                                           reinterpret_cast<float4*>(Y), T, C / 4, total);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_gather_rows(const float* table, const int32_t* ids, int rows, int width, int vocab, const uint8_t* keep,
                     float keep_scale, float* Y, void* stream) {
    TACO_CHECK(table && ids && Y && vocab > 0, "taco_gather_rows: bad arguments");
    int64_t total = (int64_t)rows * width;
    if (total == 0) return 0;
    gather_rows_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(table, ids, rows, width, vocab, keep, keep_scale, Y);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_mask_rows(const float* X, const int32_t* length, float* Y, int B, int T, int C, void* stream) {
    TACO_CHECK(X && Y && length, "taco_mask_rows: NULL");
    TACO_CHECK((C % 4) == 0 && taco_aligned16(X) && taco_aligned16(Y), "taco_mask_rows: C %% 4 != 0 or unaligned");
    int64_t total = (int64_t)B * T * (C / 4);
    if (total == 0) return 0;
    mask_rows_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(X), length,
                                                                             reinterpret_cast<float4*>(Y), T, C / 4, total);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_l1_loss_fwd(const float* a, const float* b, int64_t n, float* partial_ws, float* out, void* stream) {
    TACO_CHECK(((a && b) || n == 0) && partial_ws && out && n >= 0, "taco_l1_loss_fwd: bad arguments");   // empty inputs may be NULL
    TACO_CHECK(taco_aligned16(a) && taco_aligned16(b), "taco_l1_loss_fwd: inputs must be 16-byte aligned");
    l1_stage1<<<L1_BLOCKS, 256, 0, (cudaStream_t)stream>>>(a, b, n, partial_ws);
    TACO_LAUNCH_CHECK();
    l1_stage2<<<1, 1024, 0, (cudaStream_t)stream>>>(partial_ws, L1_BLOCKS, out);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_l1_partial_count(void) { return L1_BLOCKS; }

unsigned long long taco_launch_count(void) { return g_taco_launches; }

}  // extern "C"
