// summary.cu -- the per-step histogram summaries of training (reference: tf.summary.histogram at models/tacotron.py:129,
// 139,152): TF 1.2's HistogramSummaryOp / histogram::Histogram::Add over one contiguous float32 tensor, reduced on the
// device.  Semantics pinned by tests/mirror_kernels_summary.py (and tests/summary_oracle.py, the sequential restatement).
//
//   hist_partial   fixed grid of HIST_BLOCKS CTAs, grid-stride over float4 chunks (HIST_UNROLL loads in flight per
//                  thread).  Each CTA bins into a shared-memory histogram (1551 counters, integer atomics) and reduces
//                  its threads' {min, max, sum, sum of squares, non-finite count} in a fixed tree; one row of the
//                  workspace per CTA.
//   hist_final     CTA c < HIST_FINAL_BUCKET_CTAS sums the counts of 32 buckets over the HIST_BLOCKS rows (integers: exact
//                  in any order); the last CTA reduces the statistics rows in a fixed order.  Grid and block sizes do not
//                  depend on n, so sum and sum of squares are bit-identical from run to run.
//
// Bucket index.  TF's default table is [-DBL_MAX, -p[773] .. -p[0], 0.0, p[0] .. p[773], DBL_MAX] with p[0] = 1e-12,
// p[k+1] = p[k]*1.1 (float64, repeated multiplication) while p < 1e20.  A value goes to upper_bound(limits, x): with
// j(a) = #{k : p[k] <= a}, that is 776 + j(x) for x > 0, 776 for x = +-0, and 775 - j(|x|) for x < 0 (no nonzero limit is
// a float32 value, so |x| never equals a p[k]).  j comes from a guess log(a/1e-12)/log(1.1) + 1 corrected against the
// float64 table in shared memory -- the correction makes it exact whatever the guess; the guess makes it 0-1 steps.
#include <float.h>
#include "common.cuh"

namespace {

constexpr int HIST_NLIM = 1551;                // TF's default bucket table
constexpr int HIST_NPOS = 774;                 // positive finite limits p[0..773]
constexpr int HIST_ZERO = 775;                 // index of the 0.0 limit
constexpr int HIST_THREADS = 512;
constexpr int HIST_BLOCKS = 2 * TACO_SMS;      // two 512-thread CTAs per SM
constexpr int HIST_UNROLL = 4;                 // float4 loads in flight per thread
constexpr int HIST_FINAL_THREADS = 256;
constexpr int HIST_FINAL_BUCKET_CTAS = (HIST_NLIM + 31) / 32;

// workspace layout (per CTA row r < HIST_BLOCKS)
struct HistWs {
    double sum[HIST_BLOCKS], sumsq[HIST_BLOCKS];
    float mn[HIST_BLOCKS], mx[HIST_BLOCKS];
    unsigned long long nonfinite[HIST_BLOCKS];
    unsigned int counts[HIST_BLOCKS][HIST_NLIM];
};

struct HistAcc {
    double sum = 0.0, sumsq = 0.0;
    float mn = INFINITY, mx = -INFINITY;
    unsigned long long nonfinite = 0;
};

__device__ __forceinline__ int hist_bucket(float x, const double* __restrict__ pos) {
    const float a = fabsf(x);
    if (a == 0.f) return HIST_ZERO + 1;
    // k = log(a/1e-12)/log(1.1) = (log2(a) + 39.863137) * 7.2725409; j = #{p[k] <= a} ~ floor(k) + 1
    float g = floorf((log2f(a) + 39.8631371386f) * 7.27254089734f) + 1.f;
    g = fminf(fmaxf(g, 0.f), (float)HIST_NPOS);
    int j = (int)g;
    const double ad = (double)a;
    while (j > 0 && pos[j - 1] > ad) --j;
    while (j < HIST_NPOS && pos[j] <= ad) ++j;
    return x > 0.f ? HIST_ZERO + 1 + j : HIST_ZERO - j;
}

__device__ __forceinline__ void hist_add(float x, HistAcc& acc, unsigned int* cnt, const double* pos) {
    if (!isfinite(x)) {
        ++acc.nonfinite;
        return;
    }
    atomicAdd(&cnt[hist_bucket(x, pos)], 1u);
    acc.mn = fminf(acc.mn, x);
    acc.mx = fmaxf(acc.mx, x);
    const double d = (double)x;
    acc.sum += d;
    acc.sumsq += d * d;
}

__global__ void __launch_bounds__(HIST_THREADS) hist_partial(const float* __restrict__ x, int64_t n,
                                                              const double* __restrict__ limits, HistWs* __restrict__ ws) {
    __shared__ double pos[HIST_NPOS];
    __shared__ unsigned int cnt[HIST_NLIM];
    __shared__ double r_sum[HIST_THREADS], r_sq[HIST_THREADS];
    __shared__ float r_mn[HIST_THREADS], r_mx[HIST_THREADS];
    __shared__ unsigned long long r_nf[HIST_THREADS];
    const int tid = threadIdx.x;
    for (int i = tid; i < HIST_NPOS; i += HIST_THREADS) pos[i] = limits[HIST_ZERO + 1 + i];
    for (int i = tid; i < HIST_NLIM; i += HIST_THREADS) cnt[i] = 0u;
    __syncthreads();

    HistAcc acc;
    const int64_t n4 = n / 4;
    const float4* x4 = reinterpret_cast<const float4*>(x);
    constexpr int64_t per_cta = (int64_t)HIST_UNROLL * HIST_THREADS;
    for (int64_t base = (int64_t)blockIdx.x * per_cta; base < n4; base += (int64_t)HIST_BLOCKS * per_cta) {
        float4 v[HIST_UNROLL];
#pragma unroll
        for (int u = 0; u < HIST_UNROLL; ++u) {
            const int64_t i = base + (int64_t)u * HIST_THREADS + tid;
            v[u] = i < n4 ? __ldcs(x4 + i) : make_float4(NAN, NAN, NAN, NAN);
        }
#pragma unroll
        for (int u = 0; u < HIST_UNROLL; ++u) {
            if (base + (int64_t)u * HIST_THREADS + tid >= n4) break;
            hist_add(v[u].x, acc, cnt, pos);
            hist_add(v[u].y, acc, cnt, pos);
            hist_add(v[u].z, acc, cnt, pos);
            hist_add(v[u].w, acc, cnt, pos);
        }
    }
    if (blockIdx.x == 0 && 4 * n4 + tid < n) hist_add(x[4 * n4 + tid], acc, cnt, pos);   // the n % 4 tail

    r_sum[tid] = acc.sum; r_sq[tid] = acc.sumsq; r_mn[tid] = acc.mn; r_mx[tid] = acc.mx; r_nf[tid] = acc.nonfinite;
    __syncthreads();
    for (int s = HIST_THREADS / 2; s > 0; s >>= 1) {
        if (tid < s) {
            r_sum[tid] += r_sum[tid + s];
            r_sq[tid] += r_sq[tid + s];
            r_mn[tid] = fminf(r_mn[tid], r_mn[tid + s]);
            r_mx[tid] = fmaxf(r_mx[tid], r_mx[tid + s]);
            r_nf[tid] += r_nf[tid + s];
        }
        __syncthreads();
    }
    const int b = blockIdx.x;
    if (tid == 0) {
        ws->sum[b] = r_sum[0]; ws->sumsq[b] = r_sq[0]; ws->mn[b] = r_mn[0]; ws->mx[b] = r_mx[0]; ws->nonfinite[b] = r_nf[0];
    }
    for (int i = tid; i < HIST_NLIM; i += HIST_THREADS) ws->counts[b][i] = cnt[i];
}

// counts[k] = sum over the CTA rows; stats = {min, max, sum, sum of squares} (TF's empty histogram: min = DBL_MAX,
// max = -DBL_MAX); nonfinite[0] = NaN/Inf elements
__global__ void __launch_bounds__(HIST_FINAL_THREADS) hist_final(const HistWs* __restrict__ ws, int64_t* __restrict__ counts,
                                                                  double* __restrict__ stats, int64_t* __restrict__ nonfinite) {
    constexpr int WARPS = HIST_FINAL_THREADS / 32;
    __shared__ unsigned long long part[WARPS][32];
    __shared__ double r_sum[HIST_FINAL_THREADS], r_sq[HIST_FINAL_THREADS], r_mn[HIST_FINAL_THREADS], r_mx[HIST_FINAL_THREADS];
    __shared__ unsigned long long r_nf[HIST_FINAL_THREADS];
    const int tid = threadIdx.x;
    if (blockIdx.x < HIST_FINAL_BUCKET_CTAS) {
        const int lane = tid % 32, w = tid / 32, k = blockIdx.x * 32 + lane;
        unsigned long long s = 0;
        if (k < HIST_NLIM)
            for (int r = w; r < HIST_BLOCKS; r += WARPS) s += ws->counts[r][k];
        part[w][lane] = s;
        __syncthreads();
        if (w == 0 && k < HIST_NLIM) {
            for (int i = 1; i < WARPS; ++i) s += part[i][lane];
            counts[k] = (int64_t)s;
        }
        return;
    }
    double sum = 0.0, sq = 0.0, mn = DBL_MAX, mx = -DBL_MAX;
    unsigned long long nf = 0;
    for (int r = tid; r < HIST_BLOCKS; r += HIST_FINAL_THREADS) {
        sum += ws->sum[r]; sq += ws->sumsq[r];
        mn = fmin(mn, (double)ws->mn[r]); mx = fmax(mx, (double)ws->mx[r]);
        nf += ws->nonfinite[r];
    }
    r_sum[tid] = sum; r_sq[tid] = sq; r_mn[tid] = mn; r_mx[tid] = mx; r_nf[tid] = nf;
    __syncthreads();
    for (int s = HIST_FINAL_THREADS / 2; s > 0; s >>= 1) {
        if (tid < s) {
            r_sum[tid] += r_sum[tid + s];
            r_sq[tid] += r_sq[tid + s];
            r_mn[tid] = fmin(r_mn[tid], r_mn[tid + s]);
            r_mx[tid] = fmax(r_mx[tid], r_mx[tid + s]);
            r_nf[tid] += r_nf[tid + s];
        }
        __syncthreads();
    }
    if (tid == 0) {
        stats[0] = r_mn[0]; stats[1] = r_mx[0]; stats[2] = r_sum[0]; stats[3] = r_sq[0];
        nonfinite[0] = (int64_t)r_nf[0];
    }
}

}  // namespace

extern "C" {

size_t taco_histogram_workspace_bytes(void) { return sizeof(HistWs); }

int taco_histogram(const float* x, int64_t n, const double* limits, int nlim, void* workspace, int64_t* counts, double* stats,
                   int64_t* nonfinite, void* stream) {
    TACO_CHECK(x && limits && workspace && counts && stats && nonfinite && n >= 0, "taco_histogram: bad arguments");
    TACO_CHECK(nlim == HIST_NLIM, "taco_histogram: nlim=%d, the kernel bins into TF's default table of %d limits", nlim,
               HIST_NLIM);
    TACO_CHECK(taco_aligned16(x), "taco_histogram: x must be 16-byte aligned");
    TACO_CHECK(taco_aligned16(workspace), "taco_histogram: workspace must be 16-byte aligned");
    // a CTA's shared counters are 32-bit
    TACO_CHECK(n / HIST_BLOCKS < (int64_t)1 << 31, "taco_histogram: n=%lld elements in one call is too many", (long long)n);
    HistWs* ws = static_cast<HistWs*>(workspace);
    TACO_LAUNCH(hist_partial, HIST_BLOCKS, HIST_THREADS, 0, (cudaStream_t)stream, x, n, limits, ws);
    TACO_LAUNCH_CHECK();
    TACO_LAUNCH(hist_final, HIST_FINAL_BUCKET_CTAS + 1, HIST_FINAL_THREADS, 0, (cudaStream_t)stream, ws, counts, stats,
                nonfinite);
    TACO_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
