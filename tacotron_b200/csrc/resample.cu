// resample.cu -- sample-rate conversion for preprocessing: the resampling inside librosa.load(f, mono=True, sr=sr)
// (reference: audio.py:39) -- librosa 0.6 resample(res_type='kaiser_best') over resampy 0.2.2's interpolation loop, as
// restated in tests/resample_oracle.py.  Semantics pinned by tests/mirror_kernels_resample.py.
//
//   resample_kernel  one thread per output sample (grid row b = utterance b, grid-stride along it): the left and right
//                    wings of the windowed-sinc table around the sample's time-register position.  Every step is one
//                    IEEE operation with round-to-nearest (no contraction), so the result is bit-identical to the loop
#include "common.cuh"

namespace {

constexpr int RS_TABLE = 512;          // table entries per zero crossing (kaiser_best: precision 9)
constexpr int RS_THREADS = 256;

// y += (win + eta*delta) * x: weight and product in float64, the sum rounded to float32 (numba's `y[t] += w * x[..]`
// on a float32 array)
__device__ __forceinline__ float rs_tap(float acc, double2 wd, double eta, float x) {
    const double w = __dadd_rn(wd.x, __dmul_rn(eta, wd.y));
    return __double2float_rn(__dadd_rn((double)acc, __dmul_rn(w, (double)x)));
}

// out_b[t] for t < n_out = int(n_in * ratio): with n = int(treg[t]), frac = scale*(treg[t] - n) (scale = min(1, ratio)),
// the left wing reads x[n - i] at table entries off + i*step, the right wing x[n + 1 + k] at the entries of scale - frac.
// n_out <= t < out_off[b+1] - out_off[b] is librosa's zero padding; t >= treg_len is a caller error, written as NaN.
__global__ void __launch_bounds__(RS_THREADS) resample_kernel(float* __restrict__ out, const float* __restrict__ in,
                                                              const int64_t* __restrict__ in_off,
                                                              const int64_t* __restrict__ out_off,
                                                              const double2* __restrict__ wd, int nwin, int step,
                                                              double ratio, const double* __restrict__ treg,
                                                              int64_t treg_len) {
    const int b = blockIdx.y;
    const int64_t n_in = in_off[b + 1] - in_off[b], n_fix = out_off[b + 1] - out_off[b];
    const int64_t n_out = (int64_t)__dmul_rn((double)n_in, ratio);
    const double scale = ratio < 1.0 ? ratio : 1.0;
    const float* x = in + in_off[b];
    float* y = out + out_off[b];
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n_fix; t += (int64_t)gridDim.x * blockDim.x) {
        if (t >= n_out || t >= treg_len) {
            y[t] = t >= n_out ? 0.f : nanf("");
            continue;
        }
        const double tr = treg[t];
        const int64_t n = (int64_t)tr;
        double frac = __dmul_rn(scale, __dadd_rn(tr, -(double)n));
        double idx = __dmul_rn(frac, (double)RS_TABLE);
        int off = (int)idx;
        double eta = __dadd_rn(idx, -(double)off);
        int taps = (nwin - off) / step;
        if (n + 1 < taps) taps = (int)(n + 1);
        float acc = 0.f;
        for (int i = 0; i < taps; ++i) acc = rs_tap(acc, wd[off + i * step], eta, x[n - i]);
        frac = __dadd_rn(scale, -frac);
        idx = __dmul_rn(frac, (double)RS_TABLE);
        off = (int)idx;
        eta = __dadd_rn(idx, -(double)off);
        taps = (nwin - off) / step;
        if (n_in - n - 1 < taps) taps = (int)(n_in - n - 1);
        for (int k = 0; k < taps; ++k) acc = rs_tap(acc, wd[off + k * step], eta, x[n + 1 + k]);
        y[t] = acc;
    }
}

}  // namespace

extern "C" {

int taco_resample(float* out, const float* in, const int64_t* in_off, const int64_t* out_off, int B, const double* win_delta,
                  int nwin, int step, double ratio, const double* treg, int64_t treg_len, void* stream) {
    TACO_CHECK(out && in && in_off && out_off && win_delta && treg && B >= 0, "taco_resample: bad arguments");
    TACO_CHECK(taco_aligned16(win_delta), "taco_resample: win_delta must be 16-byte aligned");
    TACO_CHECK(B <= 65535, "taco_resample: B=%d utterances in one call (at most 65535)", B);
    TACO_CHECK(ratio > 0.0 && step >= 1 && step <= RS_TABLE && nwin > RS_TABLE && treg_len >= 1,
               "taco_resample: need ratio=%g > 0, 1 <= step=%d <= %d, nwin=%d > %d, treg_len=%lld >= 1", ratio, step,
               RS_TABLE, nwin, RS_TABLE, (long long)treg_len);
    if (B == 0) return 0;
    // sized for the longest output the register covers (n_fix <= n_out + 1 <= treg_len + 1); grid-stride beyond that
    int64_t gx = (treg_len + RS_THREADS) / RS_THREADS;
    if (gx > 65535) gx = 65535;
    TACO_LAUNCH(resample_kernel, dim3((unsigned)gx, (unsigned)B), RS_THREADS, 0, (cudaStream_t)stream, out, in, in_off, out_off,
                reinterpret_cast<const double2*>(win_delta), nwin, step, ratio, treg, treg_len);
    TACO_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
