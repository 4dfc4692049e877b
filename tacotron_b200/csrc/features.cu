// features.cu -- feature extraction for preprocessing: the analysis half of the STFT, around the library's own
// taco_rfft2048 (reference: preprocess.py:168-208 preprocess, audio.py:38-65 process_audio; librosa effects.trim / stft /
// feature.melspectrogram as restated in tests/feature_oracle.py).  Semantics pinned by tests/mirror_kernels_features.py.
//
//   trim_kernel            librosa.effects.trim: frame energies in fp64, their maximum, first / last non-silent frame
//   feature_frames_kernel  trim offset, zero padding, pre-emphasis, reflect padding, framing, window (one thread per
//                          output element, like gl_frame_kernel); the output goes straight into taco_rfft2048
//   feature_spec_kernel    |X|, the complex mel product, log(. + 1e-8), scattered into the reshape_frames layout
#include <cuda_fp16.h>
#include <limits.h>
#include "common.cuh"

namespace {

constexpr int NBINS = 1025;            // bins of taco_rfft2048 (n_fft = 2048)
constexpr int TRIM_THREADS = 256;
constexpr int TRIM_MAX_PER = 16;       // frame_length / hop the trim kernel supports

inline int grid_for(int64_t total, int block) {
    int64_t g = (total + block - 1) / block;
    if (g > TACO_SMS * 32) g = TACO_SMS * 32;
    if (g < 1) g = 1;
    return (int)g;
}

// sum of squares, in fp64, of block k (samples [k*hop, (k+1)*hop)) of x reflect-padded by `pad` on both sides
__device__ double block_sumsq(const float* x, int64_t len, int pad, int hop, int64_t k) {
    double s = 0.0;
    const int64_t p0 = k * hop - pad;
    for (int i = 0; i < hop; ++i) {
        int64_t q = p0 + i;
        if (q < 0) q = -q;
        if (q >= len) q = 2 * (len - 1) - q;
        const double v = (double)x[q];
        s = fma(v, v, s);
    }
    return s;
}

// mean-square energies of the frames f0 + tid (frame f = blocks f .. f+per-1); every thread of the CTA calls this
__device__ double tile_energy(double* blk, const float* x, int64_t len, int pad, int hop, int per, int64_t f0, int64_t nblk) {
    const int tid = threadIdx.x;
    for (int i = tid; i < TRIM_THREADS + per - 1; i += TRIM_THREADS) {
        const int64_t k = f0 + i;
        blk[i] = (k < nblk) ? block_sumsq(x, len, pad, hop, k) : 0.0;
    }
    __syncthreads();
    double e = 0.0;
    for (int j = 0; j < per; ++j) e += blk[tid + j];
    __syncthreads();                                                   // blk is refilled by the next tile
    return e / (double)(per * hop);
}

__device__ double block_max(double* red, double v) {
    const int tid = threadIdx.x;
    red[tid] = v;
    __syncthreads();
    for (int s = TRIM_THREADS / 2; s > 0; s >>= 1) {
        if (tid < s) red[tid] = fmax(red[tid], red[tid + s]);
        __syncthreads();
    }
    const double out = red[0];
    __syncthreads();
    return out;
}

// one CTA per utterance.  Frame f (f < 1 + len/hop) of the signal reflect-padded by frame_length/2 is non-silent when
// 10 log10(max(1e-10, e_f)) - 10 log10(max(1e-10, max e)) > -top_db; bounds = [first*hop, min(len, (last+1)*hop)),
// or [0, 0) if no frame is (librosa.effects.trim, frames_to_samples)
__global__ void __launch_bounds__(TRIM_THREADS) trim_kernel(int* __restrict__ bounds, const float* __restrict__ y,
                                                            const int64_t* __restrict__ offsets, int frame_length, int hop,
                                                            float top_db) {
    __shared__ double blk[TRIM_THREADS + TRIM_MAX_PER];
    __shared__ double red[TRIM_THREADS];
    __shared__ int ifirst[TRIM_THREADS], ilast[TRIM_THREADS];
    const int b = blockIdx.x, tid = threadIdx.x;
    const int64_t len = offsets[b + 1] - offsets[b];
    const float* x = y + offsets[b];
    const int pad = frame_length / 2, per = frame_length / hop;
    if (len <= pad) {                       // too short to reflect-pad: the host rejects these; keep the reads in bounds
        if (tid == 0) { bounds[2 * b] = 0; bounds[2 * b + 1] = (int)len; }
        return;
    }
    const int64_t nf = 1 + len / hop, nblk = nf + per - 1;
    double emax = 0.0;
    for (int64_t f0 = 0; f0 < nf; f0 += TRIM_THREADS) {
        const double e = tile_energy(blk, x, len, pad, hop, per, f0, nblk);
        if (f0 + tid < nf) emax = fmax(emax, e);
    }
    emax = block_max(red, emax);
    const double ref_db = 10.0 * log10(fmax(1e-10, emax));
    int first = INT_MAX, last = -1;
    for (int64_t f0 = 0; f0 < nf; f0 += TRIM_THREADS) {
        const double e = tile_energy(blk, x, len, pad, hop, per, f0, nblk);
        const int f = (int)(f0 + tid);
        if (f < nf && 10.0 * log10(fmax(1e-10, e)) - ref_db > -(double)top_db) {
            first = min(first, f);
            last = max(last, f);
        }
    }
    ifirst[tid] = first;
    ilast[tid] = last;
    __syncthreads();
    for (int s = TRIM_THREADS / 2; s > 0; s >>= 1) {
        if (tid < s) {
            ifirst[tid] = min(ifirst[tid], ifirst[tid + s]);
            ilast[tid] = max(ilast[tid], ilast[tid + s]);
        }
        __syncthreads();
    }
    if (tid == 0) {
        if (ilast[0] < 0) {
            bounds[2 * b] = 0; bounds[2 * b + 1] = 0;
        } else {
            const int64_t end = (int64_t)(ilast[0] + 1) * hop;
            bounds[2 * b] = ifirst[0] * hop;
            bounds[2 * b + 1] = (int)(end < len ? end : len);
        }
    }
}

// frw[b,t,j] = w[j] * e_b[reflect(t*hop + j - n_fft/2)],  e_b = pre-emphasis of w_b = y[start_b : start_b + len_b] zero-padded
// to max_len: e[0] = w[0], e[q] = w[q] - preemph*w[q-1] (two float32 roundings, as numpy evaluates audio.py:54)
__global__ void feature_frames_kernel(float* __restrict__ frw, const float* __restrict__ y, const int64_t* __restrict__ start,
                                      const int* __restrict__ len, int n_frames, int max_len, int hop, int n_fft, int win_length,
                                      float preemph, int64_t total) {
    const int lpad = (n_fft - win_length) / 2;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int j = (int)(i % n_fft);
        const int t = (int)((i / n_fft) % n_frames);
        const int b = (int)(i / ((int64_t)n_fft * n_frames));
        const float w = hann_at(j, lpad, win_length);
        float v = 0.f;
        if (w != 0.f) {
            int q = t * hop + j - n_fft / 2;
            if (q < 0) q = -q;
            if (q >= max_len) q = 2 * (max_len - 1) - q;
            const float* x = y + start[b];
            const int L = len[b];
            float e = q < L ? x[q] : 0.f;
            if (q > 0) e = __fsub_rn(e, __fmul_rn(preemph, q - 1 < L ? x[q - 1] : 0.f));
            v = w * e;
        }
        frw[i] = v;
    }
}

__device__ __forceinline__ void store_out(void* out, int out_f16, int64_t i, float v) {
    if (out_f16) reinterpret_cast<__half*>(out)[i] = __float2half_rn(v);
    else reinterpret_cast<float*>(out)[i] = v;
}

// one CTA per (utterance, frame f < 4r*(n_frames/4r)).  Frame f = 4r*b4 + 4c + tl lands in row 4*b4 + tl, column block c
// (reshape_frames(forward=True), audio.py:23-28).  stft = log(|X| + 1e-8); mel[m] = log(|sum_{k in [lo_m, hi_m)} basis[m][k]
// X[k]| + 1e-8): the basis multiplies the complex spectrum (melspectrogram(S=stft), audio.py:57).  One warp per filter.
__global__ void __launch_bounds__(256) feature_spec_kernel(void* __restrict__ stft_out, void* __restrict__ mel_out, int out_f16,
                                                           const float2* __restrict__ X, const float* __restrict__ basis,
                                                           const int* __restrict__ mel_lo, const int* __restrict__ mel_hi,
                                                           int n_frames, int nf_used, int r, int n_mels) {
    __shared__ float2 xs[NBINS];
    const int f = blockIdx.x % nf_used, b = blockIdx.x / nf_used;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int rows = nf_used / r;
    const int b4 = f / (4 * r), rem = f % (4 * r), c = rem >> 2, tl = rem & 3;
    const int64_t row = (int64_t)b * rows + 4 * b4 + tl;
    const float2* Xf = X + ((int64_t)b * n_frames + f) * NBINS;
    const int64_t so = row * ((int64_t)NBINS * r) + (int64_t)c * NBINS;
    for (int k = tid; k < NBINS; k += 256) {
        const float2 z = Xf[k];
        xs[k] = z;
        store_out(stft_out, out_f16, so + k, logf(hypotf(z.x, z.y) + 1e-8f));
    }
    __syncthreads();
    const int64_t mo = row * ((int64_t)n_mels * r) + (int64_t)c * n_mels;
    for (int m = warp; m < n_mels; m += 8) {
        const float* wm = basis + (int64_t)m * NBINS;
        float re = 0.f, im = 0.f;
        for (int k = mel_lo[m] + lane; k < mel_hi[m]; k += 32) {
            const float wk = wm[k];
            re = fmaf(wk, xs[k].x, re);
            im = fmaf(wk, xs[k].y, im);
        }
        for (int s = 16; s > 0; s >>= 1) {
            re += __shfl_xor_sync(0xffffffffu, re, s);
            im += __shfl_xor_sync(0xffffffffu, im, s);
        }
        if (lane == 0) store_out(mel_out, out_f16, mo + m, logf(hypotf(re, im) + 1e-8f));
    }
}

}  // namespace

extern "C" {

int taco_trim_bounds(int* bounds, const float* y, const int64_t* offsets, int B, int frame_length, int hop, float top_db,
                     void* stream) {
    TACO_CHECK(bounds && y && offsets && B >= 0, "taco_trim_bounds: bad arguments");
    TACO_CHECK(hop >= 1 && frame_length % 2 == 0 && frame_length % hop == 0 && frame_length / hop <= TRIM_MAX_PER,
               "taco_trim_bounds: frame_length=%d must be an even multiple of hop=%d, at most %d hops", frame_length, hop,
               TRIM_MAX_PER);
    if (B == 0) return 0;
    TACO_LAUNCH(trim_kernel, B, TRIM_THREADS, 0, (cudaStream_t)stream, bounds, y, offsets, frame_length, hop, top_db);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_feature_frames(float* frw, const float* y, const int64_t* start, const int* len, int B, int n_frames, int max_len,
                        int hop, int n_fft, int win_length, float preemph, void* stream) {
    TACO_CHECK(frw && y && start && len && B >= 0, "taco_feature_frames: bad arguments");
    TACO_CHECK(hop >= 1 && win_length >= 1 && win_length <= n_fft && n_frames == 1 + max_len / hop,
               "taco_feature_frames: n_frames=%d must be 1 + max_len/hop (max_len=%d, hop=%d)", n_frames, max_len, hop);
    TACO_CHECK(max_len > n_fft / 2, "taco_feature_frames: max_len=%d shorter than the reflect padding (%d)", max_len, n_fft / 2);
    const int64_t total = (int64_t)B * n_frames * n_fft;
    if (total == 0) return 0;
    TACO_LAUNCH(feature_frames_kernel, grid_for(total, 256), 256, 0, (cudaStream_t)stream, frw, y, start, len, n_frames, max_len,
                hop, n_fft, win_length, preemph, total);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_feature_spec(void* stft_out, void* mel_out, int out_f16, const float* X_c64, const float* mel_basis, const int* mel_lo,
                      const int* mel_hi, int B, int n_frames, int r, int n_mels, void* stream) {
    TACO_CHECK(stft_out && mel_out && X_c64 && mel_basis && mel_lo && mel_hi && B >= 0, "taco_feature_spec: bad arguments");
    TACO_CHECK(r >= 1 && n_mels >= 1 && n_frames >= 4 * r, "taco_feature_spec: need n_frames=%d >= 4r (r=%d), n_mels=%d >= 1",
               n_frames, r, n_mels);
    const int nf_used = 4 * r * (n_frames / (4 * r));
    const int64_t grid = (int64_t)B * nf_used;
    if (grid == 0) return 0;
    TACO_CHECK(grid <= 0x7fffffff, "taco_feature_spec: too many frames in one call");
    TACO_LAUNCH(feature_spec_kernel, (int)grid, 256, 0, (cudaStream_t)stream, stft_out, mel_out, out_f16,
                reinterpret_cast<const float2*>(X_c64), mel_basis, mel_lo, mel_hi, n_frames, nf_used, r, n_mels);
    TACO_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
