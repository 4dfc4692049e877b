// audio.cu -- Griffin-Lim spectrogram inversion: the fused steps between the two FFTs of an iteration, and the FFTs
// (reference: audio.py:67-97 invert_spectrogram / griffinlim, audio.py:30-35 reshape_frames(forward=False);
// librosa.stft / librosa.istft conventions as restated in oracle/audio_oracle.py).  SURVEY.md section 8(f) rank 1.
//
// All four kernels are bandwidth-bound gathers with one thread per output element; consecutive threads touch
// consecutive addresses of every operand.  Semantics pinned by tests/mirror_kernels.py (gl_init, gl_ola, gl_frame,
// gl_phase).  n = frames, NB = n_fft/2 + 1 bins, L = hop*(n-1) samples; the hann window (periodic, win_length
// samples, centred in n_fft) is evaluated on the fly.
#include <float.h>
#include "common.cuh"

namespace {

inline int grid_for(int64_t total, int block) {
    int64_t g = (total + block - 1) / block;
    if (g > TACO_SMS * 32) g = TACO_SMS * 32;
    if (g < 1) g = 1;
    return (int)g;
}

// mag[b,f,k] = exp(spec[b, t(f), c(f)*F + k] * scale + shift);  full = mag * exp(2 pi i u)
__global__ void gl_init_kernel(float2* __restrict__ full, float* __restrict__ mag, const float* __restrict__ spec,
                               const float* __restrict__ phase_u, int T, int n, int r, int F, const float* __restrict__ scale,
                               const float* __restrict__ shift, int64_t total) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int k = (int)(i % F);
        const int f = (int)((i / F) % n);
        const int b = (int)(i / ((int64_t)F * n));
        const int b4 = f / (4 * r), rem = f % (4 * r);
        const int c = rem >> 2, tl = rem & 3;
        const int t = 4 * b4 + tl;
        const int col = c * F + k;
        float v = spec[((int64_t)b * T + t) * ((int64_t)F * r) + col];
        if (scale) v = fmaf(v, scale[col], shift[col]);
        const float m = expf(v);
        float s, co;
        sincospif(2.0f * phase_u[i], &s, &co);
        mag[i] = m;
        full[i] = make_float2(m * co, m * s);
    }
}

// y[b,s] = sum_t w[j] fr[b,t,j] / sum_t w[j]^2,  j = s + n_fft/2 - t*hop inside the window support
__global__ void gl_ola_kernel(float* __restrict__ y, const float* __restrict__ fr, int n, int L, int hop, int n_fft, int win_length,
                              int64_t total) {
    const int lpad = (n_fft - win_length) / 2;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int s = (int)(i % L);
        const int b = (int)(i / L);
        const int p = s + n_fft / 2;
        // frames whose window support [t*hop + lpad, t*hop + lpad + win_length) contains p
        int tmax = (p - lpad) / hop;
        if (tmax > n - 1) tmax = n - 1;
        int tmin = (p - lpad - win_length + hop) / hop;             // ceil((p - lpad - win_length + 1) / hop)
        if (p - lpad - win_length + 1 <= 0) tmin = 0;
        float acc = 0.f, ss = 0.f;
        for (int t = tmin; t <= tmax; ++t) {
            const int j = p - t * hop;
            const float w = hann_at(j, lpad, win_length);
            acc = fmaf(w, fr[((int64_t)b * n + t) * n_fft + j], acc);
            ss = fmaf(w, w, ss);
        }
        y[i] = (ss > FLT_MIN) ? acc / ss : acc;
    }
}

// frw[b,t,j] = w[j] * ypad[t*hop + j],  ypad = y reflect-padded by n_fft/2 on both sides
__global__ void gl_frame_kernel(float* __restrict__ frw, const float* __restrict__ y, int n, int L, int hop, int n_fft, int win_length,
                                int64_t total) {
    const int lpad = (n_fft - win_length) / 2;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int j = (int)(i % n_fft);
        const int t = (int)((i / n_fft) % n);
        const int b = (int)(i / ((int64_t)n_fft * n));
        const float w = hann_at(j, lpad, win_length);
        float v = 0.f;
        if (w != 0.f) {
            int q = t * hop + j - n_fft / 2;
            if (q < 0) q = -q;
            if (q >= L) q = 2 * (L - 1) - q;
            v = w * y[(int64_t)b * L + q];
        }
        frw[i] = v;
    }
}

// full = mag * rebuilt / |rebuilt|   (angle(0) = 0 -> unit phasor 1)
__global__ void gl_phase_kernel(float2* __restrict__ full, const float* __restrict__ mag, const float2* __restrict__ rebuilt, int64_t total) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const float2 z = rebuilt[i];
        const float a = hypotf(z.x, z.y);
        const float m = mag[i];
        full[i] = (a > 0.f) ? make_float2(m * (z.x / a), m * (z.y / a)) : make_float2(m, 0.f);
    }
}


// ---------------------------------------------------------------------------------------------------------------------
// 2048-point REAL FFT pair in shared memory.  The real row is transformed as a 1024-point COMPLEX sequence
// z[n] = x[2n] + i x[2n+1] (half the arithmetic), with a radix-4 Stockham autosort FFT: 1024 = 4^5, so a CTA of 256
// threads does exactly one radix-4 butterfly per thread and stage, five stages, natural order in and out, ping-pong
// buffers; the twiddles exp(-2 pi i t / 1024) are tabulated once per CTA with sincospi.  A pre / post pass converts between
// Z = FFT(z) and the 1025 bins of the real transform:
//   rfft : X[k] = E[k] + w^k O[k],  E = (Z[k] + conj Z[M-k]) / 2,  O = (Z[k] - conj Z[M-k]) / 2i,  w = exp(-2 pi i / 2048)
//   irfft: Z[k] = E[k] + i w^-k O'[k],  E = (X[k] + conj X[M-k]) / 2,  O' = (X[k] - conj X[M-k]) / 2;  x = IFFT(Z) / 1024
//   INV = false: in = x [rows][2048] real,       out = X [rows][1025] complex (unnormalised)
//   INV = true : in = X [rows][1025] complex,    out = x [rows][2048] real  (1/n scaling; imaginary parts of DC / Nyquist ignored)
// ---------------------------------------------------------------------------------------------------------------------
constexpr int FN = 2048, FM = FN / 2;
__device__ __forceinline__ float2 cmul(const float2 a, const float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

template <bool INV>
__global__ void __launch_bounds__(256) fft2048_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t rows) {
    __shared__ float2 buf_a[FM];
    __shared__ float2 buf_b[FM];
    __shared__ float2 tw[FM];          // exp(-+ 2 pi i t / 1024)
    const int tid = threadIdx.x;
    for (int i = tid; i < FM; i += 256) {
        float sn, cs;
        sincospif(-2.0f * (float)i / (float)FM, &sn, &cs);
        tw[i] = make_float2(cs, INV ? -sn : sn);
    }
    for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
        // ---- load (+ pre-pass of the inverse transform) ----
        if (!INV) {
            const float2* x2 = reinterpret_cast<const float2*>(in + row * FN);     // (x[2n], x[2n+1]) = z[n]
            for (int i = tid; i < FM; i += 256) buf_a[i] = x2[i];
        } else {
            const float2* X = reinterpret_cast<const float2*>(in) + row * (FM + 1);
            for (int k = tid; k < FM; k += 256) {
                float2 xk = X[k], xm = X[FM - k];
                if (k == 0) { xk.y = 0.f; xm.y = 0.f; }                   // DC and Nyquist bins of a real signal are real
                const float2 e = make_float2(0.5f * (xk.x + xm.x), 0.5f * (xk.y - xm.y));          // (X[k] + conj X[M-k]) / 2
                const float2 o = make_float2(0.5f * (xk.x - xm.x), 0.5f * (xk.y + xm.y));          // (X[k] - conj X[M-k]) / 2
                float sn, cs;
                sincospif((float)k / (float)FM, &sn, &cs);                // w^-k = exp(+2 pi i k / 2048)
                const float2 ow = cmul(o, make_float2(cs, sn));
                buf_a[k] = make_float2(e.x - ow.y, e.y + ow.x);            // E + i * (w^-k O')
            }
        }
        __syncthreads();
        // ---- five radix-4 Stockham stages ----
        float2* src = buf_a;
        float2* dst = buf_b;
#pragma unroll
        for (int Ns = 1; Ns < FM; Ns <<= 2) {
            const int j = tid;                                             // FM / 4 = 256 butterflies
            const int k = j & (Ns - 1);
            const int ts = k * (FM / (4 * Ns));
            const float2 v0 = src[j];
            const float2 v1 = cmul(src[j + FM / 4], tw[ts]);
            const float2 v2 = cmul(src[j + 2 * (FM / 4)], tw[2 * ts]);
            const float2 v3 = cmul(src[j + 3 * (FM / 4)], tw[3 * ts]);
            const float2 a0 = make_float2(v0.x + v2.x, v0.y + v2.y), a1 = make_float2(v0.x - v2.x, v0.y - v2.y);
            const float2 a2 = make_float2(v1.x + v3.x, v1.y + v3.y);
            const float2 d = make_float2(v1.x - v3.x, v1.y - v3.y);
            const float2 a3 = INV ? make_float2(-d.y, d.x) : make_float2(d.y, -d.x);              // (v1 - v3) * (+-i)
            const int j0 = ((j - k) << 2) + k;
            dst[j0] = make_float2(a0.x + a2.x, a0.y + a2.y);
            dst[j0 + Ns] = make_float2(a1.x + a3.x, a1.y + a3.y);
            dst[j0 + 2 * Ns] = make_float2(a0.x - a2.x, a0.y - a2.y);
            dst[j0 + 3 * Ns] = make_float2(a1.x - a3.x, a1.y - a3.y);
            __syncthreads();
            float2* t = src; src = dst; dst = t;
        }
        // ---- store (+ post-pass of the forward transform) ----
        if (!INV) {
            float2* X = reinterpret_cast<float2*>(out) + row * (FM + 1);
            for (int k = tid; k <= FM; k += 256) {
                const float2 zk = src[k & (FM - 1)], zm = src[(FM - k) & (FM - 1)];
                const float2 e = make_float2(0.5f * (zk.x + zm.x), 0.5f * (zk.y - zm.y));          // (Z[k] + conj Z[M-k]) / 2
                const float2 o = make_float2(0.5f * (zk.y + zm.y), -0.5f * (zk.x - zm.x));         // (Z[k] - conj Z[M-k]) / 2i
                float sn, cs;
                sincospif(-(float)k / (float)FM, &sn, &cs);               // w^k = exp(-2 pi i k / 2048)
                const float2 ow = cmul(o, make_float2(cs, sn));
                X[k] = make_float2(e.x + ow.x, e.y + ow.y);
            }
        } else {
            float2* x2 = reinterpret_cast<float2*>(out + row * FN);
            for (int i = tid; i < FM; i += 256) x2[i] = make_float2(src[i].x * (1.0f / FM), src[i].y * (1.0f / FM));
        }
        __syncthreads();
    }
}

}  // namespace

extern "C" {

int taco_gl_init(float* full_c64, float* mag, const float* spec, const float* phase_u, int B, int T, int n, int r, int F,
                 const float* scale, const float* shift, void* stream) {
    TACO_CHECK(full_c64 && mag && spec && phase_u, "taco_gl_init: NULL");
    TACO_CHECK(r >= 1 && n == 4 * r * (T / 4) && F >= 1, "taco_gl_init: n=%d must be 4*r*(T/4) (r=%d, T=%d)", n, r, T);
    TACO_CHECK((scale == nullptr) == (shift == nullptr), "taco_gl_init: scale and shift go together");
    const int64_t total = (int64_t)B * n * F;
    if (total == 0) return 0;
    TACO_LAUNCH(gl_init_kernel, grid_for(total, 256), 256, 0, (cudaStream_t)stream, reinterpret_cast<float2*>(full_c64), mag, spec, phase_u, T, n, r, F,
                                                                           scale, shift, total);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_gl_ola(float* y, const float* fr, int B, int n, int hop, int n_fft, int win_length, void* stream) {
    TACO_CHECK(y && fr, "taco_gl_ola: NULL");
    TACO_CHECK(n >= 2 && hop >= 1 && win_length >= 1 && win_length <= n_fft, "taco_gl_ola: bad sizes");
    const int L = hop * (n - 1);
    const int64_t total = (int64_t)B * L;
    if (total == 0) return 0;
    TACO_LAUNCH(gl_ola_kernel, grid_for(total, 256), 256, 0, (cudaStream_t)stream, y, fr, n, L, hop, n_fft, win_length, total);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_gl_frame(float* frw, const float* y, int B, int n, int hop, int n_fft, int win_length, void* stream) {
    TACO_CHECK(frw && y, "taco_gl_frame: NULL");
    const int L = hop * (n - 1);
    TACO_CHECK(n >= 2 && L > n_fft / 2, "taco_gl_frame: signal (%d samples) shorter than the reflect padding (%d)", L, n_fft / 2);
    const int64_t total = (int64_t)B * n * n_fft;
    TACO_LAUNCH(gl_frame_kernel, grid_for(total, 256), 256, 0, (cudaStream_t)stream, frw, y, n, L, hop, n_fft, win_length, total);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_gl_phase(float* full_c64, const float* mag, const float* rebuilt_c64, int64_t count, void* stream) {
    TACO_CHECK(full_c64 && mag && rebuilt_c64 && count >= 0, "taco_gl_phase: bad arguments");
    if (count == 0) return 0;
    TACO_LAUNCH(gl_phase_kernel, grid_for(count, 256), 256, 0, (cudaStream_t)stream, reinterpret_cast<float2*>(full_c64), mag,
                                                                            reinterpret_cast<const float2*>(rebuilt_c64), count);
    TACO_LAUNCH_CHECK();
    return 0;
}

// real FFT / inverse real FFT of length 2048 over `rows` contiguous rows: x [rows][2048] -> X [rows][1025] complex
// (interleaved re, im; unnormalised, like numpy / torch rfft) and X -> x (scaled by 1/2048, imaginary parts of the DC
// and Nyquist bins ignored, like irfft).  Replaces the two cuFFT calls of a Griffin-Lim iteration (audio.py:84-86).
int taco_rfft2048(float* X_c64, const float* x, int64_t rows, void* stream) {
    TACO_CHECK(X_c64 && x && rows >= 0, "taco_rfft2048: bad arguments");
    if (rows == 0) return 0;
    const int grid = (int)(rows < TACO_SMS * 4 ? rows : TACO_SMS * 4);
    TACO_LAUNCH(fft2048_kernel<false>, grid, 256, 0, (cudaStream_t)stream, x, X_c64, rows);
    TACO_LAUNCH_CHECK();
    return 0;
}
int taco_irfft2048(float* x, const float* X_c64, int64_t rows, void* stream) {
    TACO_CHECK(X_c64 && x && rows >= 0, "taco_irfft2048: bad arguments");
    if (rows == 0) return 0;
    const int grid = (int)(rows < TACO_SMS * 4 ? rows : TACO_SMS * 4);
    TACO_LAUNCH(fft2048_kernel<true>, grid, 256, 0, (cudaStream_t)stream, X_c64, x, rows);
    TACO_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
