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

// The three kernels below that need to know which utterance an element belongs to take `off`:
//   off == nullptr: the padded layout, utterance b = rows [b*n, (b+1)*n), samples [b*L, (b+1)*L); a 1-D grid-stride loop
//                   over every element of the batch.
//   off != nullptr: the packed layout of taco_*_packed, utterance b = blockIdx.y = rows [off[b], off[b+1]) (n_b of them)
//                   and L_b = hop*(n_b - 1) samples from hop*(off[b] - b); the grid-stride loop runs over that
//                   utterance's elements only.
// The per-element arithmetic is the same code in both layouts, so a packed utterance is bit-identical to the padded
// path run on it alone.

// mag[b,f,k] = exp(spec[b, t(f), c(f)*F + k] * scale + shift);  full = mag * exp(2 pi i u)
__global__ void gl_init_kernel(float2* __restrict__ full, float* __restrict__ mag, const float* __restrict__ spec,
                               const float* __restrict__ phase_u, int T, int n, int r, int F, const float* __restrict__ scale,
                               const float* __restrict__ shift, const int64_t* __restrict__ off, int64_t total) {
    int64_t base = 0;                                                   // first output element of this utterance
    if (off) {
        base = off[blockIdx.y] * F;
        total = (off[blockIdx.y + 1] - off[blockIdx.y]) * F;
    }
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int k = (int)(i % F);
        const int f = off ? (int)(i / F) : (int)((i / F) % n);
        const int b = off ? (int)blockIdx.y : (int)(i / ((int64_t)F * n));
        const int64_t o = base + i;
        const int b4 = f / (4 * r), rem = f % (4 * r);
        const int c = rem >> 2, tl = rem & 3;
        const int t = 4 * b4 + tl;
        const int col = c * F + k;
        float v = spec[((int64_t)b * T + t) * ((int64_t)F * r) + col];
        if (scale) v = fmaf(v, scale[col], shift[col]);
        const float m = expf(v);
        float s, co;
        sincospif(2.0f * phase_u[o], &s, &co);
        mag[o] = m;
        full[o] = make_float2(m * co, m * s);
    }
}

// y[b,s] = sum_t w[j] fr[b,t,j] / sum_t w[j]^2,  j = s + n_fft/2 - t*hop inside the window support
__global__ void gl_ola_kernel(float* __restrict__ y, const float* __restrict__ fr, int n, int L, int hop, int n_fft, int win_length,
                              const int64_t* __restrict__ off, int64_t total) {
    const int lpad = (n_fft - win_length) / 2;
    int64_t row0 = 0, ybase = 0;
    if (off) {
        row0 = off[blockIdx.y];
        n = (int)(off[blockIdx.y + 1] - row0);
        L = hop * (n - 1);
        ybase = (int64_t)hop * (row0 - blockIdx.y);
        total = n >= 2 ? L : 0;
    }
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int s = (int)(i % L);
        const int b = (int)(i / L);
        const int64_t frow = off ? row0 : (int64_t)b * n;
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
            acc = fmaf(w, fr[(frow + t) * n_fft + j], acc);
            ss = fmaf(w, w, ss);
        }
        y[ybase + i] = (ss > FLT_MIN) ? acc / ss : acc;
    }
}

// frw[b,t,j] = w[j] * ypad[t*hop + j],  ypad = y reflect-padded by n_fft/2 on both sides
__global__ void gl_frame_kernel(float* __restrict__ frw, const float* __restrict__ y, int n, int L, int hop, int n_fft, int win_length,
                                const int64_t* __restrict__ off, int64_t total) {
    const int lpad = (n_fft - win_length) / 2;
    int64_t base = 0, ybase = 0;
    if (off) {
        const int64_t row0 = off[blockIdx.y];
        n = (int)(off[blockIdx.y + 1] - row0);
        L = hop * (n - 1);
        base = row0 * n_fft;
        ybase = (int64_t)hop * (row0 - blockIdx.y);
        total = L > n_fft / 2 ? (int64_t)n * n_fft : 0;             // the host rejects shorter ones; keep the reads in bounds
    }
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
            v = w * y[ybase + (int64_t)b * L + q];
        }
        frw[base + i] = v;
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

// fast Griffin-Lim's phase update: full = mag * d/|d|, d = rebuilt - beta * prev (angle(0) = 0 -> unit phasor 1).
// gl_phase's arithmetic on d, so beta = 0 gives gl_phase's values.
__global__ void gl_phase_momentum_kernel(float2* __restrict__ full, const float* __restrict__ mag, const float2* __restrict__ rebuilt,
                                         const float2* __restrict__ prev, float beta, int64_t total) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const float2 z = rebuilt[i], p = prev[i];
        const float2 d = make_float2(fmaf(-beta, p.x, z.x), fmaf(-beta, p.y, z.y));
        const float a = hypotf(d.x, d.y);
        const float m = mag[i];
        full[i] = (a > 0.f) ? make_float2(m * (d.x / a), m * (d.y / a)) : make_float2(m, 0.f);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// De-emphasis of synthesised waveforms (taco_de_emphasis): y[i] = x[i] + c y[i-1] in place over each segment
// [start[s], start[s+1]), zero state before start[s].  One CTA per segment walks it in tiles of DE_TILE samples, carrying
// the last output of a tile into the next; no CTA waits on another.  Within a tile:
//   - the tile is staged in shared memory (coalesced; one pad word per DE_ITEMS samples keeps the per-thread reads
//     conflict-free) while the next tile's loads are already in flight in registers;
//   - thread t runs the recurrence over its DE_ITEMS consecutive samples from zero state: loc[i], and the affine map
//     y_in -> c^len y_in + loc[len-1] its run applies to the state it receives;
//   - a block scan composes those maps in order (warp shuffles, then the warp totals serially), so thread t learns the
//     state y_in before its first sample from the carry; it writes loc[i] + c^(i+1) y_in.
// Every reduction has a fixed order: the same bits every run.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int DE_THREADS = 512, DE_ITEMS = 16, DE_TILE = DE_THREADS * DE_ITEMS;
constexpr int DE_WARPS = DE_THREADS / 32;

__device__ __forceinline__ int de_slot(int e) { return e + e / DE_ITEMS; }

__global__ void __launch_bounds__(DE_THREADS) de_emphasis_kernel(float* __restrict__ y, const int64_t* __restrict__ start, float c) {
    __shared__ float sm[DE_TILE + DE_TILE / DE_ITEMS];
    __shared__ float wa[DE_WARPS], wb[DE_WARPS];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t s0 = start[blockIdx.x], s1 = start[blockIdx.x + 1];
    float v[DE_ITEMS];
#pragma unroll
    for (int j = 0; j < DE_ITEMS; ++j) {
        const int64_t g = s0 + j * DE_THREADS + tid;
        v[j] = g < s1 ? y[g] : 0.f;
    }
    float carry = 0.f;                                                  // the output just before the tile
    for (int64_t t0 = s0; t0 < s1; t0 += DE_TILE) {
        const int len = (int)(s1 - t0 < DE_TILE ? s1 - t0 : DE_TILE);
#pragma unroll
        for (int j = 0; j < DE_ITEMS; ++j) sm[de_slot(j * DE_THREADS + tid)] = v[j];
        __syncthreads();
        const int64_t t1 = t0 + DE_TILE;                                // prefetch the next tile
#pragma unroll
        for (int j = 0; j < DE_ITEMS; ++j) {
            const int64_t g = t1 + j * DE_THREADS + tid;
            v[j] = g < s1 ? y[g] : 0.f;
        }
        int mine = len - tid * DE_ITEMS;                                // samples of this thread in the tile
        mine = mine < 0 ? 0 : (mine > DE_ITEMS ? DE_ITEMS : mine);
        const float* xs = sm + tid * (DE_ITEMS + 1);                    // = sm + de_slot(tid * DE_ITEMS)
        float loc[DE_ITEMS];
        float acc = 0.f, a = 1.f;
#pragma unroll
        for (int i = 0; i < DE_ITEMS; ++i) {
            if (i < mine) {
                acc = fmaf(c, acc, xs[i]);
                a *= c;
            }
            loc[i] = acc;
        }
        // This run's map is y_in -> a y_in + b.  Butterfly scan of the maps over the warp: at step m, (a, b) is the
        // composition of this lane's aligned block of m lanes, and (ea, eb) that of the lanes before it in the block; the
        // partner block (lane ^ m) is composed in front when it comes first, behind otherwise.  Both halves spell the
        // composition with the same operands, so every lane ends with the same warp total.
        float b = acc, ea = 1.f, eb = 0.f;
#pragma unroll
        for (int m = 1; m < 32; m <<= 1) {
            const float oa = __shfl_xor_sync(0xffffffffu, a, m), ob = __shfl_xor_sync(0xffffffffu, b, m);
            if (lane & m) {                                             // partner block first: (oa, ob) then ours
                eb = fmaf(ea, ob, eb);
                ea *= oa;
                b = fmaf(a, ob, b);
            } else {                                                    // ours first, then the partner's
                b = fmaf(oa, b, ob);
            }
            a *= oa;
        }
        if (lane == 31) { wa[warp] = a; wb[warp] = b; }
        __syncthreads();
        float yw = carry;                                               // the state entering this warp's first lane
        for (int w = 0; w < warp; ++w) yw = fmaf(wa[w], yw, wb[w]);
        const float yin = fmaf(ea, yw, eb);
        float* ys = sm + tid * (DE_ITEMS + 1);
        float p = 1.f;
#pragma unroll
        for (int i = 0; i < DE_ITEMS; ++i) {
            if (i < mine) {
                p *= c;
                ys[i] = fmaf(p, yin, loc[i]);
            }
        }
        __syncthreads();
        carry = sm[de_slot(len - 1)];
#pragma unroll
        for (int j = 0; j < DE_ITEMS; ++j) {
            const int e = j * DE_THREADS + tid;
            if (e < len) y[t0 + e] = sm[de_slot(e)];
        }
        __syncthreads();                                                // sm, wa and wb are rewritten by the next tile
    }
}


// ---------------------------------------------------------------------------------------------------------------------
// Where an utterance's speech ends (taco_speech_frames).  Two launches: frame_power_kernel spreads the read of the
// spectrogram over the whole device, one warp per frame; speech_end_kernel then reduces each utterance's n powers with
// one CTA.  Both reductions run in a fixed order, so the result does not change from run to run.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int SF_THREADS = 256;

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, m));
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
    return v;
}

// e[b*n + f] = log sum_k exp(2 v[f,k]),  v[f,k] = spec[b, t(f), c(f)*F + k] * scale + shift (gl_init's frame space),
// as max-shifted sums: m = max_k 2v, e = m + log sum_k exp(2v - m).  NaN or +Inf in v, or a frame of -Inf only, makes
// e non-finite.  Lane l sums bins l, l+32, ... in order, then the warp combines by butterfly.
__global__ void __launch_bounds__(SF_THREADS) frame_power_kernel(float* __restrict__ e, const float* __restrict__ spec, int T,
                                                                 int n, int r, int F, const float* __restrict__ scale,
                                                                 const float* __restrict__ shift, int64_t frames) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (SF_THREADS / 32);
    for (int64_t g = blockIdx.x * (int64_t)(SF_THREADS / 32) + threadIdx.x / 32; g < frames; g += warps) {
        const int f = (int)(g % n);
        const int64_t b = g / n;
        const int b4 = f / (4 * r), rem = f % (4 * r);
        const int c = rem >> 2, tl = rem & 3;
        const int t = 4 * b4 + tl;
        const float* row = spec + (b * T + t) * ((int64_t)F * r) + (int64_t)c * F;
        const float* sc = scale ? scale + c * F : nullptr;
        const float* sh = scale ? shift + c * F : nullptr;
        float m = -INFINITY;
        for (int k = lane; k < F; k += 32) {
            float v = row[k];
            if (sc) v = fmaf(v, sc[k], sh[k]);
            m = fmaxf(m, 2.0f * v);
        }
        m = warp_max(m);
        float s = 0.f;
        for (int k = lane; k < F; k += 32) {
            float v = row[k];
            if (sc) v = fmaf(v, sc[k], sh[k]);
            s += expf(2.0f * v - m);
        }
        s = warp_sum(s);
        if (lane == 0) e[g] = m + logf(s);
    }
}

// one CTA per utterance: E = max_f e[f]; f* = the last f with e[f] >= E - top_db ln(10)/10;
// frames[b] = 4r * clamp(ceil((f* + 1) / 4r), ceil(5 / 4r), T/4), or n if any e[f] is not finite
__global__ void __launch_bounds__(SF_THREADS) speech_end_kernel(int* __restrict__ frames, const float* __restrict__ e, int n, int r,
                                                                int T, float top_db) {
    __shared__ float rmax[SF_THREADS];
    __shared__ int rlast[SF_THREADS];
    const int tid = threadIdx.x;
    const float* eb = e + (int64_t)blockIdx.x * n;
    float m = -INFINITY;
    int bad = 0;
    for (int f = tid; f < n; f += SF_THREADS) {
        const float x = eb[f];
        if (fabsf(x) <= FLT_MAX) m = fmaxf(m, x);                    // finite (false for NaN and +-Inf)
        else bad = 1;
    }
    rmax[tid] = m;
    rlast[tid] = bad;
    __syncthreads();
    for (int s = SF_THREADS / 2; s > 0; s >>= 1) {
        if (tid < s) {
            rmax[tid] = fmaxf(rmax[tid], rmax[tid + s]);
            rlast[tid] |= rlast[tid + s];
        }
        __syncthreads();
    }
    const float thr = rmax[0] - top_db * 0.230258509299404568f;       // ln(10) / 10: dB of power -> natural log
    bad = rlast[0];
    __syncthreads();
    int last = -1;
    for (int f = tid; f < n; f += SF_THREADS)
        if (eb[f] >= thr) last = f;
    rlast[tid] = last;
    __syncthreads();
    for (int s = SF_THREADS / 2; s > 0; s >>= 1) {
        if (tid < s) rlast[tid] = max(rlast[tid], rlast[tid + s]);
        __syncthreads();
    }
    if (tid == 0) {
        const int blk = 4 * r;
        int k = (rlast[0] + blk) / blk;                                 // ceil((f* + 1) / 4r)
        const int kmin = (5 + blk - 1) / blk;                           // the inversion's reflect padding needs 5 frames
        if (k < kmin) k = kmin;
        if (k > T / 4) k = T / 4;
        frames[blockIdx.x] = bad ? n : blk * k;
    }
}

// one CTA per utterance, speech_end_kernel's rule plus the first voiced frame: bounds[b] = {f0, f1, frames} with
// f0 = the first f with e[f] >= thr, f1 = the last such f + 1, frames = speech_end_kernel's frames[b]; {0, n, n} if any
// e[f] is not finite.  The max is order-independent and thr is the same expression, so frames is bit for bit the same.
__global__ void __launch_bounds__(SF_THREADS) speech_bounds_kernel(int* __restrict__ bounds, const float* __restrict__ e, int n,
                                                                   int r, int T, float top_db) {
    __shared__ float rmax[SF_THREADS];
    __shared__ int rfirst[SF_THREADS], rlast[SF_THREADS];
    const int tid = threadIdx.x;
    const float* eb = e + (int64_t)blockIdx.x * n;
    float m = -INFINITY;
    int bad = 0;
    for (int f = tid; f < n; f += SF_THREADS) {
        const float x = eb[f];
        if (fabsf(x) <= FLT_MAX) m = fmaxf(m, x);
        else bad = 1;
    }
    rmax[tid] = m;
    rlast[tid] = bad;
    __syncthreads();
    for (int s = SF_THREADS / 2; s > 0; s >>= 1) {
        if (tid < s) {
            rmax[tid] = fmaxf(rmax[tid], rmax[tid + s]);
            rlast[tid] |= rlast[tid + s];
        }
        __syncthreads();
    }
    const float thr = rmax[0] - top_db * 0.230258509299404568f;       // ln(10) / 10, as in speech_end_kernel
    bad = rlast[0];
    __syncthreads();
    int first = n, last = -1;
    for (int f = tid; f < n; f += SF_THREADS)
        if (eb[f] >= thr) {
            first = min(first, f);
            last = f;
        }
    rfirst[tid] = first;
    rlast[tid] = last;
    __syncthreads();
    for (int s = SF_THREADS / 2; s > 0; s >>= 1) {
        if (tid < s) {
            rfirst[tid] = min(rfirst[tid], rfirst[tid + s]);
            rlast[tid] = max(rlast[tid], rlast[tid + s]);
        }
        __syncthreads();
    }
    if (tid == 0) {
        const int blk = 4 * r;
        int k = (rlast[0] + blk) / blk;
        const int kmin = (5 + blk - 1) / blk;
        if (k < kmin) k = kmin;
        if (k > T / 4) k = T / 4;
        int* o = bounds + 3 * (int64_t)blockIdx.x;
        o[0] = bad ? 0 : rfirst[0];
        o[1] = bad ? n : rlast[0] + 1;
        o[2] = bad ? n : blk * k;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Joining synthesised pieces (taco_join_segments): blockIdx.y = segment s = {src_start, dst_start, len}, a grid-stride
// loop over its samples; out[dst_start + i] = src[src_start + i] * w(i), w(i) = min(1, c(i), c(len-1-i)),
// c(j) = 0.5 - 0.5 cos(pi (j + 0.5) / fade) for j < fade, 1 otherwise.  c is evaluated as sin^2(pi (j + 0.5) / (2 fade))
// in double: the same raised cosine without the cancellation of 1 - cos near j = 0, so the product is rounded once from
// a weight exact to ~1e-15.  A segment outside [0, out_len) is skipped (the host has validated them all).
// ---------------------------------------------------------------------------------------------------------------------
#ifdef TACO_HOST_EMU
inline double sinpi(double x) { return std::sin(M_PI * x); }
#endif
__device__ __forceinline__ double fade_weight(int64_t j, int fade) {
    if (j >= fade) return 1.0;
    const double s = sinpi(0.5 * ((double)j + 0.5) / (double)fade);     // sinpi: no argument reduction, no stack frame
    return s * s;
}

__global__ void join_segments_kernel(float* __restrict__ out, int64_t out_len, const float* __restrict__ src,
                                     const int64_t* __restrict__ seg, int fade) {
    const int64_t s0 = seg[3 * (int64_t)blockIdx.y], d0 = seg[3 * (int64_t)blockIdx.y + 1], len = seg[3 * (int64_t)blockIdx.y + 2];
    if (s0 < 0 || d0 < 0 || len < 0 || d0 > out_len - len) return;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < len; i += (int64_t)gridDim.x * blockDim.x) {
        const double w = fmin(1.0, fmin(fade_weight(i, fade), fade_weight(len - 1 - i, fade)));
        out[d0 + i] = (float)((double)src[s0 + i] * w);
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
                                                                           scale, shift, nullptr, total);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_gl_ola(float* y, const float* fr, int B, int n, int hop, int n_fft, int win_length, void* stream) {
    TACO_CHECK(y && fr, "taco_gl_ola: NULL");
    TACO_CHECK(n >= 2 && hop >= 1 && win_length >= 1 && win_length <= n_fft, "taco_gl_ola: bad sizes");
    const int L = hop * (n - 1);
    const int64_t total = (int64_t)B * L;
    if (total == 0) return 0;
    TACO_LAUNCH(gl_ola_kernel, grid_for(total, 256), 256, 0, (cudaStream_t)stream, y, fr, n, L, hop, n_fft, win_length, nullptr, total);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_gl_frame(float* frw, const float* y, int B, int n, int hop, int n_fft, int win_length, void* stream) {
    TACO_CHECK(frw && y, "taco_gl_frame: NULL");
    const int L = hop * (n - 1);
    TACO_CHECK(n >= 2 && L > n_fft / 2, "taco_gl_frame: signal (%d samples) shorter than the reflect padding (%d)", L, n_fft / 2);
    const int64_t total = (int64_t)B * n * n_fft;
    TACO_LAUNCH(gl_frame_kernel, grid_for(total, 256), 256, 0, (cudaStream_t)stream, frw, y, n, L, hop, n_fft, win_length, nullptr, total);
    TACO_LAUNCH_CHECK();
    return 0;
}

// grid of a packed launch: blockIdx.y = utterance, enough x-blocks for the longest one, the whole grid capped like grid_for
static dim3 packed_grid(int64_t per_utt, int B) {
    int64_t gx = (per_utt + 255) / 256;
    const int64_t cap = TACO_SMS * 32 / B;
    if (gx > cap) gx = cap;
    if (gx < 1) gx = 1;
    return dim3((unsigned)gx, (unsigned)B);
}

int taco_gl_init_packed(float* full_c64, float* mag, const float* spec, const float* phase_u, const int64_t* off, int B, int T,
                        int r, int F, int max_frames, const float* scale, const float* shift, void* stream) {
    TACO_CHECK(full_c64 && mag && spec && phase_u && off, "taco_gl_init_packed: NULL");
    TACO_CHECK(B >= 1 && B <= 65535 && r >= 1 && T >= 4 && F >= 1, "taco_gl_init_packed: bad sizes (B=%d, T=%d, r=%d, F=%d)", B, T, r, F);
    TACO_CHECK(max_frames >= 1 && max_frames <= 4 * r * (T / 4), "taco_gl_init_packed: max_frames=%d outside [1, 4*r*(T/4)]", max_frames);
    TACO_CHECK((scale == nullptr) == (shift == nullptr), "taco_gl_init_packed: scale and shift go together");
    TACO_LAUNCH(gl_init_kernel, packed_grid((int64_t)max_frames * F, B), 256, 0, (cudaStream_t)stream, reinterpret_cast<float2*>(full_c64),
                mag, spec, phase_u, T, 4 * r * (T / 4), r, F, scale, shift, off, (int64_t)0);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_gl_ola_packed(float* y, const float* fr, const int64_t* off, int B, int max_frames, int hop, int n_fft, int win_length,
                       void* stream) {
    TACO_CHECK(y && fr && off, "taco_gl_ola_packed: NULL");
    TACO_CHECK(B >= 1 && B <= 65535 && max_frames >= 2 && hop >= 1 && win_length >= 1 && win_length <= n_fft,
               "taco_gl_ola_packed: bad sizes");
    TACO_LAUNCH(gl_ola_kernel, packed_grid((int64_t)hop * (max_frames - 1), B), 256, 0, (cudaStream_t)stream, y, fr, 0, 0, hop, n_fft,
                win_length, off, (int64_t)0);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_gl_frame_packed(float* frw, const float* y, const int64_t* off, int B, int max_frames, int hop, int n_fft, int win_length,
                         void* stream) {
    TACO_CHECK(frw && y && off, "taco_gl_frame_packed: NULL");
    TACO_CHECK(B >= 1 && B <= 65535 && hop >= 1 && win_length >= 1 && win_length <= n_fft && max_frames >= 2 &&
               hop * (max_frames - 1) > n_fft / 2, "taco_gl_frame_packed: bad sizes (max_frames=%d)", max_frames);
    TACO_LAUNCH(gl_frame_kernel, packed_grid((int64_t)max_frames * n_fft, B), 256, 0, (cudaStream_t)stream, frw, y, 0, 0, hop, n_fft,
                win_length, off, (int64_t)0);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_speech_frames(int* frames, const float* spec, int B, int T, int r, int F, const float* scale, const float* shift,
                       float top_db, void* stream) {
    TACO_CHECK(frames && spec, "taco_speech_frames: NULL");
    TACO_CHECK(B >= 1 && r >= 1 && T >= 4 && F >= 1, "taco_speech_frames: bad sizes (B=%d, T=%d, r=%d, F=%d)", B, T, r, F);
    TACO_CHECK(top_db > 0.f && top_db <= FLT_MAX, "taco_speech_frames: top_db=%g must be finite and positive", (double)top_db);
    TACO_CHECK((scale == nullptr) == (shift == nullptr), "taco_speech_frames: scale and shift go together");
    const int n = 4 * r * (T / 4);
    const int64_t total = (int64_t)B * n;
    cudaStream_t st = (cudaStream_t)stream;
    float* e = nullptr;                                                 // e[B][n], stream-ordered: no host synchronisation
#ifdef TACO_HOST_EMU
    e = static_cast<float*>(malloc((size_t)total * sizeof(float)));
    TACO_CHECK(e, "taco_speech_frames: out of memory");
#else
    TACO_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&e), (size_t)total * sizeof(float), st));
#endif
    int64_t g = (total + SF_THREADS / 32 - 1) / (SF_THREADS / 32);
    if (g > TACO_SMS * 16) g = TACO_SMS * 16;
    TACO_LAUNCH(frame_power_kernel, (int)g, SF_THREADS, 0, st, e, spec, T, n, r, F, scale, shift, total);
    TACO_LAUNCH_CHECK();
    TACO_LAUNCH(speech_end_kernel, B, SF_THREADS, 0, st, frames, e, n, r, T, top_db);
    TACO_LAUNCH_CHECK();
#ifdef TACO_HOST_EMU
    free(e);
#else
    TACO_CUDA(cudaFreeAsync(e, st));
#endif
    return 0;
}

int taco_speech_bounds(int* bounds, const float* spec, int B, int T, int r, int F, const float* scale, const float* shift,
                       float top_db, void* stream) {
    TACO_CHECK(bounds && spec, "taco_speech_bounds: NULL");
    TACO_CHECK(B >= 1 && r >= 1 && T >= 4 && F >= 1, "taco_speech_bounds: bad sizes (B=%d, T=%d, r=%d, F=%d)", B, T, r, F);
    TACO_CHECK(top_db > 0.f && top_db <= FLT_MAX, "taco_speech_bounds: top_db=%g must be finite and positive", (double)top_db);
    TACO_CHECK((scale == nullptr) == (shift == nullptr), "taco_speech_bounds: scale and shift go together");
    const int n = 4 * r * (T / 4);
    const int64_t total = (int64_t)B * n;
    cudaStream_t st = (cudaStream_t)stream;
    float* e = nullptr;                                                 // e[B][n], stream-ordered, as in taco_speech_frames
#ifdef TACO_HOST_EMU
    e = static_cast<float*>(malloc((size_t)total * sizeof(float)));
    TACO_CHECK(e, "taco_speech_bounds: out of memory");
#else
    TACO_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&e), (size_t)total * sizeof(float), st));
#endif
    int64_t g = (total + SF_THREADS / 32 - 1) / (SF_THREADS / 32);
    if (g > TACO_SMS * 16) g = TACO_SMS * 16;
    TACO_LAUNCH(frame_power_kernel, (int)g, SF_THREADS, 0, st, e, spec, T, n, r, F, scale, shift, total);
    TACO_LAUNCH_CHECK();
    TACO_LAUNCH(speech_bounds_kernel, B, SF_THREADS, 0, st, bounds, e, n, r, T, top_db);
    TACO_LAUNCH_CHECK();
#ifdef TACO_HOST_EMU
    free(e);
#else
    TACO_CUDA(cudaFreeAsync(e, st));
#endif
    return 0;
}

int taco_join_segments(float* out, int64_t out_len, const float* src, const int64_t* seg, int S, int max_len, int fade,
                       void* stream) {
    TACO_CHECK(out && src && seg, "taco_join_segments: NULL");
    TACO_CHECK(S >= 1 && S <= 65535 && out_len >= 0 && max_len >= 0 && fade >= 1,
               "taco_join_segments: bad sizes (S=%d, out_len=%lld, max_len=%d, fade=%d)", S, (long long)out_len, max_len, fade);
    if (max_len == 0) return 0;
    TACO_LAUNCH(join_segments_kernel, packed_grid(max_len, S), 256, 0, (cudaStream_t)stream, out, out_len, src, seg, fade);
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

int taco_gl_phase_momentum(float* full_c64, const float* mag, const float* rebuilt_c64, const float* prev_c64, float beta,
                           int64_t count, void* stream) {
    TACO_CHECK(full_c64 && mag && rebuilt_c64 && prev_c64 && count >= 0, "taco_gl_phase_momentum: bad arguments");
    TACO_CHECK(beta >= 0.f && beta <= 0.5f, "taco_gl_phase_momentum: beta=%g outside [0, 0.5]", (double)beta);
    if (count == 0) return 0;
    TACO_LAUNCH(gl_phase_momentum_kernel, grid_for(count, 256), 256, 0, (cudaStream_t)stream, reinterpret_cast<float2*>(full_c64),
                mag, reinterpret_cast<const float2*>(rebuilt_c64), reinterpret_cast<const float2*>(prev_c64), beta, count);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_de_emphasis(float* y, const int64_t* start, int S, float coef, void* stream) {
    TACO_CHECK(y && start, "taco_de_emphasis: NULL");
    TACO_CHECK(S >= 0, "taco_de_emphasis: S=%d segments", S);
    TACO_CHECK(coef >= 0.f && coef < 1.f, "taco_de_emphasis: coef=%g outside [0, 1)", (double)coef);
    if (S == 0) return 0;
    TACO_LAUNCH(de_emphasis_kernel, S, DE_THREADS, 0, (cudaStream_t)stream, y, start, coef);
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
