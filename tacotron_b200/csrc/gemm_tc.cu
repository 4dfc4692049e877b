// gemm_tc.cu -- TMA + wgmma implementation of taco_linear_fwd (TACO_IMPL_TC / TACO_IMPL_TC3), of the tensor-core
// weight gradient taco_conv_dw and of the fused CBHG highway stack taco_highway_stack_fwd, sm_90a.
//
// One kernel serves every feed-forward contraction of the model (conv bank as ONE grouped
// implicit GEMM, conv projections, highway, GRU input products, attention memory layer,
// post dense):  Y[(b,t), n] = epi( sum_j sum_c X[b, t+tap0+j, c] * W[j,c,n] ).
//
//  * A operand: activations stay in their NWC layout in HBM; a 3-D TMA tensor map (C, T, B)
//    with a {32 ch, 128 rows, 1} box loads the tile for tap j at time offset t0+tap0+j.
//    TMA out-of-bounds zero fill IS the TF 'same' padding (rows < 0 or >= T, per utterance),
//    and also pads C up to a multiple of 32 (C=80 in the post-net).
//  * B operand: weights pre-packed K-major [N][taps*Cpad], TF32-rounded (taco_pack_weight).
//  * both land in shared memory in the 128B-swizzled K-major layout that wgmma reads, in a ring of STAGES k-blocks.
//    One thread fills the ring through TMA (full barriers count the transaction bytes; empty barriers take one arrival
//    per warp once that warp's products have read the stage).
//  * 256 threads = two warpgroups; warpgroup w multiplies rows [64w, 64w+64) of the 128-row tile with wgmma m64nBNk8
//    (TF32 inputs, fp32 accumulators in registers).
//  * bank mode: CTA n-tile = filter k (BN == bank_cout), K loop runs over that filter's k taps
//    only -- no zero-padded taps are multiplied.
//  * X3 = true (TACO_IMPL_TC3, precision 'fp32x3'): error-compensated 3xTF32 -- fp32-grade products on the tensor cores.
//    Weights arrive pre-split (hi = TF32 head, lo = remainder: taco_pack_weight_x3); each thread reads its A fragment out
//    of the swizzled activation tile, splits it into hi + lo in registers, and every k-step issues lo.hi + hi.lo + hi.hi
//    into the same accumulators with the A operand taken from registers.
//  * epilogue: the accumulators are staged through shared memory (the pipeline buffers, idle by then) so that a thread
//    owns one output row: bias / activation / batch-norm affine / max-pool / dropout / residual / highway fused, then
//    16-byte row stores.
#include <cuda.h>
#include "epilogue.cuh"

namespace {

constexpr int TC_BM = 128;
constexpr int TC_BK = 32;                       // floats: one 128-byte swizzle row
constexpr int TC_THREADS = 256;                 // two warpgroups
constexpr int A_STAGE_BYTES = TC_BM * TC_BK * 4;   // 16 KB

struct TcArgs {
    int B, T;
    int cchunks;       // round_up(C,32)/32
    int Cpad;
    int taps, tap0;    // dense / plain conv
    int bank;          // 1: taps = n_tile+1, tap0 = -(taps-1)/2
    int N;             // valid output columns (highway: 2U)
    int tiles_per_seq; // M tiles per utterance
    int tile_stride;   // 128, or 127 when pooling
    int pool;
    int lo_row0;       // X3: first row of the lo half in the packed weight buffer (= rows of the hi half)
    int direct;        // 1: register-direct vectorised epilogue (all row strides multiples of 4 floats), 0: transposing epilogue
    EpiParams e;
};

template <int BN, int STAGES, bool X3 = false>
struct SmemLayout {
    static constexpr int B_STAGE_BYTES = BN * TC_BK * 4;
    static constexpr int STAGE_BYTES = A_STAGE_BYTES + (X3 ? 2 : 1) * B_STAGE_BYTES;     // A (raw fp32) | B_hi | (X3) B_lo
    static constexpr int PIPE_BYTES = STAGES * STAGE_BYTES;
    static constexpr int ACC_BYTES = TC_BM * BN / 32 * 33 * 4;   // accumulators staged as [32 rows][33] blocks for the epilogue
    static constexpr int BODY = PIPE_BYTES > ACC_BYTES ? PIPE_BYTES : ACC_BYTES;
    static constexpr int BAR_OFFSET = BODY;
    static constexpr int CONST_OFFSET = BODY + 128;       // direct epilogue: bias[256] | scale[256] | shift[256] | first rows [2][4][32]
    static constexpr int TOTAL = BODY + 128 + 3072 + 1024 + 1024;   // barriers + epilogue constants + alignment slack
    static_assert(STAGE_BYTES % 1024 == 0 && ACC_BYTES % 16 == 0, "stages must keep the 1024-byte swizzle alignment");
    static_assert(TOTAL <= 227 * 1024, "shared memory per block exceeds 227 KB");
};

// fp32 -> nearest TF32-representable value (ties away from zero), two integer instructions.  Adding 0x1000 carries the
// canonical NaN 0x7fffffff (what GPU arithmetic produces) into the sign bit: that NaN becomes -0.  Used for the lo half
// of a split, where the hi half carries any NaN.
__device__ __forceinline__ float rn_tf32(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u); }

// rn_tf32 for the hi half of a split: the signed max (one VIADDMNMX in place of the add) returns a positive NaN as a NaN,
// so a NaN computed by one layer stays NaN in the next contraction.  Every non-NaN value (infinities included) and every
// negative NaN but 0xfffff000..0xffffffff, which arithmetic does not produce, rounds exactly as rn_tf32.
__device__ __forceinline__ float rn_tf32_hi(float x) {
    const uint32_t u = __float_as_uint(x);
    return __uint_as_float((uint32_t)max((int)(u + 0x1000u), (int)u) & 0xffffe000u);
}

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// one k8 step of this warpgroup's m64 x BN product (BN = 256: two n128 halves, B rows 128.. at +16 KB = descriptor + 1024)
template <int BN>
__device__ __forceinline__ void mma_ss(float (&acc)[BN == 32 ? 16 : 64], float (&acc2)[BN == 256 ? 64 : 1], uint64_t ad, uint64_t bd) {
    if constexpr (BN == 32) {
        wgmma_m64n32k8_ss(acc, ad, bd);
    } else {
        wgmma_m64n128k8_ss(acc, ad, bd);
        if constexpr (BN == 256) wgmma_m64n128k8_ss(acc2, ad, bd + 1024);
    }
}
template <int BN>
__device__ __forceinline__ void mma_rs(float (&acc)[BN == 32 ? 16 : 64], float (&acc2)[BN == 256 ? 64 : 1], const uint32_t (&af)[4], uint64_t bd) {
    if constexpr (BN == 32) {
        wgmma_m64n32k8_rs(acc, af, bd);
    } else {
        wgmma_m64n128k8_rs(acc, af, bd);
        if constexpr (BN == 256) wgmma_m64n128k8_rs(acc2, af, bd + 1024);
    }
}

// accumulator fragment (row 16*warp + g (+8), column c0 + 8j + 2tg (+1) of this warpgroup's rows) -> the epilogue's scratch
// blocks; MODE 1 (NSLOT 2): columns [0,128) are the H half (slot 0), [128,256) the T half (slot 1)
template <int NSLOT, int NA>
__device__ __forceinline__ void stage_acc(float* scratch, int frow, int col0, int c0, const float (&acc)[NA]) {
#pragma unroll
    for (int j = 0; j < NA / 4; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int r = frow + 8 * (e >> 1);
            const int c = c0 + col0 + 8 * j + (e & 1);
            const int slot = NSLOT == 2 ? (c >> 7) : 0;
            const int ch = NSLOT == 2 ? ((c & 127) >> 5) : (c >> 5);
            scratch[((ch * 4 + (r >> 5)) * NSLOT + slot) * (32 * 33) + (r & 31) * 33 + (c & 31)] = acc[4 * j + e];
        }
    }
}

// MODE 0: normal epilogue (optional fused max-pool), MODE 1: highway (BN = 2U = 256)
template <int BN, int STAGES, int MODE, bool X3>
__global__ void __launch_bounds__(TC_THREADS, MODE == 1 ? 1 : 2) gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                                 const __grid_constant__ CUtensorMap tmB, TcArgs a) {
    using L = SmemLayout<BN, STAGES, X3>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFFSET);
    uint64_t* empty_bar = full_bar + STAGES;

    const int tid = threadIdx.x;
    const int warp = tid >> 5;
    const int lane = tid & 31;

    // tile coordinates
    const int n_tile = blockIdx.x;
    const int m_tile = blockIdx.y;
    const int b = m_tile / a.tiles_per_seq;
    const int t0 = (m_tile % a.tiles_per_seq) * a.tile_stride;
    const int n0 = n_tile * BN;
    int taps = a.taps, tap0 = a.tap0;
    if (a.bank) { taps = n_tile + 1; tap0 = -((taps - 1) / 2); }
    const int n_iters = taps * a.cchunks;

    if (tid == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], TC_THREADS / 32); }
        mbar_fence_init();
    }
    __syncthreads();

    auto issue = [&](int it) {
        const int s = it % STAGES;
        uint8_t* As = smem + s * L::STAGE_BYTES;
        uint8_t* Bs = As + A_STAGE_BYTES;
        const int j = it / a.cchunks;
        const int c0 = (it - j * a.cchunks) * TC_BK;
        mbar_arrive_expect_tx(&full_bar[s], L::STAGE_BYTES);
        tma_load_3d(As, &tmA, &full_bar[s], c0, t0 + tap0 + j, b);
        tma_load_2d(Bs, &tmB, &full_bar[s], j * a.Cpad + c0, n0);
        if (X3) tma_load_2d(Bs + L::B_STAGE_BYTES, &tmB, &full_bar[s], j * a.Cpad + c0, a.lo_row0 + n0);
    };
    if (tid == 0)
        for (int it = 0; it < STAGES && it < n_iters; ++it) issue(it);

    // ================= main loop: both warpgroups multiply, thread 0 refills the ring =================
    float acc[BN == 32 ? 16 : 64];
    float acc2[BN == 256 ? 64 : 1];
#pragma unroll
    for (int i = 0; i < (BN == 32 ? 16 : 64); ++i) acc[i] = 0.f;
#pragma unroll
    for (int i = 0; i < (BN == 256 ? 64 : 1); ++i) acc2[i] = 0.f;
    const int wg = tid >> 7;
    const int g = lane >> 2, tg = lane & 3;
    const int frow = wg * 64 + (warp & 3) * 16 + g;      // first tile row of this thread's A / accumulator fragments
    for (int it = 0; it < n_iters; ++it) {
        const int s = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1;
        mbar_wait(&full_bar[s], ph);
        const uint8_t* As = smem + s * L::STAGE_BYTES;
        const uint32_t a_addr = smem_u32(As);
        const uint64_t bhi = wgmma_desc_sw128(a_addr + A_STAGE_BYTES);
        if constexpr (X3) {
            const uint64_t blo = wgmma_desc_sw128(a_addr + A_STAGE_BYTES + L::B_STAGE_BYTES);
            // A fragment of k-step k: (row frow (+8), column 8k + tg (+4)), read out of the swizzled tile (16-byte chunk
            // c/4 of row r sits at chunk (c/4) ^ (r%8): the 8 row groups of a warp hit 8 different chunks, conflict-free).
            // x = hi + lo with hi = the nearest TF32 value (so that the result does not depend on how the tensor core
            // narrows fp32) and lo = the remainder, itself rounded to TF32.
            uint32_t ah[TC_BK / 8][4], al[TC_BK / 8][4];
#pragma unroll
            for (int k = 0; k < TC_BK / 8; ++k) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int r = frow + 8 * (e & 1);
                    const int c = 8 * k + tg + 4 * (e >> 1);
                    const float x = *reinterpret_cast<const float*>(As + r * 128 + (((c >> 2) ^ (r & 7)) << 4) + (c & 3) * 4);
                    const float hv = rn_tf32_hi(x);
                    ah[k][e] = __float_as_uint(hv);
                    al[k][e] = __float_as_uint(rn_tf32(x - hv));
                }
            }
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < TC_BK / 8; ++k) {
                // advance 8 tf32 along K: +32 bytes inside the swizzle row = +2 in 16-byte descriptor units
                mma_rs<BN>(acc, acc2, al[k], bhi + (uint64_t)(2 * k));     // lo . hi
                mma_rs<BN>(acc, acc2, ah[k], blo + (uint64_t)(2 * k));     // hi . lo
                mma_rs<BN>(acc, acc2, ah[k], bhi + (uint64_t)(2 * k));     // hi . hi
            }
        } else {
            const uint64_t adesc = wgmma_desc_sw128(a_addr + wg * 64 * 128);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < TC_BK / 8; ++k) mma_ss<BN>(acc, acc2, adesc + (uint64_t)(2 * k), bhi + (uint64_t)(2 * k));
        }
        wgmma_commit();
        wgmma_wait_all();
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[s]);           // this warp's products have read the stage
        if (tid == 0 && it + STAGES < n_iters) {
            mbar_wait(&empty_bar[s], ph);
            issue(it + STAGES);
        }
    }

    // ================= accumulators -> shared memory (the pipeline buffers are idle once every warp is here) =================
    // scratch: [chunk of 32 columns][4 row quarters][MODE ? 2 : 1][32 rows][33] floats -- what the epilogue below walks
    float* scratch_base = reinterpret_cast<float*>(smem);
    constexpr int SCR = 32 * 33;
    constexpr int NSLOT = MODE == 1 ? 2 : 1;
    __syncthreads();
    stage_acc<NSLOT>(scratch_base, frow, 2 * tg, 0, acc);
    if constexpr (BN == 256) stage_acc<NSLOT>(scratch_base, frow, 2 * tg, 128, acc2);
    __syncthreads();

    {
        const int q = warp & 3;                       // row quarter of this warp
        const int eh = tid >> 7;                      // column-chunk half
        if (a.direct) {
            // ================= register-direct epilogue =================
            // lane = output row: a lane reads 32 consecutive columns of ITS row.  The fused epilogue runs on those registers
            // and the row segment leaves as eight 16-byte stores -- ~4 instructions per element less than the transposing
            // epilogue below.  The two halves of the block take alternate 32-column chunks.
            float* cst = reinterpret_cast<float*>(smem + L::CONST_OFFSET);
            float* frow = cst + 768 + eh * 128;
            for (int i = tid; i < BN; i += TC_THREADS) {
                if (MODE == 1) {
                    cst[i] = a.e.bias ? __ldg(a.e.bias + i) : 0.f;
                } else {
                    const int col = n0 + i;
                    const bool cv = col < a.N;
                    cst[i] = (cv && a.e.bias) ? __ldg(a.e.bias + col) : 0.f;
                    if (cv && a.e.bias_utt) cst[i] += __ldg(a.e.bias_utt + (int64_t)b * a.e.ldbu + col);   // one utterance per tile
                    cst[256 + i] = (cv && a.e.scale) ? __ldg(a.e.scale + col) : 1.f;
                    cst[512 + i] = (cv && a.e.shift) ? __ldg(a.e.shift + col) : 0.f;
                }
            }
            __syncthreads();
            const int row = q * 32 + lane;
            const int t = t0 + row;
            const bool row_ok = (t < a.T) && (!a.pool || row < TC_BM - 1 || t == a.T - 1);
            const int64_t grow = (int64_t)b * a.T + t;
            constexpr int NCH = (MODE == 1) ? (BN / 2) / 32 : BN / 32;
            for (int ch = eh; ch < NCH; ch += 2) {
                const float* my_scr = scratch_base + (ch * 4 + q) * NSLOT * SCR;
                uint32_t v[32];
                float y[32];
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] = __float_as_uint(my_scr[lane * 33 + j]);
                const int c0 = ch * 32;                       // column offset inside the tile
                if (MODE == 1) {
                    uint32_t w[32];
#pragma unroll
                    for (int j = 0; j < 32; ++j) w[j] = __float_as_uint(my_scr[SCR + lane * 33 + j]);
                    const float* hx = a.e.hx + grow * a.e.ldhx + c0;
#pragma unroll
                    for (int j = 0; j < 32; j += 4) {
                        const float4 bh = *reinterpret_cast<const float4*>(cst + c0 + j);
                        const float4 bt = *reinterpret_cast<const float4*>(cst + BN / 2 + c0 + j);
                        const float4 x = row_ok ? __ldg(reinterpret_cast<const float4*>(hx + j)) : make_float4(0.f, 0.f, 0.f, 0.f);
                        const float xs[4] = {x.x, x.y, x.z, x.w}, bhs[4] = {bh.x, bh.y, bh.z, bh.w}, bts[4] = {bt.x, bt.y, bt.z, bt.w};
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            const float H = fmaxf(__uint_as_float(v[j + k]) + bhs[k], 0.f);
                            const float Tg = sigmoidf_acc(__uint_as_float(w[j + k]) + bts[k]);
                            y[j + k] = H * Tg + xs[k] * (1.0f - Tg);
                        }
                    }
                } else {
                    const int act = a.e.act;
#pragma unroll
                    for (int j = 0; j < 32; j += 4) {
                        const float4 cb = *reinterpret_cast<const float4*>(cst + c0 + j);
                        const float4 sc = *reinterpret_cast<const float4*>(cst + 256 + c0 + j);
                        const float4 sh = *reinterpret_cast<const float4*>(cst + 512 + c0 + j);
                        const float cbs[4] = {cb.x, cb.y, cb.z, cb.w}, scs[4] = {sc.x, sc.y, sc.z, sc.w}, shs[4] = {sh.x, sh.y, sh.z, sh.w};
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            float u = __uint_as_float(v[j + k]) + cbs[k];
                            u = (act == TACO_ACT_RELU) ? fmaxf(u, 0.f) : (act == TACO_ACT_NONE) ? u : apply_act(u, act);
                            y[j + k] = fmaf(u, scs[k], shs[k]);
                        }
                    }
                    if (a.pool) {
                        // max_pooling1d(2,1,'same') over t: row t needs row t+1 = the next lane; lane 31 takes the first row of
                        // the next quarter from shared memory (tiles advance by 127 rows, so row 127 never needs a successor)
                        named_bar_sync(1 + eh, 128);          // previous chunk's first rows have been consumed
                        if (lane == 0) {
#pragma unroll
                            for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(frow + q * 32 + j) = make_float4(y[j], y[j + 1], y[j + 2], y[j + 3]);
                        }
                        named_bar_sync(1 + eh, 128);
                        const bool has_next = (t + 1 < a.T) && (row + 1 < TC_BM);
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
                            float nx = __shfl_down_sync(0xffffffffu, y[j], 1);
                            if (lane == 31) nx = frow[((q + 1) & 3) * 32 + j];
                            if (has_next) y[j] = fmaxf(y[j], nx);
                        }
                    }
                    if (a.e.keep) {
                        const uint4* kp = reinterpret_cast<const uint4*>(a.e.keep + grow * (int64_t)a.e.N + n0 + c0);
                        if (row_ok) {
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                // N % 16 == 0 here: a 16-column half is either all inside the row or all past its end
                                // (the next row's mask, or past the buffer on the last row) and then not loaded
                                if (n0 + c0 + 16 * h >= a.e.N) break;
                                const uint4 kk = kp[h];
                                const uint32_t ks[4] = {kk.x, kk.y, kk.z, kk.w};
#pragma unroll
                                for (int k = 0; k < 16; ++k)
                                    y[16 * h + k] = ((ks[k >> 2] >> (8 * (k & 3))) & 0xffu) ? y[16 * h + k] * a.e.keep_scale : 0.f;
                            }
                        }
                    }
                    if (a.e.residual && row_ok) {
                        const float* rp = a.e.residual + grow * a.e.ldr + n0 + c0;
#pragma unroll
                        for (int j = 0; j < 32; j += 4) {
                            if (n0 + c0 + j < a.N) {
                                const float4 r4 = __ldg(reinterpret_cast<const float4*>(rp + j));
                                y[j] += r4.x; y[j + 1] += r4.y; y[j + 2] += r4.z; y[j + 3] += r4.w;
                            }
                        }
                    }
                }
                if (row_ok) {
                    float* yp = a.e.Y + grow * a.e.ldy + (MODE == 1 ? 0 : n0) + c0;
                    const int ncols = (MODE == 1) ? BN / 2 : a.N;
                    const int cbase = (MODE == 1 ? 0 : n0) + c0;
#pragma unroll
                    for (int j = 0; j < 32; j += 4)
                        if (cbase + j < ncols) *reinterpret_cast<float4*>(yp + j) = make_float4(y[j], y[j + 1], y[j + 2], y[j + 3]);
                }
            }
        } else {
        const int64_t seq_row0 = (int64_t)b * a.T;
        constexpr int NCHUNK = (MODE == 1) ? (BN / 2) / 32 : BN / 32;
        constexpr int EPB = (MODE == 1) ? 8 : 16;     // epilogue rows per load batch (independent global loads in flight per lane)

        for (int ch = eh; ch < NCHUNK; ch += 2) {
            const float* my_scr = scratch_base + (ch * 4 + q) * NSLOT * SCR;
            const int col = n0 + ch * 32 + lane;     // MODE 1: n0 == 0, col in [0,U)
            int nrows = a.T - (t0 + q * 32);          // valid rows of this warp's quarter
            nrows = nrows < 0 ? 0 : (nrows > 32 ? 32 : nrows);
            const int64_t row0 = seq_row0 + t0 + q * 32;
            // The row loops below are written "all loads of a batch first, then math + stores" so that 8
            // independent global loads are in flight per lane (a naive row-at-a-time loop serialises on
            // L2 latency).
            if (MODE == 1) {
                const int U = BN / 2;
                const float bH = a.e.bias ? __ldg(a.e.bias + col) : 0.f;
                const float bT = a.e.bias ? __ldg(a.e.bias + U + col) : 0.f;
                for (int rr0 = 0; rr0 < nrows; rr0 += EPB) {
                    float xin[EPB];
#pragma unroll
                    for (int i = 0; i < EPB; ++i)
                        xin[i] = (rr0 + i < nrows) ? __ldg(a.e.hx + (row0 + rr0 + i) * a.e.ldhx + col) : 0.f;
#pragma unroll
                    for (int i = 0; i < EPB; ++i) {
                        if (rr0 + i < nrows) {
                            const float H = fmaxf(my_scr[(rr0 + i) * 33 + lane] + bH, 0.f);
                            const float Tg = sigmoidf_acc(my_scr[SCR + (rr0 + i) * 33 + lane] + bT);
                            a.e.Y[(row0 + rr0 + i) * a.e.ldy + col] = H * Tg + xin[i] * (1.0f - Tg);
                        }
                    }
                }
            } else {
                const bool cvalid = col < a.N;
                float cb = (cvalid && a.e.bias) ? __ldg(a.e.bias + col) : 0.f;
                if (cvalid && a.e.bias_utt) cb += __ldg(a.e.bias_utt + (int64_t)b * a.e.ldbu + col);
                const float csc = (cvalid && a.e.scale) ? __ldg(a.e.scale + col) : 1.f;
                const float csh = (cvalid && a.e.shift) ? __ldg(a.e.shift + col) : 0.f;
                const int act = a.e.act;
                auto affine = [&](float v) { return apply_act(v + cb, act) * csc + csh; };
                if (!a.pool && !a.e.keep && !a.e.residual) {
                    // fast path (the 1025-wide spectrogram projection lands here: its rows are not 16-byte aligned, so
                    // the register-direct epilogue cannot be used): pointer stepping, no per-element index arithmetic
                    if (cvalid) {
                        float* yp = a.e.Y + row0 * a.e.ldy + col;
                        const int64_t ys = a.e.ldy;
                        if (act == TACO_ACT_RELU) {
#pragma unroll 8
                            for (int rr = 0; rr < nrows; ++rr) { *yp = fmaf(fmaxf(my_scr[rr * 33 + lane] + cb, 0.f), csc, csh); yp += ys; }
                        } else if (act == TACO_ACT_NONE) {
#pragma unroll 8
                            for (int rr = 0; rr < nrows; ++rr) { *yp = fmaf(my_scr[rr * 33 + lane] + cb, csc, csh); yp += ys; }
                        } else {
#pragma unroll 4
                            for (int rr = 0; rr < nrows; ++rr) { *yp = affine(my_scr[rr * 33 + lane]); yp += ys; }
                        }
                    }
                } else if (!a.pool) {
                    if (cvalid) {
                        for (int rr0 = 0; rr0 < nrows; rr0 += EPB) {
                            float res[EPB];
                            float kp[EPB];
#pragma unroll
                            for (int i = 0; i < EPB; ++i) {
                                const bool ok = rr0 + i < nrows;
                                res[i] = (ok && a.e.residual) ? __ldg(a.e.residual + (row0 + rr0 + i) * a.e.ldr + col) : 0.f;
                                kp[i] = (ok && a.e.keep) ? (a.e.keep[(row0 + rr0 + i) * (int64_t)a.e.N + col] ? a.e.keep_scale : 0.f) : 1.f;
                            }
#pragma unroll
                            for (int i = 0; i < EPB; ++i) {
                                if (rr0 + i < nrows)
                                    a.e.Y[(row0 + rr0 + i) * a.e.ldy + col] = affine(my_scr[(rr0 + i) * 33 + lane]) * kp[i] + res[i];
                            }
                        }
                    }
                } else {
                    // fused max_pooling1d(2,1,'same') over t (models/ops.py:66-71): out[t] = max(e[t], e[t+1]),
                    // out[T-1] = e[T-1].  Tiles advance by 127 rows so row r+1 is always in this tile.
                    if (cvalid && nrows > 0) {
                        const float* nxt_scr = scratch_base + (ch * 4 + ((q + 1) & 3)) * SCR;   // first row of the next quarter
                        float cur = affine(my_scr[lane]);
#pragma unroll 8
                        for (int rr = 0; rr < nrows; ++rr) {
                            const int r = q * 32 + rr;
                            const int t = t0 + r;
                            const bool has_next = (t + 1 < a.T) && (r + 1 < TC_BM);
                            float nxt = 0.f;
                            if (has_next) nxt = affine((rr < 31) ? my_scr[(rr + 1) * 33 + lane] : nxt_scr[lane]);
                            // rows 0..126 of the tile are produced here; row 127 only if it is the sequence end
                            if ((r < TC_BM - 1) || (t == a.T - 1))
                                a.e.Y[(seq_row0 + t) * a.e.ldy + col] = (t + 1 < a.T) ? fmaxf(cur, nxt) : cur;
                            cur = nxt;
                        }
                    }
                }
            }
        }
        }   // transposing epilogue
    }

}

// ---- weight packing: TF [taps][C][N] -> K-major [N][taps*Cpad], TF32 round-to-nearest ----
__global__ void pack_weight_kernel(const float* __restrict__ W, int taps, int C, int N, int Cpad,
                                   float* __restrict__ dst, int64_t ld) {
    // one thread per (n, j, cpad-index); reads are strided by N but this runs once per weight update
    int64_t total = (int64_t)N * taps * Cpad;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int c = (int)(i % Cpad);
        int64_t r = i / Cpad;
        int j = (int)(r % taps);
        int n = (int)(r / taps);
        float v = 0.0f;
        if (c < C) {
            v = W[((int64_t)j * C + c) * N + n];
            uint32_t u;
            asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
            v = __uint_as_float(u);
        }
        dst[(int64_t)n * ld + (int64_t)j * Cpad + c] = v;
    }
}

// X3: hi = TF32 round-to-nearest head (ties away from zero), lo = (W - hi) rounded to the nearest TF32 value (ties away
// from zero; W - hi is exact and has at most 13 significant bits, so the rounding drops at most 2^-22 |W|) -- both
// exactly representable, so the tensor core's own fp32 -> tf32 narrowing cannot change them
__global__ void pack_weight_x3_kernel(const float* __restrict__ W, int taps, int C, int N, int Cpad,
                                      float* __restrict__ dst_hi, float* __restrict__ dst_lo, int64_t ld) {
    int64_t total = (int64_t)N * taps * Cpad;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int c = (int)(i % Cpad);
        int64_t r = i / Cpad;
        int j = (int)(r % taps);
        int n = (int)(r / taps);
        float hi = 0.0f, lo = 0.0f;
        if (c < C) {
            const float v = W[((int64_t)j * C + c) * N + n];
            uint32_t u;
            asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
            hi = __uint_as_float(u & 0xffffe000u);
            lo = __uint_as_float((__float_as_uint(v - hi) + 0x1000u) & 0xffffe000u);    // nearest, not cut: no systematic bias
        }
        dst_hi[(int64_t)n * ld + (int64_t)j * Cpad + c] = hi;
        dst_lo[(int64_t)n * ld + (int64_t)j * Cpad + c] = lo;
    }
}

// ---- driver entry point for cuTensorMapEncodeTiled (no link-time libcuda dependency) ----
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn) return fn;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p) return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
    return fn;
}




// =====================================================================================================================
// Weight gradient of conv1d('same') / dense on the tensor cores (3xTF32, fp32-grade):
//     dW[j][c][n] += sum_{b,t} X[b, t+tap0+j, c] * dZ[b, t, n]
// The contraction runs over the ROWS of both operands (what a BLAS calls a TN product).  Neither operand is
// transposed in HBM:
//   * a k-block = 32 consecutive rows t of one utterance.  TMA (3-D maps (C,T,B) / (N,T,B), no swizzle, OOB rows and
//     columns zero-filled = the 'same' padding and the ragged edges) lands X[32 rows][128 c] and dZ[32 rows][128 n];
//   * the A operand (M = c, K = rows) comes from registers: each thread reads its fragment as a column of the X tile
//     and splits it into hi / lo TF32 halves (as in the forward kernel);
//   * wgmma takes TF32 B operands only K-major, so all 256 threads transpose + split the dZ tile into two K-major
//     SWIZZLE_128B tiles (hi, lo): thread = n reads 4 consecutive rows (conflict-free) and writes one 16-byte chunk per
//     tile (8 lanes of a store phase hit 8 different chunks: conflict-free);
//   * each warpgroup issues lo.hi + hi.lo + hi.hi wgmma m64n128k8 per 8 rows into its [64 c][128 n] register accumulator;
//   * split-K over the (b, t-block) list: grid.y CTAs each reduce a contiguous range and add their tile into dW with
//     vector reductions (red.global.add.v2.f32) -- same accumulate-with-atomics contract as taco_gemm's ta=1 path;
//   * chains are cut at 1024 rows: the accumulators are added into dW and restart, so that no single tensor-core
//     accumulation chain runs over more than 1024 rows.
// =====================================================================================================================
constexpr int DW_THREADS = 256;
constexpr int DW_STAGES = 4;
constexpr int DW_TILE_BYTES = 32 * 128 * 4;               // every staged tile is 16 KB
constexpr int DW_STAGE_BYTES = 2 * DW_TILE_BYTES;         // X raw | dZ raw
constexpr int DW_CONV_OFFSET = DW_STAGES * DW_STAGE_BYTES;   // dZ hi | dZ lo (K-major): one pair, a k-block's products complete before the next is converted
constexpr int DW_DRAIN = 32;                             // k-blocks (1024 rows) summed in registers before the partial tile is added to dW
constexpr int DW_SMEM = DW_CONV_OFFSET + 2 * DW_TILE_BYTES + 256 + 1024;

struct DwArgs {
    int T, C, N, taps, tap0;
    int c_tiles, n_tiles;
    int blocks_per_seq;      // ceil(T / 32)
    int total_blocks;        // B * blocks_per_seq
    int per_split;
    float* dW; int64_t ldw; int64_t tap_stride;
    int vec2;                // dW pairs (n, n+1) 8-byte aligned
};

__global__ void __launch_bounds__(DW_THREADS, 1) dw_tc_kernel(const __grid_constant__ CUtensorMap tmX,
                                                              const __grid_constant__ CUtensorMap tmZ, DwArgs a) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* zconv = smem + DW_CONV_OFFSET;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(zconv + 2 * DW_TILE_BYTES);
    uint64_t* empty_bar = full_bar + DW_STAGES;

    const int tid = threadIdx.x;
    const int warp = tid >> 5;
    const int lane = tid & 31;

    const int tiles = a.c_tiles * a.n_tiles;
    const int j = blockIdx.x / tiles;
    const int rem = blockIdx.x - j * tiles;
    const int c0 = (rem / a.n_tiles) * 128;
    const int n0 = (rem % a.n_tiles) * 128;
    const int g0 = blockIdx.y * a.per_split;
    const int g1 = min(a.total_blocks, g0 + a.per_split);
    const int n_iters = g1 - g0;                                   // >= 1 (host)

    if (tid == 0) {
        tma_prefetch_desc(&tmX);
        tma_prefetch_desc(&tmZ);
        for (int s = 0; s < DW_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], DW_THREADS / 32); }
        mbar_fence_init();
    }
    __syncthreads();

    auto issue = [&](int it) {
        const int s = it % DW_STAGES;
        uint8_t* st = smem + s * DW_STAGE_BYTES;
        const int gb = g0 + it;
        const int b = gb / a.blocks_per_seq;
        const int t = (gb - b * a.blocks_per_seq) * 32;
        mbar_arrive_expect_tx(&full_bar[s], 2 * DW_TILE_BYTES);
        tma_load_3d(st, &tmX, &full_bar[s], c0, t + a.tap0 + j, b);
        tma_load_3d(st + DW_TILE_BYTES, &tmZ, &full_bar[s], n0, t, b);
    };
    if (tid == 0)
        for (int it = 0; it < DW_STAGES && it < n_iters; ++it) issue(it);

    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    const int wg = tid >> 7;
    const int g = lane >> 2, tg = lane & 3;
    const int mrow = wg * 64 + (warp & 3) * 16 + g;                // accumulator row (c - c0) of this thread's fragments
    const int cn = tid & 127;                                      // dZ column this thread transposes ...
    const int kc0 = (tid >> 7) * 4;                                // ... for 16-byte k chunks kc0 .. kc0+3
    const uint64_t bhi = wgmma_desc_sw128(smem_u32(zconv));
    const uint64_t blo = wgmma_desc_sw128(smem_u32(zconv + DW_TILE_BYTES));

    // add the register accumulators into dW and restart the chain
    auto drain = [&]() {
        float* dWj = a.dW + (int64_t)j * a.tap_stride;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int c = c0 + mrow + 8 * h;
            if (c < a.C) {
                float* drow = dWj + (int64_t)c * a.ldw;
#pragma unroll
                for (int jj = 0; jj < 16; ++jj) {
                    const int n = n0 + 8 * jj + 2 * tg;
                    const float v0 = acc[4 * jj + 2 * h], v1 = acc[4 * jj + 2 * h + 1];
                    if (a.vec2 && n + 1 < a.N) {
                        asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(drow + n), "f"(v0), "f"(v1) : "memory");
                    } else {
                        if (n < a.N) atomicAdd(drow + n, v0);
                        if (n + 1 < a.N) atomicAdd(drow + n + 1, v1);
                    }
                }
            }
        }
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    };

    for (int chain0 = 0; chain0 < n_iters; chain0 += DW_DRAIN) {
        const int chain1 = min(n_iters, chain0 + DW_DRAIN);
        for (int it = chain0; it < chain1; ++it) {
            const int s = it % DW_STAGES;
            const uint32_t ph = (it / DW_STAGES) & 1;
            mbar_wait(&full_bar[s], ph);
            const float* xs = reinterpret_cast<const float*>(smem + s * DW_STAGE_BYTES);     // [32 rows][128 c]
            const float* zs = xs + DW_TILE_BYTES / 4;                                         // [32 rows][128 n]
            __syncthreads();                       // every warpgroup's products of the previous k-block have read the hi / lo tiles
    #pragma unroll
            for (int kc = kc0; kc < kc0 + 4; ++kc) {
                float4 h4, l4;
                const float z0 = zs[(4 * kc + 0) * 128 + cn], z1 = zs[(4 * kc + 1) * 128 + cn], z2 = zs[(4 * kc + 2) * 128 + cn], z3 = zs[(4 * kc + 3) * 128 + cn];
                h4.x = rn_tf32_hi(z0); l4.x = rn_tf32(z0 - h4.x);
                h4.y = rn_tf32_hi(z1); l4.y = rn_tf32(z1 - h4.y);
                h4.z = rn_tf32_hi(z2); l4.z = rn_tf32(z2 - h4.z);
                h4.w = rn_tf32_hi(z3); l4.w = rn_tf32(z3 - h4.w);
                const int off = cn * 128 + ((kc ^ (cn & 7)) << 4);
                *reinterpret_cast<float4*>(zconv + off) = h4;
                *reinterpret_cast<float4*>(zconv + DW_TILE_BYTES + off) = l4;
            }
            fence_proxy_async();                   // generic-proxy tile writes -> visible to the tensor core's async-proxy reads
            __syncthreads();
            // A fragment of k-step k: element (m = mrow (+8), k = 8k + tg (+4)) = X[row 8k + tg (+4)][c0 + m]
            uint32_t ah[4][4], al[4][4];
    #pragma unroll
            for (int k = 0; k < 4; ++k) {
    #pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float x = xs[(8 * k + tg + 4 * (e >> 1)) * 128 + mrow + 8 * (e & 1)];
                    const float hv = rn_tf32_hi(x);
                    ah[k][e] = __float_as_uint(hv);
                    al[k][e] = __float_as_uint(rn_tf32(x - hv));
                }
            }
            wgmma_fence();
    #pragma unroll
            for (int k = 0; k < 4; ++k) {
                wgmma_m64n128k8_rs(acc, al[k], bhi + (uint64_t)(2 * k));   // lo . hi
                wgmma_m64n128k8_rs(acc, ah[k], blo + (uint64_t)(2 * k));   // hi . lo
                wgmma_m64n128k8_rs(acc, ah[k], bhi + (uint64_t)(2 * k));   // hi . hi
            }
            wgmma_commit();
            wgmma_wait_all();
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[s]);
            if (tid == 0 && it + DW_STAGES < n_iters) {
                mbar_wait(&empty_bar[s], ph);
                issue(it + DW_STAGES);
            }
        }
        drain();
    }
}

// =====================================================================================================================
// taco_highway_stack_fwd: the pointwise tail of a CBHG inference (width-fixing dense, the highway layers, the bi-GRU
// input products) as ONE kernel, 3xTF32 (TACO_IMPL_TC3) only.
//
// Every layer of that chain is a dense (taps = 1), so a tile of flat rows (utterance boundaries do not matter) can run
// the whole chain without its activations leaving the SM:
//  * one CTA per 128-row tile: TMA loads the input rows once over a 2-D map of the flat rows, as 32-channel k-blocks in
//    the 128B-swizzled K-major layout the X3 A-fragment reader of gemm_tc_kernel reads (rows past M and channels past C are
//    zero-filled: C = 80 in the post-net is padded to 96);
//  * the activation tile (128 rows x 128 channels, 64 KB) stays in shared memory between layers, in two buffers: a
//    highway layer's carry x is its own input tile, so each layer reads one buffer and writes the other;
//  * the weights stream through a 3-deep TMA ring from the packed hi / lo buffers of taco_pack_weight_x3, one stage =
//    the hi and lo halves of 128 output columns x one k-block (32 KB).  The ring runs through the whole chain in one
//    order (layer, 128-column chunk, k-block), so the next layer's weights load under the current layer's epilogue;
//  * warpgroup w multiplies rows [64w, 64w+64) with wgmma m64n128k8 exactly as gemm_tc_kernel<.., X3 = true> does
//    (same rn_tf32 hi / lo split of A, same lo.hi + hi.lo + hi.hi order per k8 step, k-blocks in order), and the
//    epilogue runs on the accumulator fragments in registers with the same expressions as that kernel's register-direct
//    epilogue.  Each output element therefore sees the same operations in the same order as on the unfused route, and
//    the result is bit-identical to it;
//  * a warp's A fragments and its epilogue cover the same 16 rows, so a layer's output is ready for the next layer
//    after a __syncwarp: the two warpgroups share only the weight ring;
//  * only xp (+ its bias) is written to HBM.  When there are fewer tiles than SMs (the encoder: 32 utterances x 128
//    characters), grid.y splits the 768 xp columns: each CTA of a tile repeats the (cheap, otherwise idle-SM) highway
//    layers and writes its share of xp.
// =====================================================================================================================

constexpr int HS_BM = 128;
constexpr int HS_BK = 32;                                  // floats: one 128-byte swizzle row
constexpr int HS_THREADS = 256;                            // two warpgroups
constexpr int HS_STAGES = 3;
constexpr int HS_TILE_BYTES = HS_BM * HS_BK * 4;           // 16 KB: 128 rows (or 128 weight columns) x one k-block
constexpr int HS_ACT_BYTES = 4 * HS_TILE_BYTES;            // 128 rows x 128 channels
constexpr int HS_STAGE_BYTES = 2 * HS_TILE_BYTES;          // weight hi | lo
constexpr int HS_RING_OFFSET = 2 * HS_ACT_BYTES;
constexpr int HS_BAR_OFFSET = HS_RING_OFFSET + HS_STAGES * HS_STAGE_BYTES;
constexpr int HS_SMEM = HS_BAR_OFFSET + 128 + 1024;        // barriers + alignment slack
static_assert(HS_SMEM <= 227 * 1024, "shared memory per block exceeds 227 KB");
constexpr int HS_XP_N = 768;
constexpr int HS_MAX_LAYERS = TACO_HIGHWAY_STACK_MAX + 2;  // width-fixing dense + highway layers + xp

struct HsMaps {
    CUtensorMap x;                       // input rows [M][C], box {32 ch, 128 rows}
    CUtensorMap w[HS_MAX_LAYERS];        // packed weights of each layer, box {32 k, 128 output columns}
};

struct HsArgs {
    int M;
    int nlayers;                         // (dense) + highway layers + xp
    int dense;                           // 1: layer 0 is the width-fixing dense (C != 128)
    int kin;                             // k-blocks of layer 0 (round_up(C, 32) / 32)
    int xp_chunks;                       // 128-column chunks of xp per CTA (6 / grid.y)
    int total_items;                     // weight stages the CTA consumes
    int lo_row0[HS_MAX_LAYERS];          // first row of the lo half in each packed buffer (= the layer's N)
    const float* bias[HS_MAX_LAYERS];    // dense [128], highway [bH | bT] (256), xp [768]
    float* Y;                            // xp [M][ldy]
    int64_t ldy;
};

// byte offset of (row r, channel col) in a 128-row activation tile: k-block col/32, 16-byte chunk (col%32)/4 of row r at
// chunk ((col%32)/4) ^ (r%8) (SWIZZLE_128B)
__device__ __forceinline__ int act_off(int r, int col) {
    const int c = col & 31;
    return (col >> 5) * HS_TILE_BYTES + r * 128 + (((c >> 2) ^ (r & 7)) << 4) + (c & 3) * 4;
}

__global__ void __launch_bounds__(HS_THREADS, 1) highway_stack_kernel(const __grid_constant__ HsMaps maps, const __grid_constant__ HsArgs a) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* ring = smem + HS_RING_OFFSET;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + HS_BAR_OFFSET);
    uint64_t* empty_bar = full_bar + HS_STAGES;
    uint64_t* in_bar = empty_bar + HS_STAGES;

    const int tid = threadIdx.x;
    const int warp = tid >> 5;
    const int lane = tid & 31;
    const int row0 = blockIdx.x * HS_BM;
    const int xp_chunk0 = blockIdx.y * a.xp_chunks;

    auto nchunks = [&](int l) { return l == a.nlayers - 1 ? a.xp_chunks : (a.dense && l == 0) ? 1 : 2; };
    auto kblocks = [&](int l) { return l == 0 ? a.kin : 4; };

    // producer cursor (thread 0 only): the next weight stage to load, in consumption order
    int pl = 0, pch = 0, pkb = 0;
    auto issue = [&](int it) {
        const int s = it % HS_STAGES;
        uint8_t* Bs = ring + s * HS_STAGE_BYTES;
        const int n0 = ((pl == a.nlayers - 1) ? xp_chunk0 + pch : pch) * 128;
        mbar_arrive_expect_tx(&full_bar[s], HS_STAGE_BYTES);
        tma_load_2d(Bs, &maps.w[pl], &full_bar[s], pkb * HS_BK, n0);
        tma_load_2d(Bs + HS_TILE_BYTES, &maps.w[pl], &full_bar[s], pkb * HS_BK, a.lo_row0[pl] + n0);
        if (++pkb == kblocks(pl)) {
            pkb = 0;
            if (++pch == nchunks(pl)) { pch = 0; ++pl; }
        }
    };

    if (tid == 0) {
        tma_prefetch_desc(&maps.x);
        for (int s = 0; s < HS_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], HS_THREADS / 32); }
        mbar_init(in_bar, 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (tid == 0) {
        mbar_arrive_expect_tx(in_bar, a.kin * HS_TILE_BYTES);
        for (int kb = 0; kb < a.kin; ++kb) tma_load_2d(smem + kb * HS_TILE_BYTES, &maps.x, in_bar, kb * HS_BK, row0);
        for (int it = 0; it < HS_STAGES && it < a.total_items; ++it) issue(it);
    }

    const int wg = tid >> 7;
    const int g = lane >> 2, tg = lane & 3;
    const int frow = wg * 64 + (warp & 3) * 16 + g;       // first tile row of this thread's A / accumulator fragments
    int it = 0;                                           // weight stage being consumed

    // one 128-column chunk of a layer: d = act_in[rows, 0 : 32 kb) . W[:, chunk], k-blocks in order (gemm_tc_kernel X3)
    auto mma_chunk = [&](float (&d)[64], const uint8_t* act_in, int kb_n) {
#pragma unroll
        for (int i = 0; i < 64; ++i) d[i] = 0.f;
        for (int kb = 0; kb < kb_n; ++kb, ++it) {
            const int s = it % HS_STAGES;
            const uint32_t ph = (it / HS_STAGES) & 1;
            mbar_wait(&full_bar[s], ph);
            const uint8_t* As = act_in + kb * HS_TILE_BYTES;
            const uint32_t b_addr = smem_u32(ring + s * HS_STAGE_BYTES);
            const uint64_t bhi = wgmma_desc_sw128(b_addr);
            const uint64_t blo = wgmma_desc_sw128(b_addr + HS_TILE_BYTES);
            uint32_t ah[HS_BK / 8][4], al[HS_BK / 8][4];
#pragma unroll
            for (int k = 0; k < HS_BK / 8; ++k) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int r = frow + 8 * (e & 1);
                    const int c = 8 * k + tg + 4 * (e >> 1);
                    const float x = *reinterpret_cast<const float*>(As + r * 128 + (((c >> 2) ^ (r & 7)) << 4) + (c & 3) * 4);
                    const float hv = rn_tf32_hi(x);
                    ah[k][e] = __float_as_uint(hv);
                    al[k][e] = __float_as_uint(rn_tf32(x - hv));
                }
            }
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < HS_BK / 8; ++k) {
                wgmma_m64n128k8_rs(d, al[k], bhi + (uint64_t)(2 * k));     // lo . hi
                wgmma_m64n128k8_rs(d, ah[k], blo + (uint64_t)(2 * k));     // hi . lo
                wgmma_m64n128k8_rs(d, ah[k], bhi + (uint64_t)(2 * k));     // hi . hi
            }
            wgmma_commit();
            wgmma_wait_all();
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[s]);           // this warp's products have read the stage
            if (tid == 0 && it + HS_STAGES < a.total_items) {
                mbar_wait(&empty_bar[s], ph);
                issue(it + HS_STAGES);
            }
        }
    };

    mbar_wait(in_bar, 0);
    uint8_t* act_in = smem;
    uint8_t* act_out = smem + HS_ACT_BYTES;
    float acc[64], acc2[64];
    // accumulator fragment i = 4j + e of this thread: row frow + 8 (e >> 1), column 8j + 2 tg + (e & 1) of the chunk
    for (int l = 0; l < a.nlayers; ++l) {
        const float* bias = a.bias[l];
        if (l == a.nlayers - 1) {
            // ---- bi-GRU input products: xp = h . Wx + bx, the only output that leaves the SM ----
            for (int ch = 0; ch < a.xp_chunks; ++ch) {
                mma_chunk(acc, act_in, kblocks(l));
                const int n0 = (xp_chunk0 + ch) * 128;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int grow = row0 + frow + 8 * h;
                    if (grow < a.M) {
                        float* yp = a.Y + (int64_t)grow * a.ldy + n0 + 2 * tg;
#pragma unroll
                        for (int j = 0; j < 16; ++j) {
                            const float b0 = __ldg(bias + n0 + 8 * j + 2 * tg), b1 = __ldg(bias + n0 + 8 * j + 2 * tg + 1);
                            *reinterpret_cast<float2*>(yp + 8 * j) =
                                make_float2(fmaf(acc[4 * j + 2 * h] + b0, 1.f, 0.f), fmaf(acc[4 * j + 2 * h + 1] + b1, 1.f, 0.f));
                        }
                    }
                }
            }
        } else if (a.dense && l == 0) {
            // ---- width-fixing dense (models/ops.py:29-30): y = x . Wd + bd ----
            mma_chunk(acc, act_in, kblocks(l));
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = frow + 8 * h;
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int col = 8 * j + 2 * tg;
                    const float b0 = __ldg(bias + col), b1 = __ldg(bias + col + 1);
                    *reinterpret_cast<float2*>(act_out + act_off(r, col)) =
                        make_float2(fmaf(acc[4 * j + 2 * h] + b0, 1.f, 0.f), fmaf(acc[4 * j + 2 * h + 1] + b1, 1.f, 0.f));
                }
            }
            __syncwarp();
            uint8_t* t = act_in; act_in = act_out; act_out = t;
        } else {
            // ---- highway (models/ops.py:32-45): H = relu(x.WH + bH), T = sigmoid(x.WT + bT), y = H T + x (1 - T) ----
            mma_chunk(acc, act_in, kblocks(l));
            mma_chunk(acc2, act_in, kblocks(l));
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = frow + 8 * h;
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int col = 8 * j + 2 * tg;
                    const float2 x = *reinterpret_cast<const float2*>(act_in + act_off(r, col));
                    const float xs[2] = {x.x, x.y};
                    float y[2];
#pragma unroll
                    for (int k = 0; k < 2; ++k) {
                        const float H = fmaxf(acc[4 * j + 2 * h + k] + __ldg(bias + col + k), 0.f);
                        const float Tg = sigmoidf_acc(acc2[4 * j + 2 * h + k] + __ldg(bias + 128 + col + k));
                        y[k] = H * Tg + xs[k] * (1.0f - Tg);
                    }
                    *reinterpret_cast<float2*>(act_out + act_off(r, col)) = make_float2(y[0], y[1]);
                }
            }
            __syncwarp();
            uint8_t* t = act_in; act_in = act_out; act_out = t;
        }
    }
}

// 2-D fp32 map [rows][cols] (row stride ld floats), box {32 columns, 128 rows}, 128-byte swizzle
int encode_2d(EncodeTiledFn enc, CUtensorMap* m, const float* base, int64_t cols, int64_t rows, int64_t ld, const char* what) {
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
    cuuint32_t box[2] = {HS_BK, HS_BM};
    cuuint32_t es[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    TACO_CHECK(r == CUDA_SUCCESS, "taco_highway_stack_fwd: cuTensorMapEncodeTiled(%s) failed: %d (cols=%lld rows=%lld ld=%lld)", what,
               (int)r, (long long)cols, (long long)rows, (long long)ld);
    return 0;
}

template <int BN, int STAGES, int MODE, bool X3 = false>
int launch_tc(const CUtensorMap& tmA, const CUtensorMap& tmB, const TcArgs& a, dim3 grid, cudaStream_t st) {
    using L = SmemLayout<BN, STAGES, X3>;
    static bool configured = false;
    if (!configured) {
        TACO_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<BN, STAGES, MODE, X3>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
        configured = true;
    }
    gemm_tc_kernel<BN, STAGES, MODE, X3><<<grid, TC_THREADS, L::TOTAL, st>>>(tmA, tmB, a);
    TACO_LAUNCH_CHECK();
    return 0;
}

}  // namespace

int taco_pack_weight_impl(const float* W, int taps, int C, int N, float* dst, int64_t ld_dst, cudaStream_t st) {
    const int Cpad = (C + 31) / 32 * 32;
    TACO_CHECK(ld_dst >= (int64_t)taps * Cpad, "taco_pack_weight: ld_dst %lld < taps*Cpad %d", (long long)ld_dst, taps * Cpad);
    int64_t total = (int64_t)N * taps * Cpad;
    int blocks = (int)((total + 255) / 256);
    if (blocks > TACO_SMS * 16) blocks = TACO_SMS * 16;
    if (blocks < 1) blocks = 1;
    pack_weight_kernel<<<blocks, 256, 0, st>>>(W, taps, C, N, Cpad, dst, ld_dst);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_pack_weight_x3_impl(const float* W, int taps, int C, int N, float* dst_hi, float* dst_lo, int64_t ld_dst, cudaStream_t st) {
    const int Cpad = (C + 31) / 32 * 32;
    TACO_CHECK(ld_dst >= (int64_t)taps * Cpad, "taco_pack_weight_x3: ld_dst %lld < taps*Cpad %d", (long long)ld_dst, taps * Cpad);
    int64_t total = (int64_t)N * taps * Cpad;
    int blocks = (int)((total + 255) / 256);
    if (blocks > TACO_SMS * 16) blocks = TACO_SMS * 16;
    if (blocks < 1) blocks = 1;
    pack_weight_x3_kernel<<<blocks, 256, 0, st>>>(W, taps, C, N, Cpad, dst_hi, dst_lo, ld_dst);
    TACO_LAUNCH_CHECK();
    return 0;
}

int taco_conv_dw_tc_impl(float* dW, int64_t ldw, int64_t tap_stride, const float* X, int64_t ldx, const float* dZ, int64_t lddz,
                         int B, int T, int C, int N, int taps, int tap0, cudaStream_t st) {
    TACO_CHECK(taco_aligned16(X) && taco_aligned16(dZ), "taco_conv_dw: X / dZ must be 16-byte aligned");
    TACO_CHECK((ldx % 4) == 0 && (lddz % 4) == 0, "taco_conv_dw: ldx and lddz must be multiples of 4 floats (TMA 16B strides)");
    TACO_CHECK(B >= 1 && T >= 1 && C >= 1 && N >= 1 && taps >= 1, "taco_conv_dw: bad shape");
    EncodeTiledFn enc = get_encode_fn();
    TACO_CHECK(enc != nullptr, "cuTensorMapEncodeTiled driver entry point not available");
    DwArgs a;
    a.T = T; a.C = C; a.N = N; a.taps = taps; a.tap0 = tap0;
    a.c_tiles = (C + 127) / 128; a.n_tiles = (N + 127) / 128;
    a.blocks_per_seq = (T + 31) / 32;
    a.total_blocks = B * a.blocks_per_seq;
    const int tiles = a.c_tiles * a.n_tiles * taps;
    int splits = TACO_SMS / tiles;
    if (splits < 1) splits = 1;
    if (splits > a.total_blocks) splits = a.total_blocks;
    a.per_split = (a.total_blocks + splits - 1) / splits;
    splits = (a.total_blocks + a.per_split - 1) / a.per_split;        // every split owns at least one block
    a.dW = dW; a.ldw = ldw; a.tap_stride = tap_stride;
    a.vec2 = ((reinterpret_cast<uintptr_t>(dW) & 7) == 0 && (ldw % 2) == 0 && (tap_stride % 2) == 0) ? 1 : 0;
    CUtensorMap tmX, tmZ;
    {
        cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)T, (cuuint64_t)B};
        cuuint64_t strides[2] = {(cuuint64_t)ldx * 4, (cuuint64_t)T * (cuuint64_t)ldx * 4};
        cuuint32_t box[3] = {128, 32, 1};
        cuuint32_t es[3] = {1, 1, 1};
        CUresult r = enc(&tmX, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(X), dims, strides, box, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        TACO_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(X) failed: %d (C=%d T=%d B=%d ldx=%lld)", (int)r, C, T, B, (long long)ldx);
    }
    {
        cuuint64_t dims[3] = {(cuuint64_t)N, (cuuint64_t)T, (cuuint64_t)B};
        cuuint64_t strides[2] = {(cuuint64_t)lddz * 4, (cuuint64_t)T * (cuuint64_t)lddz * 4};
        cuuint32_t box[3] = {128, 32, 1};
        cuuint32_t es[3] = {1, 1, 1};
        CUresult r = enc(&tmZ, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(dZ), dims, strides, box, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        TACO_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(dZ) failed: %d (N=%d T=%d B=%d lddz=%lld)", (int)r, N, T, B, (long long)lddz);
    }
    static bool configured = false;
    if (!configured) {
        TACO_CUDA(cudaFuncSetAttribute(dw_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DW_SMEM));
        configured = true;
    }
    dw_tc_kernel<<<dim3((unsigned)tiles, (unsigned)splits), DW_THREADS, DW_SMEM, st>>>(tmX, tmZ, a);
    TACO_LAUNCH_CHECK();
    return 0;
}

// The dispatch decision of taco_linear_tc, host only (no CUDA call): every check of a tensor-core descriptor that needs no
// device, then which kernel instantiation and which epilogue the launch uses.
int taco_linear_tc_route(const taco_linear_desc* d, TcRoute* r) {
    TACO_CHECK(d->Wp != nullptr, "taco_linear_fwd(TC): Wp (packed weights) is NULL");
    TACO_CHECK(taco_aligned16(d->X) && taco_aligned16(d->Wp), "taco_linear_fwd(TC): X / Wp must be 16-byte aligned");
    TACO_CHECK((d->ldx % 4) == 0 && (d->ldwp % 4) == 0, "taco_linear_fwd(TC): ldx and ldwp must be multiples of 4 floats (TMA 16B strides)");
    const bool highway = d->epilogue == TACO_EPI_HIGHWAY;
    if (highway) TACO_CHECK(d->N == 256 && d->taps == 1 && d->bank_K == 0 && d->hx, "highway (TC): needs N == 256 (U = 128), dense, hx");
    if (d->bank_K > 0) TACO_CHECK(d->bank_cout == 128 && d->N == d->bank_K * 128, "bank (TC): bank_cout must be 128");
    if (d->pool) TACO_CHECK(!highway && !d->residual && !d->keep, "pool cannot be combined with highway / residual / dropout");
    const int Cpad = (d->C + 31) / 32 * 32;
    const int max_taps = d->bank_K > 0 ? d->bank_K : d->taps;
    TACO_CHECK(d->ldwp >= (int64_t)max_taps * Cpad, "taco_linear_fwd(TC): ldwp too small for taps*Cpad");

    const bool x3 = d->impl == TACO_IMPL_TC3;
    r->mode = highway ? 1 : 0;
    r->bn = highway ? 256 : 128;
    // few output tiles (encoder-side contractions: 32 utterances x 128 characters = 32 m-tiles): 32-column n-tiles put
    // four times as many CTAs on the machine, each with a 6-deep ring (with 128-column tiles the long-K conv projection
    // 2048x3 -> 128 would run on 32 of the 132 SMs)
    {
        const int64_t mt = (int64_t)((d->T + TC_BM - 1) / TC_BM) * d->B;
        if (x3 && !highway && d->bank_K == 0 && !d->pool && mt * ((d->N + 127) / 128) <= TACO_SMS / 4 && d->N >= 64) r->bn = 32;
    }
    if (x3) r->stages = r->bn == 32 ? 6 : 2;
    // tf32: short K loops (<= 8 k-iterations: dense 128/256-wide inputs) are epilogue/latency bound: a 2-stage ring suffices
    else r->stages = (highway || (d->bank_K == 0 && d->taps * (Cpad / 32) <= 8)) ? 2 : 3;
    // register-direct epilogue: needs 16-byte aligned row segments everywhere it touches
    {
        const int nout = highway ? d->N / 2 : d->N;
        bool ok = (d->ldy % 4) == 0 && (nout % 4) == 0 && taco_aligned16(d->Y);
        if (d->residual) ok = ok && (d->ldr % 4) == 0 && taco_aligned16(d->residual);
        if (d->hx) ok = ok && (d->ldhx % 4) == 0 && taco_aligned16(d->hx);
        if (d->keep) ok = ok && (nout % 16) == 0 && taco_aligned16(d->keep);
        r->direct = ok ? 1 : 0;
    }
    r->tile_stride = d->pool ? (TC_BM - 1) : TC_BM;
    return 0;
}

int taco_linear_tc(const taco_linear_desc* d, cudaStream_t st) {
    TcRoute r;
    if (int rc = taco_linear_tc_route(d, &r)) return rc;
    EncodeTiledFn enc = get_encode_fn();
    TACO_CHECK(enc != nullptr, "cuTensorMapEncodeTiled driver entry point not available");
    const int64_t M = (int64_t)d->B * d->T;
    if (M == 0 || d->N == 0) return 0;

    const bool highway = r.mode == 1;
    const int BN = r.bn;
    TcArgs a;
    a.B = d->B; a.T = d->T;
    a.Cpad = (d->C + 31) / 32 * 32;
    a.cchunks = a.Cpad / 32;
    a.taps = d->taps; a.tap0 = d->tap0; a.bank = d->bank_K > 0 ? 1 : 0;
    a.N = d->N;
    a.pool = d->pool ? 1 : 0;
    const bool x3 = d->impl == TACO_IMPL_TC3;
    a.direct = r.direct;
    a.lo_row0 = d->N;                                    // packed buffer = [hi rows 0..N) | lo rows N..2N)
    a.tile_stride = r.tile_stride;
    a.tiles_per_seq = a.pool ? ((d->T - 1 + a.tile_stride - 1) / a.tile_stride) : ((d->T + TC_BM - 1) / TC_BM);
    if (a.tiles_per_seq < 1) a.tiles_per_seq = 1;
    a.e.Y = d->Y; a.e.ldy = d->ldy; a.e.bias = d->bias; a.e.scale = d->scale; a.e.shift = d->shift;
    a.e.keep = d->keep; a.e.keep_scale = d->keep_scale; a.e.residual = d->residual; a.e.ldr = d->ldr;
    a.e.hx = d->hx; a.e.ldhx = d->ldhx; a.e.act = d->act; a.e.N = highway ? d->N / 2 : d->N;
    a.e.bias_utt = d->bias_utt; a.e.ldbu = d->ldbu; a.e.T = d->T;

    CUtensorMap tmA, tmB;
    {
        cuuint64_t dims[3] = {(cuuint64_t)d->C, (cuuint64_t)d->T, (cuuint64_t)d->B};
        cuuint64_t strides[2] = {(cuuint64_t)d->ldx * 4, (cuuint64_t)d->T * (cuuint64_t)d->ldx * 4};
        cuuint32_t box[3] = {TC_BK, TC_BM, 1};
        cuuint32_t es[3] = {1, 1, 1};
        CUresult r = enc(&tmA, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(d->X), dims, strides, box, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        TACO_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(A) failed: %d (C=%d T=%d B=%d ldx=%lld)", (int)r, d->C, d->T, d->B, (long long)d->ldx);
    }
    {
        cuuint64_t dims[2] = {(cuuint64_t)d->ldwp, (cuuint64_t)d->N * (x3 ? 2u : 1u)};
        cuuint64_t strides[1] = {(cuuint64_t)d->ldwp * 4};
        cuuint32_t box[2] = {TC_BK, (cuuint32_t)BN};
        cuuint32_t es[2] = {1, 1};
        CUresult r = enc(&tmB, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(d->Wp), dims, strides, box, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        TACO_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(B) failed: %d (N=%d ldwp=%lld)", (int)r, d->N, (long long)d->ldwp);
    }
    dim3 grid((d->N + BN - 1) / BN, (unsigned)(a.tiles_per_seq * d->B));
    if (x3) {
        if (highway) return launch_tc<256, 2, 1, true>(tmA, tmB, a, grid, st);
        if (BN == 32) return launch_tc<32, 6, 0, true>(tmA, tmB, a, grid, st);
        // 2 stages x 48 KB per CTA: two CTAs per SM (4 loads in flight per SM, the epilogue of one under the main loop of
        // the other)
        return launch_tc<128, 2, 0, true>(tmA, tmB, a, grid, st);
    }
    if (highway) return launch_tc<256, 2, 1>(tmA, tmB, a, grid, st);
    if (r.stages == 2) return launch_tc<128, 2, 0>(tmA, tmB, a, grid, st);
    return launch_tc<128, 3, 0>(tmA, tmB, a, grid, st);
}

// the checks of a descriptor that need no device
static int taco_highway_stack_check(const taco_highway_stack_desc* d) {
    TACO_CHECK(d != nullptr, "taco_highway_stack_fwd: NULL descriptor");
    TACO_CHECK(d->impl == TACO_IMPL_TC3, "taco_highway_stack_fwd: only TACO_IMPL_TC3 (fp32x3) is implemented (impl %d)", d->impl);
    TACO_CHECK(d->M >= 0 && d->C >= 1 && d->C <= 128, "taco_highway_stack_fwd: bad sizes M=%d C=%d (1 <= C <= 128)", d->M, d->C);
    TACO_CHECK(d->L >= 1 && d->L <= TACO_HIGHWAY_STACK_MAX, "taco_highway_stack_fwd: L=%d highway layers (1..%d)", d->L,
               TACO_HIGHWAY_STACK_MAX);
    TACO_CHECK(d->X && d->Y && d->xp_p && d->xp_b, "taco_highway_stack_fwd: X, Y, xp_p or xp_b is NULL");
    TACO_CHECK((d->C == 128) == (d->Wd_p == nullptr), "taco_highway_stack_fwd: the width-fixing dense (Wd_p, bd) is used iff C != 128");
    TACO_CHECK(d->C == 128 || d->bd, "taco_highway_stack_fwd: bd is NULL");
    for (int l = 0; l < d->L; ++l)
        TACO_CHECK(d->hw_p[l] && d->hw_b[l] && taco_aligned16(d->hw_p[l]), "taco_highway_stack_fwd: highway layer %d: NULL or unaligned", l);
    TACO_CHECK(taco_aligned16(d->X) && taco_aligned16(d->xp_p) && taco_aligned16(d->Y) && (!d->Wd_p || taco_aligned16(d->Wd_p)),
               "taco_highway_stack_fwd: X, Y and the packed weights must be 16-byte aligned");
    const int Cpad = (d->C + 31) / 32 * 32;
    TACO_CHECK(d->ldx >= d->C && (d->ldx % 4) == 0, "taco_highway_stack_fwd: ldx %lld (>= C, multiple of 4)", (long long)d->ldx);
    TACO_CHECK(d->ldy >= HS_XP_N && (d->ldy % 4) == 0, "taco_highway_stack_fwd: ldy %lld (>= 768, multiple of 4)", (long long)d->ldy);
    TACO_CHECK(d->ldhw >= 128 && (d->ldhw % 4) == 0 && d->ldxp >= 128 && (d->ldxp % 4) == 0,
               "taco_highway_stack_fwd: ldhw / ldxp must be >= 128 and multiples of 4");
    TACO_CHECK(!d->Wd_p || (d->ldwd >= Cpad && (d->ldwd % 4) == 0), "taco_highway_stack_fwd: ldwd %lld (>= round_up(C,32), multiple of 4)",
               (long long)d->ldwd);
    return 0;
}

// xp column splits per tile: the most (of 1, 2, 3, 6) that keep every CTA on its own SM
static int taco_highway_stack_split(int M) {
    const int tiles = (M + HS_BM - 1) / HS_BM;
    for (int s : {6, 3, 2})
        if (tiles * s <= TACO_SMS) return s;
    return 1;
}

int taco_highway_stack(const taco_highway_stack_desc* d, cudaStream_t st) {
    if (int rc = taco_highway_stack_check(d)) return rc;
    if (d->M == 0) return 0;
    EncodeTiledFn enc = get_encode_fn();
    TACO_CHECK(enc != nullptr, "cuTensorMapEncodeTiled driver entry point not available");
    const bool dense = d->C != 128;
    const int split = taco_highway_stack_split(d->M);
    HsMaps maps;
    HsArgs a;
    a.M = d->M;
    a.dense = dense ? 1 : 0;
    a.nlayers = a.dense + d->L + 1;
    a.kin = (d->C + 31) / 32;
    a.xp_chunks = HS_XP_N / 128 / split;
    if (int rc = encode_2d(enc, &maps.x, d->X, d->C, d->M, d->ldx, "X")) return rc;
    int l = 0;
    if (dense) {
        if (int rc = encode_2d(enc, &maps.w[l], d->Wd_p, d->ldwd, 2 * 128, d->ldwd, "Wd")) return rc;
        a.lo_row0[l] = 128; a.bias[l] = d->bd; ++l;
    }
    for (int h = 0; h < d->L; ++h, ++l) {
        if (int rc = encode_2d(enc, &maps.w[l], d->hw_p[h], d->ldhw, 2 * 256, d->ldhw, "highway")) return rc;
        a.lo_row0[l] = 256; a.bias[l] = d->hw_b[h];
    }
    if (int rc = encode_2d(enc, &maps.w[l], d->xp_p, d->ldxp, 2 * HS_XP_N, d->ldxp, "xp")) return rc;
    a.lo_row0[l] = HS_XP_N; a.bias[l] = d->xp_b;
    a.total_items = (dense ? a.kin : 0) + d->L * 2 * 4 + a.xp_chunks * 4;    // (without the dense, kin = 4)
    a.Y = d->Y; a.ldy = d->ldy;
    static bool configured = false;
    if (!configured) {
        TACO_CUDA(cudaFuncSetAttribute(highway_stack_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, HS_SMEM));
        configured = true;
    }
    dim3 grid((unsigned)((d->M + HS_BM - 1) / HS_BM), (unsigned)split);
    highway_stack_kernel<<<grid, HS_THREADS, HS_SMEM, st>>>(maps, a);
    TACO_LAUNCH_CHECK();
    return 0;
}
