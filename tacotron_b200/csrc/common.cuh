// common.cuh -- shared helpers for libtaco_b200 (sm_90a only).
//
// TACO_HOST_EMU: the functional host emulation used by tests/cuda_emu/ (the SAME kernel sources compiled with g++ and
// run thread by thread on the CPU, so that indexing of a new kernel can be checked without a GPU).  It only removes
// what cannot exist on a host (inline PTX, the CUDA runtime error plumbing) -- nothing below changes under nvcc.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include "../../include/taco_b200.h"

// ---------------------------------------------------------------------------------------------
// error plumbing: nothing throws across the C-ABI; message is thread-local
// ---------------------------------------------------------------------------------------------
void taco_set_error(const char* fmt, ...);

#define TACO_CHECK(cond, ...)                                    \
    do {                                                         \
        if (!(cond)) {                                           \
            taco_set_error(__VA_ARGS__);                         \
            return 1;                                            \
        }                                                        \
    } while (0)

#define TACO_CUDA(expr)                                                                     \
    do {                                                                                    \
        cudaError_t _e = (expr);                                                            \
        if (_e != cudaSuccess) {                                                            \
            taco_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return 2;                                                                       \
        }                                                                                   \
    } while (0)

extern unsigned long long g_taco_launches;   // kernels launched by this library (bench.py reports it)

// kernel launch: <<<>>> under nvcc; the emulation header pre-defines TACO_LAUNCH to run the grid on host threads
#ifndef TACO_LAUNCH
#define TACO_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#endif

#ifdef TACO_HOST_EMU
#define TACO_LAUNCH_CHECK() do { ++g_taco_launches; } while (0)
#else
#define TACO_LAUNCH_CHECK()                                                                 \
    do {                                                                                    \
        ++g_taco_launches;                                                                  \
        cudaError_t _e = cudaGetLastError();                                                \
        if (_e != cudaSuccess) {                                                            \
            taco_set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
            return 3;                                                                       \
        }                                                                                   \
    } while (0)
#endif

static inline bool taco_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// launch route of a tensor-core taco_linear_fwd (gemm_tc.cu taco_linear_tc_route; reported by taco_linear_route)
struct TcRoute {
    int bn;            // n-tile width: 32, 128 or 256 (highway)
    int stages;        // k-block ring depth
    int mode;          // 0 normal epilogue, 1 highway
    int direct;        // 1 register-direct epilogue, 0 transposing epilogue
    int tile_stride;   // rows between consecutive m-tiles of an utterance: 128, or 127 with the fused max-pool
};

// SMs of the H100 SXM: sizes grid-stride launches and the split-K of the weight-gradient kernel
constexpr int TACO_SMS = 132;

// ---------------------------------------------------------------------------------------------
// device math
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float sigmoidf_acc(float x) {
    // 1/(1+exp(-x)) with the fast exp2 path (rel. err ~1e-7 after the division; abs err <= 2.5e-7 for any finite x:
    // __expf's error grows with |x| only where sigmoid'(x) is small, and __fdividef adds 2 ulp)
    return __fdividef(1.0f, 1.0f + __expf(-x));
}
__device__ __forceinline__ float tanhf_acc(float x) {
    // tanh(x) = 1 - 2/(exp(2x)+1); exact limits at +-inf, abs err ~2e-7 (<= 5e-7: 2 ulp of the quotient in [1, 2) for
    // x < 0, plus __expf's error)
    float e = __expf(2.0f * x);
    return 1.0f - __fdividef(2.0f, e + 1.0f);
}
// periodic hann window of win_length samples centred in the n_fft-sample frame (lpad = (n_fft - win_length)/2), as
// librosa's stft / istft build it; j in [0, n_fft), 0 outside the support
__device__ __forceinline__ float hann_at(int j, int lpad, int win_length) {
    const int i = j - lpad;
    if (i < 0 || i >= win_length) return 0.f;
    return 0.5f - 0.5f * cospif(2.0f * (float)i / (float)win_length);
}
__device__ __forceinline__ float apply_act(float v, int act) {
    switch (act) {
        case TACO_ACT_RELU:    return fmaxf(v, 0.0f);
        case TACO_ACT_SIGMOID: return sigmoidf_acc(v);
        case TACO_ACT_TANH:    return tanhf_acc(v);
        default:               return v;
    }
}

#ifndef TACO_HOST_EMU
// ---------------------------------------------------------------------------------------------
// PTX wrappers (mbarrier / TMA / wgmma / grid sync primitives)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a wedged pipeline traps (context error, reported to the host) instead of
// hanging the GPU.  ~2^28 polls of a HW-sleeping try_wait is many seconds.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > (1u << 28)) { __trap(); }
    }
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// TMA: 3D tiled load global -> shared, completion on an mbarrier
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
// plain bulk copy global -> shared (contiguous bytes, multiple of 16)
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

// wgmma (Hopper warpgroup MMA): 128 threads (four consecutive warps, the first a multiple of 4) issue one m64nNk8 TF32
// product together.  Operands: A from a shared-memory descriptor or from registers, B from a shared-memory descriptor;
// the fp32 accumulator fragment lives in registers (row 16*warp + lane/4 (+8), column 8*j + 2*(lane%4) (+1)).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// Shared-memory matrix descriptor of a K-major, 128-byte-swizzled tile (what TMA writes with CU_TENSOR_MAP_SWIZZLE_128B):
// rows of 128 bytes (32 tf32), 8-row groups 1024 bytes apart (stride byte offset), leading byte offset unused.  The tile
// must be 1024-byte aligned; the next 8 K elements (32 bytes) inside the swizzle row are at descriptor + 2.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFF) >> 4);          // start address
    d |= (uint64_t)1 << 16;                           // leading byte offset (ignored for swizzled K-major)
    d |= (uint64_t)(1024 >> 4) << 32;                 // stride byte offset
    d |= (uint64_t)1 << 62;                           // SWIZZLE_128B
    return d;
}
__device__ __forceinline__ void wgmma_m64n32k8_ss(float (&d)[16], uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc)
        : "memory");
}
__device__ __forceinline__ void wgmma_m64n32k8_rs(float (&d)[16], const uint32_t (&a)[4], uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "{%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc)
        : "memory");
}
__device__ __forceinline__ void wgmma_m64n128k8_ss(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc)
        : "memory");
}
__device__ __forceinline__ void wgmma_m64n128k8_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc)
        : "memory");
}


// acquire / release at gpu scope for the software grid barrier and flags
__device__ __forceinline__ void red_release_add(unsigned int* p, unsigned int v) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
#endif  // !TACO_HOST_EMU
