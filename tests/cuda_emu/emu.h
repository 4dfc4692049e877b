// emu.h -- TEST INFRASTRUCTURE ONLY.  A functional host emulation of the CUDA execution model, just large enough to run
// this repository's kernels (the SAME .cu sources, compiled with g++) thread by thread on a CPU.  Purpose: check the
// index algebra of a new kernel -- the thing a kernel written without GPU access gets wrong -- before it ever sees
// hardware.  It says nothing about performance, memory ordering or the real instruction semantics beyond their
// arithmetic definition.
//
// Model: one launch = blocks run one after the other; the threads of a block are real OS threads, so __syncthreads()
// (std::barrier), __shared__ (static storage, valid because blocks are sequential), shuffles and the warp-collective
// mma (per-warp exchange buffers + a per-warp barrier) behave as on the device.  Kernels without block-level
// synchronisation could run sequentially, but one code path keeps the emulation simple.
#pragma once
#define TACO_HOST_EMU 1
#include <cuda_runtime.h>          // vector types, dim3 (host-compatible headers of the toolkit)
#include <atomic>
#include <barrier>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <memory>
#include <thread>
#include <vector>

#ifndef __launch_bounds__
#define __launch_bounds__(...)
#endif
#undef __shared__
#define __shared__ static            // blocks are emulated sequentially, so block-shared storage can be static

namespace emu {
struct Ctx {
    std::barrier<>* block_bar = nullptr;
    std::barrier<>* warp_bar = nullptr;       // barrier of this thread's warp
    float* warp_xf = nullptr;                 // per-warp exchange buffer, 32 x 8 words
    int lane = 0;
};
inline thread_local Ctx ctx;
}  // namespace emu

inline thread_local uint3 threadIdx, blockIdx;
inline dim3 blockDim, gridDim;

inline void __syncthreads() { emu::ctx.block_bar->arrive_and_wait(); }
inline void __syncwarp(unsigned = 0xffffffffu) { emu::ctx.warp_bar->arrive_and_wait(); }

template <class T> inline T __ldg(const T* p) { return *p; }
template <class T> inline T __ldcg(const T* p) { return *p; }
template <class T> inline T __ldcs(const T* p) { return *p; }
inline float __expf(float x) { return expf(x); }
inline float __fdividef(float a, float b) { return a / b; }
inline float __fdiv_rn(float a, float b) { return a / b; }
// sin(pi x) and cos(pi x) as the device computes them: exact at multiples of 1/2 (sinpi(1) = 0, cospi(1/2) = 0, where
// sin(M_PI) in double is 1.2e-16), otherwise the double value rounded once.  The argument is reduced exactly mod 2 first.
inline void emu_sincospi(double x, double* s, double* c) {
    const double r = std::fmod(x, 2.0);                                  // exact, in (-2, 2), sign of x
    const double a = std::fabs(r);
    if (a == 0.0 || a == 1.0) { *s = std::copysign(0.0, r); *c = a == 0.0 ? 1.0 : -1.0; return; }
    if (a == 0.5 || a == 1.5) { *s = (a == 0.5) == (r > 0) ? 1.0 : -1.0; *c = 0.0; return; }
    *s = std::sin(M_PI * r);
    *c = std::cos(M_PI * r);
}
inline float cospif(float x) { double s, c; emu_sincospi(x, &s, &c); return (float)c; }
inline void sincospif(float x, float* s, float* c) { double sd, cd; emu_sincospi(x, &sd, &cd); *s = (float)sd; *c = (float)cd; }
inline uint32_t __float_as_uint(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
inline float __uint_as_float(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
inline int min(int a, int b) { return a < b ? a : b; }
inline int max(int a, int b) { return a > b ? a : b; }
inline float atomicAdd(float* p, float v) { return std::atomic_ref<float>(*p).fetch_add(v, std::memory_order_relaxed); }

// warp shuffle: every lane publishes its value, then reads the partner's
inline float __shfl_xor_sync(unsigned, float v, int lane_mask) {
    auto& c = emu::ctx;
    c.warp_xf[c.lane] = v;
    c.warp_bar->arrive_and_wait();
    const float r = c.warp_xf[c.lane ^ lane_mask];
    c.warp_bar->arrive_and_wait();
    return r;
}
inline double __shfl_xor_sync(unsigned, double v, int lane_mask) {      // two exchange words per lane
    auto& c = emu::ctx;
    memcpy(c.warp_xf + 2 * c.lane, &v, sizeof v);
    c.warp_bar->arrive_and_wait();
    double r;
    memcpy(&r, c.warp_xf + 2 * (c.lane ^ lane_mask), sizeof r);
    c.warp_bar->arrive_and_wait();
    return r;
}

// mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 by its PTX definition:
//   A (16x8, row): a0 (g, tg) a1 (g+8, tg) a2 (g, tg+4) a3 (g+8, tg+4);  B (8x8, col): b0 (k=tg, n=g) b1 (k=tg+4, n=g)
//   C/D (16x8): c0 (g, 2tg) c1 (g, 2tg+1) c2 (g+8, 2tg) c3 (g+8, 2tg+1);   g = lane>>2, tg = lane&3
// Operands are read as TF32: the low 13 mantissa bits are ignored.
inline void emu_mma_m16n8k8_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    auto& c = emu::ctx;
    auto tf32 = [](uint32_t u) { return __uint_as_float(u & 0xffffe000u); };
    float* mine = c.warp_xf + c.lane * 8;
    for (int i = 0; i < 4; ++i) mine[i] = tf32(a[i]);
    mine[4] = tf32(b0); mine[5] = tf32(b1);
    c.warp_bar->arrive_and_wait();
    const int g = c.lane >> 2, tg = c.lane & 3;
    auto A = [&](int row, int k) {            // element (row, k) of the 16x8 A tile
        const int l = (row & 7) * 4 + (k & 3);
        return c.warp_xf[l * 8 + (row >> 3) + 2 * (k >> 2)];
    };
    auto Bm = [&](int k, int n) {             // element (k, n) of the 8x8 B tile
        const int l = n * 4 + (k & 3);
        return c.warp_xf[l * 8 + 4 + (k >> 2)];
    };
    float out[4];
    for (int e = 0; e < 4; ++e) {
        const int row = g + ((e >> 1) ? 8 : 0), col = 2 * tg + (e & 1);
        double s = 0.0;
        for (int k = 0; k < 8; ++k) s += (double)A(row, k) * (double)Bm(k, col);
        out[e] = d[e] + (float)s;
    }
    c.warp_bar->arrive_and_wait();
    for (int e = 0; e < 4; ++e) d[e] = out[e];
}

namespace emu {
// run `body` for every thread of every block of the grid
template <class F>
inline void launch(dim3 grid, dim3 block, F body) {
    gridDim = grid; blockDim = block;
    const int nthreads = (int)(block.x * block.y * block.z);
    const int nwarps = (nthreads + 31) / 32;
    for (unsigned bz = 0; bz < grid.z; ++bz)
        for (unsigned by = 0; by < grid.y; ++by)
            for (unsigned bx = 0; bx < grid.x; ++bx) {
                std::barrier<> bb(nthreads);
                std::vector<std::unique_ptr<std::barrier<>>> wb;
                std::vector<std::vector<float>> xf(nwarps, std::vector<float>(32 * 8, 0.f));
                for (int w = 0; w < nwarps; ++w) {
                    const int in_warp = std::min(32, nthreads - 32 * w);
                    wb.emplace_back(new std::barrier<>(in_warp));
                }
                std::vector<std::thread> th;
                th.reserve(nthreads);
                for (int t = 0; t < nthreads; ++t) {
                    th.emplace_back([&, t, bx, by, bz] {
                        threadIdx = uint3{(unsigned)(t % block.x), (unsigned)((t / block.x) % block.y), (unsigned)(t / (block.x * block.y))};
                        blockIdx = uint3{bx, by, bz};
                        ctx.block_bar = &bb;
                        ctx.warp_bar = wb[t / 32].get();
                        ctx.warp_xf = xf[t / 32].data();
                        ctx.lane = t % 32;
                        body();
                    });
                }
                for (auto& x : th) x.join();
            }
}
inline dim3 as_dim3(dim3 d) { return d; }
inline dim3 as_dim3(int x) { return dim3((unsigned)x); }
}  // namespace emu

namespace emu {
// dynamic shared memory of the (single) running block; large enough for every kernel of this repository
inline float* dynamic_smem() { static float buf[64 * 1024]; return buf; }
}  // namespace emu

// cooperative groups for a ONE-block grid (kernels written for any grid size are emulated with gridDim = 1):
// grid.sync() is then a block barrier
namespace cg {
struct grid_group { void sync() const { __syncthreads(); } };
inline grid_group this_grid() { return grid_group(); }
}  // namespace cg

#define TACO_LAUNCH(kernel, grid, block, smem, stream, ...) \
    emu::launch(emu::as_dim3(grid), emu::as_dim3(block), [&] { kernel(__VA_ARGS__); })
