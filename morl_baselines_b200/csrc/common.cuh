// common.cuh -- shared device helpers + argument checking for libmorl_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/morl_b200.h"

namespace morl {

// ---- error plumbing (thread-local message, see morl_last_error) --------------------------------
void set_error(const char* fmt, ...);
int check_launch(const char* what);

#define MORL_REQUIRE(cond, code, ...)    \
    do {                                 \
        if (!(cond)) {                   \
            ::morl::set_error(__VA_ARGS__); \
            return (code);               \
        }                                \
    } while (0)

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// ---- programmatic dependent launch (PDL) -----------------------------------------------------------
// Every kernel of the captured Envelope update is launched through launch_k() and starts with pdl_enter(): the grid may become resident
// while its predecessor in the stream is still draining (the launch latency and the block scheduling of kernel n+1 overlap the tail of
// kernel n; in a CUDA graph the edge is captured as a programmatic dependency), and `griddepcontrol.wait` then blocks until the
// predecessor has COMPLETED and its writes are visible.  Rules that keep this equivalent to plain stream order:
//   * pdl_enter() is the first statement of the kernel, executed by every thread, before any global-memory access;
//   * a kernel launched with the attribute always executes the wait (the chain kernel n-1 -> n -> n+1 stays transitively ordered).
// Without the launch attribute both instructions are no-ops.  The attribute is OPT-IN (MORL_PDL=1): on every kernel of the update it
// measured 4.5 % slower than plain stream order (api.cu: pdl_enabled); the GEMM chain has its own switch (MORL_GEMM_PDL, default on).
__device__ __forceinline__ void pdl_enter() {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
}

bool pdl_enabled();  // api.cu

template <typename... KArgs, typename... Args>
static inline void launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// ---- scalarisation w . q in the three documented arithmetics (include/morl_b200.h) --------------
// All intrinsics are the _rn forms so nvcc can never contract or reorder them.
template <int D, int MODE>
__device__ __forceinline__ float dotw(const float (&w)[D], const float (&q)[D]) {
    if constexpr (MODE == MORL_DOT_UNFUSED) {
        float acc = __fmul_rn(w[0], q[0]);
#pragma unroll
        for (int r = 1; r < D; ++r) acc = __fadd_rn(acc, __fmul_rn(w[r], q[r]));
        return acc;
    } else if constexpr (MODE == MORL_DOT_FMA) {
        float acc = __fmul_rn(w[0], q[0]);
#pragma unroll
        for (int r = 1; r < D; ++r) acc = __fmaf_rn(w[r], q[r], acc);
        return acc;
    } else {  // MORL_DOT_PAIRFMA: pairs (fma(w1,q1,w0*q0)) summed left to right, odd tail product added last
        float acc = 0.f;
#pragma unroll
        for (int r = 0; r + 1 < D; r += 2) {
            float p = __fmaf_rn(w[r + 1], q[r + 1], __fmul_rn(w[r], q[r]));
            acc = (r == 0) ? p : __fadd_rn(acc, p);
        }
        if constexpr (D % 2 == 1) {
            float t = __fmul_rn(w[D - 1], q[D - 1]);
            acc = (D == 1) ? t : __fadd_rn(acc, t);
        }
        return acc;
    }
}

// vector Bellman line, unfused exactly like the reference's elementwise ops (envelope.py:298):
//   r + ((1 - done) * gamma) * q
__device__ __forceinline__ float bellman(float r, float done, float gamma, float q) {
    float nd = __fmul_rn(__fsub_rn(1.0f, done), gamma);
    return __fadd_rn(r, __fmul_rn(nd, q));
}

__device__ __forceinline__ int map_row(int k, int rows, int n, int map) {
    if (rows == n) return k;
    if (rows == 1) return 0;
    return map == MORL_MAP_TILE ? (k % rows) : (k / (n / rows));
}

// ---- ReLU bit masks (include/morl_b200.h "ReLU bit masks"): the one place that knows the layout ---------------------------------
// A row of an activation `width` columns wide is 8 uint32 words (width <= 256) or 16 (width <= 512).  Column c lies in chunk k = c / 32;
// within each 256-column half the word order is (k & 1) * 4 + ((k >> 1) & 3), so the four chunks one epilogue thread owns are one
// 16-byte load; the second half's words follow the first's.
__host__ __device__ __forceinline__ int relu_bits_words(int width) { return width > 256 ? 16 : 8; }
__host__ __device__ __forceinline__ int relu_bits_word(int col) {
    const int k = col >> 5;
    return 8 * (k >> 3) + (k & 1) * 4 + ((k >> 1) & 3);
}

// (value desc, index asc) total order used when partial argmaxes are merged: keeps first occurrence.
__device__ __forceinline__ void argmax_merge(float& v, int& i, float v2, int i2) {
    if (v2 > v || (v2 == v && i2 < i)) {
        v = v2;
        i = i2;
    }
}

__device__ __forceinline__ void warp_argmax(float& v, int& i) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        float v2 = __shfl_xor_sync(0xffffffffu, v, off);
        int i2 = __shfl_xor_sync(0xffffffffu, i, off);
        argmax_merge(v, i, v2, i2);
    }
}

}  // namespace morl

// Dispatch helpers: D in 1..8, dot mode in 0..2.
#define MORL_DISPATCH_D(D_, ...)                                         \
    switch (D_) {                                                        \
        case 1: { constexpr int kD = 1; __VA_ARGS__; } break;            \
        case 2: { constexpr int kD = 2; __VA_ARGS__; } break;            \
        case 3: { constexpr int kD = 3; __VA_ARGS__; } break;            \
        case 4: { constexpr int kD = 4; __VA_ARGS__; } break;            \
        case 5: { constexpr int kD = 5; __VA_ARGS__; } break;            \
        case 6: { constexpr int kD = 6; __VA_ARGS__; } break;            \
        case 7: { constexpr int kD = 7; __VA_ARGS__; } break;            \
        case 8: { constexpr int kD = 8; __VA_ARGS__; } break;            \
        default: break;                                                  \
    }

#define MORL_DISPATCH_MODE(M_, ...)                                                  \
    switch (M_) {                                                                    \
        case MORL_DOT_UNFUSED: { constexpr int kMode = MORL_DOT_UNFUSED; __VA_ARGS__; } break; \
        case MORL_DOT_FMA: { constexpr int kMode = MORL_DOT_FMA; __VA_ARGS__; } break;         \
        case MORL_DOT_PAIRFMA: { constexpr int kMode = MORL_DOT_PAIRFMA; __VA_ARGS__; } break; \
        default: break;                                                              \
    }
