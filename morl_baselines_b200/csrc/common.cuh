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
// Every kernel of the captured Envelope update starts with pdl_enter().  A kernel launched with the PDL attribute may become resident
// while its predecessor in the stream is still draining (the launch latency and the block scheduling of kernel n+1 overlap the tail of
// kernel n; in a CUDA graph the edge is captured as a programmatic dependency), and `griddepcontrol.wait` then blocks until the
// predecessor has COMPLETED and its writes are visible.  Rules that keep this equivalent to plain stream order:
//   * pdl_enter() is the first statement of the kernel, executed by every thread, before any global-memory access;
//   * a kernel launched with the attribute always executes the wait (the chain kernel n-1 -> n -> n+1 stays transitively ordered).
// Without the launch attribute both instructions are no-ops.  The tensor-core GEMM, chain and fused-head (qhead_envelope) launches set it
// (launch_k_pdl(true, ...)), where the prologue that overlaps (barrier initialisation, tensor-map prefetch) is long.  Every other kernel
// is launched in plain stream order (launch_k): with the attribute on every kernel of the update, the update measured 4.5 % slower than
// plain stream order (the early-resident CTAs of the small kernels take issue slots and shared memory from the draining grid).
__device__ __forceinline__ void pdl_enter() {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
}

// Launch with the PDL attribute iff `pdl`.
template <typename... KArgs, typename... Args>
static inline void launch_k_pdl(bool pdl, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
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
    cfg.numAttrs = pdl ? 1 : 0;
    cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

template <typename... KArgs, typename... Args>
static inline void launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
    launch_k_pdl(false, kernel, grid, block, smem, stream, static_cast<Args&&>(args)...);
}

// Raises the dynamic-shared-memory limit of kernel K to `bytes` once per process (the first call of each instantiation).
template <auto K>
static inline void set_smem_limit_once(size_t bytes) {
    static const bool done = (cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes), true);
    (void)done;
}

// SMs of the current device, 132 (H100 SXM) when it cannot be queried
static inline int sm_count() {
    const int n = morl_device_sm_count();
    return n > 0 ? n : 132;
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

// ---- warp and block reductions (butterfly trees: every lane gets the same value) ------------------------------------------------
__device__ __forceinline__ float warp_sum_f32(float v) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    return v;
}

__device__ __forceinline__ float warp_max_f32(float v) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, off));
    return v;
}

// Sum of one double per thread of a kThreads-thread block in a fixed order: the warp tree, then the warp sums in warp order.  `red`
// holds kThreads / 32 doubles of shared memory; the first barrier frees it from a previous call.  Every thread gets the same value.
template <int kThreads>
__device__ __forceinline__ double block_sum_f64(double v, double* red) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
#pragma unroll
    for (int i = 0; i < kThreads / 32; ++i) t += red[i];
    return t;
}

__device__ __forceinline__ float sigmoid_f32(float z) { return 1.0f / (1.0f + expf(-z)); }

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
