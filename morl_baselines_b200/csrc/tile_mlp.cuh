// tile_mlp.cuh -- the row-tile MLP layers of the CUDA-core policy kernels (eupg.cu, nl_ppo.cu, pcn.cu).
//
// A tile is kTileRows rows of a batch; one CTA of kTileThreads threads holds every activation of the tile in shared memory, row-major
// [kTileRows, width], and reads the weights through the read-only cache.  A layer's gradient is folded into a per-CTA partial laid out as
// the parameter tensors back to back (ParamLayout); partial_sum_kernel then sums the partials in CTA order into the .grad storages.  No
// float atomics: every sum has a fixed order, so results depend on neither the SM count nor the run.
#pragma once
#include "common.cuh"

namespace morl {

constexpr int kTileRows = 16;
constexpr int kTileThreads = 256;
constexpr int kTileWarps = kTileThreads / 32;

enum class Act { None, Tanh, Relu, Sigmoid };

template <int kMax>
struct ParamTable {
    const float* p[kMax];
};
template <int kMax>
struct GradTable {
    float* g[kMax];
};

// The first n entries of size[] are the element counts of the parameter tensors, in table order; a gradient partial holds them back to back.
template <int kMax>
struct ParamLayout {
    int n;
    int size[kMax];
    __host__ __device__ int offset(int t) const {
        int o = 0;
        for (int i = 0; i < t; ++i) o += size[i];
        return o;
    }
    __host__ __device__ int total() const { return offset(n); }
};

// Row groups of a layer with n outputs: the largest power of two <= kTileThreads / n, at most kTileRows, so that job (j, g) of the n * groups
// jobs owns rows g, g + groups, ... (rpj = kTileRows / groups of them) and every job runs in one pass of the block.
__device__ __forceinline__ int tile_groups(int n) {
    int g = kTileThreads / n;
    g = g > kTileRows ? kTileRows : g;
    return 1 << (31 - __clz(g));
}

// The rows of a job, unrolled to kTileRows so that the per-row accumulators stay in registers.
#define MORL_TILE_ROWS(i) _Pragma("unroll") for (int i = 0; i < kTileRows; ++i) if (i < rpj)

__device__ __forceinline__ float tile_act(float v, Act act) {
    switch (act) {
        case Act::Tanh: return tanhf(v);
        case Act::Relu: return fmaxf(v, 0.f);
        case Act::Sigmoid: return sigmoid_f32(v);
        default: return v;
    }
}

// out[r, j] = act(b[j] + sum_k W[j, k] in[r, k]) for the tile's rows (k ascending, one fmaf each, then the bias).  Job (j, g) walks weight
// row j once and applies it to its rows.  Not inlined: NL-PPO's six layers inlined with their unrolled row loops take 202 registers, called
// they take 80.
static __device__ __noinline__ void tile_linear(const float* __restrict__ W, const float* __restrict__ b, const float* in, int K, float* out, int N,
                                               Act act) {
    const int groups = tile_groups(N), rpj = kTileRows / groups;
    const int job = threadIdx.x;
    if (job < N * groups) {
        const int j = job % N, g = job / N;
        float acc[kTileRows];
        MORL_TILE_ROWS(i) acc[i] = 0.f;
        const float* wr = W + (size_t)j * K;
        for (int k = 0; k < K; ++k) {
            const float wv = __ldg(wr + k);
            MORL_TILE_ROWS(i) acc[i] = fmaf(wv, in[(g + groups * i) * K + k], acc[i]);
        }
        const float bj = __ldg(b + j);
        MORL_TILE_ROWS(i) out[(g + groups * i) * N + j] = acc[i] + bj;
        // the activation in a rolled loop over the job's own outputs: one copy of its code rather than one per unrolled row
        if (act != Act::None)
            for (int i = 0; i < rpj; ++i) out[(g + groups * i) * N + j] = tile_act(out[(g + groups * i) * N + j], act);
    }
    __syncthreads();
}

// Backward of the layer z = W a + b from dz [kTileRows, N], a [kTileRows, K]: the weight and bias gradients summed over the tile's rows in
// order are written to gw / gb when `init` (the CTA's first tile) and added otherwise; with `dnext`, the gradient w.r.t. the layer's
// pre-activation input, dnext[r, k] = (sum_j W[j, k] dz[r, j]) * act'(a[r, k]), where `act` produced a: 1 - a^2 for Tanh, a > 0 for Relu,
// 1 for None.  The folds and dnext read the same buffers and write different ones, so they share one barrier.
static __device__ __noinline__ void tile_backward(const float* __restrict__ W, const float* a, int K, const float* dz, int N, float* gw, float* gb,
                                                 bool init, float* dnext, Act act) {
    for (int idx = threadIdx.x; idx < N * K; idx += kTileThreads) {
        const int j = idx / K, k = idx % K;
        float s = 0.f;
#pragma unroll
        for (int r = 0; r < kTileRows; ++r) s = fmaf(dz[r * N + j], a[r * K + k], s);
        gw[idx] = init ? s : gw[idx] + s;
    }
    for (int j = threadIdx.x; j < N; j += kTileThreads) {
        float s = 0.f;
#pragma unroll
        for (int r = 0; r < kTileRows; ++r) s += dz[r * N + j];
        gb[j] = init ? s : gb[j] + s;
    }
    if (dnext) {
        const int groups = tile_groups(K), rpj = kTileRows / groups;
        const int job = threadIdx.x;
        if (job < K * groups) {
            const int k = job % K, g = job / K;
            float s[kTileRows];
            MORL_TILE_ROWS(i) s[i] = 0.f;
            for (int j = 0; j < N; ++j) {
                const float wv = __ldg(W + (size_t)j * K + k);
                MORL_TILE_ROWS(i) s[i] = fmaf(wv, dz[(g + groups * i) * N + j], s[i]);
            }
            MORL_TILE_ROWS(i) {
                const int r = g + groups * i;
                const float y = a[r * K + k];
                dnext[r * K + k] = act == Act::Tanh ? s[i] * (1.0f - y * y) : (act == Act::Relu ? (y > 0.f ? s[i] : 0.f) : s[i]);
            }
        }
    }
    __syncthreads();
}

// The tiles [first, first + count) of CTA c when n_tiles are split in contiguous ranges over the grid, the first n_tiles % gridDim.x CTAs
// taking one more.
__device__ __forceinline__ void tile_range(int n_tiles, int c, int& first, int& count) {
    const int ctas = gridDim.x;
    const int q = n_tiles / ctas, rem = n_tiles % ctas;
    first = c * q + min(c, rem);
    count = q + (c < rem ? 1 : 0);
}

// Sum of the n_parts gradient partials (partial c at part + c * L.total()), c ascending, into the .grad storages; then block 0 runs the
// caller's `fin(n_parts)` with all its threads (the loss and statistics of the update).
template <int kMax, typename Finish>
__global__ void __launch_bounds__(kTileThreads) partial_sum_kernel(const __grid_constant__ GradTable<kMax> G, const __grid_constant__ ParamLayout<kMax> L,
                                                                   const float* __restrict__ part, int n_parts, const Finish fin) {
    const int total = L.total();
    int off = 0;
#pragma unroll
    for (int t = 0; t < kMax; ++t) {  // unrolled: G.g[t] stays a kernel parameter, not a stack array
        if (t < L.n) {
            const int n = L.size[t];
            for (int q = blockIdx.x * kTileThreads + threadIdx.x; q < n; q += gridDim.x * kTileThreads) {
                float s = 0.f;
                for (int c = 0; c < n_parts; ++c) s += __ldg(part + (size_t)c * total + off + q);
                G.g[t][q] = s;
            }
            off += n;
        }
    }
    if (blockIdx.x == 0) fin(n_parts);
}

template <int kMax, typename Finish>
static void launch_partial_sum(const GradTable<kMax>& G, const ParamLayout<kMax>& L, const float* part, int n_parts, const Finish& fin,
                               cudaStream_t st) {
    const int blocks = min((L.total() + kTileThreads - 1) / kTileThreads, 4 * sm_count());
    partial_sum_kernel<kMax, Finish><<<blocks, kTileThreads, 0, st>>>(G, L, part, n_parts, fin);
}

// Copies the n pointers of `params` (and of `grads` when given) into the kernel tables, NULL past n.  A NULL one of the n sets entry
// point `what`'s error and returns MORL_ERR_NULL.
template <int kMax>
static int load_tables(const char* what, int n, const float* const* params, ParamTable<kMax>& P, float* const* grads = nullptr,
                       GradTable<kMax>* G = nullptr) {
    for (int t = 0; t < n; ++t) {
        MORL_REQUIRE(params[t] && (!grads || grads[t]), MORL_ERR_NULL,
                     grads ? "%s: NULL parameter or gradient pointer %d" : "%s: NULL parameter pointer %d", what, t);
    }
    for (int t = 0; t < kMax; ++t) {
        P.p[t] = t < n ? params[t] : nullptr;
        if (G) G->g[t] = t < n ? grads[t] : nullptr;
    }
    return MORL_OK;
}

}  // namespace morl
