// sumtree.cu -- device-resident prioritised-replay sum tree (SURVEY.md 8(f)1), bit-identical to the reference's numpy tree.
//
// Replaces SumTree.sample / set / batch_set and PrioritizedReplayBuffer.update_priorities (reference common/prioritized_buffer.py:30-82,
// 186-195) for a buffer whose transitions already live in HBM: the sampled indices feed the replay gather and the new priorities come
// out of the TD-loss kernel, so with the tree on the device one update needs no device->host->device round trip and the whole update
// (sample -> gather -> ... -> priorities -> tree) is ONE captured CUDA graph.
//
// Layout = the reference's (and csrc/host_replay.cu's): float64, level l (2^l nodes) at element 2^l - 1, root first, leaves last.
// The reference's arithmetic is order dependent (inner nodes are updated INCREMENTALLY, node += new - old, in array order), so the
// kernels reproduce its orders exactly:
//   walk      : query = root * u  (np.random.uniform(0, root) = 0 + (root - 0) * u, one IEEE multiply), then per level
//               left = node[2 i]; right = query > left; i = 2 i + right; query -= left * right                           (:40-54)
//   batch_set : np.unique(index, return_index=True) -> sorted unique leaves, each with the priority of its FIRST occurrence;
//               diff = new - leaf; per level np.add.at(level, index >> k, diff) = for i in array order: level[..] += diff[i]   (:66-82)
//               -- every node's additions happen in sorted-leaf order; distinct nodes are independent, so one thread per (level, node)
//               run performs that node's additions sequentially, all runs in parallel;
//   set       : one leaf, diff added to its ancestor on every level (replay_buffer.add, :56-64, 149-151)
//   priorities: p = fl32(fl32(|w . td| + min_p) ** alpha)  and  min_p = max(min_p, max p)                                 (envelope.py:329-334,
//               prioritized_buffer.py:194); the power is evaluated in float64 and rounded once to float32 (numpy's float32 power is
//               within 1 ulp of that, but not reproducible across its own SIMD / libm back ends).
#include "sumtree.cuh"

namespace morl {

__global__ void __launch_bounds__(256) sumtree_walk_kernel(const double* __restrict__ tree, int n_levels, const double* __restrict__ u, int n,
                                                           int scale_by_root, long long* __restrict__ out) {
    pdl_enter();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = st_walk(tree, n_levels, scale_by_root ? __dmul_rn(tree[0], u[i]) : u[i]);
}

constexpr int kStMaxBatch = 2048;  // (44 KB of static shared memory)
constexpr int kStThreads = 1024;

// one block.  idx [n] leaf indices, prio [n] new priorities (float64), n <= kStMaxBatch.
__global__ void __launch_bounds__(kStThreads) sumtree_batch_set_kernel(double* __restrict__ tree, int n_levels, const long long* __restrict__ idx,
                                                                       const double* __restrict__ prio, int n, int* __restrict__ err) {
    pdl_enter();
    __shared__ unsigned long long key[kStMaxBatch];  // (leaf << 13 | position), sorted ascending; position < 2^13
    __shared__ double diff[kStMaxBatch];             // diff of the i-th UNIQUE leaf (compacted)
    __shared__ int leaf[kStMaxBatch];                // the i-th unique leaf
    __shared__ int scan[kStThreads];
    __shared__ int m_s;
    const long long n_leaves = (long long)1 << (n_levels - 1);
    int np2 = 1;
    while (np2 < n) np2 <<= 1;
    for (int i = threadIdx.x; i < np2; i += blockDim.x) {
        unsigned long long k = ~0ULL;
        if (i < n) {
            const long long v = idx[i];
            if (v < 0 || v >= n_leaves)
                *err = 1;  // flagged, and left as padding: never dereferenced
            else
                k = ((unsigned long long)v << 13) | (unsigned long long)i;
        }
        key[i] = k;
    }
    __syncthreads();
    // bitonic sort, ascending (n <= 2048: at most 2 elements per thread per pass)
    for (int size = 2; size <= np2; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = threadIdx.x; i < np2; i += blockDim.x) {
                const int j = i ^ stride;
                if (j > i) {
                    const bool up = (i & size) == 0;
                    const unsigned long long a = key[i], b = key[j];
                    if ((a > b) == up) {
                        key[i] = b;
                        key[j] = a;
                    }
                }
            }
            __syncthreads();
        }
    }
    // unique leaves (first occurrence = smallest position, which sorts first inside a run of equal leaves): block-wide compaction
    const int per = (n + blockDim.x - 1) / blockDim.x;
    const int b0 = threadIdx.x * per, b1 = min(n, b0 + per);
    int cnt = 0;
    for (int i = b0; i < b1; ++i) cnt += (key[i] != ~0ULL && (i == 0 || (key[i] >> 13) != (key[i - 1] >> 13))) ? 1 : 0;
    scan[threadIdx.x] = cnt;
    __syncthreads();
    for (int off = 1; off < (int)blockDim.x; off <<= 1) {  // inclusive Hillis-Steele scan
        const int v = threadIdx.x >= off ? scan[threadIdx.x - off] : 0;
        __syncthreads();
        scan[threadIdx.x] += v;
        __syncthreads();
    }
    int pos = scan[threadIdx.x] - cnt;
    if (threadIdx.x == blockDim.x - 1) m_s = scan[threadIdx.x];
    double* leaves = st_level(tree, n_levels - 1);
    for (int i = b0; i < b1; ++i) {
        if (key[i] != ~0ULL && (i == 0 || (key[i] >> 13) != (key[i - 1] >> 13))) {
            const int lf = (int)(key[i] >> 13);
            leaf[pos] = lf;
            diff[pos] = __dsub_rn(prio[key[i] & 0x1FFFULL], leaves[lf]);  // diff = new - old, before any level is touched
            ++pos;
        }
    }
    __syncthreads();
    const int m = m_s;
    // every (level, node) run: one thread adds the run's diffs to the node, in array order
    const long long total = (long long)n_levels * m;
    for (long long w = threadIdx.x; w < total; w += blockDim.x) {
        const int l = (int)(w / m), i = (int)(w - (long long)l * m);
        const int shift = n_levels - 1 - l;
        const int node = leaf[i] >> shift;
        if (i > 0 && (leaf[i - 1] >> shift) == node) continue;  // not the head of its run
        double* p = st_level(tree, l) + node;
        double acc = *p;
        for (int j = i; j < m && (leaf[j] >> shift) == node; ++j) acc = __dadd_rn(acc, diff[j]);
        *p = acc;
    }
}

// SumTree.set (one leaf; replay_buffer.add): diff = new - leaf, every level += diff.  Scalar kernel arguments -- no staging buffer, so a
// call per environment step is just a launch.  use_min != 0: new = the buffer's current min_priority (device float32).
__global__ void __launch_bounds__(32) sumtree_set_kernel(double* __restrict__ tree, int n_levels, long long index, double priority, int use_min,
                                                         const double* __restrict__ min_priority, int* __restrict__ err) {
    const long long n_leaves = (long long)1 << (n_levels - 1);
    if (index < 0 || index >= n_leaves) {
        if (threadIdx.x == 0) *err = 1;
        return;
    }
    st_set_warp(tree, n_levels, index, use_min ? *min_priority : priority);
}

// p32[i] = fl32( (fl32(raw[i] + fl32(min_p))) ** alpha ), p64 = (double) p32, then min_p = max(min_p, max_i p32[i]).  One block.
// min_p is a DOUBLE: the reference starts it as a python float (1e-5, not float32-representable: new transitions enter the tree with that
// double) and it becomes a float32 value the first time a priority exceeds it (python max(float, np.float32)).
__global__ void __launch_bounds__(kStThreads) per_priority_kernel(const float* __restrict__ raw, int n, float alpha, double* __restrict__ min_priority,
                                                                  double* __restrict__ p64, float* __restrict__ p32) {
    pdl_enter();
    __shared__ float red[kStThreads / 32];
    const double mp64 = *min_priority;
    const float mp = (float)mp64;
    float mx = 0.f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float x = __fadd_rn(raw[i], mp);
        const float p = (float)pow((double)x, (double)alpha);  // correctly rounded float32 power (double evaluation, one rounding)
        if (p32) p32[i] = p;
        p64[i] = (double)p;
        mx = fmaxf(mx, p);  // (NaN priorities do not ratchet min_priority: fmaxf drops them, as python's max(min_p, nan) keeps min_p)
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x < 32) {
        mx = threadIdx.x < kStThreads / 32 ? red[threadIdx.x] : 0.f;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
        if (threadIdx.x == 0 && (double)mx > mp64) *min_priority = (double)mx;
    }
}

}  // namespace morl

extern "C" int morl_sumtree_walk_f64(const double* tree, int n_levels, const double* u, int n, int scale_by_root, long long* out_index, void* stream) {
    using namespace morl;
    MORL_REQUIRE(tree && u && out_index, MORL_ERR_NULL, "morl_sumtree_walk_f64: NULL pointer argument");
    MORL_REQUIRE(n_levels >= 1 && n_levels <= 31 && n >= 0, MORL_ERR_SHAPE, "morl_sumtree_walk_f64: bad shape n_levels=%d n=%d", n_levels, n);
    if (n == 0) return MORL_OK;
    launch_k(sumtree_walk_kernel, dim3((n + 255) / 256), dim3(256), 0, static_cast<cudaStream_t>(stream), tree, n_levels, u, n, scale_by_root, out_index);
    return check_launch("morl_sumtree_walk_f64");
}

extern "C" int morl_sumtree_batch_set_f64(double* tree, int n_levels, const long long* index, const double* priority, int n, int* err_flag,
                                          void* stream) {
    using namespace morl;
    MORL_REQUIRE(tree && index && priority && err_flag, MORL_ERR_NULL, "morl_sumtree_batch_set_f64: NULL pointer argument");
    MORL_REQUIRE(n_levels >= 1 && n_levels <= 31 && n >= 0 && n <= kStMaxBatch, MORL_ERR_SHAPE,
                 "morl_sumtree_batch_set_f64: bad shape n_levels=%d n=%d (at most %d indices per call)", n_levels, n, kStMaxBatch);
    if (n == 0) return MORL_OK;
    launch_k(sumtree_batch_set_kernel, dim3(1), dim3(kStThreads), 0, static_cast<cudaStream_t>(stream), tree, n_levels, index, priority, n, err_flag);
    return check_launch("morl_sumtree_batch_set_f64");
}

extern "C" int morl_sumtree_set_f64(double* tree, int n_levels, long long index, double priority, int use_min_priority, const double* min_priority,
                                    int* err_flag, void* stream) {
    using namespace morl;
    MORL_REQUIRE(tree && err_flag && (min_priority || !use_min_priority), MORL_ERR_NULL, "morl_sumtree_set_f64: NULL pointer argument");
    MORL_REQUIRE(n_levels >= 1 && n_levels <= 31, MORL_ERR_SHAPE, "morl_sumtree_set_f64: bad n_levels=%d", n_levels);
    sumtree_set_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(tree, n_levels, index, priority, use_min_priority, min_priority, err_flag);
    return check_launch("morl_sumtree_set_f64");
}

extern "C" int morl_per_priority_f32(const float* raw, int n, float alpha, double* min_priority, double* prio64, float* prio32, void* stream) {
    using namespace morl;
    MORL_REQUIRE(raw && min_priority && prio64, MORL_ERR_NULL, "morl_per_priority_f32: NULL pointer argument");
    MORL_REQUIRE(n > 0, MORL_ERR_SHAPE, "morl_per_priority_f32: bad n=%d", n);
    launch_k(per_priority_kernel, dim3(1), dim3(kStThreads), 0, static_cast<cudaStream_t>(stream), raw, n, alpha, min_priority, prio64, prio32);
    return check_launch("morl_per_priority_f32");
}
