// sumtree.cuh -- the reference SumTree's walk and single-leaf set (common/prioritized_buffer.py:30-64) as device functions, shared by
// sumtree.cu (the replay buffer's tree) and moq.cu (the tabular Dyna model's prioritised pair sampling).
// Layout: float64, level l (2^l nodes) at element 2^l - 1, root first, leaves last.
#pragma once
#include "common.cuh"

namespace morl {

__device__ __forceinline__ double* st_level(double* tree, int l) { return tree + (((size_t)1) << l) - 1; }
__device__ __forceinline__ const double* st_level(const double* tree, int l) { return tree + (((size_t)1) << l) - 1; }

// leaf index the query q descends to: per level left = node[2 i]; right = q > left; i = 2 i + right; q -= left * right   (:40-54)
__device__ __forceinline__ long long st_walk(const double* tree, int n_levels, double q) {
    long long node = 0;
    for (int l = 1; l < n_levels; ++l) {
        const double left = st_level(tree, l)[2 * node];
        const bool right = q > left;
        node = 2 * node + (right ? 1 : 0);
        q = __dsub_rn(q, __dmul_rn(left, right ? 1.0 : 0.0));  // query -= left_sum * is_greater
    }
    return node;
}

// SumTree.set of one leaf (:56-64) by the 32 lanes of one warp: diff = p - leaf, then every level += diff (lane l takes levels l, l + 32).
// index must be a leaf (0 <= index < 2^(n_levels - 1)).
__device__ __forceinline__ void st_set_warp(double* tree, int n_levels, long long index, double p) {
    const int lane = threadIdx.x & 31;
    const double d = __dsub_rn(p, st_level(tree, n_levels - 1)[index]);  // (every lane reads the old leaf before any lane writes it)
    __syncwarp();
    for (int l = lane; l < n_levels; l += 32) {
        double* node = st_level(tree, l) + (index >> (n_levels - 1 - l));
        *node = __dadd_rn(*node, d);
    }
}

}  // namespace morl
