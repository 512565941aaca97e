// pql.cu -- Pareto Q-learning's set table on the device: the per-step set update and the greedy step's action scores.
//
// Replaces the Python-set work of the reference's PQL (multi_policy/pareto_q_learning/pql.py): get_q_set, calc_non_dominated and the
// update of pql.py:260-262, score_hypervolume (pymoo's exact HV, pql.py:143-154) and score_pareto_cardinality (pql.py:122-141).
// Layout (caller-owned, nothing allocated here): nd f64 [S, A, K, d] with nd_count int32 [S, A] (the stored set ND[s][a], its first
// nd_count rows valid), avg_reward f64 [S, A, d], counts f64 [S, A], status int32 [3].
//
// Rounding: every operation is one IEEE float64 operation in numpy's order (gamma * v, then avg + that; r - avg, then / counts, then
// avg + that), spelled with the _rn intrinsics so no FMA contraction can change a bit.  Prune: keep a point iff no distinct point is >= it
// in every coordinate, and only the first copy of equal points (morl_pareto_mask_f64 with remove_duplicates).  Canonical order: descending
// coordinate sum (added left to right), ties lexicographically descending; the kept points are distinct, so the order is total and equal
// sets are stored as equal bytes.
#include "common.cuh"
#include "hv.cuh"

namespace morl {

constexpr int kPqlThreads = 1024;
constexpr int kPqlMaxA = 16;
constexpr int kPqlMaxK = 256;
constexpr int kPqlMaxUnion = 2048;  // A * K: the union of one state's Q-sets

struct PqlVec {
    double v[MORL_MAX_D];
};

// Q-set(state, a') of every action, concatenated in action order, into pts [n, d] of shared memory; returns n.  off [A + 1] (shared)
// receives each action's first row.  Reads the stored sets and avg_reward of `state` only.
__device__ __forceinline__ int pql_stage_union(const double* nd, const int* nd_count, const double* avg,
                                               int A, int K, int d, int state, double gamma, double* pts, int* off) {
    if (threadIdx.x == 0) {
        int o = 0;
        for (int b = 0; b < A; ++b) {
            off[b] = o;
            o += min(max(nd_count[(size_t)state * A + b], 0), K);
        }
        off[A] = o;
    }
    __syncthreads();
    for (int t = threadIdx.x; t < A * K; t += blockDim.x) {
        const int b = t / K, i = t - b * K;
        if (off[b] + i >= off[b + 1]) continue;
        const double* v = nd + (((size_t)state * A + b) * K + i) * d;
        const double* r = avg + ((size_t)state * A + b) * d;
        double* q = pts + (size_t)(off[b] + i) * d;
        for (int c = 0; c < d; ++c) q[c] = __dadd_rn(r[c], __dmul_rn(gamma, v[c]));
    }
    __syncthreads();
    return off[A];
}

// point i of pts [n, d] survives the prune: no distinct point is >= it everywhere, and no earlier index in [first, n) holds its value
__device__ __forceinline__ bool pql_survives(const double* pts, int n, int d, int i, int first) {
    const double* p = pts + (size_t)i * d;
    for (int j = 0; j < n; ++j) {
        const double* o = pts + (size_t)j * d;
        bool ge = true, eq = true;
        for (int c = 0; c < d; ++c) {
            ge = ge && (o[c] >= p[c]);
            eq = eq && (o[c] == p[c]);
        }
        if ((ge && !eq) || (eq && j >= first && j < i)) return false;
    }
    return true;
}

// canonical order: does p come before q (descending coordinate sum, then lexicographically descending)?  p != q.
__device__ __forceinline__ bool pql_before(const double* p, double sp, const double* q, double sq, int d) {
    if (sp != sq) return sp > sq;
    for (int c = 0; c < d; ++c)
        if (p[c] != q[c]) return p[c] > q[c];
    return false;
}

// One reference step (pql.py:260-262) in one CTA.  The whole union of ND[s'][.] is staged in shared memory before anything is written,
// so s' == s (a wall of a grid world) reads the old sets (no __restrict__ here: the table is read and written by the same launch).  On overflow (more than K points survive) nothing but `status` is written.
__global__ void __launch_bounds__(kPqlThreads, 1) pql_update_kernel(double* nd, int* nd_count, double* avg, double* counts, int* status, int A, int K, int d,
                                                                    int s, int a, int s_next, double gamma, PqlVec reward) {
    extern __shared__ double pql_smem[];
    __shared__ int off[kPqlMaxA + 1];
    double* pts = pql_smem;                          // [A * K, d]
    double* sum = pts + (size_t)A * K * d;           // [A * K]
    int* keep = reinterpret_cast<int*>(sum + A * K);  // [A * K]
    const int n = pql_stage_union(nd, nd_count, avg, A, K, d, s_next, gamma, pts, off);

    int m = 0;
    for (int i0 = 0; i0 < n; i0 += blockDim.x) {
        const int i = i0 + threadIdx.x;
        bool k = false;
        if (i < n) {
            k = pql_survives(pts, n, d, i, 0);
            keep[i] = k ? 1 : 0;
            double acc = pts[(size_t)i * d];
            for (int c = 1; c < d; ++c) acc = __dadd_rn(acc, pts[(size_t)i * d + c]);
            sum[i] = acc;
        }
        m += __syncthreads_count(k);
    }
    // every thread holds the same m here
    const size_t sa = (size_t)s * A + a;
    if (m > K) {
        if (threadIdx.x == 0 && status[0] == 0) {
            status[0] = m;
            status[1] = s;
            status[2] = a;
        }
        return;
    }
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        if (!keep[i]) continue;
        const double* p = pts + (size_t)i * d;
        int rank = 0;
        for (int j = 0; j < n; ++j)
            rank += (keep[j] && j != i && pql_before(pts + (size_t)j * d, sum[j], p, sum[i], d)) ? 1 : 0;
        double* dst = nd + (sa * K + rank) * d;
        for (int c = 0; c < d; ++c) dst[c] = p[c];
    }
    if (threadIdx.x == 0) {
        nd_count[sa] = m;
        const double cnt = __dadd_rn(counts[sa], 1.0);
        counts[sa] = cnt;
        double* r = avg + sa * d;
#pragma unroll
        for (int c = 0; c < MORL_MAX_D; ++c)  // unrolled: the reward stays in parameter space, no stack copy
            if (c < d) r[c] = __dadd_rn(r[c], __ddiv_rn(__dsub_rn(reward.v[c], r[c]), cnt));
    }
}

// scores[a] (block a) = exact volume of Q-set(state, a) above ref, as morl_hypervolume_batch_f64 counts it (d <= 4)
__global__ void __launch_bounds__(kHvThreads, 1) pql_score_hv_kernel(const double* __restrict__ nd, const int* __restrict__ nd_count,
                                                                     const double* __restrict__ avg, int A, int K, int d, int state, double gamma,
                                                                     PqlVec ref, double* __restrict__ scores) {
    extern __shared__ double pql_smem[];
    const int a = blockIdx.x;
    const size_t sa = (size_t)state * A + a;
    const int n = min(max(nd_count[sa], 0), K);
    const HvSmem s = hv_carve(pql_smem, n);
    double rp[4];
    for (int c = 0; c < 4; ++c) rp[c] = c < d ? ref.v[c] : 0.0;
    const double* r = avg + sa * d;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const double* v = nd + (sa * K + i) * d;
        double q[4];
        for (int c = 0; c < 4; ++c) q[c] = c < d ? __dadd_rn(r[c], __dmul_rn(gamma, v[c])) : 0.0;
        hv_stage(s, i, q, true, d, rp);
    }
    __syncthreads();
    const double v = hv_sweep(s, n, d == 4);
    if (threadIdx.x == 0) scores[a] = v;
}

// scores[a] (block a) = number of points of ND(union of the state's Q-sets) equal to a point of Q-set(state, a): the distinct values of
// Q-set(state, a) that no distinct point of the union is >= in every coordinate
__global__ void __launch_bounds__(kPqlThreads, 1) pql_score_card_kernel(const double* __restrict__ nd, const int* __restrict__ nd_count,
                                                                        const double* __restrict__ avg, int A, int K, int d, int state,
                                                                        double gamma, double* __restrict__ scores) {
    extern __shared__ double pql_smem[];
    __shared__ int off[kPqlMaxA + 1];
    const int n = pql_stage_union(nd, nd_count, avg, A, K, d, state, gamma, pql_smem, off);
    const int a = blockIdx.x, lo = off[a], hi = off[a + 1];
    int m = 0;
    for (int i0 = lo; i0 < hi; i0 += blockDim.x) {
        const int i = i0 + threadIdx.x;
        m += __syncthreads_count(i < hi && pql_survives(pql_smem, n, d, i, lo));
    }
    if (threadIdx.x == 0) scores[a] = (double)m;
}

static size_t pql_update_smem(int A, int K, int d) { return (size_t)A * K * ((size_t)d + 1) * sizeof(double) + (size_t)A * K * sizeof(int); }
static size_t pql_card_smem(int A, int K, int d) { return (size_t)A * K * d * sizeof(double); }

static PqlVec pql_vec(const double* p, int d) {
    PqlVec v = {};
    for (int c = 0; c < d; ++c) v.v[c] = p[c];
    return v;
}

}  // namespace morl

extern "C" int morl_pql_supported(int n_actions, int cap, int d, int mode) {
    using namespace morl;
    const bool base = n_actions >= 1 && n_actions <= kPqlMaxA && cap >= 1 && cap <= kPqlMaxK && n_actions * cap <= kPqlMaxUnion && d >= 1 &&
                      d <= MORL_MAX_D;
    if (mode == MORL_PQL_HYPERVOLUME) return base && d <= 4 ? 1 : 0;
    if (mode == MORL_PQL_CARDINALITY) return base ? 1 : 0;
    return 0;
}

extern "C" int morl_pql_update_f64(double* nd, int* nd_count, double* avg_reward, double* counts, int* status, int S, int A, int K, int d,
                                   int s, int a, int s_next, double gamma, const double* reward, void* stream) {
    using namespace morl;
    MORL_REQUIRE(nd && nd_count && avg_reward && counts && status && reward, MORL_ERR_NULL, "morl_pql_update_f64: NULL pointer argument");
    MORL_REQUIRE(S >= 1, MORL_ERR_SHAPE, "morl_pql_update_f64: bad shape S=%d", S);
    MORL_REQUIRE(morl_pql_supported(A, K, d, MORL_PQL_CARDINALITY), MORL_ERR_UNSUPPORTED,
                 "morl_pql_update_f64: supports 1 <= A <= %d, 1 <= K <= %d, A * K <= %d, 1 <= d <= %d (got A=%d, K=%d, d=%d)", kPqlMaxA, kPqlMaxK,
                 kPqlMaxUnion, MORL_MAX_D, A, K, d);
    MORL_REQUIRE(s >= 0 && s < S && s_next >= 0 && s_next < S && a >= 0 && a < A, MORL_ERR_SHAPE,
                 "morl_pql_update_f64: s=%d, s_next=%d outside [0, %d) or a=%d outside [0, %d)", s, s_next, S, a, A);
    set_smem_limit_once<pql_update_kernel>(pql_update_smem(kPqlMaxA, kPqlMaxUnion / kPqlMaxA, MORL_MAX_D));
    pql_update_kernel<<<1, kPqlThreads, pql_update_smem(A, K, d), static_cast<cudaStream_t>(stream)>>>(nd, nd_count, avg_reward, counts, status, A,
                                                                                                        K, d, s, a, s_next, gamma,
                                                                                                        pql_vec(reward, d));
    return check_launch("morl_pql_update_f64");
}

extern "C" int morl_pql_score_f64(const double* nd, const int* nd_count, const double* avg_reward, int S, int A, int K, int d, int state,
                                  double gamma, int mode, const double* ref, double* scores, void* stream) {
    using namespace morl;
    MORL_REQUIRE(nd && nd_count && avg_reward && scores && (ref || mode != MORL_PQL_HYPERVOLUME), MORL_ERR_NULL,
                 "morl_pql_score_f64: NULL pointer argument");
    MORL_REQUIRE(S >= 1, MORL_ERR_SHAPE, "morl_pql_score_f64: bad shape S=%d", S);
    MORL_REQUIRE(morl_pql_supported(A, K, d, mode), MORL_ERR_UNSUPPORTED,
                 "morl_pql_score_f64: mode %d supports 1 <= A <= %d, 1 <= K <= %d, A * K <= %d and 1 <= d <= %d (got A=%d, K=%d, d=%d)", mode,
                 kPqlMaxA, kPqlMaxK, kPqlMaxUnion, mode == MORL_PQL_HYPERVOLUME ? 4 : MORL_MAX_D, A, K, d);
    MORL_REQUIRE(state >= 0 && state < S, MORL_ERR_SHAPE, "morl_pql_score_f64: state=%d outside [0, %d)", state, S);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (mode == MORL_PQL_HYPERVOLUME) {
        pql_score_hv_kernel<<<A, kHvThreads, hv_smem_bytes(K), st>>>(nd, nd_count, avg_reward, A, K, d, state, gamma, pql_vec(ref, d), scores);
    } else {
        set_smem_limit_once<pql_score_card_kernel>(pql_card_smem(kPqlMaxA, kPqlMaxUnion / kPqlMaxA, MORL_MAX_D));
        pql_score_card_kernel<<<A, kPqlThreads, pql_card_smem(A, K, d), st>>>(nd, nd_count, avg_reward, A, K, d, state, gamma, scores);
    }
    return check_launch("morl_pql_score_f64");
}
