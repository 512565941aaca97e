// linear_support.cu -- corner weights of a convex coverage set by exact vertex enumeration (float64).
//
// Replaces compute_corner_weights (reference multi_policy/linear_support/linear_support.py:295-349), which hands the polyhedron
//     { x = (w, u) in R^{d+1} :  v_i . w - u <= 0 (i < n),  -w_j <= 0 (j < d),  sum_j w_j = 1 }
// to cdd and keeps the generators that are vertices.  The polyhedron has one ray (+u) and no lines, so its vertices are exactly the
// feasible points where sum w = 1 and d linearly independent inequality rows are tight.
//
// Enumeration: rows 0..n-1 are the value rows, rows n..n+d-1 the non-negativity rows; a candidate is a sorted d-subset S of the
// n + d rows (lexicographic order, C(n+d, d) candidates).  A subset without a value row leaves u free: skipped (value rows have the
// lowest indices, so this is s_0 >= n).  Otherwise u is eliminated through the first value row i0 = s_0, leaving the d x d system
//     R w = e_0,   R = [ 1 ;  v_s - v_i0 (value rows s in S, s != i0) ;  e_j (non-negativity rows n + j in S) ]
// solved by LU with partial pivoting in registers; u = v_i0 . w.  Rejected: |pivot| <= kPivotEps * scale (rank deficient),
// w_j < -kWTol, or v_k . w > u + kVTol * scale for some k, with scale = max(1, max |V|).
//
// Degenerate vertices (more than d tight rows) are reachable from several subsets but are emitted once: with T the tight rows of the
// solution, S must be the lexicographically first basis of T, taken greedily in row order after the sum row.  For a matroid that
// holds iff every tight row r outside S lies in the span of the sum row and the rows of S below r.  r < s_0 is never in that span
// (span{sum row} contains no value or non-negativity row for d >= 2).  For r > s_0, the coefficients of r in the basis {sum row, S}
// are those of the transposed reduced system R^T c = b_r (b_r = v_r - v_i0, or e_j), the coefficient of i0 being implied by the
// u-component; S is canonical iff c_k ~ 0 for every row s_k > r of S.  The LU factors are reused for these solves.
//
// Mapping: each thread walks a contiguous range of candidate indices (unranked once with exact binomials, then lexicographic
// successors); vertices are appended with one atomicAdd on *count, which is NOT clipped to cap.
#include "common.cuh"

namespace morl {

constexpr int kCornerThreads = 128;
constexpr double kPivotEps = 1e-11;  // relative to scale: smaller pivots are a rank-deficient subset
constexpr double kWTol = 1e-9;       // w_j >= -kWTol; w_j <= kWTol counts as tight
constexpr double kVTol = 1e-9;       // v_k . w <= u + kVTol * scale; |u - v_k . w| <= kVTol * scale counts as tight
constexpr double kCoefEps = 1e-9;    // basis coefficients below this (relative to scale) are zero

// C(a, b) for the small b used here; every value asked for is <= the candidate count, and each partial product C(a, i) * (a - i) stays
// below 8 * kCornerMaxCandidates, so uint64 is exact.  Returns UINT64_MAX when the value exceeds `limit` (host-side bound check).
__host__ __device__ inline unsigned long long binom_capped(long long a, int b, unsigned long long limit) {
    if (b < 0 || a < b) return 0ull;
    unsigned long long c = 1ull;
    for (int i = 0; i < b; ++i) {
        c = c * (unsigned long long)(a - i) / (unsigned long long)(i + 1);
        if (c > limit) return ~0ull;
    }
    return c;
}

template <int D>
__global__ void __launch_bounds__(kCornerThreads) corner_weights_kernel(const double* __restrict__ V, int n, unsigned long long total,
                                                                        unsigned long long per_thread, double* __restrict__ verts, int cap,
                                                                        int* __restrict__ count) {
    __shared__ double red[kCornerThreads];
    double mx = 0.0;
    for (int e = threadIdx.x; e < n * D; e += blockDim.x) mx = fmax(mx, fabs(__ldg(V + e)));
    red[threadIdx.x] = mx;
    __syncthreads();
    for (int off = kCornerThreads / 2; off > 0; off >>= 1) {
        if (threadIdx.x < off) red[threadIdx.x] = fmax(red[threadIdx.x], red[threadIdx.x + off]);
        __syncthreads();
    }
    const double scale = fmax(1.0, red[0]);
    const double piv_eps = kPivotEps * scale, v_tol = kVTol * scale, c_eps = kCoefEps * scale;

    const unsigned long long tid = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long idx = tid * per_thread;
    if (idx >= total) return;
    const unsigned long long end = idx + per_thread < total ? idx + per_thread : total;
    const int m = n + D;

    // unrank idx: lexicographic order of sorted D-subsets of {0..m-1}
    int s[D];
    {
        unsigned long long r = idx;
        int c = 0;
#pragma unroll
        for (int i = 0; i < D; ++i) {
            for (;; ++c) {
                const unsigned long long cnt = binom_capped(m - c - 1, D - i - 1, ~0ull);
                if (r < cnt) break;
                r -= cnt;
            }
            s[i] = c++;
        }
    }

    for (; idx < end; ++idx) {
        if (s[0] < n) {
            const int i0 = s[0];
            double v0[D];
#pragma unroll
            for (int j = 0; j < D; ++j) v0[j] = __ldg(V + (size_t)i0 * D + j);
            // reduced system, rows permuted in place by the pivoting; rid = subset row held at each position (-1: the sum row)
            double a[D][D];
            int rid[D];
#pragma unroll
            for (int j = 0; j < D; ++j) a[0][j] = 1.0;
            rid[0] = -1;
#pragma unroll
            for (int k = 1; k < D; ++k) {
                const int r = s[k];
                rid[k] = r;
                if (r < n) {
#pragma unroll
                    for (int j = 0; j < D; ++j) a[k][j] = __ldg(V + (size_t)r * D + j) - v0[j];
                } else {
#pragma unroll
                    for (int j = 0; j < D; ++j) a[k][j] = (j == r - n) ? 1.0 : 0.0;
                }
            }
            // LU with partial pivoting: P R = L U, L unit lower (below the diagonal), U on and above it
            bool ok = true;
            double rdiag[D];  // 1 / U[k][k]
#pragma unroll
            for (int k = 0; k < D; ++k) {
                int p = k;
                double best = fabs(a[k][k]);
#pragma unroll
                for (int i = k + 1; i < D; ++i)
                    if (fabs(a[i][k]) > best) { best = fabs(a[i][k]); p = i; }
                ok = ok && best > piv_eps;
#pragma unroll
                for (int i = k + 1; i < D; ++i) {
                    if (i == p) {
#pragma unroll
                        for (int j = 0; j < D; ++j) { const double t = a[k][j]; a[k][j] = a[i][j]; a[i][j] = t; }
                        const int t = rid[k]; rid[k] = rid[i]; rid[i] = t;
                    }
                }
                const double inv = ok ? __drcp_rn(a[k][k]) : 0.0;
                rdiag[k] = inv;
#pragma unroll
                for (int i = k + 1; i < D; ++i) {
                    const double f = a[i][k] * inv;
                    a[i][k] = f;
#pragma unroll
                    for (int j = k + 1; j < D; ++j) a[i][j] = fma(-f, a[k][j], a[i][j]);
                }
            }
            if (ok) {
                // R w = e_0: the right-hand side is 1 at the position the sum row was moved to, 0 elsewhere
                double w[D];
#pragma unroll
                for (int i = 0; i < D; ++i) {
                    double y = rid[i] == -1 ? 1.0 : 0.0;
#pragma unroll
                    for (int j = 0; j < i; ++j) y = fma(-a[i][j], w[j], y);
                    w[i] = y;
                }
#pragma unroll
                for (int i = D - 1; i >= 0; --i) {
                    double y = w[i];
#pragma unroll
                    for (int j = i + 1; j < D; ++j) y = fma(-a[i][j], w[j], y);
                    w[i] = y * rdiag[i];
                }
#pragma unroll
                for (int j = 0; j < D; ++j) ok = ok && w[j] >= -kWTol;
                double u = 0.0;
#pragma unroll
                for (int j = 0; j < D; ++j) u = fma(v0[j], w[j], u);
                for (int k = 0; ok && k < n; ++k) {
                    double vw = 0.0;
#pragma unroll
                    for (int j = 0; j < D; ++j) vw = fma(__ldg(V + (size_t)k * D + j), w[j], vw);
                    ok = vw <= u + v_tol;
                }
                // canonical-basis test over the tight rows outside S (rows in S are tight by construction); a bit mask keeps w in
                // registers (a select over w[r - n] compiles to an indexed local-memory load)
                unsigned w_tight = 0u;
#pragma unroll
                for (int j = 0; j < D; ++j) w_tight |= (w[j] <= kWTol ? 1u : 0u) << j;
                for (int r = 0; ok && r < m; ++r) {
                    bool in_s = false;
#pragma unroll
                    for (int k = 0; k < D; ++k) in_s = in_s || s[k] == r;
                    if (in_s) continue;
                    double b[D];
                    bool tight;
                    if (r < n) {
                        double vw = 0.0;
#pragma unroll
                        for (int j = 0; j < D; ++j) {
                            const double vr = __ldg(V + (size_t)r * D + j);
                            vw = fma(vr, w[j], vw);
                            b[j] = vr - v0[j];
                        }
                        tight = u - vw <= v_tol;
                    } else {
#pragma unroll
                        for (int j = 0; j < D; ++j) b[j] = (j == r - n) ? 1.0 : 0.0;
                        tight = (w_tight >> (r - n)) & 1u;
                    }
                    if (!tight) continue;
                    if (r < i0) { ok = false; break; }
                    // R^T c = b with P R = L U:  U^T y = b,  L^T z = y,  c = P^T z (z[i] is the coefficient of subset row rid[i])
#pragma unroll
                    for (int i = 0; i < D; ++i) {
                        double y = b[i];
#pragma unroll
                        for (int j = 0; j < i; ++j) y = fma(-a[j][i], b[j], y);
                        b[i] = y * rdiag[i];
                    }
#pragma unroll
                    for (int i = D - 1; i >= 0; --i) {
                        double y = b[i];
#pragma unroll
                        for (int j = i + 1; j < D; ++j) y = fma(-a[j][i], b[j], y);
                        b[i] = y;
                    }
#pragma unroll
                    for (int i = 0; i < D; ++i) ok = ok && !(rid[i] > r && fabs(b[i]) > c_eps);
                }
                if (ok) {
                    const int slot = atomicAdd(count, 1);
                    if (slot < cap) {
#pragma unroll
                        for (int j = 0; j < D; ++j) verts[(size_t)slot * (D + 1) + j] = w[j];
                        verts[(size_t)slot * (D + 1) + D] = u;
                    }
                }
            }
        }
        // lexicographic successor: bump the rightmost position that can still grow, reset the positions after it
        int p = -1;
#pragma unroll
        for (int i = 0; i < D; ++i)
            if (s[i] < m - D + i) p = i;
        if (p < 0) break;
        int sp = 0;
#pragma unroll
        for (int i = 0; i < D; ++i) sp = i == p ? s[i] : sp;
#pragma unroll
        for (int i = 0; i < D; ++i)
            if (i >= p) s[i] = sp + 1 + (i - p);
    }
}

}  // namespace morl

extern "C" int morl_corner_weights_f64(const double* V, int n, int d, double* verts, int cap, int* count, void* stream) {
    using namespace morl;
    const char* fn = "morl_corner_weights_f64";
    MORL_REQUIRE(V && count && (verts || cap == 0), MORL_ERR_NULL, "%s: NULL pointer argument", fn);
    MORL_REQUIRE(n >= 1 && cap >= 0, MORL_ERR_SHAPE, "%s: bad shape n=%d cap=%d", fn, n, cap);
    MORL_REQUIRE(d >= 2 && d <= MORL_MAX_D, MORL_ERR_UNSUPPORTED, "%s: d=%d outside 2..%d", fn, d, MORL_MAX_D);
    const unsigned long long total = binom_capped((long long)n + d, d, MORL_CORNER_MAX_CANDIDATES);
    MORL_REQUIRE(total <= MORL_CORNER_MAX_CANDIDATES, MORL_ERR_UNSUPPORTED,
                 "%s: C(n+d, d) candidate subsets exceed %llu (n=%d, d=%d)", fn, (unsigned long long)MORL_CORNER_MAX_CANDIDATES, n, d);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e = cudaMemsetAsync(count, 0, sizeof(int), st);
    if (e != cudaSuccess) return check_launch(fn);
    // about 8 resident blocks of 128 threads per SM; each thread walks a contiguous range of candidates
    const unsigned long long max_threads = (unsigned long long)sm_count() * 8ull * kCornerThreads;
    const unsigned long long threads = total < max_threads ? total : max_threads;
    const unsigned long long per_thread = (total + threads - 1) / threads;
    const unsigned long long used = (total + per_thread - 1) / per_thread;
    const int blocks = (int)((used + kCornerThreads - 1) / kCornerThreads);
    switch (d) {
        case 2: corner_weights_kernel<2><<<blocks, kCornerThreads, 0, st>>>(V, n, total, per_thread, verts, cap, count); break;
        case 3: corner_weights_kernel<3><<<blocks, kCornerThreads, 0, st>>>(V, n, total, per_thread, verts, cap, count); break;
        case 4: corner_weights_kernel<4><<<blocks, kCornerThreads, 0, st>>>(V, n, total, per_thread, verts, cap, count); break;
        case 5: corner_weights_kernel<5><<<blocks, kCornerThreads, 0, st>>>(V, n, total, per_thread, verts, cap, count); break;
        case 6: corner_weights_kernel<6><<<blocks, kCornerThreads, 0, st>>>(V, n, total, per_thread, verts, cap, count); break;
        case 7: corner_weights_kernel<7><<<blocks, kCornerThreads, 0, st>>>(V, n, total, per_thread, verts, cap, count); break;
        default: corner_weights_kernel<8><<<blocks, kCornerThreads, 0, st>>>(V, n, total, per_thread, verts, cap, count); break;
    }
    return check_launch(fn);
}
