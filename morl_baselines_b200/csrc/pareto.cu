// pareto.cu -- warp-ballot Pareto dominance mask (SURVEY.md K10).
//
// Replaces get_non_pareto_dominated_inds (reference common/pareto.py:34-57), whose all-pairs broadcast builds two
// N x N x D boolean temporaries plus a lexicographic np.unique.  Rule reproduced (SURVEY Appendix A.5):
//   keep[i] = no row j holds a DIFFERENT value that is >= pts[i] in every coordinate
//             AND (remove_duplicates == 0 OR no j < i holds exactly the same value)
//             AND pts[i] contains no NaN.
// Comparisons are exact in the input dtype (fp32 or fp64); output order = input order.
//
// Mapping: grid = (i-tiles, j-splits).  A CTA stages a tile of IT candidate rows i in shared memory; each lane holds
// one potential dominator row j in registers (coalesced global load), the warp walks the i-tile with broadcast
// shared-memory reads, and one __ballot_sync per (i, 32 j's) tells the whole warp whether i was just killed.
#include "common.cuh"
#include "hv.cuh"

namespace morl {

constexpr int kParetoThreads = 256;
constexpr int kParetoTile = 256;  // rows i per CTA

template <typename T, int D>
__global__ void __launch_bounds__(kParetoThreads) pareto_init_kernel(const T* __restrict__ pts, int N, uint8_t* __restrict__ keep) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    bool ok = true;
#pragma unroll
    for (int r = 0; r < D; ++r) {
        const T v = pts[(size_t)i * D + r];
        ok = ok && (v == v);
    }
    keep[i] = ok ? 1 : 0;
}

template <typename T, int D>
__global__ void __launch_bounds__(kParetoThreads) pareto_mask_kernel(const T* __restrict__ pts, int N, int remove_duplicates,
                                                                     int j_per_split, uint8_t* __restrict__ keep) {
    __shared__ T xi_s[kParetoTile * D];
    __shared__ uint8_t killed[kParetoTile];
    const int i0 = blockIdx.x * kParetoTile;
    const int ni = min(kParetoTile, N - i0);
    for (int t = threadIdx.x; t < ni * D; t += blockDim.x) xi_s[t] = pts[(size_t)i0 * D + t];
    for (int t = threadIdx.x; t < kParetoTile; t += blockDim.x) killed[t] = 0;
    __syncthreads();

    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int nwarps = blockDim.x >> 5;
    const int jbeg = blockIdx.y * j_per_split;
    const int jend = min(N, jbeg + j_per_split);

    for (int jc = jbeg + warp * 32; jc < jend; jc += nwarps * 32) {
        const int j = jc + lane;
        const bool jvalid = j < jend;
        T xj[D];
#pragma unroll
        for (int r = 0; r < D; ++r) xj[r] = jvalid ? pts[(size_t)j * D + r] : T(0);
        for (int ii = 0; ii < ni; ++ii) {
            bool ge = jvalid, eq = jvalid;
#pragma unroll
            for (int r = 0; r < D; ++r) {
                const T xi = xi_s[ii * D + r];  // warp-wide broadcast
                ge = ge && (xj[r] >= xi);
                eq = eq && (xj[r] == xi);
            }
            const bool kill = (ge && !eq) || (remove_duplicates && eq && (j < i0 + ii));
            const unsigned m = __ballot_sync(0xffffffffu, kill);
            if (m != 0u && lane == 0) killed[ii] = 1;  // benign same-value race between warps
        }
    }
    __syncthreads();
    for (int t = threadIdx.x; t < ni; t += blockDim.x)
        if (killed[t]) keep[i0 + t] = 0;  // only ever cleared after pareto_init_kernel set it
}

template <typename T>
static int pareto_launch(const char* fn, const T* pts, int N, int D, int remove_duplicates, uint8_t* keep, void* stream) {
    MORL_REQUIRE(pts && keep, MORL_ERR_NULL, "%s: NULL pointer argument", fn);
    MORL_REQUIRE(N >= 0 && D > 0, MORL_ERR_SHAPE, "%s: bad shape N=%d D=%d", fn, N, D);
    MORL_REQUIRE(D <= MORL_MAX_D, MORL_ERR_UNSUPPORTED, "%s: D=%d > %d", fn, D, MORL_MAX_D);
    if (N == 0) return MORL_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int itiles = (N + kParetoTile - 1) / kParetoTile;
    // enough CTAs for ~4 waves of 132 SMs, but never split j finer than one pass of the CTA's 8 warps
    int jsplits = (4 * 132 + itiles - 1) / itiles;
    const int max_splits = (N + kParetoThreads - 1) / kParetoThreads;
    if (jsplits > max_splits) jsplits = max_splits;
    if (jsplits < 1) jsplits = 1;
    int j_per_split = (N + jsplits - 1) / jsplits;
    j_per_split = (j_per_split + 31) / 32 * 32;
    jsplits = (N + j_per_split - 1) / j_per_split;
    const dim3 grid((unsigned)itiles, (unsigned)jsplits, 1);
    MORL_DISPATCH_D(D, {
        pareto_init_kernel<T, kD><<<(N + kParetoThreads - 1) / kParetoThreads, kParetoThreads, 0, st>>>(pts, N, keep);
        pareto_mask_kernel<T, kD><<<grid, kParetoThreads, 0, st>>>(pts, N, remove_duplicates, j_per_split, keep);
    });
    return check_launch(fn);
}

// ---- front records for the one-collective exchange of non-dominated fronts (SURVEY.md 8(e)) ----------------------------------------------
// record = [ count | cap x d rows | n_extra extras ] (float64).  Everything stays on the device and on one stream: no host-visible count,
// fixed shapes, so the evaluation round is  prune -> pack -> ONE all-gather -> unpack -> prune -> pack -> one device->host copy.
constexpr int kPackThreads = 1024;

// count = number of rows with keep != 0 (NOT clipped to cap, so overflow is visible to every rank); the first `cap` kept rows follow in
// input order; unused rows are -inf in every coordinate (dominated by any real point: harmless in the global prune).
__global__ void __launch_bounds__(kPackThreads) front_pack_kernel(const double* __restrict__ pts, const uint8_t* __restrict__ keep, int n, int d, int cap,
                                                                  const double* __restrict__ extras, int n_extra, double* __restrict__ rec) {
    __shared__ int warp_cnt[kPackThreads / 32];
    __shared__ int base_s;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) base_s = 0;
    __syncthreads();
    for (int i0 = 0; i0 < n; i0 += kPackThreads) {
        const int i = i0 + threadIdx.x;
        const bool k = i < n && (keep == nullptr || keep[i] != 0);
        const unsigned m = __ballot_sync(0xffffffffu, k);
        if (lane == 0) warp_cnt[warp] = __popc(m);
        __syncthreads();
        int before = base_s;
        for (int w = 0; w < warp; ++w) before += warp_cnt[w];
        const int pos = before + __popc(m & ((1u << lane) - 1u));
        if (k && pos < cap)
            for (int r = 0; r < d; ++r) rec[1 + (size_t)pos * d + r] = pts[(size_t)i * d + r];
        __syncthreads();
        if (threadIdx.x == 0) {
            int tot = 0;
            for (int w = 0; w < kPackThreads / 32; ++w) tot += warp_cnt[w];
            base_s += tot;
        }
        __syncthreads();
    }
    const int count = base_s;
    const double ninf = -__longlong_as_double(0x7FF0000000000000LL);
    for (long long e = (long long)min(count, cap) * d + threadIdx.x; e < (long long)cap * d; e += kPackThreads) rec[1 + e] = ninf;
    for (int e = threadIdx.x; e < n_extra; e += kPackThreads) rec[1 + (size_t)cap * d + e] = extras[e];
    if (threadIdx.x == 0) rec[0] = (double)count;
}

// gathered [world][rec_len] -> pts_out [world * cap, d] (rows as packed, -inf padding included) and meta_out [world][1 + n_extra]
// (count and extras of every rank, contiguous)
__global__ void __launch_bounds__(256) front_unpack_kernel(const double* __restrict__ gathered, int world, int rec_len, int d, int cap, int n_extra,
                                                           double* __restrict__ pts_out, double* __restrict__ meta_out) {
    const long long per = (long long)cap * d;
    const long long total = (long long)world * per;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(e / per);
        pts_out[e] = gathered[(size_t)r * rec_len + 1 + (e - (long long)r * per)];
    }
    const int m = world * (1 + n_extra);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < m; e += gridDim.x * blockDim.x) {
        const int r = e / (1 + n_extra), k = e - r * (1 + n_extra);
        meta_out[e] = k == 0 ? gathered[(size_t)r * rec_len] : gathered[(size_t)r * rec_len + 1 + per + (k - 1)];
    }
}

// one set: the points with keep[i] != 0 (keep NULL = all), d <= 3
__global__ void __launch_bounds__(kHvThreads, 1) hypervolume_kernel(const double* __restrict__ pts, const uint8_t* __restrict__ keep, int n, int d,
                                                                 const double* __restrict__ ref, double* __restrict__ out) {
    extern __shared__ double hv_smem[];
    const HvSmem s = hv_carve(hv_smem, n);
    for (int i = threadIdx.x; i < n; i += blockDim.x) hv_stage(s, i, pts + (size_t)i * d, keep == nullptr || keep[i] != 0, d, ref);
    __syncthreads();
    const double v = hv_sweep(s, n, false);
    if (threadIdx.x == 0) *out = v;
}

// block b: the set base [n_base] plus cand[b] (cand NULL: base alone), d <= 4
__global__ void __launch_bounds__(kHvThreads, 1) hypervolume_batch_kernel(const double* __restrict__ base, int n_base, const double* __restrict__ cand,
                                                                       int d, const double* __restrict__ ref, double* __restrict__ out) {
    extern __shared__ double hv_smem[];
    const int n = n_base + (cand != nullptr ? 1 : 0);
    const HvSmem s = hv_carve(hv_smem, n);
    for (int i = threadIdx.x; i < n; i += blockDim.x)
        hv_stage(s, i, i < n_base ? base + (size_t)i * d : cand + (size_t)blockIdx.x * d, true, d, ref);
    __syncthreads();
    const double v = hv_sweep(s, n, d == 4);
    if (threadIdx.x == 0) out[blockIdx.x] = v;
}

static int hv_batch_cap(int d) { return d >= 1 && d <= 3 ? kHvMaxN : d == 4 ? kHvMaxN4 : -1; }

}  // namespace morl

extern "C" int morl_pareto_mask_f32(const float* pts, int N, int D, int remove_duplicates, uint8_t* keep, void* stream) {
    return morl::pareto_launch<float>("morl_pareto_mask_f32", pts, N, D, remove_duplicates, keep, stream);
}

extern "C" int morl_pareto_mask_f64(const double* pts, int N, int D, int remove_duplicates, uint8_t* keep, void* stream) {
    return morl::pareto_launch<double>("morl_pareto_mask_f64", pts, N, D, remove_duplicates, keep, stream);
}

extern "C" int morl_front_pack_f64(const double* pts, const uint8_t* keep, int n, int d, int cap, const double* extras, int n_extra, double* rec,
                                   void* stream) {
    using namespace morl;
    MORL_REQUIRE(rec && (pts || n == 0) && (extras || n_extra == 0), MORL_ERR_NULL, "morl_front_pack_f64: NULL pointer argument");
    MORL_REQUIRE(n >= 0 && d > 0 && cap > 0 && n_extra >= 0, MORL_ERR_SHAPE, "morl_front_pack_f64: bad shape n=%d d=%d cap=%d n_extra=%d", n, d, cap, n_extra);
    front_pack_kernel<<<1, kPackThreads, 0, static_cast<cudaStream_t>(stream)>>>(pts, keep, n, d, cap, extras, n_extra, rec);
    return check_launch("morl_front_pack_f64");
}

extern "C" int morl_front_unpack_f64(const double* gathered, int world, int d, int cap, int n_extra, double* pts_out, double* meta_out, void* stream) {
    using namespace morl;
    MORL_REQUIRE(gathered && pts_out && meta_out, MORL_ERR_NULL, "morl_front_unpack_f64: NULL pointer argument");
    MORL_REQUIRE(world > 0 && d > 0 && cap > 0 && n_extra >= 0, MORL_ERR_SHAPE, "morl_front_unpack_f64: bad shape world=%d d=%d cap=%d n_extra=%d", world, d,
                 cap, n_extra);
    const int rec_len = 1 + cap * d + n_extra;
    long long blocks = ((long long)world * cap * d + 255) / 256;
    if (blocks > 132 * 4) blocks = 132 * 4;
    front_unpack_kernel<<<(int)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(gathered, world, rec_len, d, cap, n_extra, pts_out, meta_out);
    return check_launch("morl_front_unpack_f64");
}

extern "C" int morl_hypervolume_f64(const double* pts, const uint8_t* keep, int n, int d, const double* ref, double* out, void* stream) {
    using namespace morl;
    MORL_REQUIRE(ref && out && (pts || n == 0), MORL_ERR_NULL, "morl_hypervolume_f64: NULL pointer argument");
    MORL_REQUIRE(n >= 0 && d >= 1 && d <= 3, MORL_ERR_UNSUPPORTED, "morl_hypervolume_f64: exact device hypervolume supports 1 <= d <= 3 (got d=%d)", d);
    MORL_REQUIRE(n <= kHvMaxN, MORL_ERR_UNSUPPORTED, "morl_hypervolume_f64: at most %d points (got %d): prune the set first", kHvMaxN, n);
    static bool configured = false;
    if (!configured) {
        cudaFuncSetAttribute(hypervolume_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hv_smem_bytes(kHvMaxN));
        configured = true;
    }
    hypervolume_kernel<<<1, kHvThreads, hv_smem_bytes(n), static_cast<cudaStream_t>(stream)>>>(pts, keep, n, d, ref, out);
    return check_launch("morl_hypervolume_f64");
}

extern "C" int morl_hypervolume_batch_supported(int n, int d) {
    const int cap = morl::hv_batch_cap(d);
    return cap > 0 && n >= 0 && n <= cap ? 1 : 0;
}

extern "C" int morl_hypervolume_batch_f64(const double* base, int n_base, const double* cand, int n_cand, int d, const double* ref, double* out,
                                          void* stream) {
    using namespace morl;
    MORL_REQUIRE(ref && out && (base || n_base == 0) && (cand || n_cand == 0), MORL_ERR_NULL, "morl_hypervolume_batch_f64: NULL pointer argument");
    MORL_REQUIRE(n_base >= 0 && n_cand >= 0, MORL_ERR_SHAPE, "morl_hypervolume_batch_f64: bad shape n_base=%d n_cand=%d", n_base, n_cand);
    MORL_REQUIRE(morl_hypervolume_batch_supported(n_base, d), MORL_ERR_UNSUPPORTED,
                 "morl_hypervolume_batch_f64: supports 1 <= d <= 4 with at most %d (d <= 3) or %d (d = 4) base points (got d=%d, n_base=%d)",
                 kHvMaxN, kHvMaxN4, d, n_base);
    static bool configured = false;
    if (!configured) {
        cudaFuncSetAttribute(hypervolume_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hv_smem_bytes(kHvMaxN + 1));
        configured = true;
    }
    const int n = n_base + (n_cand > 0 ? 1 : 0);
    hypervolume_batch_kernel<<<n_cand > 0 ? n_cand : 1, kHvThreads, hv_smem_bytes(n), static_cast<cudaStream_t>(stream)>>>(
        base, n_base, n_cand > 0 ? cand : nullptr, d, ref, out);
    return check_launch("morl_hypervolume_batch_f64");
}
