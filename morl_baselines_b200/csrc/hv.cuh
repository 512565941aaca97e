// hv.cuh -- exact hypervolume sweep shared by pareto.cu (single and batched sets) and pql.cu (Pareto Q-learning's action scores).
#pragma once
#include "common.cuh"

namespace morl {

// ---- exact hypervolume (maximisation) of one set, or of a batch of sets "base plus one candidate", above a reference point -----------------
// Replaces the host-side exact sweep behind `hypervolume(ref_point, points)` (reference common/performance_indicators.py:15-25, which
// delegates to pymoo's exact HV) for fronts that already live on the device, and IPRO's hypervolume improvements of the sampled lower points
// (reference multi_policy/ipro/ipro.py:212-226: one exact volume per candidate, all of them in one launch here).
// q_i = p_i - ref clipped at 0 (a point that does not exceed ref in some objective spans no volume; nor does a NaN); missing objectives get
// a unit extent, so every set is treated as 4-D.  Volume of the union of the boxes [0, q_i]: slabs in w-descending order (only one slab of
// height 1 when d <= 3), each slab a 3-D volume of the points with w-rank <= j; that volume is a sum over z-descending slabs of the 2-D
// staircase area of the points with z-rank <= k (and w-rank <= j), integrated over the x-descending order.  Thread t of the block takes the
// (w-slab, z-slab) pairs t, t + blockDim, ... (an O(n) loop each: n^2 work for d <= 3, n^3 for d = 4, no scans, no atomics); the slab
// volumes are added by a fixed-shape tree reduction (deterministic).  Ranks come from counting (ties by index).
constexpr int kHvMaxN = 2048;     // points per set, d <= 3
constexpr int kHvMaxN4 = 512;     // points per set, d = 4 (O(n^3) per set)
constexpr int kHvThreads = 1024;

// shared-memory carve for sets of up to n points: red [kHvThreads] | rx ry rz rw [n] (input order) | qx qy [n] (x-descending order) |
// zs ws [n + 1] (descending, then 0) | zr wr [n] shorts (z- and w-rank of the point at x-position i)
struct HvSmem {
    double *red, *rx, *ry, *rz, *rw, *qx, *qy, *zs, *ws;
    short *zr, *wr;
};

__host__ __device__ constexpr size_t hv_smem_bytes(int n) { return ((size_t)kHvThreads + 8 * (size_t)n + 2) * sizeof(double) + 2 * (size_t)n * sizeof(short); }

__device__ __forceinline__ HvSmem hv_carve(double* smem, int n) {
    HvSmem s;
    s.red = smem;
    s.rx = s.red + kHvThreads; s.ry = s.rx + n; s.rz = s.ry + n; s.rw = s.rz + n;
    s.qx = s.rw + n; s.qy = s.qx + n;
    s.zs = s.qy + n; s.ws = s.zs + n + 1;
    s.zr = reinterpret_cast<short*>(s.ws + n + 1); s.wr = s.zr + n;
    return s;
}

// stage point i: its clipped offsets from ref (all zero unless it exceeds ref in every objective and `keep`)
__device__ __forceinline__ void hv_stage(const HvSmem& s, int i, const double* __restrict__ p, bool keep, int d, const double* __restrict__ ref) {
    double c[4] = {0.0, 1.0, 1.0, 1.0};
    bool ok = keep;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        if (r < d) {
            const double v = p[r] - ref[r];
            c[r] = v > 0.0 ? v : 0.0;  // (NaN fails the comparison: contributes nothing)
            ok = ok && (v > 0.0);
        }
    }
    s.rx[i] = ok ? c[0] : 0.0; s.ry[i] = ok ? c[1] : 0.0; s.rz[i] = ok ? c[2] : 0.0; s.rw[i] = ok ? c[3] : 0.0;
}

// the volume of the n staged points (every thread returns it); `sliced_w`: the w-slabs of d = 4, else one slab of height 1
__device__ __forceinline__ double hv_sweep(const HvSmem& s, int n, bool sliced_w) {
    // rank by counting: position of point i in x-descending order (ties by index), its z- and w-descending ranks
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const double xi = s.rx[i], zi = s.rz[i], wi = s.rw[i];
        int px = 0, pz = 0, pw = 0;
        for (int j = 0; j < n; ++j) {
            px += (s.rx[j] > xi || (s.rx[j] == xi && j < i)) ? 1 : 0;
            pz += (s.rz[j] > zi || (s.rz[j] == zi && j < i)) ? 1 : 0;
            if (sliced_w) pw += (s.rw[j] > wi || (s.rw[j] == wi && j < i)) ? 1 : 0;
        }
        s.qx[px] = xi; s.qy[px] = s.ry[i]; s.zr[px] = (short)pz; s.wr[px] = (short)pw;
        s.zs[pz] = zi; s.ws[pw] = wi;
    }
    if (threadIdx.x == 0) { s.zs[n] = 0.0; s.ws[n] = 0.0; }
    __syncthreads();
    const int nw = sliced_w ? n : 1;
    double acc = 0.0;
    for (int t = threadIdx.x; t < nw * n; t += blockDim.x) {
        const int j = t / n, k = t - j * n;           // w-slab j, z-slab k
        const double zh = s.zs[k] - s.zs[k + 1];      // slab between the k-th and (k+1)-th largest z
        const double wh = sliced_w ? s.ws[j] - s.ws[j + 1] : 1.0;
        if (zh > 0.0 && wh > 0.0) {
            double m = 0.0, area = 0.0;
            for (int i = 0; i < n; ++i) {
                if ((int)s.zr[i] <= k && (int)s.wr[i] <= j) m = fmax(m, s.qy[i]);
                const double xn = i + 1 < n ? s.qx[i + 1] : 0.0;
                area = __fma_rn(s.qx[i] - xn, m, area);
            }
            acc = __fma_rn(__dmul_rn(area, wh), zh, acc);  // (wh = 1 is exact: the d <= 3 sum is area * zh)
        }
    }
    s.red[threadIdx.x] = acc;
    __syncthreads();
    for (int off = kHvThreads / 2; off > 0; off >>= 1) {
        if (threadIdx.x < off) s.red[threadIdx.x] += s.red[threadIdx.x + off];
        __syncthreads();
    }
    return s.red[0];
}

}  // namespace morl
