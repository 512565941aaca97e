// envelope_wp.cuh -- the "weight pair" envelope scan of ONE transition by a group of 128 threads, as a device function, so that the
// operator can run inside another kernel's epilogue (qhead_envelope.cu: the Q tiles are produced in shared memory by the output layer's
// tensor-core GEMMs and never exist in HBM).  Same algorithm, arithmetic and tie rules as envelope_td_wp_kernel (envelope_td.cu):
//   scan   : lane = weight pair (two scalarising weights packed in f32x2 registers), warp = candidate quarter, groups of 16 candidates,
//            FMA-chain scores (the FILTER), best / runner-up group maxima per weight;
//   finish : thread pair (2k, 2k+1) re-evaluates weight k's winning group in the CONTRACT arithmetic (first occurrence), near ties
//            (runner-up within 2^-19 * sum|w| * max|Q| of the best) are re-scanned exactly by the whole warp;
//   output : r + ((1 - done) gamma) Q_tg[b, j*, a*, :]  (reference multi_policy/envelope/envelope.py:422-440, 298).
// Bit-identical to the standalone operator on identical Q tiles (tests/test_qhead_envelope_gpu.py).
#pragma once
#include <limits.h>

#include "common.cuh"

namespace morl {
namespace wp {

typedef unsigned long long u64;
__device__ __forceinline__ u64 pk2(float lo, float hi) {
    u64 r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
    return r;
}
__device__ __forceinline__ void upk2(u64 v, float& lo, float& hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
// Hopper has no packed-fp32 arithmetic and no 3-input max: the pair forms below are two scalar IEEE operations on the halves of the
// register pair (the same values a packed instruction would give), the 3-input max two FMNMX
__device__ __forceinline__ u64 mul2(u64 a, u64 b) {
    float a0, a1, b0, b1;
    upk2(a, a0, a1);
    upk2(b, b0, b1);
    return pk2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ u64 fma2(u64 a, u64 b, u64 c) {
    float a0, a1, b0, b1, c0, c1;
    upk2(a, a0, a1);
    upk2(b, b0, b1);
    upk2(c, c0, c1);
    return pk2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ float max3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }

// per-group scratch in shared memory: [4][64] best group maximum, runner-up, group of best; [4] max |Q| bits per warp
struct Scratch {
    float red_v[256];
    float red_s[256];
    int red_g[256];
    unsigned red_amax[4];
};

// per-thread constants of a group member (the weight set does not change between transitions)
template <int D>
struct Role {
    u64 wp2[D];    // scan role: weights 2*lane, 2*lane + 1
    float fw[D];   // finish role: weight tid >> 1
    float wsum;
    int fi;        // finish weight index
    bool f_active;
};

template <int D>
__device__ __forceinline__ void load_role(Role<D>& ro, const float* __restrict__ wset, int W, int tid) {
    const int lane = tid & 31;
    const int i0 = 2 * lane, i1 = i0 + 1;
#pragma unroll
    for (int r = 0; r < D; ++r) ro.wp2[r] = pk2(i0 < W ? __ldg(wset + (size_t)i0 * D + r) : 0.f, i1 < W ? __ldg(wset + (size_t)i1 * D + r) : 0.f);
    ro.fi = tid >> 1;
    ro.f_active = ro.fi < W;
    ro.wsum = 0.f;
#pragma unroll
    for (int r = 0; r < D; ++r) {
        ro.fw[r] = ro.f_active ? __ldg(wset + (size_t)ro.fi * D + r) : 0.f;
        ro.wsum += fabsf(ro.fw[r]);
    }
}

// One transition.  Qa / Qt: AoS [C][D] tiles of Q_on[b] / Q_tg[b] in shared memory (C = W*A candidates, c = j*A + a, C % 16 == 0,
// C*D % 4 == 0, 16-byte aligned).  `tid` in [0, 128) is the thread's index in its group, `sync()` a barrier over exactly the group.
// Returns the winning candidate c* (valid when ro.f_active); the caller writes the outputs.  Ends with the group in step (one barrier
// inside); the caller must barrier once more before Qa / Qt / the scratch are rewritten.
template <int D, int MODE, typename SyncF>
__device__ __forceinline__ int scan_transition(const float* __restrict__ Qa, Scratch& sc, const Role<D>& ro, int tid, int C, SyncF sync) {
    constexpr bool FILTER = (MODE != MORL_DOT_FMA);
    const int lane = tid & 31, warp = tid >> 5;
    const int ngroups = C >> 4;
    const int gpw = (ngroups + 3) >> 2;
    const int g_begin = warp * gpw, g_end = min(g_begin + gpw, ngroups);

    // ---- max |Q_on[b]| for the filter threshold (integer max of the magnitude bits: NaN / inf sort above every finite value) ----
    if (FILTER) {
        unsigned am = 0u;
        for (int t = tid; t < (C * D) >> 2; t += 128) {
            const uint4 x = *reinterpret_cast<const uint4*>(Qa + 4 * t);
            am = max(max(am, x.x & 0x7FFFFFFFu), max(x.y & 0x7FFFFFFFu, max(x.z & 0x7FFFFFFFu, x.w & 0x7FFFFFFFu)));
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) am = max(am, __shfl_xor_sync(0xffffffffu, am, off));
        if (lane == 0) sc.red_amax[warp] = am;
    }

    // ---- scan: groups of 16 candidates, two weights per thread, FMA-chain scores ----
    float best0 = -INFINITY, second0 = -INFINITY, best1 = -INFINITY, second1 = -INFINITY;
    int bg0 = INT_MAX, bg1 = INT_MAX;
#pragma unroll 1
    for (int g = g_begin; g < g_end; ++g) {
        const float4* src = reinterpret_cast<const float4*>(Qa + (size_t)g * 16 * D);
        float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
        for (int sub = 0; sub < 4; ++sub) {
            float f[4 * D];
#pragma unroll
            for (int v = 0; v < D; ++v) {
                const float4 x = src[sub * D + v];
                f[4 * v + 0] = x.x;
                f[4 * v + 1] = x.y;
                f[4 * v + 2] = x.z;
                f[4 * v + 3] = x.w;
            }
            float lo[4], hi[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                u64 acc = mul2(ro.wp2[0], pk2(f[k * D], f[k * D]));
#pragma unroll
                for (int r = 1; r < D; ++r) acc = fma2(ro.wp2[r], pk2(f[k * D + r], f[k * D + r]), acc);
                upk2(acc, lo[k], hi[k]);
            }
            m0 = max3(max3(m0, lo[0], lo[1]), lo[2], lo[3]);
            m1 = max3(max3(m1, hi[0], hi[1]), hi[2], hi[3]);
        }
        if (FILTER) {
            second0 = fmaxf(second0, fminf(best0, m0));
            second1 = fmaxf(second1, fminf(best1, m1));
        }
        if (m0 > best0) {
            best0 = m0;
            bg0 = g;
        }
        if (m1 > best1) {
            best1 = m1;
            bg1 = g;
        }
    }
    {
        const int k0 = warp * 64 + 2 * lane;
        *reinterpret_cast<float2*>(sc.red_v + k0) = make_float2(best0, best1);
        *reinterpret_cast<int2*>(sc.red_g + k0) = make_int2(bg0, bg1);
        if (FILTER) *reinterpret_cast<float2*>(sc.red_s + k0) = make_float2(second0, second1);
    }
    sync();

    // ---- finish weight fi: merge the four quarters (candidate order), exact re-check of the winning group ----
    const int fl = tid >> 1, part = tid & 1;
    float bb = -INFINITY, ss = -INFINITY;
    int g = INT_MAX;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float pb = sc.red_v[k * 64 + fl];
        if (FILTER) ss = fmaxf(fmaxf(ss, sc.red_s[k * 64 + fl]), fminf(bb, pb));
        if (pb > bb) {
            bb = pb;
            g = sc.red_g[k * 64 + fl];
        }
    }
    bool amb = false;
    if (FILTER) {
        const unsigned am = max(max(sc.red_amax[0], sc.red_amax[1]), max(sc.red_amax[2], sc.red_amax[3]));
        const float qmax = am >= 0x7F800000u ? INFINITY : __uint_as_float(am);
        const float thr = 1.9073486328125e-06f * ro.wsum * qmax;  // 2^-19 * sum|w| * max|Q|
        amb = ro.f_active && !(ss < bb - thr);                    // also true for NaN / inf
    }
    int cstar = 0;
    {
        const int gg = (g == INT_MAX) ? 0 : g;  // every candidate was -inf / NaN: th.argmax returns 0 (found by the re-check below)
        const int c0 = 16 * gg + 8 * part;
        float ev = -INFINITY;
        int ei = INT_MAX;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            float q[D];
#pragma unroll
            for (int r = 0; r < D; ++r) q[r] = Qa[(c0 + k) * D + r];
            const float s = dotw<D, MODE>(ro.fw, q);
            if (s > ev) {
                ev = s;
                ei = c0 + k;
            }
        }
        const float ev2 = __shfl_xor_sync(0xffffffffu, ev, 1);
        const int ei2 = __shfl_xor_sync(0xffffffffu, ei, 1);
        argmax_merge(ev, ei, ev2, ei2);
        cstar = (ei == INT_MAX) ? 0 : ei;
    }
    if (FILTER) {
        // near ties: the whole warp re-scans the row exactly (rare)
        unsigned ambmask = __ballot_sync(0xffffffffu, amb && part == 0);
        while (ambmask) {
            const int L = __ffs(ambmask) - 1;
            ambmask &= ambmask - 1;
            float wl[D];
#pragma unroll
            for (int r = 0; r < D; ++r) wl[r] = __shfl_sync(0xffffffffu, ro.fw[r], L);
            float bv = -INFINITY;
            int bc = INT_MAX;
            for (int c = lane; c < C; c += 32) {
                float q[D];
#pragma unroll
                for (int r = 0; r < D; ++r) q[r] = Qa[c * D + r];
                const float s = dotw<D, MODE>(wl, q);
                if (s > bv) {
                    bv = s;
                    bc = c;
                }
            }
            warp_argmax(bv, bc);
            if ((lane & ~1) == L) cstar = (bc == INT_MAX) ? 0 : bc;
        }
    }
    return cstar;
}

}  // namespace wp
}  // namespace morl
