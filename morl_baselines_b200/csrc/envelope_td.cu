// envelope_td.cu -- fused envelope-max TD target (SURVEY.md K3+K4).
//
// Replaces Envelope.envelope_target (reference multi_policy/envelope/envelope.py:404-440) and the vector Bellman
// line (envelope.py:298).  The reference runs both Q-nets on B*W^2 tiled rows; here the operator consumes the
// Q tensors of the B*W DISTINCT (s'_b, w_j) rows and performs, per output row (i, b),
//     (j*, a*) = first argmax_{j,a} wset[i] . Q_on[b, j, a, :]        (joint first-occurrence == th.max(dim=2) then th.argmax(dim=1))
//     out      = r[b] + ((1 - done[b]) * gamma) * Q_tg[b, j*, a*, :]
//
// Mapping (one CTA per transition b): the Q_on[b] block (W*A*D floats, 6 KB at the north-star shape) is staged in
// shared memory with 128-bit loads; thread (js, i) owns scalarising weight i and scans the j = js, js+JS, ...
// candidates, so every shared-memory read is a warp-wide broadcast (all lanes of a warp share js) and no shuffle
// is needed in the hot loop; the JS partial results per weight are merged through shared memory with the
// (value desc, flat index asc) order, which preserves first-occurrence semantics.  Q_tg is only touched at the
// winning (j*, a*) (a D-float gather per output row), never streamed.
#include <limits.h>
#include <stdlib.h>

#include "envelope_wp.cuh"
#include "gemm_tc.cuh"

namespace morl {

template <int D, int MODE, bool VEC4>
__global__ void __launch_bounds__(512) envelope_td_kernel(const float* __restrict__ q_on, const float* __restrict__ q_tg,
                                                          const float* __restrict__ wset, const float* __restrict__ reward,
                                                          const float* __restrict__ done, float gamma, int B, int W, int A,
                                                          int Wc, int JS, int JT, int row_order,
                                                          float* __restrict__ target_out, int32_t* __restrict__ pref_out,
                                                          int32_t* __restrict__ act_out) {
    extern __shared__ __align__(16) float smem[];
    const int AD = A * D;
    const int tile_floats = (JT * AD + 3) & ~3;
    float* tile = smem;
    float* pv = smem + tile_floats;                         // [JS][Wc] partial best values
    int* pi = reinterpret_cast<int*>(pv + JS * Wc);         // [JS][Wc] partial best flat indices

    const int b = blockIdx.x;
    const int il = threadIdx.x % Wc;
    const int js = threadIdx.x / Wc;
    const int i = blockIdx.y * Wc + il;
    const bool active = i < W;

    float w[D];
#pragma unroll
    for (int r = 0; r < D; ++r) w[r] = active ? __ldg(wset + (size_t)i * D + r) : 0.f;

    float best = -INFINITY;
    int bidx = INT_MAX;

    const float* qb = q_on + (size_t)b * W * AD;
    for (int j0 = 0; j0 < W; j0 += JT) {
        const int jt = min(JT, W - j0);
        const int n = jt * AD;
        const float* src = qb + (size_t)j0 * AD;
        if (j0 > 0) __syncthreads();  // previous tile fully consumed
        if (((reinterpret_cast<uintptr_t>(src) & 15u) == 0) && (n % 4 == 0)) {
            const float4* s4 = reinterpret_cast<const float4*>(src);
            float4* d4 = reinterpret_cast<float4*>(tile);
            for (int t = threadIdx.x; t < n / 4; t += blockDim.x) d4[t] = __ldg(s4 + t);
        } else {
            for (int t = threadIdx.x; t < n; t += blockDim.x) tile[t] = __ldg(src + t);
        }
        __syncthreads();
        if (active) {
            for (int jj = js; jj < jt; jj += JS) {
                const float* qj = tile + jj * AD;
                const int base = (j0 + jj) * A;
                if constexpr (VEC4) {
                    for (int a4 = 0; a4 < A; a4 += 4) {
                        float f[4 * D];
                        const float4* p = reinterpret_cast<const float4*>(qj + a4 * D);
#pragma unroll
                        for (int v = 0; v < D; ++v) {
                            const float4 x = p[v];
                            f[4 * v + 0] = x.x;
                            f[4 * v + 1] = x.y;
                            f[4 * v + 2] = x.z;
                            f[4 * v + 3] = x.w;
                        }
#pragma unroll
                        for (int t = 0; t < 4; ++t) {
                            float q[D];
#pragma unroll
                            for (int r = 0; r < D; ++r) q[r] = f[t * D + r];
                            const float s = dotw<D, MODE>(w, q);
                            if (s > best) {
                                best = s;
                                bidx = base + a4 + t;
                            }
                        }
                    }
                } else {
                    for (int a = 0; a < A; ++a) {
                        float q[D];
#pragma unroll
                        for (int r = 0; r < D; ++r) q[r] = qj[a * D + r];
                        const float s = dotw<D, MODE>(w, q);
                        if (s > best) {
                            best = s;
                            bidx = base + a;
                        }
                    }
                }
            }
        }
    }

    if (JS > 1) {
        pv[js * Wc + il] = best;
        pi[js * Wc + il] = bidx;
        __syncthreads();
    }
    if (js == 0 && active) {
        for (int s = 1; s < JS; ++s) argmax_merge(best, bidx, pv[s * Wc + il], pi[s * Wc + il]);
        if (bidx == INT_MAX) bidx = 0;  // every candidate was -inf (or NaN): th.argmax returns 0
        const int jstar = bidx / A;
        const int astar = bidx - jstar * A;
        const float* qt = q_tg + (((size_t)b * W + jstar) * A + astar) * D;
        const size_t k = (row_order == MORL_ROWS_REFERENCE) ? ((size_t)i * B + b) : ((size_t)b * W + i);
        const float dn = __ldg(done + b);
#pragma unroll
        for (int r = 0; r < D; ++r)
            target_out[k * D + r] = bellman(__ldg(reward + (size_t)b * D + r), dn, gamma, __ldg(qt + r));
        if (pref_out) pref_out[k] = jstar;
        if (act_out) act_out[k] = astar;
    }
}


// =================================================================================================================
// v3 kernel: CUDA-core fast path for the shapes the weight-pair kernel below does not take (|W| <= 32, W*A not a multiple of 16).
//   * Q_on[b] arrives by a 1-D bulk async copy (AoS staging) and is transposed once, smem -> smem, into SoA planes Qs[r][c]
//     (c = j*A + a), so one LDS.128 yields the r-th objective of four consecutive candidates.  The transposing pass walks
//     candidates (no div/mod) and is bank-conflict free for odd D;
//   * candidates are scanned in groups of 8: eight FMA-chain scores, max of 8, and only the GROUP index of the running maximum is
//     tracked (strict '>' keeps the first group); the exact (first) position inside the winning group is recovered afterwards by
//     re-evaluating its 8 scores in the contract arithmetic and taking the first strict maximum;
//   * FILTER (MODE != FMA): the scan uses the 3-op FMA chain t = fma(w2,q2, fma(w1,q1, w0*q0)) as an approximation of the
//     contract arithmetic e (5 roundings).  |t - e| <= 6u * sum_r |w_r q_r| < eps := 2^-21 * (sum_r |w_r|) * max|Q_on[b]|.
//     Per weight the scan keeps the best group maximum, its (first) group, and the runner-up group maximum.  If
//     runner_up < best - thr (thr = 2^-19 * ..., a 4x margin over 2 eps) every candidate outside the best group is exactly
//     smaller than the best group's maximum, so the exact first argmax lies in that group and is found by evaluating its 8
//     candidates in the contract arithmetic.  Otherwise (near tie, ~1e-4 of the rows on continuous data; always for constant
//     or non-finite Q) the row is re-scanned exactly by its whole warp.  The result is bit-identical to the exact scan.
//   * Q_tg[b] is staged with one 1-D bulk async copy that overlaps the scan; reward/done are pre-loaded.
// =================================================================================================================
template <int D, int MODE>
__global__ void __launch_bounds__(256) envelope_td_v3_kernel(const float* __restrict__ q_on, const float* __restrict__ q_tg,
                                                             const float* __restrict__ wset, const float* __restrict__ reward,
                                                             const float* __restrict__ done, float gamma, int B, int W, int A,
                                                             int Cp, int CS, int gps, int row_order, float* __restrict__ target_out,
                                                             int32_t* __restrict__ pref_out, int32_t* __restrict__ act_out) {
    constexpr bool FILTER = (MODE != MORL_DOT_FMA);
    constexpr int SCAN_MODE = MORL_DOT_FMA;  // arithmetic of the scan: the FMA chain (exact when MODE == FMA)
    extern __shared__ __align__(16) float smem[];
    const int C = W * A;
    const int plane = Cp;
    float* Qs = smem;                                        // [D][Cp] SoA planes of Q_on[b]
    float* Qt = smem + D * plane;                            // [C*D] AoS copy of Q_tg[b] (bulk async copy)
    const int WI = blockDim.x / CS;
    float* red_v = Qt + ((C * D + 3) & ~3);                  // [CS][WI] best
    float* red_s = red_v + CS * WI;                          // [CS][WI] runner-up
    int* red_g = reinterpret_cast<int*>(red_s + CS * WI);    // [CS][WI] group of best
    float* red_amax = reinterpret_cast<float*>(red_g + CS * WI);  // [32] per-warp max |Q|
    uint64_t* bar = reinterpret_cast<uint64_t*>(red_amax + 32);
    uint64_t* bar_on = bar + 1;
    float* Qa = reinterpret_cast<float*>(bar + 2);           // [C*D] AoS staging of Q_on[b] (bulk async copy)

    const int il = threadIdx.x % WI;
    const int cs = threadIdx.x / WI;
    const int i = blockIdx.y * WI + il;
    const bool active = i < W;
    const int lane = threadIdx.x & 31;
    const int nwarps = blockDim.x >> 5;

    float w[D];
    float wsum = 0.f;
#pragma unroll
    for (int r = 0; r < D; ++r) {
        w[r] = active ? __ldg(wset + (size_t)i * D + r) : 0.f;
        wsum += fabsf(w[r]);
    }
    const int ngroups = (C + 7) / 8;
    const int g_begin = cs * gps;
    const int g_end = min(g_begin + gps, ngroups);
    const int g_full = min(g_end, C / 8);
    const uint32_t qt_bytes = (uint32_t)(C * D) * 4u;  // multiple of 16 (launcher)

    if (threadIdx.x == 0) {
        g_mbar_init(bar, 1);
        g_mbar_init(bar_on, 1);
        g_mbar_init_fence();
    }
    for (int t = threadIdx.x; t < (Cp - C) * D; t += blockDim.x) Qs[(t / (Cp - C)) * plane + C + t % (Cp - C)] = 0.f;
    __syncthreads();

    uint32_t parity = 0;
    for (int b = blockIdx.x; b < B; b += gridDim.x, parity ^= 1u) {
        if (threadIdx.x == 0) {
            g_mbar_expect_tx(bar_on, qt_bytes);
            bulk_g2s(Qa, q_on + (size_t)b * C * D, qt_bytes, bar_on);
            g_mbar_expect_tx(bar, qt_bytes);
            bulk_g2s(Qt, q_tg + (size_t)b * C * D, qt_bytes, bar);
        }
        // pre-load the per-transition scalars of the epilogue
        float rw[D];
        float dn = 0.f;
        if (cs == 0) {
            dn = __ldg(done + b);
#pragma unroll
            for (int r = 0; r < D; ++r) rw[r] = __ldg(reward + (size_t)b * D + r);
        }
        // ---- Q_on[b] arrives by the same bulk async copy (AoS staging); transpose smem -> smem into the SoA planes ----
        // (reads at stride D words are bank-conflict free for odd D; the running max |q| feeds the filter threshold)
        float amax = 0.f;
        {
            g_mbar_wait(bar_on, parity);
            for (int c = threadIdx.x; c < C; c += blockDim.x) {
                float x[D];
#pragma unroll
                for (int r = 0; r < D; ++r) x[r] = Qa[c * D + r];
#pragma unroll
                for (int r = 0; r < D; ++r) {
                    Qs[r * plane + c] = x[r];
                    amax = fmaxf(amax, fabsf(x[r]));
                    if (!(x[r] == x[r])) amax = INFINITY;  // NaN in the block: force the exact path
                }
            }
            if (FILTER) {
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, off));
                if (lane == 0) red_amax[threadIdx.x >> 5] = amax;
            }
        }
        __syncthreads();
        float qmax = 0.f;
        if (FILTER)
            for (int k = 0; k < nwarps; ++k) qmax = fmaxf(qmax, red_amax[k]);

        // ---- scan: groups of 8 candidates, FMA-chain scores, best / runner-up group maxima ----
        float best = -INFINITY, second = -INFINITY;
        int bg = INT_MAX;
        auto scan_group = [&](int g, bool tail) {
            const int c0 = 8 * g;
            float q[8][D];
#pragma unroll
            for (int r = 0; r < D; ++r) {
                const float4 lo = *reinterpret_cast<const float4*>(Qs + r * plane + c0);
                const float4 hi = *reinterpret_cast<const float4*>(Qs + r * plane + c0 + 4);
                q[0][r] = lo.x;
                q[1][r] = lo.y;
                q[2][r] = lo.z;
                q[3][r] = lo.w;
                q[4][r] = hi.x;
                q[5][r] = hi.y;
                q[6][r] = hi.z;
                q[7][r] = hi.w;
            }
            float x[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) x[k] = dotw<D, SCAN_MODE>(w, q[k]);
            if (tail) {
#pragma unroll
                for (int k = 0; k < 8; ++k)
                    if (c0 + k >= C) x[k] = -INFINITY;
            }
            const float m = fmaxf(wp::max3(x[0], x[1], x[2]), wp::max3(wp::max3(x[3], x[4], x[5]), x[6], x[7]));
            if (FILTER) second = fmaxf(second, fminf(best, m));
            if (m > best) {
                best = m;
                bg = g;
            }
        };
#pragma unroll 2
        for (int g = g_begin; g < g_full; ++g) scan_group(g, false);
        for (int g = max(g_begin, g_full); g < g_end; ++g) scan_group(g, true);

        if (CS > 1) {
            red_v[cs * WI + il] = best;
            red_g[cs * WI + il] = bg;
            if (FILTER) red_s[cs * WI + il] = second;
            __syncthreads();
        }
        if (cs == 0) {  // warp-uniform: WI is a multiple of 32
            for (int s = 1; s < CS; ++s) {
                const float v2 = red_v[s * WI + il];
                const int g2 = red_g[s * WI + il];
                if (FILTER) second = fmaxf(fmaxf(second, red_s[s * WI + il]), fminf(best, v2));
                argmax_merge(best, bg, v2, g2);
            }
            int cstar = 0;
            bool amb = false;
            if (FILTER) {
                const float thr = 1.9073486328125e-06f * wsum * qmax;  // 2^-19 * sum|w| * max|Q|
                amb = active && !(second < best - thr);                // also true for NaN / inf
            }
            if (!amb && bg != INT_MAX) {
                // exact first argmax inside the winning group, contract arithmetic (strict '>' from the left)
                const int c0 = 8 * bg;
                float ev = -INFINITY;
                int kf = 0;
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    float q[D];
#pragma unroll
                    for (int r = 0; r < D; ++r) q[r] = Qs[r * plane + c0 + k];
                    const float s = dotw<D, MODE>(w, q);
                    if (c0 + k < C && s > ev) {
                        ev = s;
                        kf = k;
                    }
                }
                cstar = c0 + kf;
            }
            if (FILTER) {
                // near ties: the whole warp re-scans the row exactly (rare)
                unsigned ambmask = __ballot_sync(0xffffffffu, amb);
                while (ambmask) {
                    const int L = __ffs(ambmask) - 1;
                    ambmask &= ambmask - 1;
                    float wl[D];
#pragma unroll
                    for (int r = 0; r < D; ++r) wl[r] = __shfl_sync(0xffffffffu, w[r], L);
                    float bv = -INFINITY;
                    int bc = INT_MAX;
                    for (int c = lane; c < C; c += 32) {
                        float q[D];
#pragma unroll
                        for (int r = 0; r < D; ++r) q[r] = Qs[r * plane + c];
                        const float s = dotw<D, MODE>(wl, q);
                        if (s > bv) {
                            bv = s;
                            bc = c;
                        }
                    }
                    warp_argmax(bv, bc);
                    if (lane == L) cstar = (bc == INT_MAX) ? 0 : bc;
                }
            }
            g_mbar_wait(bar, parity);  // Q_tg[b] has landed in shared memory
            if (active) {
                const int jstar = cstar / A;
                const int astar = cstar - jstar * A;
                const float* qt = Qt + (size_t)cstar * D;
                const size_t k = (row_order == MORL_ROWS_REFERENCE) ? ((size_t)i * B + b) : ((size_t)b * W + i);
#pragma unroll
                for (int r = 0; r < D; ++r) target_out[k * D + r] = bellman(rw[r], dn, gamma, qt[r]);
                if (pref_out) pref_out[k] = jstar;
                if (act_out) act_out[k] = astar;
            }
        }
        __syncthreads();  // Qs / Qt / red_* are rewritten by the next transition
    }
}

// =================================================================================================================
// Weight-pair kernel, the default whenever the shape fits: one 128-thread CTA per block of 64 scalarising weights (blockIdx.y),
// persistent over the transitions b.  Q_on[b] and Q_tg[b] arrive by 1-D bulk async copies and are consumed as delivered (AoS, no
// transposition); the scan of a transition is wp::scan_transition (envelope_wp.cuh), the same code as in the fused head of
// qhead_envelope.cu.  Shapes: W*A a multiple of 16, 16-byte multiple Q blocks, |W| > 32 (below that half of the lanes would idle and
// v3 is used).
// =================================================================================================================
template <int D, int MODE>
__global__ void __launch_bounds__(128) envelope_td_wp_kernel(const float* __restrict__ q_on, const float* __restrict__ q_tg,
                                                             const float* __restrict__ wset, const float* __restrict__ reward,
                                                             const float* __restrict__ done, float gamma, int B, int W, int A,
                                                             int row_order, float* __restrict__ target_out,
                                                             int32_t* __restrict__ pref_out, int32_t* __restrict__ act_out) {
    extern __shared__ __align__(16) float smem[];
    const int C = W * A;
    const int CDp = (C * D + 3) & ~3;
    float* Qa = smem;                                              // [C*D] AoS Q_on[b]  (bulk async copy)
    float* Qt = Qa + CDp;                                          // [C*D] AoS Q_tg[b]  (bulk async copy)
    wp::Scratch* sc = reinterpret_cast<wp::Scratch*>(Qt + CDp);
    uint64_t* bar_on = reinterpret_cast<uint64_t*>(sc + 1);
    uint64_t* bar_tg = bar_on + 1;

    const int tid = threadIdx.x, part = tid & 1;
    const int wbase = blockIdx.y * 64;
    wp::Role<D> role;
    wp::load_role<D>(role, wset + (size_t)wbase * D, W - wbase, tid);
    const int fi = wbase + role.fi;
    const uint32_t q_bytes = (uint32_t)(C * D) * 4u;  // multiple of 16 (launcher)

    if (tid == 0) {
        g_mbar_init(bar_on, 1);
        g_mbar_init(bar_tg, 1);
        g_mbar_init_fence();
    }
    __syncthreads();

    uint32_t parity = 0;
    for (int b = blockIdx.x; b < B; b += gridDim.x, parity ^= 1u) {
        if (tid == 0) {
            g_mbar_expect_tx(bar_on, q_bytes);
            bulk_g2s(Qa, q_on + (size_t)b * C * D, q_bytes, bar_on);
            g_mbar_expect_tx(bar_tg, q_bytes);
            bulk_g2s(Qt, q_tg + (size_t)b * C * D, q_bytes, bar_tg);
        }
        float rw[D];
        const float dn = __ldg(done + b);
#pragma unroll
        for (int r = 0; r < D; ++r) rw[r] = __ldg(reward + (size_t)b * D + r);
        g_mbar_wait(bar_on, parity);
        const int cstar = wp::scan_transition<D, MODE>(Qa, *sc, role, tid, C, [] { __syncthreads(); });
        g_mbar_wait(bar_tg, parity);  // Q_tg[b] has landed in shared memory
        if (role.f_active) {
            const size_t k = (row_order == MORL_ROWS_REFERENCE) ? ((size_t)fi * B + b) : ((size_t)b * W + fi);
            if (part == 0) {
                const float* qt = Qt + (size_t)cstar * D;
#pragma unroll
                for (int r = 0; r < D; ++r) target_out[k * D + r] = bellman(rw[r], dn, gamma, qt[r]);
            } else {
                const int jstar = cstar / A;
                if (pref_out) pref_out[k] = jstar;
                if (act_out) act_out[k] = cstar - jstar * A;
            }
        }
        __syncthreads();  // Qa / Qt / the scratch are rewritten by the next transition
    }
}

struct EnvelopeV3Plan {
    bool ok;
    int Cp, CS, gps;
    dim3 grid, block;
    size_t smem;
};

static EnvelopeV3Plan plan_envelope_v3(int W, int A, int D) {
    EnvelopeV3Plan p{};
    const long long C = (long long)W * A;
    p.ok = false;
    if ((C * D) % 4 != 0) return p;  // Q_tg[b] must be a 16-byte multiple for the bulk copy
    const int Wp = (W + 31) / 32 * 32;
    const int WI = Wp < 256 ? Wp : 256;
    const int warps_i = WI / 32;
    int cs = 4 / warps_i;
    if (cs < 1) cs = 1;
    const int ngroups = (int)((C + 7) / 8);
    if (cs > ngroups) cs = ngroups;
    p.CS = cs;
    p.gps = (ngroups + cs - 1) / cs;
    p.Cp = ngroups * 8;
    p.block = dim3((unsigned)(WI * p.CS), 1, 1);
    const size_t qs = (size_t)D * p.Cp * sizeof(float);
    const size_t qt = (((size_t)C * D + 3) & ~(size_t)3) * sizeof(float);
    p.smem = qs + 2 * qt + 3 * (size_t)p.CS * WI * sizeof(float) + 32 * sizeof(float) + 16;
    if (p.smem > 96 * 1024) return p;
    p.grid = dim3(1u, (unsigned)((W + WI - 1) / WI), 1);  // grid.x is set by the launcher from the measured occupancy
    p.ok = true;
    return p;
}

struct EnvelopePlan {
    int Wc, JS, JT;
    dim3 grid, block;
    size_t smem;
};

static EnvelopePlan plan_envelope(int B, int W, int A, int D) {
    EnvelopePlan p;
    const int Wp = (W + 31) / 32 * 32;
    p.Wc = Wp < 256 ? Wp : 256;
    int js = 256 / p.Wc;
    if (js > 8) js = 8;
    if (js > W) js = W;
    if (js < 1) js = 1;
    p.JS = js;
    const int AD = A * D;
    int jt = 10240 / AD;  // <= 40 KB of tile
    if (jt < 1) jt = 1;
    if (jt > W) jt = W;
    p.JT = jt;
    p.grid = dim3((unsigned)B, (unsigned)((W + p.Wc - 1) / p.Wc), 1);
    p.block = dim3((unsigned)(p.Wc * p.JS), 1, 1);
    const size_t tile_floats = ((size_t)jt * AD + 3) & ~(size_t)3;
    p.smem = (tile_floats + 2 * (size_t)p.JS * p.Wc) * sizeof(float);
    return p;
}

// grid.x of the persistent kernels: every transition co-resident in one wave when they fit, else CTAs striding over b
static unsigned persistent_grid_x(int sms, int occ, unsigned gy, int B) {
    long long gx = (long long)sms * (occ < 1 ? 1 : occ) / gy;
    if (gx < 1) gx = 1;
    if (gx > B) gx = B;
    return (unsigned)gx;
}

// Path selection, read on every call: MORL_ENVELOPE_PATH = "v1" (generic kernel), "v3" (CUDA-core fast path), "wp" (weight-pair
// kernel).  Unset: "wp" whenever the shape fits, then "v3", then "v1".
enum EnvelopePath { kPathAuto, kPathV1, kPathV3, kPathWp };

static EnvelopePath envelope_path_override() {
    const char* e = getenv("MORL_ENVELOPE_PATH");
    if (!e) return kPathAuto;
    if (e[0] == 'v' && e[1] == '1') return kPathV1;
    if (e[0] == 'v' && e[1] == '3') return kPathV3;
    if (e[0] == 'w' && e[1] == 'p') return kPathWp;
    return kPathAuto;
}

}  // namespace morl

extern "C" int morl_envelope_td_f32(const float* q_online, const float* q_target, const float* wset, const float* reward,
                                    const float* done, float gamma, int B, int W, int A, int D, int dot_mode,
                                    int row_order, float* target_out, int32_t* pref_out, int32_t* act_out, void* stream) {
    using namespace morl;
    MORL_REQUIRE(q_online && q_target && wset && reward && done && target_out, MORL_ERR_NULL,
                 "morl_envelope_td_f32: NULL pointer argument");
    MORL_REQUIRE(B > 0 && W > 0 && A > 0 && D > 0, MORL_ERR_SHAPE, "morl_envelope_td_f32: bad shape B=%d W=%d A=%d D=%d", B,
                 W, A, D);
    MORL_REQUIRE(D <= MORL_MAX_D && A * D <= 10240, MORL_ERR_UNSUPPORTED,
                 "morl_envelope_td_f32: unsupported D=%d (max %d) or A*D=%d (max 10240)", D, MORL_MAX_D, A * D);
    MORL_REQUIRE((long long)W * A < INT_MAX, MORL_ERR_UNSUPPORTED, "morl_envelope_td_f32: W*A overflows int32");
    MORL_REQUIRE(dot_mode >= 0 && dot_mode <= 2, MORL_ERR_UNSUPPORTED, "morl_envelope_td_f32: bad dot_mode %d", dot_mode);
    MORL_REQUIRE(row_order == MORL_ROWS_REFERENCE || row_order == MORL_ROWS_BMAJOR, MORL_ERR_UNSUPPORTED,
                 "morl_envelope_td_f32: bad row_order %d", row_order);
    MORL_REQUIRE(aligned16(q_online) && aligned16(q_target) && aligned16(target_out), MORL_ERR_ALIGN,
                 "morl_envelope_td_f32: q_online/q_target/target_out must be 16-byte aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int sms = morl_device_sm_count();
    if (sms <= 0) sms = 132;
    const EnvelopePath path = envelope_path_override();
    const long long Cw = (long long)W * A;
    const size_t wp_smem = (size_t)(2 * ((Cw * D + 3) & ~3LL) + 3 * 256 + 16) * 4;  // Q_on[b], Q_tg[b], wp::Scratch, barriers
    const bool wp_ok = W > 32 && (Cw % 16) == 0 && ((Cw * D) % 4) == 0 && wp_smem <= 96 * 1024;
    MORL_REQUIRE(path != kPathWp || wp_ok, MORL_ERR_UNSUPPORTED, "morl_envelope_td_f32: MORL_ENVELOPE_PATH=wp but the shape W=%d A=%d D=%d is outside the weight-pair path", W, A, D);
    if (wp_ok && (path == kPathAuto || path == kPathWp)) {
        bool launched = false;
        MORL_DISPATCH_D(D, MORL_DISPATCH_MODE(dot_mode, {
                            auto kern = envelope_td_wp_kernel<kD, kMode>;
                            if (wp_smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wp_smem);
                            int occ = 0;
                            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, 128, wp_smem);
                            const unsigned gy = (unsigned)((W + 63) / 64);
                            kern<<<dim3(persistent_grid_x(sms, occ, gy, B), gy, 1), 128, wp_smem, st>>>(
                                q_online, q_target, wset, reward, done, gamma, B, W, A, row_order, target_out, pref_out, act_out);
                            launched = true;
                        }));
        MORL_REQUIRE(launched, MORL_ERR_UNSUPPORTED, "morl_envelope_td_f32: no weight-pair kernel for D=%d mode=%d", D, dot_mode);
        return check_launch("morl_envelope_td_f32(wp)");
    }
    EnvelopeV3Plan p3 = plan_envelope_v3(W, A, D);
    if (p3.ok && path != kPathV1) {
        bool launched = false;
        MORL_DISPATCH_D(D, MORL_DISPATCH_MODE(dot_mode, {
                            auto kern = envelope_td_v3_kernel<kD, kMode>;
                            if (p3.smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p3.smem);
                            int occ = 0;
                            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, (int)p3.block.x, p3.smem);
                            p3.grid.x = persistent_grid_x(sms, occ, p3.grid.y, B);
                            kern<<<p3.grid, p3.block, p3.smem, st>>>(q_online, q_target, wset, reward, done, gamma, B, W, A, p3.Cp, p3.CS, p3.gps,
                                                                      row_order, target_out, pref_out, act_out);
                            launched = true;
                        }));
        MORL_REQUIRE(launched, MORL_ERR_UNSUPPORTED, "morl_envelope_td_f32: no fast-path kernel for D=%d mode=%d", D, dot_mode);
        return check_launch("morl_envelope_td_f32(v3)");
    }
    const EnvelopePlan p = plan_envelope(B, W, A, D);
    const bool vec4 = (A % 4 == 0);
    bool launched = false;
    MORL_DISPATCH_D(D, MORL_DISPATCH_MODE(dot_mode, {
                        if (vec4)
                            envelope_td_kernel<kD, kMode, true><<<p.grid, p.block, p.smem, st>>>(
                                q_online, q_target, wset, reward, done, gamma, B, W, A, p.Wc, p.JS, p.JT, row_order,
                                target_out, pref_out, act_out);
                        else
                            envelope_td_kernel<kD, kMode, false><<<p.grid, p.block, p.smem, st>>>(
                                q_online, q_target, wset, reward, done, gamma, B, W, A, p.Wc, p.JS, p.JT, row_order,
                                target_out, pref_out, act_out);
                        launched = true;
                    }));
    MORL_REQUIRE(launched, MORL_ERR_UNSUPPORTED, "morl_envelope_td_f32: no kernel for D=%d mode=%d", D, dot_mode);
    return check_launch("morl_envelope_td_f32");
}
